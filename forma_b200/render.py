"""Headless front end: render an SVG file to PPM / PNG on the GPU.

    python -m forma_b200.render in.svg out.ppm [--width W --height H --scale S --device 0] [--ids ids.npy] [--linear out.npy]
                                               [--over image.{ppm,png}] [--masks masks.npy --mask-orders A:B [--mask-u8]]
                                               [--stats stats.npz [--stats-orders A:B] [--stats-min-coverage C]]

The equivalent of the reference's `demo svg --file in.svg --scale S` + the `S` key's
capture.ppm (demo/src/main.rs, demo/src/runner.rs:193-219: a binary P6 file with the
frame's RGB bytes), without a window. The output format follows the extension (.ppm, or
.png when Pillow is available). There is no CPU fallback: without a CUDA device the
renderer cannot be created and the command fails. `--ids` also writes the frame's ID frame (per pixel
the order of the top-most layer drawn there, 0xFFFFFFFF for none) as an H x W uint32 .npy.
`--linear` also writes the frame's linear colour before the sRGB encode (RGBA, float32) as an
H x W x 4 .npy.
`--over` draws the SVG over an image instead of a white frame: the image (binary PPM, or PNG with
Pillow) goes to the GPU as an H x W x 4 uint8 tensor, Renderer.render_over_device draws over it, and
its size replaces --width / --height.
`--masks` also writes the layer coverage masks of orders [A, B) (`--mask-orders A:B`, Renderer.render_masks):
per layer its anti-aliased coverage, whatever lies above it, as a (B - A) x H x W float32 .npy, or uint8 with
`--mask-u8`.
`--stats` also writes the layer statistics of orders [A, B) (`--stats-orders A:B`, default every order;
Renderer.render_stats) to an .npz: per order its amodal `area` (sum of mask values x 2^18), the `pixels`
its mask exceeds `--stats-min-coverage` on and their `box` (x0, y0, x1, y1), the `visible` pixels its
ID owns and their `visible_box`, and the window's `first_order`.
"""
from __future__ import annotations

import argparse
import sys
import time

import numpy as np


def write_ppm(path: str, rgba: np.ndarray, width: int, height: int) -> None:
    """runner.rs:193-219: "P6\\n{w} {h}\\n255\\n" + RGB triples."""
    rgb = np.ascontiguousarray(rgba.reshape(height, width, 4)[:, :, :3])
    with open(path, "wb") as f:
        f.write(f"P6\n{width} {height}\n255\n".encode())
        f.write(rgb.tobytes())


def read_image(path: str) -> np.ndarray:
    """An H x W x 4 uint8 RGBA array of a binary PPM (alpha 255) or, with Pillow, a PNG."""
    if path.lower().endswith(".png"):
        from PIL import Image
        return np.asarray(Image.open(path).convert("RGBA"), np.uint8).copy()
    with open(path, "rb") as f:
        data = f.read()
    fields, pos = [], 0
    while len(fields) < 4:  # magic, width, height, maxval; '#' comments between them
        while data[pos:pos + 1].isspace():
            pos += 1
        if data[pos:pos + 1] == b"#":
            pos = data.index(b"\n", pos)
            continue
        end = pos
        while not data[end:end + 1].isspace():
            end += 1
        fields.append(data[pos:end])
        pos = end
    if fields[0] != b"P6" or int(fields[3]) != 255:
        raise ValueError(f"{path}: not a binary 8-bit PPM")
    w, h = int(fields[1]), int(fields[2])
    rgb = np.frombuffer(data, np.uint8, 3 * w * h, pos + 1).reshape(h, w, 3)
    out = np.full((h, w, 4), 255, np.uint8)
    out[..., :3] = rgb
    return out


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="python -m forma_b200.render", description=__doc__.split("\n\n")[0])
    ap.add_argument("svg")
    ap.add_argument("out")
    ap.add_argument("--width", type=int, default=1000)   # App::width / height of the demo (svg.rs:860-868)
    ap.add_argument("--height", type=int, default=1000)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--frames", type=int, default=1, help="render this many times and report the last frame's timings")
    ap.add_argument("--ids", help="also write the ID frame (H x W uint32, Renderer.render_ids) to this .npy file")
    ap.add_argument("--linear", help="also write the linear float frame (H x W x 4 float32, Renderer.render_linear) to this .npy file")
    ap.add_argument("--over", help="draw over this image (.ppm or .png, Renderer.render_over_device) instead of a white frame; its size "
                                   "replaces --width / --height")
    ap.add_argument("--masks", help="also write the layer coverage masks (K x H x W, Renderer.render_masks) to this .npy file")
    ap.add_argument("--mask-orders", default="0:1", help="the masks' layer orders A:B, i.e. [A, B) (default 0:1)")
    ap.add_argument("--mask-u8", action="store_true", help="masks as uint8 (the alpha byte of sRGB8 frames) instead of float32")
    ap.add_argument("--stats", help="also write the layer statistics (Renderer.render_stats) to this .npz file")
    ap.add_argument("--stats-orders", help="the statistics' layer orders A:B, i.e. [A, B) (default: every order)")
    ap.add_argument("--stats-min-coverage", type=float, default=0.0,
                    help="the coverage a pixel's mask must exceed to count for pixels / box, as for ID frames (default 0)")
    args = ap.parse_args(argv)
    mask_lo, mask_hi = (int(v) for v in args.mask_orders.split(":"))
    if args.masks and mask_hi <= mask_lo:
        ap.error("--mask-orders A:B needs A < B")

    import forma_b200
    from forma_b200 import svg
    from forma_b200.binding import RGBA, Color

    image = None
    if args.over:
        image = read_image(args.over)
        args.height, args.width = image.shape[:2]
    t0 = time.perf_counter()
    paths = svg.parse_svg(args.svg)
    t1 = time.perf_counter()
    api = forma_b200.load()
    renderer = api.Renderer(args.device)  # raises without a usable GPU
    comp = api.Composition()
    svg.compose(api, comp, paths, scale=args.scale)
    buf = np.zeros(args.width * args.height * 4, np.uint8)
    t2 = time.perf_counter()
    if image is None:
        for _ in range(max(args.frames, 1)):
            t = renderer.render(comp, buf, args.width, args.height, RGBA, Color(1.0, 1.0, 1.0, 1.0))  # the demo clears to white
    else:
        import torch
        frame = torch.empty((args.height, args.width, 4), dtype=torch.uint8, device=f"cuda:{args.device}")
        src = torch.from_numpy(image).to(frame.device)
        for _ in range(max(args.frames, 1)):
            frame.copy_(src)
            torch.cuda.synchronize(frame.device)
            t = renderer.render_over_device(comp, frame.data_ptr(), args.width, args.height, RGBA)
        buf = frame.cpu().numpy().reshape(-1)
    t3 = time.perf_counter()
    if args.out.lower().endswith(".png"):
        from PIL import Image
        Image.fromarray(buf.reshape(args.height, args.width, 4), "RGBA").save(args.out)
    else:
        write_ppm(args.out, buf, args.width, args.height)
    if args.ids:
        ids = np.zeros(args.width * args.height, np.uint32)
        renderer.render_ids(comp, ids, args.width, args.height)
        np.save(args.ids, ids.reshape(args.height, args.width))
    if args.linear:
        linear = np.zeros((args.height, args.width, 4), np.float32)
        renderer.render_linear(comp, linear, args.width, args.height, RGBA, Color(1.0, 1.0, 1.0, 1.0), format="f32")
        np.save(args.linear, linear)
    if args.masks:
        masks = np.zeros((mask_hi - mask_lo, args.height, args.width), np.uint8 if args.mask_u8 else np.float32)
        renderer.render_masks(comp, masks, args.width, args.height, mask_lo)
        np.save(args.masks, masks)
    if args.stats:
        if args.stats_orders:
            stats_lo, stats_hi = (int(v) for v in args.stats_orders.split(":"))
        else:
            stats_lo, stats_hi, found = 0, 0, 0  # every order: up to the last of the composition's layers
            while found < len(comp):
                found += comp.get(stats_hi) is not None
                stats_hi += 1
            stats_hi = max(stats_hi, 1)
        if stats_hi <= stats_lo:
            ap.error("--stats-orders A:B needs A < B")
        rec = renderer.render_stats(comp, args.width, args.height, stats_lo, stats_hi - stats_lo, args.stats_min_coverage)
        np.savez(args.stats, first_order=stats_lo, **{name: rec[name] for name in rec.dtype.names})
    print(f"{len(paths)} paths parsed in {t1 - t0:.2f} s, composed in {t2 - t1:.2f} s; {t.n_segments} pixel segments; "
          f"last frame: line setup {t.line_setup_ms:.3f} ms, rasterize {t.rasterize_ms:.3f} ms, sort {t.sort_ms:.3f} ms, "
          f"paint {t.paint_ms:.3f} ms ({(t3 - t2) / max(args.frames, 1) * 1e3:.2f} ms per call) -> {args.out}", file=sys.stderr)
    return 0


if __name__ == "__main__":
    sys.exit(main())
