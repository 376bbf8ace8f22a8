"""Device time of frames over a background next to their twins, in alternating runs timed with
CUDA events: per case and format the over call (render_over_device / render_batch_over_device)
and its twin with a clear colour (render_device / render_linear_device, render_batch_device /
render_batch_linear_device), each with the paint kernel's time (kernel_times()["paint"]) and the
bytes the over call's paint kernel reads in addition to its twin's (the frames' pixels x bytes per
pixel: the background). Prints the card and its power limit from the same run, then one JSON line
per case:

- paris4k: the 3840 x 2160 paris scene (tests/workloads.py);
- random_511x64: 511 distinct resident 64 x 64 synth.random_mixed compositions as one batch.

    python tools/bench_over.py [--steps 20] [--runs 3] [--cases paris4k,random_511x64] [--formats srgb8,f16,f32]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--cases", default="paris4k,random_511x64")
    ap.add_argument("--formats", default="srgb8,f16,f32")
    args = ap.parse_args(argv)
    import numpy as np
    import torch

    import forma_b200
    import synth
    import workloads
    from bench_linear import card
    from forma_b200.binding import RGBA, Color

    print(f"card: {card()}", flush=True)
    api = forma_b200.load()
    clear = Color(1.0, 1.0, 1.0, 1.0)
    dtypes = {"srgb8": (torch.uint8, 4), "f16": (torch.float16, 8), "f32": (torch.float32, 16)}
    for name in args.cases.split(","):
        r = api.Renderer(0)
        if name == "random_511x64":
            comps, w, h = [], 64, 64
            for k in range(511):
                comps.append(api.Composition())
                synth.random_mixed(api, comps[-1], 24, w, h, 1000 + k)
            n = len(comps)
        else:
            comp, w, h = workloads.build_scene(api, name)
            n = 1
        line = {"case": name, "width": w, "height": h, "frames": n, "steps": args.steps}
        for fmt in args.formats.split(","):
            dtype, bpp = dtypes[fmt]
            gen = torch.Generator(device="cuda:0").manual_seed(1)
            if fmt == "srgb8":
                bg = torch.randint(0, 256, (n * h * w * 4,), dtype=torch.uint8, device="cuda:0", generator=gen)
            else:
                bg = torch.rand(n * h * w * 4, device="cuda:0", generator=gen).to(dtype)
            over_buf, twin_buf = bg.clone(), torch.empty_like(bg)
            po, pt = over_buf.data_ptr(), twin_buf.data_ptr()
            if n > 1:
                over = lambda: r.render_batch_over_device(comps, po, w, h, RGBA, format=fmt, timings=False)
                twin = ((lambda: r.render_batch_device(comps, pt, w, h, RGBA, clear, timings=False)) if fmt == "srgb8" else
                        (lambda: r.render_batch_linear_device(comps, pt, w, h, RGBA, clear, format=fmt, timings=False)))
            else:
                over = lambda: r.render_over_device(comp, po, w, h, RGBA, format=fmt, timings=False)
                twin = ((lambda: r.render_device(comp, pt, w, h, RGBA, clear, timings=False)) if fmt == "srgb8" else
                        (lambda: r.render_linear_device(comp, pt, w, h, RGBA, clear, format=fmt, timings=False)))
            calls = {"over": over, "twin": twin}
            for f in calls.values():  # warm-up: uploads, buffers, sync-free bounds
                f(), f()
            res = {k: {"ms": [], "kernel_ms": []} for k in calls}
            for _ in range(args.runs):
                for k, f in calls.items():
                    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    kern = []
                    torch.cuda.synchronize()
                    ev0.record()
                    for _ in range(args.steps):
                        f()
                        kern.append(r.kernel_times()["paint"]["ms"])
                    ev1.record()
                    torch.cuda.synchronize()
                    res[k]["ms"].append(ev0.elapsed_time(ev1) / args.steps)
                    res[k]["kernel_ms"].append(float(np.median(kern)))
            line[fmt] = {k: {"ms_per_call": [round(v, 4) for v in d["ms"]], "paint_kernel_ms": [round(v, 4) for v in d["kernel_ms"]]}
                         for k, d in res.items()}
            line[fmt]["over_extra_read_bytes"] = n * w * h * bpp
            del over_buf, twin_buf, bg
        print(json.dumps(line), flush=True)
        del r
        torch.cuda.empty_cache()
    return 0


if __name__ == "__main__":
    sys.exit(main())
