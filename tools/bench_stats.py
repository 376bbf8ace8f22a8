"""Device time of layer statistics, in alternating runs timed with CUDA events, next to the plain RGBA
call of the same frame: per case the statistics call alone and with the RGBA frame from the same pass,
with the time of each statistics kernel (torch.profiler, one extra profiled run: the records'
initialisation, the amodal walk, the visible walk, the empty boxes' fix-up). Prints the card and its
power limit from the same run, then one JSON line per case:

- paris4k: the 3840 x 2160 paris scene (tests/workloads.py), every order, min_coverage 0;
- random_511x64: 511 distinct resident 64 x 64 synth.random_mixed compositions (24 layers each) as one
  batch, every order, against render_batch_device;
- background4k: one layer over the whole 3840 x 2160 frame, so that each of its 32 400 tiles adds into
  the same record: the statistics kernels against the ID kernel, which walks the same tiles without
  atomics (render_ids_device);
- masks64: the way a caller gets the same numbers without this call: one 64-order F32 mask call of
  paris4k plus its torch reduction (area, pixels, box), timed, and that time scaled to every order
  (a scaled estimate, not a measurement of all orders).

    python tools/bench_stats.py [--steps 20] [--runs 3] [--cases paris4k,random_511x64,background4k,masks64]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

KERNELS = ("init_stats_kernel", "stats_amodal", "stats_visible", "fix_stats_kernel", "paint_ids", "paint_kernel")


def kernel_ms(fn, steps):
    """Mean device time per call of each statistics kernel and of the paint / ID kernels (torch.profiler)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        us = e.cuda_time_total if us is None else us
        for k in KERNELS:
            if k in e.key:
                out[k] = out.get(k, 0.0) + us / 1e3 / steps
    return {k: round(v, 4) for k, v in out.items()}


def timed(calls, steps, runs):
    import torch
    for f in calls.values():  # warm-up: uploads, buffers, sync-free bounds
        f(), f()
    res = {k: [] for k in calls}
    for _ in range(runs):
        for k, f in calls.items():
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            ev0.record()
            for _ in range(steps):
                f()
            ev1.record()
            torch.cuda.synchronize()
            res[k].append(round(ev0.elapsed_time(ev1) / steps, 4))
    return res


def n_orders(comp):
    import batch_scenes
    return max(batch_scenes.n_orders(comp), 1)


def mask_reduction(planes, threshold):
    """area, pixels and box of [K, H, W] F32 planes in torch: what render_stats gives without its visible half."""
    import torch
    area = (planes.double() * 262144.0).sum(dim=(1, 2)).long()
    hit = planes > threshold
    pixels = hit.sum(dim=(1, 2))
    cols, rows = hit.any(dim=1), hit.any(dim=2)
    w, h = planes.shape[2], planes.shape[1]
    x0 = torch.argmax(cols.int(), dim=1)
    x1 = w - torch.argmax(cols.flip(1).int(), dim=1)
    y0 = torch.argmax(rows.int(), dim=1)
    y1 = h - torch.argmax(rows.flip(1).int(), dim=1)
    return area, pixels, torch.stack([x0, y0, x1, y1], 1) * (pixels > 0)[:, None]


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--cases", default="paris4k,random_511x64,background4k,masks64")
    args = ap.parse_args(argv)
    import torch

    import forma_b200
    import style_scenes as ss
    import synth
    import workloads
    from bench_linear import card
    from forma_b200.binding import RGBA, Color, Fill

    print(f"card: {card()}", flush=True)
    api = forma_b200.load()
    clear = Color(1.0, 1.0, 1.0, 1.0)
    for name in args.cases.split(","):
        r = api.Renderer(0)
        if name == "random_511x64":
            comps, w, h = [], 64, 64
            for i in range(511):
                comps.append(api.Composition())
                synth.random_mixed(api, comps[-1], 24, w, h, 1000 + i)
            n, k = len(comps), max(n_orders(c) for c in comps)
        elif name == "background4k":
            comp, w, h = api.Composition(), 3840, 2160
            ss.add(api, comp, ss.Built(), 0, [ss.rect(0, 0, w, h)], ss.draw(Fill.Solid(Color(0.2, 0.4, 0.6, 1.0))))
            n, k = 1, 1
        else:
            comp, w, h = workloads.build_scene(api, "paris4k")
            n, k = 1, n_orders(comp)
        line = {"case": name, "width": w, "height": h, "frames": n, "orders": k, "steps": args.steps}
        rgba = torch.empty((n, h, w, 4), dtype=torch.uint8, device="cuda:0")
        rec = torch.empty((n, k, 12), dtype=torch.int32, device="cuda:0")
        pr, ps = rgba.data_ptr(), rec.data_ptr()
        if name == "masks64":
            planes = torch.empty((64, h, w), dtype=torch.float32, device="cuda:0")
            pm = planes.data_ptr()

            def masks_and_reduction():
                r.render_masks_device(comp, pm, w, h, 0, 64, "f32", timings=False)
                return mask_reduction(planes, 0.0)
            calls = {"plain": lambda: r.render_device(comp, pr, w, h, RGBA, clear, timings=False),
                     "stats_all_orders": lambda: r.render_stats_device(comp, ps, w, h, 0, k, timings=False),
                     "masks64_and_reduction": masks_and_reduction}
            line["ms_per_call"] = timed(calls, args.steps, args.runs)
            per64 = min(line["ms_per_call"]["masks64_and_reduction"])
            line["masks_all_orders_ms_scaled_estimate"] = round(per64 * k / 64, 1)
            print(json.dumps(line), flush=True)
            del planes, r
            torch.cuda.empty_cache()
            continue
        if n > 1:
            calls = {"plain": lambda: r.render_batch_device(comps, pr, w, h, RGBA, clear, timings=False),
                     "stats": lambda: r.render_batch_stats_device(comps, ps, w, h, 0, k, timings=False),
                     "stats_rgba": lambda: r.render_batch_stats_device(comps, ps, w, h, 0, k, rgba_ptr=pr, clear_color=clear,
                                                                       timings=False)}
        else:
            calls = {"plain": lambda: r.render_device(comp, pr, w, h, RGBA, clear, timings=False),
                     "stats": lambda: r.render_stats_device(comp, ps, w, h, 0, k, timings=False),
                     "stats_rgba": lambda: r.render_stats_device(comp, ps, w, h, 0, k, rgba_ptr=pr, clear_color=clear, timings=False)}
        if name == "background4k":
            ids = torch.empty((h, w), dtype=torch.int32, device="cuda:0")
            calls["ids"] = lambda: r.render_ids_device(comp, ids.data_ptr(), w, h, timings=False)
            line["ids_kernels_ms"] = kernel_ms(calls["ids"], args.steps)
        line["ms_per_call"] = timed(calls, args.steps, args.runs)
        line["kernels_ms"] = kernel_ms(calls["stats"], args.steps)
        print(json.dumps(line), flush=True)
        del r
        torch.cuda.empty_cache()
    return 0


if __name__ == "__main__":
    sys.exit(main())
