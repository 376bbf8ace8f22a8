"""Device time of layer coverage masks, in alternating runs timed with CUDA events, next to the plain
RGBA call of the same frame: per case the mask call alone and with the RGBA frame from the same pass,
in F32 and U8, with the zero-fill and mask kernels' times (torch.profiler, one extra profiled run) and
the bytes the mask planes take. Prints the card and its power limit from the same run, then one JSON
line per case:

- paris4k: the 3840 x 2160 paris scene (tests/workloads.py), a window of 64 orders;
- random_511x64: 511 distinct resident 64 x 64 synth.random_mixed compositions (24 layers each) as one
  batch, K = 24, against render_batch_device;
- diy16: the masks of 16 paris4k layers the way a caller gets them without this call: one linear
  render per layer with every other layer disabled and the layer solid white (device time of the 16
  renders, and the host time of the whole loop with its set_props / set_is_enabled calls).

    python tools/bench_masks.py [--steps 20] [--runs 3] [--cases paris4k,random_511x64,diy16]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]


def kernel_ms(fn, steps):
    """Mean device time per call of the zero-fill and mask kernels (torch.profiler)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    out = {"zero_fill": 0.0, "masks": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        us = e.cuda_time_total if us is None else us
        if "zero_masks_kernel" in e.key:
            out["zero_fill"] += us / 1e3 / steps
        elif "paint_masks" in e.key:
            out["masks"] += us / 1e3 / steps
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


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--cases", default="paris4k,random_511x64,diy16")
    args = ap.parse_args(argv)
    import torch

    import forma_b200
    import synth
    import workloads
    from bench_linear import card
    from forma_b200.binding import RGBA, BlendMode, Color, Fill, Func, Props, Style

    print(f"card: {card()}", flush=True)
    api = forma_b200.load()
    clear = Color(1.0, 1.0, 1.0, 1.0)
    for name in args.cases.split(","):
        r = api.Renderer(0)
        if name == "random_511x64":
            comps, w, h, k, first = [], 64, 64, 24, 0
            for i in range(511):
                comps.append(api.Composition())
                synth.random_mixed(api, comps[-1], 24, w, h, 1000 + i)
            n = len(comps)
        else:
            comp, w, h = workloads.build_scene(api, "paris4k")
            n, k, first = 1, 64, 20000
        line = {"case": name, "width": w, "height": h, "frames": n, "steps": args.steps}
        rgba = torch.empty((n, h, w, 4), dtype=torch.uint8, device="cuda:0")
        pr = rgba.data_ptr()
        if name == "diy16":
            lin = torch.empty((h, w, 4), dtype=torch.float32, device="cuda:0")
            orders = range(first, first + 16)
            saved = {o: comp.get(o).is_enabled() for o in range(len(comp)) if comp.get(o) is not None}
            for o in saved:
                comp.get(o).set_is_enabled(False)
            white = Props(func=Func.Draw(Style(fill=Fill.Solid(Color(1.0, 1.0, 1.0, 1.0)), blend_mode=BlendMode.Over)))

            def diy():
                for o in orders:
                    layer = comp.get(o)
                    layer.set_props(white).set_is_enabled(True)
                    r.render_linear_device(comp, lin.data_ptr(), w, h, RGBA, Color(0.0, 0.0, 0.0, 0.0), format="f32", timings=False)
                    layer.set_is_enabled(False)
            diy()
            t0 = time.perf_counter()
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for _ in range(max(args.steps // 4, 1)):
                diy()
            ev1.record()
            torch.cuda.synchronize()
            steps = max(args.steps // 4, 1)
            line["diy_16_layers"] = {"device_ms_per_16": round(ev0.elapsed_time(ev1) / steps, 3),
                                     "host_ms_per_16": round((time.perf_counter() - t0) * 1e3 / steps, 3)}
            print(json.dumps(line), flush=True)
            del r
            continue
        for fmt, dtype in (("f32", torch.float32), ("u8", torch.uint8)):
            planes = torch.empty((n, k, h, w), dtype=dtype, device="cuda:0")
            pm = planes.data_ptr()
            if n > 1:
                calls = {"plain": lambda: r.render_batch_device(comps, pr, w, h, RGBA, clear, timings=False),
                         "masks": lambda: r.render_batch_masks_device(comps, pm, w, h, first, k, fmt, timings=False),
                         "masks_rgba": lambda: r.render_batch_masks_device(comps, pm, w, h, first, k, fmt, rgba_ptr=pr,
                                                                           clear_color=clear, timings=False)}
            else:
                calls = {"plain": lambda: r.render_device(comp, pr, w, h, RGBA, clear, timings=False),
                         "masks": lambda: r.render_masks_device(comp, pm, w, h, first, k, fmt, timings=False),
                         "masks_rgba": lambda: r.render_masks_device(comp, pm, w, h, first, k, fmt, rgba_ptr=pr, clear_color=clear,
                                                                     timings=False)}
            line[fmt] = {"ms_per_call": timed(calls, args.steps, args.runs), "kernels_ms": kernel_ms(calls["masks"], args.steps),
                         "mask_bytes": n * k * w * h * planes.element_size(), "orders": [first, first + k]}
            del planes
        print(json.dumps(line), flush=True)
        del r
        torch.cuda.empty_cache()
    return 0


if __name__ == "__main__":
    sys.exit(main())
