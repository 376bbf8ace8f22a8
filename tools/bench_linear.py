"""Device time of linear float frames next to sRGB8 frames, in alternating runs timed with CUDA
events: per case the sRGB8 call and its RGBA16F / RGBA32F twin, each with the paint kernel's time
(kernel_times()["paint"], summed over the call's paint launches) and the bytes that kernel
writes (the frame's pixels x bytes per pixel). Prints the card and its power limit from the same
run, then one JSON line per case:

- paris4k: the 3840 x 2160 paris scene (tests/workloads.py), render_device vs render_linear_device;
- random_511x64: 511 distinct resident 64 x 64 synth.random_mixed compositions as one batch,
  render_batch_device vs render_batch_linear_device.

    python tools/bench_linear.py [--steps 20] [--runs 3] [--cases paris4k,random_511x64]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    import torch
    return out or torch.cuda.get_device_name(0)


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--cases", default="paris4k,random_511x64")
    args = ap.parse_args(argv)
    import numpy as np
    import torch

    import forma_b200
    import synth
    import workloads
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
        outs = {k: torch.empty(n * h * w * 4, dtype=t, device="cuda:0") for k, (t, _) in dtypes.items()}  # [n, h, w, 4]

        def call(kind):
            p = outs[kind].data_ptr()
            if n > 1:
                if kind == "srgb8":
                    return lambda: r.render_batch_device(comps, p, w, h, RGBA, clear, timings=False)
                return lambda: r.render_batch_linear_device(comps, p, w, h, RGBA, clear, format=kind, timings=False)
            if kind == "srgb8":
                return lambda: r.render_device(comp, p, w, h, RGBA, clear, timings=False)
            return lambda: r.render_linear_device(comp, p, w, h, RGBA, clear, format=kind, timings=False)

        calls = {k: call(k) for k in dtypes}
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
        line = {"case": name, "width": w, "height": h, "frames": n, "steps": args.steps}
        for k, d in res.items():
            nbytes = n * w * h * dtypes[k][1]
            kms = float(np.median(d["kernel_ms"]))
            line[k] = {"ms_per_call": [round(v, 4) for v in d["ms"]], "paint_kernel_ms": [round(v, 4) for v in d["kernel_ms"]],
                       "frame_bytes": nbytes, "paint_store_GBps": round(nbytes / kms / 1e6, 1) if kms > 0 else None}
        print(json.dumps(line), flush=True)
        del r, outs
        torch.cuda.empty_cache()
    return 0


if __name__ == "__main__":
    sys.exit(main())
