"""Device time of ID frames next to RGBA frames: render_device, render_ids_device and
render_device_with_ids on paris4k, cubics100k and circles8k_1m (tests/workloads.py), in
alternating runs, timed with CUDA events; the paint / ID kernel stage (stage_times()
"paint_kernel") of every call as well. Prints the card and its power limit from the same run,
then one JSON line per workload.

    python tools/bench_ids.py [--steps 20] [--runs 3] [--workloads paris4k,cubics100k,circles8k_1m]
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
    ap.add_argument("--workloads", default="paris4k,cubics100k,circles8k_1m")
    args = ap.parse_args(argv)
    import numpy as np
    import torch

    import forma_b200
    import workloads
    from forma_b200.binding import RGBA, Color

    print(f"card: {card()}", flush=True)
    api = forma_b200.load()
    clear = Color(1.0, 1.0, 1.0, 1.0)
    for name in args.workloads.split(","):
        comp, w, h = workloads.build_scene(api, name)
        r = api.Renderer(0)
        rgba = torch.empty(w * h * 4, dtype=torch.uint8, device="cuda:0")
        ids = torch.empty(w * h, dtype=torch.int32, device="cuda:0")
        calls = {
            "render_device": lambda: r.render_device(comp, rgba.data_ptr(), w, h, RGBA, clear, timings=False),
            "render_ids_device": lambda: r.render_ids_device(comp, ids.data_ptr(), w, h, timings=False),
            "render_device_with_ids": lambda: r.render_device_with_ids(comp, rgba.data_ptr(), ids.data_ptr(), w, h, RGBA, clear,
                                                                       timings=False),
        }
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
                    kern.append(r.stage_times()["paint_kernel"])
                ev1.record()
                torch.cuda.synchronize()
                res[k]["ms"].append(ev0.elapsed_time(ev1) / args.steps)
                res[k]["kernel_ms"].append(float(np.median(kern)))
        print(json.dumps({"workload": name, "width": w, "height": h, "steps": args.steps,
                          **{k: {"ms_per_frame": [round(v, 4) for v in d["ms"]],
                                 "paint_or_id_kernel_ms": [round(v, 4) for v in d["kernel_ms"]]} for k, d in res.items()}}),
              flush=True)
        del comp, r, rgba, ids
        torch.cuda.empty_cache()
    return 0


if __name__ == "__main__":
    sys.exit(main())
