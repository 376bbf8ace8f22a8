"""A/B of the segment sort's tile counts from the kernels that write its keys (option sort_counts)
against an upsweep pass per digit: alternating fresh processes, one per (round, workload, value),
each rendering the workload with render_device, L2 flushed between steps as bench.py does. Prints
the card, its power limit and SM clock, then one JSON line per run with frames per second (CUDA
events around render_device, the bench's `value`), the mean stage times (stage_times) and the sort's
kernel times per frame (kernel_times), and per workload whether both values gave the same bytes.

    python tools/ab_sort_counts.py [--rounds 3] [--steps 20] [--warmup 3] [--workloads paris4k,cubics100k,circles8k_1m]
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return ""


def child(workload: str, value: int, steps: int, warmup: int) -> dict:
    import numpy as np
    import torch

    import forma_b200
    import workloads
    from forma_b200.binding import RGBA, Color

    api = forma_b200.load()
    api.set_option("sort_counts", value)
    comp, w, h = workloads.build_scene(api, workload)
    fb = torch.zeros(h * w * 4, dtype=torch.uint8, device="cuda:0")
    flush = torch.empty(384 << 20, dtype=torch.uint8, device="cuda:0")
    clear = Color(1.0, 1.0, 1.0, 0.0)
    r = api.Renderer(0)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(warmup):
        r.render_device(comp, fb.data_ptr(), w, h, RGBA, clear, timings=False)
    dev_ms = 0.0
    stages = np.zeros(8)
    kernels = {}
    for _ in range(steps):
        flush.zero_()
        torch.cuda.synchronize()
        ev[0].record()
        r.render_device(comp, fb.data_ptr(), w, h, RGBA, clear, timings=False)
        ev[1].record()
        torch.cuda.synchronize()
        dev_ms += ev[0].elapsed_time(ev[1])
        stages += np.array(list(r.stage_times().values()))
        for k, v in r.kernel_times().items():
            acc = kernels.setdefault(k, {"ms": 0.0, "launches": 0})
            acc["ms"] += v["ms"] / steps
            acc["launches"] = v["launches"]
    return {"workload": workload, "sort_counts": value, "value": steps / (dev_ms * 1e-3), "ms_per_step": dev_ms / steps,
            "stage_ms": dict(zip(r.STAGES, (stages / steps).round(4).tolist())),
            "kernel_ms": {k: {"ms": round(v["ms"], 4), "launches": v["launches"]} for k, v in kernels.items()},
            "source": r.sort_counts()["source"], "segments": r.counters()["segments"],
            "frame_sha1": hashlib.sha1(fb.cpu().numpy().tobytes()).hexdigest()}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workloads", default="paris4k,cubics100k,circles8k_1m")
    ap.add_argument("--values", default="0,1")
    ap.add_argument("--child", nargs=2, metavar=("WORKLOAD", "VALUE"), help=argparse.SUPPRESS)
    args = ap.parse_args(argv)
    if args.child:
        print(json.dumps(child(args.child[0], int(args.child[1]), args.steps, args.warmup)), flush=True)
        return 0
    print(f"card (name, power limit, SM clock, max SM clock): {card()}", flush=True)
    values = [int(v) for v in args.values.split(",")]
    frames = {}
    for rnd in range(args.rounds):
        for wl in args.workloads.split(","):
            for v in values:
                out = subprocess.run([sys.executable, os.path.abspath(__file__), "--steps", str(args.steps), "--warmup",
                                      str(args.warmup), "--child", wl, str(v)], capture_output=True, text=True)
                if out.returncode != 0:
                    print(out.stdout + out.stderr, file=sys.stderr)
                    return out.returncode
                res = json.loads(out.stdout.strip().splitlines()[-1])
                res["round"] = rnd
                frames.setdefault(wl, set()).add(res.pop("frame_sha1"))
                print(json.dumps(res), flush=True)
    for wl, shas in frames.items():
        print(json.dumps({"workload": wl, "frames_equal_across_values": len(shas) == 1}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
