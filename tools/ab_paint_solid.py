"""A/B of the paint kernel's lean build for solid `Over` frames (option paint_solid) against the
general build, in one process: every round renders each workload with each value of the option in
turn, L2 flushed between steps as bench.py does. Prints the card and its power limit, then one JSON
line per (round, workload, value) with frames per second of render_device (CUDA events, the
bench's `value`) and the paint kernel's ms per launch (kernel_times), and per workload whether every
value gave the same bytes.

    python tools/ab_paint_solid.py [--rounds 3] [--steps 20] [--warmup 3] [--workloads paris4k,cubics100k] [--values 0,1]
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
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workloads", default="paris4k,cubics100k")
    ap.add_argument("--values", default="0,1")
    args = ap.parse_args(argv)
    import torch

    import forma_b200
    import workloads
    from forma_b200.binding import RGBA, Color

    name = card()
    print(f"card: {name}", flush=True)
    api = forma_b200.load()
    values = [int(v) for v in args.values.split(",")]
    saved = api.get_option("paint_solid")
    clear = Color(1.0, 1.0, 1.0, 0.0)
    flush = torch.empty(384 << 20, dtype=torch.uint8, device="cuda:0")
    scenes = {}
    for wl in args.workloads.split(","):
        comp, w, h = workloads.build_scene(api, wl)
        scenes[wl] = (comp, w, h, torch.zeros(h * w * 4, dtype=torch.uint8, device="cuda:0"), {})
    r = api.Renderer(0)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    try:
        for rnd in range(args.rounds):
            for wl, (comp, w, h, fb, frames) in scenes.items():
                for v in values:
                    api.set_option("paint_solid", v)
                    for _ in range(args.warmup):
                        r.render_device(comp, fb.data_ptr(), w, h, RGBA, clear, timings=False)
                    dev_ms = paint_ms = 0.0
                    for _ in range(args.steps):
                        flush.zero_()
                        torch.cuda.synchronize()
                        ev[0].record()
                        r.render_device(comp, fb.data_ptr(), w, h, RGBA, clear, timings=False)
                        ev[1].record()
                        torch.cuda.synchronize()
                        dev_ms += ev[0].elapsed_time(ev[1])
                        k = r.kernel_times()["paint"]
                        paint_ms += k["ms"] / max(k["launches"], 1)
                    frame = fb.cpu()
                    same = bool(torch.equal(frame, frames.setdefault(v, frame)))
                    print(json.dumps({"round": rnd, "workload": wl, "paint_solid": v, "value": args.steps / (dev_ms * 1e-3),
                                      "ms_per_step": dev_ms / args.steps, "paint_ms_per_launch": paint_ms / args.steps,
                                      "frame_same_as_round_0": same, "card": name}), flush=True)
        for wl, (*_, frames) in scenes.items():
            ref = frames[values[0]]
            print(json.dumps({"workload": wl, "frames_equal_across_values": all(torch.equal(ref, f) for f in frames.values())}),
                  flush=True)
    finally:
        api.set_option("paint_solid", saved)
    return 0


if __name__ == "__main__":
    sys.exit(main())
