"""Where a paris@4K `render_device` step spends its time outside the frame's device time, with the
segment count read back mid-frame (option sync_free_sort 0) and without it (1), alternating in
one process.

Timed leg (no profiler): steps as bench.py times them - the L2 flushed between steps, CUDA events
on the render stream around the call, and a host clock closed by a synchronisation. Per setting:
wall ms per step, the a -> b event ms and the renderer's stage_ms.total.

Profiled leg (separate, torch.profiler with CUDA activities): the idle device time between the
frame's first and last stage event (tools/frame_gaps.py's trace parsing) and the host time spent in
cudaEventSynchronize and cudaStreamSynchronize per step.

Prints the card, its power limit and its SM clock from the same run.

    python tools/host_share.py [--workload paris4k] [--steps 200] [--rounds 3] [--frames 6]
"""
from __future__ import annotations

import argparse
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

import frame_gaps  # noqa: E402


def host_sync_us(trace_path, label):
    """Host microseconds in cudaEventSynchronize / cudaStreamSynchronize inside each range `label`."""
    import json
    with open(trace_path) as f:
        evs = json.load(f)["traceEvents"]
    frames = [e for e in evs if e.get("name") == label and e.get("ph") == "X" and e.get("cat") == "user_annotation"]
    out = []
    for fr in frames:
        t0, t1, tid = fr["ts"], fr["ts"] + fr["dur"], fr["tid"]
        acc = {"cudaEventSynchronize": 0.0, "cudaStreamSynchronize": 0.0}
        for e in evs:
            if e.get("cat") == "cuda_runtime" and e.get("ph") == "X" and e.get("tid") == tid and t0 <= e["ts"] <= t1 \
                    and e.get("name") in acc:
                acc[e["name"]] += e["dur"]
        out.append(acc)
    return out


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="paris4k")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=6, help="profiled steps per setting")
    args = ap.parse_args(argv)
    import torch
    from torch.profiler import ProfilerActivity, profile, record_function

    import forma_b200
    from forma_b200.binding import RGBA, Color
    from workloads import build_scene

    print(f"card (name, power limit, max SM clock): {frame_gaps.card()}", flush=True)
    api = forma_b200.load()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    clear = Color(1.0, 1.0, 1.0, 0.0)
    legs = {}
    for mode in (0, 1):  # a renderer and a composition per setting
        comp, w, h = build_scene(api, args.workload)
        r = api.Renderer(0)
        r.set_stream(stream.cuda_stream)
        fb = torch.zeros((h, w * 4), dtype=torch.uint8, device=dev)
        legs[mode] = (comp, w, h, r, fb)

    def step(mode):
        comp, w, h, r, fb = legs[mode]
        api.set_option("sync_free_sort", mode)
        r.render_device(comp, fb.data_ptr(), w, h, RGBA, clear, None, None, w * 4, timings=False)

    for mode in (0, 1):
        for _ in range(5):
            step(mode)
    torch.cuda.synchronize()
    res = {0: {"wall": [], "event": [], "total": []}, 1: {"wall": [], "event": [], "total": []}}
    for _ in range(args.rounds):
        for mode in (0, 1):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            wall = ev = tot = 0.0
            for _ in range(args.steps):
                with torch.cuda.stream(stream):
                    flush.zero_()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                a.record(stream)
                step(mode)
                b.record(stream)
                torch.cuda.synchronize()
                wall += time.perf_counter() - t0
                ev += a.elapsed_time(b)
                tot += legs[mode][3].stage_times()["total"]
            res[mode]["wall"].append(wall * 1e3 / args.steps)
            res[mode]["event"].append(ev / args.steps)
            res[mode]["total"].append(tot / args.steps)
    print(f"sync modes after the timed leg: {[legs[m][3].sort_mode() for m in (0, 1)]}")
    for mode in (0, 1):
        d = res[mode]
        print(f"sync_free_sort {mode}: wall ms/step " + ", ".join(f"{v:.4f}" for v in d["wall"]) +
              " | event ms/step " + ", ".join(f"{v:.4f}" for v in d["event"]) +
              " | stage_ms.total " + ", ".join(f"{v:.4f}" for v in d["total"]), flush=True)
    for mode in (0, 1):
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, "trace.json")
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                for _ in range(args.frames):
                    with torch.cuda.stream(stream):
                        flush.zero_()
                    torch.cuda.synchronize()
                    with record_function("forma_step"):
                        step(mode)
                    torch.cuda.synchronize()
            prof.export_chrome_trace(path)
            ops = frame_gaps.frame_ops(path, "forma_step")
            syncs = host_sync_us(path, "forma_step")
        import contextlib
        import io
        with contextlib.redirect_stdout(io.StringIO()):
            idle, boundaries = frame_gaps.report(ops)
        big = sorted(boundaries, reverse=True)[:3]
        ev_sync = sum(s["cudaEventSynchronize"] for s in syncs) / len(syncs)
        st_sync = sum(s["cudaStreamSynchronize"] for s in syncs) / len(syncs)
        print(f"sync_free_sort {mode} (profiled, last step): idle inside the frame {idle:.1f} us over {len(boundaries)} boundaries, "
              f"largest " + ", ".join(f"{g:.1f} us before {n}" for g, n in big) +
              f" | host us/step in cudaEventSynchronize {ev_sync:.1f}, cudaStreamSynchronize {st_sync:.1f}", flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
