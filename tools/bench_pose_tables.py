"""Time per frame of poses calls whose tables are CUDA tensors (Poses with torch CUDA tensors),
against the same tables in host memory and against the way a PyTorch pipeline gets there without
them: tables made on the GPU, `.cpu()`, then the host-table call. Alternating runs; device time
from CUDA events around each call sequence, host wall time from the host clock around the same
sequence, which ends in a synchronisation. Prints the card and its power limit from the same run,
then one JSON line per case with, for each way, host wall and device ms per frame, the upload
stage of the last chunk (stage_times()["upload"]: window records, table copies, fold, pose style
table) and the bytes sent host-to-device per call. The frames of the three ways are compared.

Cases (tests/pose_fill_scenes.py, as tools/bench_pose_fills.py): spaceship_200 (200 frames at
1920 x 1080, transforms and colours), library_511x64 (511 frames, transforms, visibility and
colours), paris_fills_16 (16 frames of 960 x 540, all 50 620 layers translated and recoloured).

    python tools/bench_pose_tables.py [--steps 3] [--runs 3] [--cases spaceship_200,library_511x64,paris_fills_16]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

SCENE = {"spaceship_200": "spaceship_filled", "library_511x64": "library_filled", "paris_fills_16": "paris_filled"}


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
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--cases", default="spaceship_200,library_511x64,paris_fills_16")
    args = ap.parse_args(argv)
    import numpy as np
    import torch

    import forma_b200
    import pose_fill_scenes as pfs
    from forma_b200.binding import RGBA, Color, Poses

    print(f"card: {card()}", flush=True)
    api = forma_b200.load()
    clear = Color(1.0, 1.0, 1.0, 1.0)
    for name in args.cases.split(","):
        sc = pfs.SCENES[SCENE[name]]
        w, h, n = sc.width, sc.height, sc.n
        comp, _ = sc.build(api)
        r = api.Renderer(0)
        out = torch.empty((n, h, w, 4), dtype=torch.uint8, device="cuda:0")
        host_tables = (sc.transforms, sc.visible, sc.colors)
        cuda_tables = tuple(None if t is None else torch.from_numpy(np.ascontiguousarray(t)).to("cuda:0") for t in host_tables)
        host_poses, cuda_poses = Poses(sc.first_order, *host_tables), Poses(sc.first_order, *cuda_tables)

        def host():
            r.render_poses_device(comp, host_poses, out.data_ptr(), w, h, RGBA, clear, timings=False)

        def cuda():
            r.render_poses_device(comp, cuda_poses, out.data_ptr(), w, h, RGBA, clear, timings=False)

        def via_cpu():  # what a caller with CUDA tables does without device tables
            tables = [None if t is None else t.cpu().numpy() for t in cuda_tables]
            r.render_poses_device(comp, Poses(sc.first_order, *tables), out.data_ptr(), w, h, RGBA, clear, timings=False)

        calls = {"host_tables": host, "cuda_tables": cuda, "cuda_tables_via_cpu": via_cpu}
        frames = {}
        for k, f in calls.items():  # warm-up: uploads, buffers, sync-free bounds
            f(), f()
            torch.cuda.synchronize()
            frames[k] = out.clone()
        same = all(bool(torch.equal(frames[k], frames["host_tables"])) for k in calls)
        h2d, upload = {}, {}
        for k, f in calls.items():
            before = r.counters()["h2d_bytes"]
            f()
            torch.cuda.synchronize()
            h2d[k] = int(r.counters()["h2d_bytes"] - before)
            upload[k] = round(r.stage_times()["upload"], 4)
        dev = {k: [] for k in calls}
        wall = {k: [] for k in calls}
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        for _ in range(args.runs):
            for k, f in calls.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                ev[0].record()
                for _ in range(args.steps):
                    f()
                ev[1].record()
                torch.cuda.synchronize()
                wall[k].append((time.perf_counter() - t0) * 1e3 / args.steps / n)
                dev[k].append(ev[0].elapsed_time(ev[1]) / args.steps / n)
        line = {"case": name, "frames": n, "width": w, "height": h, "n_orders": sc.n_orders, "frames_equal": same,
                "tables": [k for k, t in zip(("transforms", "visible", "colors"), host_tables) if t is not None],
                "h2d_bytes_per_call": h2d, "upload_stage_ms_last_chunk": upload,
                "host_wall_ms_per_frame": {k: round(float(np.median(v)), 5) for k, v in wall.items()},
                "device_ms_per_frame": {k: round(float(np.median(v)), 5) for k, v in dev.items()},
                "host_wall_ms_per_frame_runs": {k: [round(x, 5) for x in v] for k, v in wall.items()}}
        print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
