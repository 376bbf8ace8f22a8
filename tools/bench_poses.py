"""Time per frame of Renderer.render_poses_device against the ways to render the same frames
without it, in alternating runs. Device time comes from CUDA events around each call sequence;
host wall time from the host clock around the same sequence, which ends in a synchronisation.
Building the pose records (and, for the other ways, setting layer state or building
compositions) is part of each call's cost. Prints the card and its power limit from the same run,
then one JSON line per case:

- spaceship_200: the 200 frames of tests/synth.py's spaceship animation at 1920 x 1080, in chunks
  of max_views(1080) = 30, against a loop of animate(f) + render_device;
- library_511x64: 511 frames of 64 x 64, each a random subset of a 64-shape library at random
  offsets, against render_batch_device of 511 compositions built anew and against a
  set_transform / set_is_enabled + render_device loop;
- paris_poses_16: 16 frames of 960 x 540 of paris, every one of its 50 620 layers with its own
  translation, against 16 x (50 620 set_transform + render_device). Also reports the bytes the
  pose records upload per call.

    python tools/bench_poses.py [--steps 3] [--runs 3] [--cases spaceship_200,library_511x64,paris_poses_16]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

SCENE = {"spaceship_200": "spaceship1080p", "library_511x64": "library_511x64", "paris_poses_16": "paris_poses"}


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
    ap.add_argument("--cases", default="spaceship_200,library_511x64,paris_poses_16")
    args = ap.parse_args(argv)
    import numpy as np
    import torch

    import forma_b200
    import pose_scenes as ps
    from forma_b200.binding import RGBA, Color

    print(f"card: {card()}", flush=True)
    api = forma_b200.load()
    clear = Color(1.0, 1.0, 1.0, 1.0)
    for name in args.cases.split(","):
        sc = ps.SCENES[SCENE[name]]
        w, h, n = sc.width, sc.height, sc.n
        comp, orders = sc.build(api)
        inside = ps.window_orders(sc, orders)
        handles = [comp.get(o)._h for o in inside]
        ks = [o - sc.first_order for o in inside]
        r = api.Renderer(0)
        out = torch.empty((n, h, w, 4), dtype=torch.uint8, device="cuda:0")

        def poses():
            r.render_poses_device(comp, ps.poses(forma_b200.binding, sc), out.data_ptr(), w, h, RGBA, clear, timings=False)

        # The loop sets each layer's state through the C ABI directly: the fastest way the binding allows.
        xf = None if sc.transforms is None else [[(C.c_float * 6)(*sc.transforms[b, k]) for k in ks] for b in range(n)]

        def loop():
            for b in range(n):
                for j, lh in enumerate(handles):
                    if xf is not None:
                        api.layer_set_transform(comp._h, lh, xf[b][j])
                    if sc.visible is not None:
                        api.layer_set_is_enabled(comp._h, lh, int(sc.visible[b, ks[j]]))
                r.render_device(comp, out[b].data_ptr(), w, h, RGBA, clear, timings=False)

        calls = {"render_poses_device": poses, "render_device_loop": loop}
        if name == "library_511x64":
            rb = api.Renderer(0)

            def batch():  # one composition per frame, built anew: the shapes of the frame at its offsets
                comps = []
                for b in range(n):
                    c, _ = sc.build(api)
                    for k in range(sc.n_orders):
                        layer = c.get(k)
                        layer.set_transform([float(x) for x in sc.transforms[b, k]])
                        layer.set_is_enabled(bool(sc.visible[b, k]))
                    comps.append(c)
                rb.render_batch_device(comps, out.data_ptr(), w, h, RGBA, clear, timings=False)
            calls["render_batch_device_built_anew"] = batch
        for f in calls.values():  # warm-up: uploads, buffers, sync-free bounds
            f(), f()
        loop()
        torch.cuda.synchronize()
        want = out.clone()
        poses()
        torch.cuda.synchronize()
        same = bool(torch.equal(out, want))  # the poses call equals the loop's frames
        h2d0 = r.counters()["h2d_bytes"]
        poses()
        upload = r.counters()["h2d_bytes"] - h2d0
        dev = {k: [] for k in calls}
        wall = {k: [] for k in calls}
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        for _ in range(args.runs):
            for k, f in calls.items():
                f()  # untimed: the loop leaves edited layer tables, which the next call of either kind re-uploads
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                ev[0].record()
                for _ in range(args.steps):
                    f()
                ev[1].record()
                torch.cuda.synchronize()
                wall[k].append((time.perf_counter() - t0) * 1e3 / args.steps / n)
                dev[k].append(ev[0].elapsed_time(ev[1]) / args.steps / n)
        line = {"case": name, "frames": n, "width": w, "height": h, "layers_posed": len(inside), "frames_equal": same,
                "pose_upload_bytes_per_call": int(upload),
                "device_ms_per_frame": {k: round(float(np.median(v)), 5) for k, v in dev.items()},
                "host_wall_ms_per_frame": {k: round(float(np.median(v)), 5) for k, v in wall.items()},
                "device_ms_per_frame_runs": {k: [round(x, 5) for x in v] for k, v in dev.items()}}
        line["speedup_vs"] = {k: round(line["host_wall_ms_per_frame"][k] / line["host_wall_ms_per_frame"]["render_poses_device"], 2)
                              for k in calls if k != "render_poses_device"}
        print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
