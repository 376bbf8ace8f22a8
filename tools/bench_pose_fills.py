"""Time per frame of pose fills (Renderer.render_poses_device with Poses(colors=...)) against the
ways to render the same frames without them, in alternating runs. Device time comes from CUDA
events around each call sequence; host wall time from the host clock around the same sequence,
which ends in a synchronisation. Building the pose records and uploading the colours (and, for
the loops, setting layer props and transforms) is part of each call's cost. Prints the card and
its power limit from the same run, then one JSON line per case:

- spaceship_200: the 200 frames of the spaceship animation at 1920 x 1080 (tests/pose_scenes.py)
  with a colour per ship and frame, against the same poses call without colours (the cost of the
  fills) and against a set_props + set_transform + render_device loop;
- library_511x64: the 511 shape-library frames with random colours, against a set_props +
  set_transform + set_is_enabled + render_device loop;
- paris_fills_16: 16 frames of 960 x 540 of paris with all 50 620 layers translated and recoloured,
  against the same call without colours. Reports the upload stage of both calls (the pose style
  table is built there), the colour bytes uploaded per call and the bytes of the table's pose
  records (112 per frame and layer, besides one record per style of the composition).

    python tools/bench_pose_fills.py [--steps 3] [--runs 3] [--cases spaceship_200,library_511x64,paris_fills_16]
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
    import pose_scenes as ps
    from forma_b200.binding import RGBA, Color, Poses, _lower_props

    print(f"card: {card()}", flush=True)
    api = forma_b200.load()
    clear = Color(1.0, 1.0, 1.0, 1.0)
    for name in args.cases.split(","):
        sc = pfs.SCENES[SCENE[name]]
        w, h, n = sc.width, sc.height, sc.n
        comp, orders = sc.build(api)
        inside = ps.window_orders(sc, orders)
        props = pfs.props_of(comp)
        r = api.Renderer(0)
        out = torch.empty((n, h, w, 4), dtype=torch.uint8, device="cuda:0")
        with_colors, without = pfs.poses(sc), Poses(sc.first_order, sc.transforms, sc.visible)

        def fills():
            r.render_poses_device(comp, with_colors, out.data_ptr(), w, h, RGBA, clear, timings=False)

        def no_fills():
            r.render_poses_device(comp, without, out.data_ptr(), w, h, RGBA, clear, timings=False)

        calls = {"render_poses_device_colors": fills, "render_poses_device_no_colors": no_fills}
        if name != "paris_fills_16":
            # The loop sets each layer's state through the C ABI directly, from props lowered ahead
            # of time: the fastest way the binding allows.
            handles = [comp.get(o)._h for o in inside]
            ks = [o - sc.first_order for o in inside]
            low = [[_lower_props(pfs.filled(props[o], sc.colors[b, o - sc.first_order])) for o in inside] for b in range(n)]
            xf = None if sc.transforms is None else [[(C.c_float * 6)(*sc.transforms[b, k]) for k in ks] for b in range(n)]

            def loop():
                for b in range(n):
                    for j, lh in enumerate(handles):
                        api.layer_set_props(comp._h, lh, C.byref(low[b][j][0]))
                        if xf is not None:
                            api.layer_set_transform(comp._h, lh, xf[b][j])
                        if sc.visible is not None:
                            api.layer_set_is_enabled(comp._h, lh, int(sc.visible[b, ks[j]]))
                    r.render_device(comp, out[b].data_ptr(), w, h, RGBA, clear, timings=False)
            calls["set_props_render_device_loop"] = loop
        for f in calls.values():  # warm-up: uploads, buffers, sync-free bounds
            f(), f()
        same = None
        if "set_props_render_device_loop" in calls:
            calls["set_props_render_device_loop"]()
            torch.cuda.synchronize()
            want = out.clone()
            fills()
            torch.cuda.synchronize()
            same = bool(torch.equal(out, want))  # the poses call equals the loop's frames
        fills()
        h2d0 = r.counters()["h2d_bytes"]
        fills()
        upload_colors = r.counters()["h2d_bytes"] - h2d0
        upload_stage = {}
        for k, f in (("colors", fills), ("no_colors", no_fills)):
            f()
            torch.cuda.synchronize()
            upload_stage[k] = round(r.stage_times()["upload"], 4)  # the last chunk's upload stage
        no_fills()
        h2d0 = r.counters()["h2d_bytes"]
        no_fills()
        upload_plain = r.counters()["h2d_bytes"] - h2d0
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
        chunk = min(n, r.max_views(h))
        line = {"case": name, "frames": n, "width": w, "height": h, "layers_recoloured": len(inside), "frames_equal_loop": same,
                "colour_upload_bytes_per_call": int(upload_colors - upload_plain),
                "pose_style_records_bytes_per_chunk": 112 * chunk * sc.n_orders,
                "upload_stage_ms_last_chunk": upload_stage,
                "device_ms_per_frame": {k: round(float(np.median(v)), 5) for k, v in dev.items()},
                "host_wall_ms_per_frame": {k: round(float(np.median(v)), 5) for k, v in wall.items()},
                "device_ms_per_frame_runs": {k: [round(x, 5) for x in v] for k, v in dev.items()}}
        base = line["host_wall_ms_per_frame"]["render_poses_device_colors"]
        line["host_wall_ratio_vs_colors"] = {k: round(v / base, 2) for k, v in line["host_wall_ms_per_frame"].items()
                                             if k != "render_poses_device_colors"}
        print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
