"""Time per frame of Renderer.render_instances_device against the ways to render the same frames
without it, in alternating runs. Device time comes from CUDA events around each call sequence;
host wall time from the host clock around the same sequence, which ends in a synchronisation.
Building the instance records (and, for the other ways, building compositions) is part of each
call's cost. Prints the card and its power limit from the same run, then one JSON line per case:

- library_511x64: tests/instance_scenes.py's 511 frames of 64 x 64, 8 slots each from a 64-shape
  library with per-instance transforms and colours, against render_batch_device of the 511
  compositions T_b built anew every step (today's way to get a fresh instance list per frame) and
  of the same compositions built once;
- glyphs_1080p: one 1920 x 1080 frame of 20 000 glyph-sized instances of 90 prototypes, against
  render_device of one composition holding the 20 000 layers. Also reports the resident points of
  the library and of that composition.

Every case reports the bytes each call sends to the device (h2d_bytes) and whether the arms give
the same frames.

    python tools/bench_instances.py [--steps 3] [--runs 3] [--cases library_511x64,glyphs_1080p]
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
    ap.add_argument("--cases", default="library_511x64,glyphs_1080p")
    args = ap.parse_args(argv)
    import numpy as np
    import torch

    import forma_b200
    import instance_scenes as ins
    from forma_b200.binding import RGBA, Color

    print(f"card: {card()}", flush=True)
    api = forma_b200.load()
    clear = Color(1.0, 1.0, 1.0, 1.0)
    for name in args.cases.split(","):
        sc = ins.SCENES[name]
        w, h, n = sc.width, sc.height, sc.n
        lib = ins.build_library(api, sc)
        inst = ins.instances(forma_b200.binding, sc)
        r = api.Renderer(0)
        out = torch.empty((n, h, w, 4), dtype=torch.uint8, device="cuda:0")
        want = torch.empty_like(out)

        def instances():
            r.render_instances_device(lib, inst, out.data_ptr(), w, h, RGBA, clear, timings=False)

        calls = {"render_instances_device": instances}
        rb = api.Renderer(0)
        if n > 1:
            built = [ins.twin(api, sc, b) for b in range(n)]

            def anew():
                rb.render_batch_device([ins.twin(api, sc, b) for b in range(n)], out.data_ptr(), w, h, RGBA, clear, timings=False)

            def prebuilt():
                rb.render_batch_device(built, out.data_ptr(), w, h, RGBA, clear, timings=False)
            calls["render_batch_device_built_anew"] = anew
            calls["render_batch_device_prebuilt"] = prebuilt
            reference = prebuilt
            points = {"library": lib.point_count(), "compositions_prebuilt": sum(c.point_count() for c in built)}
        else:
            page = ins.twin(api, sc, 0)

            def single():
                rb.render_device(page, out.data_ptr(), w, h, RGBA, clear, timings=False)
            calls["render_device_one_composition"] = single
            reference = single
            points = {"library": lib.point_count(), "one_composition": page.point_count()}
        for f in calls.values():  # warm-up: uploads, buffers, sync-free bounds
            f(), f()
        reference()
        torch.cuda.synchronize()
        want.copy_(out)
        instances()
        torch.cuda.synchronize()
        same = bool(torch.equal(out, want))
        upload = {}
        for k, f in calls.items():
            rr = r if k == "render_instances_device" else rb
            h0 = rr.counters()["h2d_bytes"]
            f()
            torch.cuda.synchronize()
            upload[k] = rr.counters()["h2d_bytes"] - h0
        dev = {k: [] for k in calls}
        wall = {k: [] for k in calls}
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        for _ in range(args.runs):
            for k, f in calls.items():
                f()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                ev[0].record()
                for _ in range(args.steps):
                    f()
                ev[1].record()
                torch.cuda.synchronize()
                wall[k].append((time.perf_counter() - t0) * 1e3 / args.steps / n)
                dev[k].append(ev[0].elapsed_time(ev[1]) / args.steps / n)
        line = {"case": name, "frames": n, "width": w, "height": h, "slots": sc.m, "prototypes": len(sc.protos), "frames_equal": same,
                "resident_points": points, "h2d_bytes_per_call": upload,
                "device_ms_per_frame": {k: round(float(np.median(v)), 5) for k, v in dev.items()},
                "host_wall_ms_per_frame": {k: round(float(np.median(v)), 5) for k, v in wall.items()},
                "device_ms_per_frame_runs": {k: [round(x, 5) for x in v] for k, v in dev.items()},
                "host_wall_ms_per_frame_runs": {k: [round(x, 5) for x in v] for k, v in wall.items()}}
        line["speedup_vs"] = {k: round(line["host_wall_ms_per_frame"][k] / line["host_wall_ms_per_frame"]["render_instances_device"], 2)
                              for k in calls if k != "render_instances_device"}
        print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
