"""Device time per view of Renderer.render_views_device against a loop of render_device calls
with the layer transforms set per frame (the way to render many views without it), in
alternating runs timed with CUDA events. Prints the card and its power limit from the same run,
then one JSON line per case:

- e2e_1024x64: 1024 views of 64 x 64 of the radial_gradient e2e scene (rotations, shears, zoom-outs);
- paris_64x512: 64 views of 512 x 512 of paris, rotated and zoomed out;
- paris_tiles_16: the 16 translated 960 x 540 tiles of tests/view_scenes.py.

    python tools/bench_views.py [--steps 5] [--runs 3] [--cases e2e_1024x64,paris_64x512,paris_tiles_16]

The loop's time includes setting every layer's transform per frame (50 620 layers for paris):
that host work is part of what the loop costs its caller.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
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


def cases():
    import view_scenes as vs
    e2e = vs.e2e_views(64)[:7]
    paris = []
    for k in range(64):
        a, s = 2.0 * math.pi * k / 64.0, 0.25 + 0.25 * (k % 3)  # rotated, zoomed out to 1/4 ... 3/4
        c, n = s * math.cos(a), s * math.sin(a)
        cx, cy = 300.0 + 20.0 * (k % 8) * 8, 200.0 + 80.0 * (k // 8)
        paris.append([c, -n, n, c, 256.0 - (c * cx - n * cy), 256.0 - (n * cx + c * cy)])
    return {
        "e2e_1024x64": (vs._e2e("radial_gradient"), 64, 64, [e2e[k % len(e2e)] for k in range(1024)]),
        "paris_64x512": (vs._paris, 512, 512, paris),
        "paris_tiles_16": (vs._paris, 960, 540, vs.SCENES["paris_tiles"].views),
    }


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--cases", default="e2e_1024x64,paris_64x512,paris_tiles_16")
    args = ap.parse_args(argv)
    import numpy as np
    import torch

    import forma_b200
    import view_scenes as vs
    from forma_b200.binding import RGBA, Color

    print(f"card: {card()}", flush=True)
    api = forma_b200.load()
    clear = Color(1.0, 1.0, 1.0, 1.0)
    table = cases()
    for name in args.cases.split(","):
        build, w, h, views = table[name]
        comp = api.Composition()
        xf = build(api, comp)
        r = api.Renderer(0)
        n = len(views)
        out = torch.empty((n, h, w, 4), dtype=torch.uint8, device="cuda:0")

        def batch():
            r.render_views_device(comp, views, out.data_ptr(), w, h, RGBA, clear, timings=False)

        # The loop sets every layer's transform through the C ABI directly (no layer of these
        # scenes has a transform of its own, so C = V): the fastest way the binding allows.
        handles = [comp.get(o)._h for o in xf]
        arrays = [(C.c_float * 6)(*vs.compose(v, None)) for v in views]
        ident = (C.c_float * 6)(*vs.IDENTITY)

        def loop():
            for b in range(n):
                for lh in handles:
                    api.layer_set_transform(comp._h, lh, arrays[b])
                r.render_device(comp, out[b].data_ptr(), w, h, RGBA, clear, timings=False)
            for lh in handles:
                api.layer_set_transform(comp._h, lh, ident)

        calls = {"render_views_device": batch, "render_device_loop": loop}
        for f in calls.values():  # warm-up: uploads, buffers, sync-free bounds
            f(), f()
        want = out.clone()
        batch()
        torch.cuda.synchronize()
        same = bool(torch.equal(out, want))  # the batch equals the loop's frames
        res = {k: [] for k in calls}
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        for _ in range(args.runs):
            for k, f in calls.items():
                f()  # untimed: the loop leaves edited layer tables, which the next call of either kind re-uploads
                torch.cuda.synchronize()
                ev[0].record()
                for _ in range(args.steps):
                    f()
                ev[1].record()
                torch.cuda.synchronize()
                res[k].append(ev[0].elapsed_time(ev[1]) / args.steps / n)
        batch()
        line = {"case": name, "views": n, "width": w, "height": h, "frames_equal": same,
                "segments": r.counters()["segments"],
                "ms_per_view": {k: round(float(np.median(v)), 5) for k, v in res.items()},
                "ms_per_view_runs": {k: [round(x, 5) for x in v] for k, v in res.items()}}
        line["speedup"] = round(line["ms_per_view"]["render_device_loop"] / line["ms_per_view"]["render_views_device"], 2)
        print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
