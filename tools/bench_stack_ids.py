"""Device time per frame of the stacked RGBA + ID calls against a loop of render_device_with_ids
calls (the way to get the frames and their ID frames without them), in alternating runs timed
with CUDA events. Prints the card and its power limit from the same run, then one JSON line per
case:

- batch/random_511x64: render_batch_ids_device of 511 distinct resident 64 x 64
  synth.random_mixed compositions (tools/bench_batch.py's case);
- batch/paris_tiles_16: render_batch_ids_device of paris split into 16 compositions, one per
  960 x 540 tile (tests/batch_scenes.py);
- views/paris_tiles_16: render_views_ids_device of the 16 translated 960 x 540 tiles of paris
  (tests/view_scenes.py); the loop sets every layer's transform per view, as tools/bench_views.py
  does.

Both arms write an RGBA stack and an ID stack; a case counts only if both produced equal frames
and equal IDs ("frames_equal", "ids_equal"). Needs a GPU.

    python tools/bench_stack_ids.py [--steps 5] [--runs 3] [--cases batch/random_511x64,batch/paris_tiles_16,views/paris_tiles_16]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

from bench_views import card  # noqa: E402


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--cases", default="batch/random_511x64,batch/paris_tiles_16,views/paris_tiles_16")
    args = ap.parse_args(argv)
    import numpy as np
    import torch

    import batch_scenes as bs
    import forma_b200
    import synth
    import view_scenes as vs
    from forma_b200.binding import RGBA, Color

    print(f"card: {card()}", flush=True)
    api = forma_b200.load()
    clear = Color(1.0, 1.0, 1.0, 1.0)

    for name in args.cases.split(","):
        r = api.Renderer(0)
        if name == "batch/random_511x64":
            comps, w, h = [], 64, 64
            for k in range(511):
                comps.append(api.Composition())
                synth.random_mixed(api, comps[-1], 24, 64, 64, 1000 + k)
        elif name == "batch/paris_tiles_16":
            comps, w, h = [b(api) for b in bs.SCENES["paris_tiles"].builders], *bs.PARIS_TILE
        elif name == "views/paris_tiles_16":
            comp, (w, h), views = api.Composition(), bs.PARIS_TILE, vs.SCENES["paris_tiles"].views
            handles = [comp.get(o)._h for o in vs._paris(api, comp)]  # no layer has a transform of its own: C = V
            arrays = [(C.c_float * 6)(*vs.compose(v, None)) for v in views]
            ident = (C.c_float * 6)(*vs.IDENTITY)
        else:
            raise SystemExit(f"unknown case {name}")
        is_views = name.startswith("views/")
        n = len(views) if is_views else len(comps)
        rgba = torch.empty((n, h, w, 4), dtype=torch.uint8, device="cuda:0")
        ids = torch.empty((n, h, w), dtype=torch.int32, device="cuda:0")

        def stacked():
            if is_views:
                r.render_views_ids_device(comp, views, ids.data_ptr(), w, h, rgba_ptr=rgba.data_ptr(), clear_color=clear, timings=False)
            else:
                r.render_batch_ids_device(comps, ids.data_ptr(), w, h, rgba_ptr=rgba.data_ptr(), clear_color=clear, timings=False)

        def loop():
            for b in range(n):
                if is_views:
                    for lh in handles:
                        api.layer_set_transform(comp._h, lh, arrays[b])
                r.render_device_with_ids(comp if is_views else comps[b], rgba[b].data_ptr(), ids[b].data_ptr(), w, h, RGBA, clear,
                                         timings=False)
            if is_views:
                for lh in handles:
                    api.layer_set_transform(comp._h, lh, ident)

        stacked_name = "render_views_ids_device" if is_views else "render_batch_ids_device"
        calls = {stacked_name: stacked, "render_device_with_ids_loop": loop}
        for f in calls.values():  # warm-up: uploads, buffers, sync-free bounds
            f(), f()
        want_rgba, want_ids = rgba.clone(), ids.clone()
        rgba.zero_(), ids.zero_()
        stacked()
        torch.cuda.synchronize()
        same_rgba, same_ids = bool(torch.equal(rgba, want_rgba)), bool(torch.equal(ids, want_ids))  # the stack equals the loop
        res = {k: [] for k in calls}
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        for _ in range(args.runs):
            for k, f in calls.items():
                f()  # untimed: a views loop leaves edited layer tables, which the next call of either kind re-uploads
                torch.cuda.synchronize()
                ev[0].record()
                for _ in range(args.steps):
                    f()
                ev[1].record()
                torch.cuda.synchronize()
                res[k].append(ev[0].elapsed_time(ev[1]) / args.steps / n)
        stacked()
        line = {"case": name, "frames": n, "width": w, "height": h, "frames_equal": same_rgba, "ids_equal": same_ids,
                "hit_pixels": int((want_ids != -1).sum()), "segments": r.counters()["segments"],
                "ms_per_frame": {k: round(float(np.median(v)), 5) for k, v in res.items()},
                "ms_per_frame_runs": {k: [round(x, 5) for x in v] for k, v in res.items()}}
        line["speedup"] = round(line["ms_per_frame"]["render_device_with_ids_loop"] / line["ms_per_frame"][stacked_name], 2)
        print(json.dumps(line), flush=True)
        if not (same_rgba and same_ids):
            return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
