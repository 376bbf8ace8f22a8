"""Device time per frame of Renderer.render_batch_device against a loop of render_device calls
(the way to render many compositions without it), in alternating runs timed with CUDA events.
Prints the card and its power limit from the same run, then one JSON line per case:

- random_511x64: 511 distinct resident 64 x 64 synth.random_mixed compositions;
- paris_tiles_16: paris split into 16 compositions, one per 960 x 540 tile (tests/batch_scenes.py);
- fresh_256x64: 256 64 x 64 compositions built anew every step, so that their construction,
  upload and flatten are part of both timings.

    python tools/bench_batch.py [--steps 5] [--runs 3] [--cases random_511x64,paris_tiles_16,fresh_256x64]
"""
from __future__ import annotations

import argparse
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
    ap.add_argument("--cases", default="random_511x64,paris_tiles_16,fresh_256x64")
    args = ap.parse_args(argv)
    import numpy as np
    import torch

    import batch_scenes as bs
    import forma_b200
    import synth
    from forma_b200.binding import RGBA, Color

    print(f"card: {card()}", flush=True)
    api = forma_b200.load()
    clear = Color(1.0, 1.0, 1.0, 1.0)

    def random_comps(n, seed0):
        out = []
        for k in range(n):
            comp = api.Composition()
            synth.random_mixed(api, comp, 24, 64, 64, seed0 + k)
            out.append(comp)
        return out

    for name in args.cases.split(","):
        fresh = name == "fresh_256x64"
        if name == "random_511x64":
            comps, w, h = random_comps(511, 1000), 64, 64
        elif name == "paris_tiles_16":
            comps, w, h = [b(api) for b in bs.SCENES["paris_tiles"].builders], *bs.PARIS_TILE
        elif fresh:
            comps, w, h = random_comps(256, 5000), 64, 64
        else:
            raise SystemExit(f"unknown case {name}")
        n = len(comps)
        r = api.Renderer(0)
        out = torch.empty((n, h, w, 4), dtype=torch.uint8, device="cuda:0")
        state = {"comps": comps}

        def step_comps():
            if fresh:  # new compositions every step: built, uploaded and flattened inside the timing
                state["comps"] = random_comps(n, 5000)
            return state["comps"]

        def batch():
            r.render_batch_device(step_comps(), out.data_ptr(), w, h, RGBA, clear, timings=False)

        def loop():
            for c, comp in enumerate(step_comps()):
                r.render_device(comp, out[c].data_ptr(), w, h, RGBA, clear, timings=False)

        calls = {"render_batch_device": batch, "render_device_loop": loop}
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
                torch.cuda.synchronize()
                ev[0].record()
                for _ in range(args.steps):
                    f()
                ev[1].record()
                torch.cuda.synchronize()
                res[k].append(ev[0].elapsed_time(ev[1]) / args.steps / n)
        batch()
        line = {"case": name, "frames": n, "width": w, "height": h, "frames_equal": same,
                "segments": r.counters()["segments"],
                "ms_per_frame": {k: round(float(np.median(v)), 5) for k, v in res.items()},
                "ms_per_frame_runs": {k: [round(x, 5) for x in v] for k, v in res.items()}}
        line["speedup"] = round(line["ms_per_frame"]["render_device_loop"] / line["ms_per_frame"]["render_batch_device"], 2)
        print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
