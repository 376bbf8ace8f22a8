#!/usr/bin/env python
"""Frames of the working-tree oracle against the oracle of an earlier commit (CPU only).

The oracle is the checker of every GPU parity test, so a change to it (e.g. a speed-up of the
CPU baseline) must leave its frames untouched. This builds `oracle/` of <rev> in a temporary
directory and compares both on random mixed / circle / cubic scenes, the 32 e2e scenes, channel
orders, a crop, the layer-cache scenarios and an animation.

usage: python tools/compare_oracles.py <git rev>
"""
import os
import subprocess
import tempfile
import sys, ctypes as C, numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
from forma_b200 import binding
from forma_b200.binding import RGBA, Color
import oracle.oracle as O
import synth, scenes
OPT = ("renderer_render_device", "renderer_stage_times", "renderer_counters", "renderer_kernel_times", "renderer_set_stream", "path_program_stats",
       "path_program_records", "shared_frame_create", "shared_frame_open", "shared_frame_close", "shared_frame_free", "composition_evict", "composition_point_count")
new = O.load()
rev = sys.argv[1]
tmp = tempfile.mkdtemp()
subprocess.check_call(f"git -C {ROOT} archive {rev} oracle | tar -x -C {tmp} && make -s -C {tmp}/oracle", shell=True)
old = binding.Api(C.CDLL(os.path.join(tmp, 'oracle', 'libforma_oracle.so')), "fo_", optional=OPT)
def frame(api, build, w, h, channels=RGBA, clear=Color(1, 1, 1, 0)):
    comp = api.Composition(); build(api, comp)
    r = api.Renderer(); buf = np.zeros(w * h * 4, np.uint8)
    r.render(comp, buf, w, h, channels, clear)
    return buf
n = 0
for seed, cnt, w, h in [(1, 200, 640, 360), (2, 800, 1280, 720), (3, 1500, 1920, 1080), (4, 60, 97, 131), (5, 3000, 1024, 1024)]:
    a = frame(new, lambda api, c: synth.random_mixed(api, c, cnt, w, h, seed), w, h)
    b = frame(old, lambda api, c: synth.random_mixed(api, c, cnt, w, h, seed), w, h)
    assert np.array_equal(a, b), (seed, int((a != b).sum())); n += 1
for seed in (7, 8):
    a = frame(new, lambda api, c: synth.random_circles(api, c, 3000, 1920, 1080, seed), 1920, 1080)
    b = frame(old, lambda api, c: synth.random_circles(api, c, 3000, 1920, 1080, seed), 1920, 1080)
    assert np.array_equal(a, b), seed; n += 1
a = frame(new, lambda api, c: synth.random_cubics(api, c, 5000, 1920, 1080, 3), 1920, 1080)
b = frame(old, lambda api, c: synth.random_cubics(api, c, 5000, 1920, 1080, 3), 1920, 1080)
assert np.array_equal(a, b); n += 1
for name in sorted(scenes.E2E):
    build = scenes.E2E[name]
    a = frame(new, lambda api, c: build(api, c), 64, 64, clear=scenes.E2E_CLEAR)
    b = frame(old, lambda api, c: build(api, c), 64, 64, clear=scenes.E2E_CLEAR)
    assert np.array_equal(a, b), name; n += 1
print("new oracle == old oracle on", n, "scenes")
from forma_b200.binding import Rect
import cache_scenarios
# channel orders + crop + stride
for ch in ([2, 1, 0, 3], [3, 2, 1, 0], [0, 1, 2, 5], [4, 1, 2, 3]):
    a = frame(new, lambda api, c: synth.random_mixed(api, c, 300, 333, 211, 11), 333, 211, channels=ch, clear=Color(0.2, 0.3, 0.4, 1.0))
    b = frame(old, lambda api, c: synth.random_mixed(api, c, 300, 333, 211, 11), 333, 211, channels=ch, clear=Color(0.2, 0.3, 0.4, 1.0))
    assert np.array_equal(a, b), ch
def cropped(api):
    comp = api.Composition(); synth.random_mixed(api, comp, 400, 640, 480, 12)
    r = api.Renderer(); buf = np.full(640 * 480 * 4, 7, np.uint8)
    r.render(comp, buf, 640, 480, RGBA, Color(1, 1, 1, 1), crop=Rect(range(100, 400), range(50, 300)))
    return buf
assert np.array_equal(cropped(new), cropped(old))
# layer-cache scenarios frame by frame
for sc in cache_scenarios.SCENARIOS:
    fa, fb = sc(new), sc(old)
    assert len(fa) == len(fb)
    for x, y in zip(fa, fb):
        assert np.array_equal(np.asarray(x), np.asarray(y)), sc.__name__
fa, fb = cache_scenarios.animated_scene(new), cache_scenarios.animated_scene(old)
for x, y in zip(fa, fb):
    assert np.array_equal(np.asarray(x), np.asarray(y))
print("channels / crop / cache scenarios / animation identical too")
