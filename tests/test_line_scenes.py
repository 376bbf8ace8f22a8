"""Line setup at its limits on the CPU (scenes: tests/line_scenes.py; model: tests/line_model.py).

- On every in-limit scene the model's line records equal the oracle's bit for bit, including
  the reference's wrapped u32 prefix sums, and the scene reaches its target and fits the budget.
- Over-limit scenes reach a true total of 2^30 or more (exactly 2^30; 2^32 + 7 in one CTA or
  spread over CTAs so that only the device-wide scan passes 2^32; a CTA sum past 2^32; a
  saturated ±3e38 line), and the model names the status the renderer returns. The oracle, in a
  process of its own, refuses those above 2^32 - 1 without writing out of bounds.
- Single-segment lines at 2^26 ... 2^30 px and through a NaN transform pin the oracle's
  `rasterize_only` to segment words derived by hand from `round_sub` (i32::MIN for NaN and
  out-of-range values, as the reference's x86 build gives).
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import flatten_model as fm
import line_model as lm
import line_scenes as ls

FIELDS = ("orders", "x0", "y0", "dx", "dy", "a", "b", "c", "d")


def _bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float32:
        na, nb = np.isnan(a), np.isnan(b)
        return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))
    return np.array_equal(a, b)


def oracle_lines(oracle_api, scene):
    comp, _, _ = ls.build(oracle_api, scene.layers)
    r = oracle_api.Renderer(0)
    segs = r.rasterize_only(comp, scene.width, scene.height)
    return r, comp, segs, r.lines()


def test_fmaf_is_exact_at_float32_midpoints():
    # 1 + 2^-24 is the midpoint between 1 and 1 + 2^-23: the error term decides.
    one, half_ulp = np.float32(1.0), np.float32(2.0 ** -24)
    assert lm.fmaf(one, one, half_ulp) == np.float32(1.0)                     # a tie, to even
    assert lm.fmaf(np.float32(1 + 2 ** -23), np.float32(1 + 2 ** -23), np.float32(-1.0)) == np.float32(2 ** -22 + 2 ** -46)
    tiny = np.float32(2.0 ** -60)
    assert lm.fmaf(half_ulp, np.float32(1 + 2 ** -23), one) == np.float32(1 + 2 ** -23)  # just above the tie
    assert lm.fmaf(half_ulp, one, one + tiny * 0) == one
    assert lm.fmaf(np.float32(3e38), np.float32(2), np.float32(-3e38)) == np.float32(3e38)


@pytest.mark.parametrize("name", ls.IN_LIMIT)
def test_model_equals_oracle_line_records(oracle_api, name):
    sc = ls.SCENES[name]
    rec = ls.model(oracle_api, sc)
    _, _, segs, lines = oracle_lines(oracle_api, sc)
    assert lines["orders"].size == rec["orders"].size
    for f in FIELDS:
        assert _bits_equal(rec[f], lines[f]), f"{name}: {f} differs from the oracle's"
    c = rec["counts"]
    assert np.array_equal(c.prefix_u32, lines["lengths"]), f"{name}: wrapped prefix sums differ"
    assert segs.size == c.total
    assert sc.reached(rec), f"{name} does not reach its target: {sc.target}"
    assert c.status == lm.FORMA_OK
    assert c.total <= fm.SEGMENT_CAP, f"{name}: {c.total} segments > {fm.SEGMENT_CAP}"
    assert int(c.emit_iterations.sum()) == c.total
    assert max(lm.max_tile(rec)) <= 4095


@pytest.mark.parametrize("name", ls.OVER_LIMIT)
def test_over_limit_scenes_are_refused(oracle_api, name):
    sc = ls.SCENES[name]
    rec = ls.model(oracle_api, sc)
    c = rec["counts"]
    assert sc.reached(rec) and c.total >= lm.SEGMENT_LIMIT, f"{name} does not reach its target ({sc.target}): {c.total}"
    # The device's emit pass stays inside any buffer: at most cap iterations in all.
    for cap in (0, 1, 1000, 2 ** 26):
        it = lm.counts(rec["length"], rec["n_points"], cap).emit_iterations
        assert int(it.sum()) <= cap
    if c.total <= lm.U32_MAX:
        return  # below 2^32: the oracle would render it (8 GB of segments); only the device refuses
    # In a process of its own: an oracle that indexed with the wrapped sums would crash this one.
    out = subprocess.run([sys.executable, "-c", _REFUSAL.format(name=name)], capture_output=True, text=True,
                         timeout=300, env=dict(os.environ, PYTHONPATH=os.pathsep.join((ROOT, os.path.join(ROOT, "tests")))))
    assert out.returncode == 0 and out.stdout.split() == ["refused", "refused"], (out.returncode, out.stdout, out.stderr[-2000:])


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_REFUSAL = """
import numpy as np
import line_scenes as ls
from forma_b200.binding import RGBA, Color, FormaError
from oracle import oracle
api = oracle.load()
sc = ls.SCENES["{name}"]
comp, _, _ = ls.build(api, sc.layers)
r = api.Renderer(0)
segs = r.rasterize_only(comp, sc.width, sc.height)
print("refused" if segs.size == 0 and "exceed" in api.last_error().decode() else "rasterized")
buf = np.zeros(sc.width * sc.height * 4, np.uint8)
try:
    r.render(comp, buf, sc.width, sc.height, RGBA, Color(1, 1, 1, 0))
    print("rendered")
except FormaError as e:
    print("refused" if "status 5" in str(e) and not buf.any() else "failed")
"""


def test_hand_derived_segment_words_at_out_of_range_positions(oracle_api):
    comp, _, _ = ls.build(oracle_api, ls.origin_layers())
    r = oracle_api.Renderer(0)
    segs = r.rasterize_only(comp, ls.ORIGIN_WIDTH, 64)
    orders = (segs >> np.uint64(20)) & np.uint64(0x1FFFFF)
    for k, (x, y0, y1) in enumerate(ls.ORIGINS):
        xs = np.float32(x) * np.float32(16)
        mine = segs[orders == k]
        # The first line of the layer: (x, y0) -> (x, y1), one segment, t0 = 0 and t1 = 1.
        if x == x:  # (a NaN line's t0, t1 are not 0 and 1: only its x fields are pinned below)
            assert int(mine[0]) == lm.segment_word(k, xs, y0 * 16, xs, y1 * 16), (k, x, hex(int(mine[0])))
        if x != x or x >= 2 ** 27:  # i32::MIN: tile column 0, local x 0, for every segment of the layer
            assert np.all((mine >> np.uint64(41)) & np.uint64(0xFFF) == 1), (k, x)
            assert np.all((mine >> np.uint64(16)) & np.uint64(0xF) == 0), (k, x)
    assert lm.round_sub(2.0 ** 31) == lm.INT_MIN and lm.round_sub(float("nan")) == lm.INT_MIN
    assert lm.round_sub(2.0 ** 31 - 128) == 2 ** 31 - 128 and lm.round_sub(-2.0 ** 31) == lm.INT_MIN

