"""The oracle's layer statistics (fo_renderer_render_stats, tests/oracle_stats.py), pinned without a GPU
to the oracles already pinned: area, pixels and box are a numpy reduction of the mask oracle's F32
planes, visible and visible_box one of the ID oracle's frame at the same min_coverage, over the
pixels the call counts (the crop's tile rectangle in the frame). tests/test_gpu_stats.py then holds
the device to these records."""
import numpy as np
import pytest

import extremes
import oracle_ids
import oracle_masks
import oracle_stats
import scenes
import style_scenes as ss
import synth
from forma_b200.binding import ID_NONE, STATS_DTYPE, FormaError, Rect, _CStats

THRESHOLDS = (0.0, 0.5, 0.998)


@pytest.fixture(autouse=True)
def _attach(oracle_api):
    oracle_stats.attach(oracle_api)
    oracle_masks.attach(oracle_api)
    oracle_ids.attach(oracle_api)


def n_orders(comp):
    import batch_scenes
    return max(batch_scenes.n_orders(comp), 1)


def check(api, comp, w, h, first, k, min_coverage, crop=None):
    """The stats oracle against the reduction of the mask and ID oracles; returns the records."""
    got = oracle_stats.render(api, comp, w, h, first, k, min_coverage, crop)
    planes = oracle_masks.render(api, comp, w, h, first, k, "f32", crop)
    ids = np.full(w * h, ID_NONE, np.uint32)
    api.Renderer(0).render_ids(comp, ids, w, h, crop=crop, min_coverage=min_coverage)
    want = oracle_stats.reduce(planes, ids.reshape(h, w), first, min_coverage, oracle_stats.region(w, h, crop))
    assert not oracle_stats.diff(got, want), oracle_stats.diff(got, want)
    return got


@pytest.mark.parametrize("threshold", THRESHOLDS)
@pytest.mark.parametrize("name", sorted(scenes.E2E))
def test_e2e(oracle_api, name, threshold):
    comp = oracle_api.Composition()
    scenes.E2E[name](oracle_api, comp)
    got = check(oracle_api, comp, 64, 64, 0, n_orders(comp) + 1, threshold)
    assert got["area"].any() or name == "empty"


@pytest.mark.parametrize("name", sorted(extremes.SCENES))
def test_extremes(oracle_api, name):
    comp, _, sc = extremes.build(oracle_api, name)
    n = n_orders(comp)
    big = sc.width * sc.height > 1 << 20
    k = min(n, 8 if big else 64)
    for first, threshold in ((0, 0.0), (max(n - k, 0), 0.5)):
        check(oracle_api, comp, sc.width, sc.height, first, k, threshold, sc.crop)


@pytest.mark.parametrize("name", sorted(ss.SCENES))
def test_styles(oracle_api, name):
    comp, _, sc = ss.build(oracle_api, name)
    check(oracle_api, comp, sc.width, sc.height, 0, min(n_orders(comp), 96), 0.5)


@pytest.mark.parametrize("threshold", THRESHOLDS)
def test_random_mixed(oracle_api, threshold):
    w, h = 120, 90  # neither a multiple of 16
    comp = oracle_api.Composition()
    synth.random_mixed(oracle_api, comp, 60, w, h, 9)
    got = check(oracle_api, comp, w, h, 0, 61, threshold)
    assert (got["pixels"] >= got["visible"]).all() or threshold > 0  # amodal covers visible at coverage 0
    assert got["visible"].sum() <= w * h


def test_crops_and_odd_sizes(oracle_api):
    for w, h, crop in ((100, 70, Rect((20, 50), (17, 40))), (97, 53, Rect((0, 97), (30, 53))), (130, 41, Rect((33, 34), (1, 2))),
                       (64, 64, Rect((70, 90), (0, 64)))):
        comp = oracle_api.Composition()
        synth.random_mixed(oracle_api, comp, 25, w, h, w + h)
        for threshold in (0.0, 0.5):
            check(oracle_api, comp, w, h, 0, 26, threshold, crop)


def test_windows(oracle_api):
    w, h = 100, 70
    comp = oracle_api.Composition()
    synth.random_mixed(oracle_api, comp, 30, w, h, 4)
    n = n_orders(comp)
    full = check(oracle_api, comp, w, h, 0, n, 0.0)
    for first, k in ((0, 1), (7, 1), (0, 5), (n - 3, 6), (n, 4), (n + 100, 2), ((1 << 21) - 2, 2), ((1 << 21) - 40, 40)):
        got = check(oracle_api, comp, w, h, first, k, 0.0)
        for j in range(k):
            want = full[first + j] if first + j < n else np.zeros((), STATS_DTYPE)
            assert got[j] == want, (first, k, j)


def test_disabled_and_clip_layers(oracle_api):
    w, h = 64, 64
    for name in ("clipping",) + tuple(n for n in sorted(scenes.E2E) if "clip" in n and n != "clipping"):
        comp = oracle_api.Composition()
        scenes.E2E[name](oracle_api, comp)
        n = n_orders(comp)
        before = check(oracle_api, comp, w, h, 0, n, 0.0)
        layer = next(comp.get(o) for o in range(n) if comp.get(o) is not None)
        order = next(o for o in range(n) if comp.get(o) is not None)
        layer.set_is_enabled(False)
        after = check(oracle_api, comp, w, h, 0, n, 0.0)
        assert after[order] == np.zeros((), STATS_DTYPE)
        assert before[order]["area"] > 0 or not before[order]["pixels"]


def test_records_layout():
    assert STATS_DTYPE.itemsize == 48
    assert [STATS_DTYPE.fields[f][1] for f in ("area", "pixels", "visible", "box", "visible_box")] == [0, 8, 12, 16, 32]


@pytest.mark.parametrize("case", ["null", "k0", "past_field", "nan", "negative", "one", "unaligned"])
def test_invalid_arguments_leave_the_records(oracle_api, case):
    import ctypes as C
    comp = oracle_api.Composition()
    scenes.E2E["clipping"](oracle_api, comp)
    buf = np.full(4 * 48 + 8, 0x5A, np.uint8)
    base = buf.ctypes.data + (-buf.ctypes.data) % 8
    args = dict(ptr=base, first_order=0, n_orders=4, min_coverage=0.0)
    args.update({"null": dict(ptr=None), "k0": dict(n_orders=0), "past_field": dict(first_order=(1 << 21) - 3),
                 "nan": dict(min_coverage=float("nan")), "negative": dict(min_coverage=-0.25), "one": dict(min_coverage=1.0),
                 "unaligned": dict(ptr=base + 4)}[case])
    s = _CStats(args["ptr"], args["first_order"], args["n_orders"], args["min_coverage"])
    r = oracle_api.Renderer(0)
    assert oracle_api.renderer_render_stats(r._h, comp._h, C.byref(s), 64, 64, None, None) != 0
    assert (buf == 0x5A).all()
    with pytest.raises(FormaError):
        r.render_stats(comp, 64, 64, 0, 0)
