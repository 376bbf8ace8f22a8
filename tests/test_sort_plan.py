"""The sort plan (make_sort_plan, exported by forma_debug_sort_plan) against tests/sort_model.py,
for every triple of field widths of both key layouts, on the CPU.

The model is pinned on its own as well: one stable counting pass per modelled digit equals a
stable sort on the virtual key. And the checks are shown to bite: each of sort_model.MUTATIONS
(a deliberate error of the model) is caught by them.
"""
import itertools

import numpy as np
import pytest

import sort_model as sm


def _triples(layout):
    return itertools.product(*[range(w + 1) for _, w in sm.LAYOUTS[layout]])


def _bound_sets(layout, widths):
    """Bounds that give `widths`, and the bounds one step around each power of two."""
    yield [(1 << w) - 1 for w in widths]
    yield [1 << w for w in widths]                       # one bit more (where the field has room)
    yield [(1 << (w - 1)) if w else 0 for w in widths]   # the smallest bound of the same width


def _random_keys(rng, n):
    return rng.integers(0, 1 << 63, size=n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=n, dtype=np.uint64)


@pytest.mark.parametrize("layout", [0, 1])
def test_library_plan_equals_model_for_every_width_triple(cuda_api, layout):
    n = 0
    for widths in _triples(layout):
        for bound in _bound_sets(layout, widths):
            raw = cuda_api.sort_plan(layout, bound)
            want = sm.make_plan(layout, bound)
            assert raw == sm.plan_bytes(want), (layout, bound, sm.parse_plan(raw).describe(), want.describe())
            faults = sm.plan_faults(sm.parse_plan(raw), layout, bound)
            assert not faults, (layout, bound, faults)
            n += 1
    assert n == 3 * np.prod([w + 1 for _, w in sm.LAYOUTS[layout]])


@pytest.mark.parametrize("layout", [0, 1])
def test_bounds_above_a_field_are_cut_to_its_width(cuda_api, layout):
    full = [(1 << w) - 1 for _, w in sm.LAYOUTS[layout]]
    for f in range(3):
        for big in (1 << sm.LAYOUTS[layout][f][1], (1 << 32) + 5, (1 << 63), (1 << 64) - 1):
            for rest in (full, [0, 0, 0], [1, 1, 1]):
                bound = list(rest)
                bound[f] = big
                raw = cuda_api.sort_plan(layout, bound)
                cut = list(bound)
                cut[f] = full[f]
                assert raw == cuda_api.sort_plan(layout, cut) == sm.plan_bytes(sm.make_plan(layout, bound)), (layout, bound)
                assert not sm.plan_faults(sm.parse_plan(raw), layout, bound)
    raw = cuda_api.sort_plan(layout, [(1 << 64) - 1] * 3)
    assert raw[0] == 6 and raw[1] == 44 and sm.parse_plan(raw).sizes() == [8, 8, 7, 7, 7, 7]
    assert cuda_api.sort_plan(layout, [0, 0, 0]) == bytes(62)


def test_layout_is_checked(cuda_api):
    from forma_b200.binding import FormaError
    for layout in (-1, 2):
        with pytest.raises(FormaError):
            cuda_api.sort_plan(layout, [1, 1, 1])


def test_known_plans(cuda_api):
    """Plans written out by hand from the layout (layer 20..40, tile_x 41..52, tile_y 53..63)."""
    # 16 layer + 8 tile_x + 8 tile_y bits: four single-run digits.
    p = sm.parse_plan(cuda_api.sort_plan(0, [0xFFFF, 0xFF, 0xFF]))
    assert [(d.shift, d.width, d.lsh, d.bits) for d in p.passes] == [
        ((20, 0, 0), (8, 0, 0), (0, 0, 0), 8), ((28, 0, 0), (8, 0, 0), (0, 0, 0), 8),
        ((41, 0, 0), (8, 0, 0), (0, 0, 0), 8), ((53, 0, 0), (8, 0, 0), (0, 0, 0), 8)]
    # 1 + 1 + 6 bits: one digit of three runs.
    p = sm.parse_plan(cuda_api.sort_plan(0, [1, 1, 63]))
    assert [(d.shift, d.width, d.lsh, d.bits) for d in p.passes] == [((20, 41, 53), (1, 1, 6), (0, 1, 2), 8)]
    # The carry layout: 5 tile_x + 12 layer bits = 17 bits = 6 + 6 + 5, the first digit straddling.
    p = sm.parse_plan(cuda_api.sort_plan(1, [31, 4095, 0]))
    assert [(d.shift, d.width, d.lsh, d.bits) for d in p.passes] == [
        ((20, 32, 0), (5, 1, 0), (0, 5, 0), 6), ((33, 0, 0), (6, 0, 0), (0, 0, 0), 6), ((39, 0, 0), (5, 0, 0), (0, 0, 0), 5)]
    # 38 bits -> 8, 8, 8, 7, 7.
    assert sm.parse_plan(cuda_api.sort_plan(0, [(1 << 21) - 1, 4095, 31])).sizes() == [8, 8, 8, 7, 7]


def _sampled_plans(seed, count):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(count):
        layout = k % 2
        widths = [int(rng.integers(0, w + 1)) for _, w in sm.LAYOUTS[layout]]
        out.append((layout, [(1 << w) - 1 for w in widths]))
    return out


def test_model_passes_sort_like_a_stable_sort_on_the_virtual_key():
    rng = np.random.default_rng(5)
    straddling = 0
    for layout, bound in _sampled_plans(17, 200):
        keys = _random_keys(rng, 10_000)
        # keep only the bits the bounds allow (and everything below bit 20)
        mask = np.uint64((1 << sm.SORT_SHIFT) - 1)
        for (pos, _), b in zip(sm.LAYOUTS[layout], bound):
            mask |= np.uint64(b << pos)
        keys &= mask
        plan = sm.make_plan(layout, bound)
        straddling += any(d.runs > 1 for d in plan.passes)
        assert np.array_equal(sm.lsd_order(keys, plan), sm.reference_order(keys, layout, bound)), (layout, bound)
        # with exact bounds the virtual key orders like bits [20, 64) for the segment layout
        if layout == 0:
            assert np.array_equal(sm.reference_order(keys, layout, bound), np.argsort(keys >> np.uint64(20), kind="stable"))
    assert straddling > 50


@pytest.mark.parametrize("mutation", sm.MUTATIONS)
def test_a_wrong_model_is_caught(cuda_api, mutation):
    """Each deliberate error of the model differs from the library's plan, breaks a plan
    property, and (when it changes digits at all) mis-sorts: the checks above can fail."""
    rng = np.random.default_rng(3)
    differs = faulty = missorts = 0
    for layout, bound in _sampled_plans(23, 200):
        bad = sm.make_plan(layout, bound, mutation)
        differs += sm.plan_bytes(bad) != cuda_api.sort_plan(layout, bound)
        faulty += bool(sm.plan_faults(bad, layout, bound))
        keys = _random_keys(rng, 2000)
        missorts += not np.array_equal(sm.lsd_order(keys, bad), sm.reference_order(keys, layout, bound))
    assert differs > 20 and faulty > 20, (mutation, differs, faulty)
    assert differs == faulty  # the property checks see every wrong plan the byte comparison sees
    if mutation != "greedy_sizes":  # (8, 8, ..., rest) still sorts; only its sizes are wrong
        assert missorts > 20, (mutation, missorts)
