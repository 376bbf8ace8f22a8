"""The pose limit scenes (tests/pose_limit_scenes.py) on the CPU, before any of them reaches a GPU:
every table is one the poses calls accept, every scene reaches the condition it is named for, every
in-limit call fits the budgets (segments, points, pose records and pose style table), the refusal
scenes are refused by their counts alone, and the checks catch errors planted in them."""
import numpy as np
import pytest

import line_model as lm
import pose_fill_scenes as pfs
import pose_limit_scenes as pls
import pose_scenes as ps

f32 = np.float32
_MODELS = {}


def geom_pres_ok(t) -> bool:
    """forma_layer_set_transform's check of [ux, vx, uy, vy, tx, ty], in separately rounded f32."""
    ux, vx, uy, vy = (f32(v) for v in t[:4])
    max_x, max_y = f32(1.0) + f32(1.0 / 16.0) / f32(65536.0), f32(1.0) + f32(1.0 / 16.0) / f32(32768.0)
    with np.errstate(all="ignore"):
        return not (f32(ux * ux) + f32(uy * uy) > max_x) and not (f32(vx * vx) + f32(vy * vy) > max_y)


def build_counting_points(api, sc):
    """(composition, orders, flattened points of every insert) of a scene: Layer.insert counted."""
    from forma_b200 import binding
    original, n = binding.Layer.insert, [0]

    def insert(layer, path):
        n[0] += len(path.segments()[0])
        return original(layer, path)
    binding.Layer.insert = insert
    try:
        comp, orders = sc.build(api)
    finally:
        binding.Layer.insert = original
    return comp, orders, n[0]


def models(oracle_api, name):
    """(points, [frame_model of every frame]) of a specs scene, computed once."""
    if name not in _MODELS:
        sc = pls.SCENES[name]
        pts = pls.points(oracle_api, sc)
        _MODELS[name] = pts, [pls.frame_model(sc, pts, b) for b in range(sc.n)]
    return _MODELS[name]


def stack_violations(sc, recs, remap=True, bound=pls.frame_bound):
    """Kept lines whose rows {-1, 0, rows - 1, rows} (where they reach them) land outside their
    frame's stacked rows [b rows + 1, bound] and are not dropped to row 0."""
    bad, rows = [], sc.rows
    for b, rec in enumerate(recs):
        lo, hi = pls.touched_rows(rec)
        for t in (-1, 0, rows - 1, rows):
            if not np.any((lo <= t) & (hi >= t)):
                continue
            s = pls.stacked_row(b, t, rows, remap)
            if s != 0 and not (b * rows + 1 <= s <= bound(b, rows)):
                bad.append((b, t, s))
    return bad


def reached_rows(sc, recs):
    """{t: number of frames with a kept line in frame tile row t}, for t = -1, rows - 1, rows."""
    out = {}
    for t in (-1, sc.rows - 1, sc.rows):
        out[t] = sum(bool(np.any((lo <= t) & (hi >= t))) for lo, hi in (pls.touched_rows(r) for r in recs))
    return out


def far_frames(recs):
    """Frames with kept lines, every one of them more than 2^19 px left of the frame."""
    out = []
    for b, rec in enumerate(recs):
        k = rec["keep"]
        if k.any():
            x_hi = np.fmax(rec["x0"][k], rec["x0"][k] + rec["dx"][k]).astype(np.float64) / 16.0
            if np.all(x_hi < pls.FAR_LEFT):
                out.append(b)
    return out


@pytest.mark.parametrize("name", list(pls.SCENES))
def test_tables_are_accepted(name):
    sc = pls.SCENES[name]
    tables = [t for t in (sc.transforms, sc.visible, sc.colors) if t is not None]
    assert len({t.shape[:2] for t in tables}) == 1 and sc.n >= 1 and sc.n_orders >= 1
    assert sc.first_order + sc.n_orders <= ps.LAYER_LIMIT
    if sc.transforms is not None:
        t = sc.transforms.reshape(-1, 6)
        assert all(geom_pres_ok(r) for r in np.unique(t, axis=0)), name


def test_full_stacks_are_at_the_limit(oracle_api):
    for name, rows, n in (("limit_h16", 1, 2046), ("limit_h1", 1, 2046), ("limit_h17", 2, 1023), ("limit_h1000", 63, 32)):
        sc = pls.SCENES[name]
        assert sc.rows == rows and sc.n == n == 2046 // rows == pls.max_views(sc.height), name
        _, recs = models(oracle_api, name)
        for b in (0, n - 1):
            lo, hi = pls.touched_rows(recs[b])
            assert np.any((hi >= 0) & (lo < rows)), (name, b)  # content in the first and the last frame
        vis = sc.visible
        assert len({bytes(v) for v in vis}) > 1 and np.all(vis[0]) and np.all(vis[-1])


@pytest.mark.parametrize("name", pls.STACKS + pls.ODD)
def test_neighbour_shifts_reach_the_adjacent_frames(oracle_api, name):
    """Lines reach the tile row above the frame and the one below it in frames with a neighbour on
    that side, and the frame's last row: a remap of every row would put them into the neighbour's
    rows, a bound one row short would miss the last. The model's rows match the oracle's segments."""
    sc = pls.SCENES[name]
    _, recs = models(oracle_api, name)
    assert stack_violations(sc, recs) == []
    got = reached_rows(sc, recs[1:-1])
    assert got[-1] > 0 and got[sc.rows] > 0 and got[sc.rows - 1] > 0, (name, got)
    if sc.height % 16:
        assert sc.height != 16 * sc.rows  # the repack path on the device
    for b in range(min(sc.n, 3)):
        assert recs[b]["counts"].total > 0


@pytest.mark.parametrize("name", [n for n in pls.IN_LIMIT if pls.SCENES[n].specs is not None])
def test_model_counts_are_the_oracles(oracle_api, name):
    """line_model's segment count of a frame equals the oracle's rasterize_only of the composition
    put into that pose (the first three frames and the last)."""
    sc = pls.SCENES[name]
    _, recs = models(oracle_api, name)
    comp, orders = sc.build(oracle_api)
    r = oracle_api.Renderer(0)
    for b in sorted({0, 1, 2, sc.n - 1} & set(range(sc.n))):
        pfs.set_pose_fill(comp, sc, orders, b)
        assert int(r.rasterize_only(comp, sc.width, sc.height).size) == recs[b]["counts"].total, (name, b)


def test_far_frames_lie_beyond_2p19(oracle_api):
    """The frames each scene lists as far are exactly those whose every line lies left of -2^19 px."""
    seen = 0
    for name in pls.IN_LIMIT:
        sc = pls.SCENES[name]
        if sc.specs is None or sc.big:
            continue
        _, recs = models(oracle_api, name)
        assert far_frames(recs) == list(sc.far), name
        seen += len(sc.far)
    assert seen >= 2


def test_far_up_line_wraps_its_rows(oracle_api):
    _, recs = models(oracle_api, "far_up")
    for b in (1, 2):
        rec = recs[b]
        lo = np.minimum(rec["y0"], rec["y0"] + rec["dy"])
        hi = np.maximum(rec["y0"], rec["y0"] + rec["dy"])
        assert np.any(rec["keep"] & (lo < -32770 * 256.0) & (hi > 0)), b
    assert not np.any(recs[0]["keep"] & (recs[0]["orders"] == 0))  # below the frame in its own state


NONFINITE = {"far_translations", "lines_translations", "lines_translations_own", "lines_nan", "lines_nan_own"}


@pytest.mark.parametrize("name", [n for n in pls.IN_LIMIT if pls.SCENES[n].specs is not None and not pls.SCENES[n].big])
def test_surviving_lines_are_finite_or_named(oracle_api, name):
    """No kept line of an in-limit scene has a non-finite end point, except in the scenes there for
    it, which do have one; no kept line's length saturates."""
    _, recs = models(oracle_api, name)
    nonfinite = 0
    for rec in recs:
        k = rec["keep"]
        ends = np.concatenate([e[k] for e in rec["end_points"]])
        nonfinite += int(np.sum(~np.isfinite(ends)))
        assert not rec["saturated"].any()
    assert (nonfinite > 0) == (name in NONFINITE), (name, nonfinite)


@pytest.mark.parametrize("name", pls.IN_LIMIT)
def test_in_limit_calls_fit_the_budgets(oracle_api, name):
    """Per call (a chunk of max_views(height) frames for the binding): at most 50 M segments, 20 M
    point pairs visited and 1 GB of pose records and pose style table; every frame below 2^30."""
    sc = pls.SCENES[name]
    comp, orders, n_points = build_counting_points(oracle_api, sc)
    assert orders and all(0 <= o < pls.ps.LAYER_LIMIT for o in orders)
    if name.startswith("crowded_"):
        assert orders[-1] < sc.first_order + sc.n_orders, (name, orders[-1])  # the window covers every layer
    n_call = min(sc.n, pls.max_views(sc.height))
    records = 32 * n_call * sc.n_orders
    styles = 112 * (len(orders) + n_call * sc.n_orders) if sc.colors is not None else 0
    assert records + styles <= pls.TABLE_BUDGET, (name, records, styles)
    assert 0 < n_points and n_call * n_points <= pls.POINT_BUDGET, (name, n_points)
    if sc.specs is not None:
        _, recs = models(oracle_api, name)
        totals = [rec["counts"].total for rec in recs]
    else:
        r = oracle_api.Renderer(0)
        totals = []
        for b in range(sc.n):
            pfs.set_pose_fill(comp, sc, orders, b)
            totals.append(int(r.rasterize_only(comp, sc.width, sc.height).size))
    assert all(t < lm.SEGMENT_LIMIT for t in totals)
    for c in range(0, sc.n, n_call):
        assert sum(totals[c:c + n_call]) <= pls.SEGMENT_BUDGET, (name, c)
    assert sum(totals) > 0


def test_refusal_scenes_are_refused_by_their_counts(oracle_api):
    """Every frame below 2^30 segments, the call's saturated total at 2^30 or more (segment_limit
    below 2^32 - 1, segment_saturate at it): refused at the count, before any buffer is sized."""
    for name in pls.OVER_LIMIT:
        sc = pls.SCENES[name]
        _, recs = models(oracle_api, name)
        totals = [rec["counts"].total for rec in recs]
        assert all(rec["counts"].status == lm.FORMA_OK for rec in recs), name
        assert all(0 < t < lm.SEGMENT_LIMIT for t in totals), (name, totals)
        device_total = min(sum(totals), lm.U32_MAX)
        assert device_total >= lm.SEGMENT_LIMIT, name
        assert (device_total == lm.U32_MAX) == (sc.kind == "saturate"), (name, sum(totals))
        assert sc.n <= pls.max_views(sc.height)


def _window_direct(order, first_order, n_orders, b):
    """The record of a layer inside [first_order, first_order + K), written out with both ends."""
    return b * n_orders + order - first_order if first_order <= order < first_order + n_orders else None


def test_window_compare(oracle_api):
    sc = pls.SCENES["window_from_1"]
    for b in range(sc.n):
        assert pls.frame_layers(sc, b) == pls.frame_layers(sc, b, _window_direct)
    assert pls.record_index(0, 1, 3, 2) is None and pls.record_index(3, 1, 3, 2) == 8
    assert pls.record_index(ps.LAYER_LIMIT - 1, 0, ps.LAYER_LIMIT, 1) == 2 * ps.LAYER_LIMIT - 1


def test_planted_errors_are_caught(oracle_api):
    """Errors planted in the checks above are reported: a frame bound of (b + 1) rows - 1, a remap of
    every row into the stack, a window compare without the unsigned wrap, a far-left rule at 2^18."""
    caught = []
    for name in pls.STACKS + pls.ODD:
        sc = pls.SCENES[name]
        _, recs = models(oracle_api, name)
        short = stack_violations(sc, recs, bound=lambda b, rows: (b + 1) * rows - 1)
        moved = stack_violations(sc, recs, remap=False)
        assert short and moved, name
        caught.append((name, len(short), len(moved)))
    sc = pls.SCENES["window_from_1"]
    signed = lambda o, f, k, b: pls.record_index(o, f, k, b, wrap=False)  # noqa: E731
    wrong = [b for b in range(sc.n) if pls.frame_layers(sc, b, signed) != pls.frame_layers(sc, b)]
    assert wrong == list(range(sc.n)), wrong
    pts, recs = models(oracle_api, "window_from_1")
    for b in range(1, sc.n):
        assert not np.array_equal(pls.frame_model(sc, pts, b, signed)["x0"], recs[b]["x0"]), b
    # A far scene whose far frames move only 2^18 px left is not one: the check does not list them.
    far = pls.SCENES["far_left"]
    t = far.transforms.copy()
    t[list(far.far), :, 4] = -(2.0 ** 18)
    near = pls.LimitScene("near_left", "", far.build, far.width, far.height, 0, lambda: (t, far.visible, None), far.specs)
    pts = pls.points(oracle_api, near)
    assert far_frames([pls.frame_model(near, pts, b) for b in range(near.n)]) == []
    print("planted errors caught:", caught, "window frames:", wrong, "near-left frames: none listed")
