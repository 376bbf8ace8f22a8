"""CPU checks of the stage-1 scenes (tests/flatten_scenes.py) before any of them reaches a
device: for every path, plain and through the transforms, tests/flatten_model.py replays the
indexing of flatten_eval_kernel over the host-built records and finds every index in range, the
kernel's quad choice equals the reference's quad walk, the point count and contour flags equal
the oracle's, and the scene passes its pre-flight budget. Each scene also reaches its target
condition, and the model itself is pinned on hand-made records."""
import numpy as np
import pytest

import flatten_model as fm
import flatten_scenes as fs
from forma_b200.binding import POINT_REC, QUAD_REC, SPLINE_REC


class Recorder:
    """Stands in for a Composition: records what the scene builders insert."""

    def __init__(self):
        self.inserts = []

    def get_mut_or_insert_default(self, order):
        return _RecordedLayer(self, order)


class _RecordedLayer:
    def __init__(self, rec, order):
        self.rec, self.order = rec, order

    def insert(self, path):
        self.rec.inserts.append((self.order, path))
        return self

    def set_props(self, props):
        return self


def recorded(api, build):
    rec = Recorder()
    build(api, rec)
    return [p for _, p in rec.inserts]


def check_path(pc, po, what, device=True, within_bounds=True):
    prog = pc.program()
    r = fm.check_program(prog)
    assert r["mismatch"] is None, f"{what}: {r['mismatch']}"
    n = prog["stats"]["points"]
    assert len(r["kind"]) == n
    x, y, c = po.segments()
    assert len(x) == n, f"{what}: {n} points in the program, {len(x)} in the oracle"
    assert np.array_equal(r["contour"], c.astype(bool)), f"{what}: contour flags differ from the oracle's"
    if prog["bounded"] and n and np.isfinite(y).all() and within_bounds:
        # the band filter's premise: every point lies within the program's bounds widened by the
        # margin Composition::layer_insert adds (0.5 px + 1e-4 of the magnitude)
        lo, hi = float(prog["bounds"][1]), float(prog["bounds"][3])
        margin = 0.5 + 1e-4 * max(abs(lo), abs(hi))
        assert lo - margin <= y.min() and y.max() <= hi + margin, f"{what}: points leave the program's bounds"
    if device:
        fm.assert_preflight(fm.preflight(n), what)
    return prog


@pytest.mark.parametrize("name", list(fs.PATHS))
def test_path_scene_replays_in_range_and_walks_like_the_reference(cuda_api, oracle_api, name):
    sc = fs.PATHS[name]
    pcs, pos = sc.build(cuda_api), sc.build(oracle_api)
    assert len(pcs) == len(pos) and pcs
    for i, (pc, po) in enumerate(zip(pcs, pos)):
        check_path(pc, po, f"{name} path {i}", sc.device)
        if sc.transforms:
            for tn, m in fs.TRANSFORMS.items():
                check_path(pc.transform(m), po.transform(m), f"{name} path {i} {tn}", within_bounds=False)
            for a, b in fs.CHAINS:
                check_path(pc.transform(fs.TRANSFORMS[a]).transform(fs.TRANSFORMS[b]),
                           po.transform(fs.TRANSFORMS[a]).transform(fs.TRANSFORMS[b]), f"{name} path {i} {a}+{b}",
                           within_bounds=False)
        if not sc.finite or sc.transforms:
            for tn, m in fs.DEGENERATE_TRANSFORMS.items():
                check_path(pc.transform(m), po.transform(m), f"{name} path {i} {tn}", device=False, within_bounds=False)


@pytest.mark.parametrize("name", list(fs.RENDER) + [f"band_{n}" for n in fs.BANDS])
def test_render_scene_batch_and_budget(cuda_api, oracle_api, oracle_renderer, name):
    """The scene's inserts staged as one batch replay in range and walk like the reference, and
    the whole frame passes the pre-flight budget."""
    sc = fs.BANDS[name[5:]] if name.startswith("band_") else fs.RENDER[name]
    progs = [p.program() for p in recorded(cuda_api, sc.build)]
    b = fm.layout(progs, geom_ids=range(1, len(progs) + 1), has_xf=[i % 2 == 0 for i in range(len(progs))])
    r = fm.replay(b)
    assert fm.reference_walk_mismatch(b, r) is None
    assert set(np.unique(r["job"])) == set(range(len(progs))) - {j for j, p in enumerate(progs) if p["stats"]["points"] == 0}
    comp = oracle_api.Composition()
    sc.build(oracle_api, comp)
    budget = fm.preflight(b.n_points, oracle_renderer, comp, sc.width, sc.height)
    fm.assert_preflight(budget, name)
    assert budget.segments > 0


# ---------------------------------------------------------------------------
# Target conditions
# ---------------------------------------------------------------------------
def _prog(api, name, i=0):
    return fs.PATHS[name].build(api)[i].program()


def test_long_spline_targets(cuda_api):
    p = _prog(cuda_api, "spiral_1e5")
    assert p["stats"]["quads"] == fs.SPIRAL_QUADS and p["splines"]["n_quads"].max() == fs.SPIRAL_QUADS, "one spline"
    assert p["stats"]["points"] > fs.SPIRAL_QUADS
    chain = _prog(cuda_api, "collinear_chain")
    t = chain["quads"]["total"]
    assert np.array_equal(t, 2.0 * np.arange(1, len(t) + 1, dtype=np.float32)), "every collinear quad adds exactly 2.0"
    for i, n in enumerate((1, 4, 64, 1000)):
        p = _prog(cuda_api, "collinear_then_curve", i)
        t, s = p["quads"]["total"], p["splines"]
        assert len(t) == n + 1 and np.array_equal(t[:-1], 2.0 * np.arange(1, n + 1, dtype=np.float32))
        if n >= 4:  # spline records: the kernel bisects, and pi meets a collinear total exactly
            assert s["step"][0] < 1.0 and (s["info"][0] & fm.EVAL_MASK) >= t[-2], "pi reaches the last collinear total"
    lag = _prog(cuda_api, "lagging_walk_small")
    t = lag["quads"]["total"]
    assert t[4095] == 8192.0 and t[4096] == 8193.0, "the quad after the chain adds exactly 1"
    assert lag["stats"]["splines"] == 0 and (lag["kinds"] == 3).any(), "the lagging walk is recorded point by point"


def test_curvature_past_2p25_targets(cuda_api):
    keeps = _prog(cuda_api, "spiral_2p25_keeps_up")
    assert keeps["quads"]["total"].max() >= 2.0 ** 25 and keeps["stats"]["points"] > 2 ** 25
    assert keeps["stats"]["splines"] > 0, "spline records while the walk keeps up"
    stalled = _prog(cuda_api, "spiral_2p25_stalled")
    t = stalled["quads"]["total"]
    assert t.max() >= 2.0 ** 25 and (t[1:] == t[:-1]).any(), "a quad past 2^25 adds nothing"
    assert stalled["stats"]["splines"] == 0 and (stalled["kinds"] == 3).any()
    assert stalled["stats"]["points"] > fm.POINT_CAP, "beyond the device budget: CPU only"


def test_encoding_crossover_targets(cuda_api):
    p47, p48 = (_prog(cuda_api, "encodings", i) for i in range(2))
    assert p47["stats"]["points"] == 47 and p47["stats"]["point_records"] == 47 and p47["stats"]["splines"] == 0
    assert p48["stats"]["points"] == 48 and p48["stats"]["splines"] == 12
    assert 36 * p48["stats"]["splines"] == 9 * p48["stats"]["points"]
    progs = [p.program() for p in recorded(cuda_api, fs.render_encodings)]
    kinds = ["points" if p["stats"]["splines"] == 0 else "splines" for p in progs]
    assert all(a != b for a, b in zip(kinds[:-2], kinds[1:-2])), "the encodings alternate job by job"
    assert [p["stats"]["points"] for p in progs[-2:]] == [47, 48]


def test_rational_targets(cuda_api):
    ps = [p.program() for p in fs.rational(cuda_api)]
    assert any(p["stats"]["rational"] for p in ps) and not all(p["stats"]["rational"] for p in ps)
    # the cubic `mult` factor: the same cubic with weights 1e3 subdivides into more quads than with 1
    cubic = {w: ps[3 * i + 1]["stats"]["quads"] for i, w in enumerate(fs.WEIGHTS)}
    assert cubic[1e3] > 100 * cubic[1.0]
    bad = [p.program() for p in fs.degenerate_weights(cuda_api)]
    negative_quads = [p for i, p in enumerate(bad) if fs.BAD_WEIGHTS[i // 3] < 0 and i % 3 == 0]
    assert negative_quads and not any(p["bounded"] for p in negative_quads), "no hull bound without positive weights"
    mixed = [p.program()["stats"]["rational"] for p in recorded(cuda_api, fs.render_rational_mix)]
    assert any(mixed) and not all(mixed)


def _shares(pc, m):
    a, b = pc.program(), pc.transform(m).program()
    return all(np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)) for k in ("splines", "points", "quads"))


def test_transform_boundary_targets(cuda_api):
    """Which transforms are geometry preserving (the transformed path shares the program)."""
    pc = fs.transform_sample(cuda_api)[0]
    expect = {"identity": True, "translate": True, "sx_at_limit": True, "sx_above_limit": False, "sx_limit_value": False,
              "sx_limit_value_up": False, "sy_at_limit": True, "sy_above_limit": False, "m8_two": True, "m8_eps": True,
              "m8_2eps": True, "m8_half": True, "m6_at_eps": True, "m6_above_eps": False, "m7_at_eps": True,
              "m7_above_eps": False, "reflect_x": True, "reflect_y": True, "swap_xy": True, "scale_up_2": False,
              "scale_down_half": True, "projective": False, "projective_strong": False, "rotate_37_shrink": True}
    got = {k: _shares(pc, fs.TRANSFORMS[k]) for k in expect}
    assert got == expect
    sx = np.float32(fs.SX_EDGE)
    assert sx * sx == np.float32(1.0 + fs.MAX_ERROR / 65536.0), "the squared scale sits exactly at the limit"
    rot = [_shares(pc, fs.TRANSFORMS[f"rotate_{15 * k}"]) for k in range(24)]
    assert any(rot), "rotations that stay geometry preserving"
    # chained: a geometry-preserving transform replaces the first one
    a = pc.transform(fs.TRANSFORMS["rotate_30"]).transform(fs.TRANSFORMS["translate"])
    assert _shares(pc, fs.TRANSFORMS["translate"]) and all(
        np.array_equal(a.program()[k].view(np.uint8), pc.program()[k].view(np.uint8)) for k in ("splines", "quads"))


def test_band_scene_targets(cuda_api):
    rot = recorded(cuda_api, fs.band_rotated)
    base = rot[0].program()
    assert all(_shares_prog(base, p.program()) for p in rot), "rotations are geometry preserving"
    rat = [p.program() for p in recorded(cuda_api, fs.band_rational_outside)]
    assert all(p["bounded"] for p in rat)
    ext = [e for e in fs._edges()]
    for (edge, body, y_ext), p in zip(ext, rat):
        q = p["quads"][0]
        y1 = q["py"][1] / q["pw"][1]
        assert (y1 - y_ext) * body < -1.0, "the control point lies beyond the curve's apex"
        assert abs(q["py"][0] - y_ext) >= 29.0, "the end points lie far from the extreme row"
    gaps = sorted({round(abs(y - e), 2) for e, _, y in ext})
    assert gaps[0] == 0.0 and gaps[-1] == 1.0 and len(gaps) == len(fs.EDGE_GAPS)
    unb = [p.program() for p in recorded(cuda_api, fs.band_unbounded)]
    assert not any(p["bounded"] for p in unb) and all(np.isfinite(p["quads"]["total"]).all() for p in unb)


def _shares_prog(a, b):
    return all(np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)) for k in ("splines", "points", "quads"))


# ---------------------------------------------------------------------------
# The model on hand-made records
# ---------------------------------------------------------------------------
def _spline(first_quad, n_quads, first_point, evaluated, start=True, ends=False, step=1.0):
    s = np.zeros(1, SPLINE_REC)
    s["first_quad"], s["n_quads"], s["first_point"], s["step"] = first_quad, n_quads, first_point, step
    s["info"] = evaluated | (int(start) << 30) | (int(ends) << 31)
    return s


def _quads(totals):
    q = np.zeros(len(totals), QUAD_REC)
    q["total"] = np.asarray(totals, np.float32)
    return q


def _prog_of(splines=(), points=None, kinds=None, quads=(), n=0):
    return {"splines": np.concatenate(splines) if len(splines) else np.zeros(0, SPLINE_REC),
            "points": points if points is not None else np.zeros(0, POINT_REC),
            "kinds": kinds if kinds is not None else np.zeros(0, np.uint8),
            "quads": _quads(quads), "stats": {"points": n}}


def test_model_bisection_and_walk_on_hand_made_records():
    # spline 0: quads totals 2, 3 (C = 3, S = 3, E = 2): pi 1, 2 -> quad 0; the walk ends there and
    # steps to quad 1, inside the same spline; spline 1 (one quad) is then walked from quad 1
    p = _prog_of([_spline(0, 2, 0, 2), _spline(2, 1, 4, 2)], quads=[2.0, 3.0, 2.5], n=8)
    r = fm.check_program(p)
    assert r["kind"].tolist() == [0, 2, 2, 0, 0, 2, 2, 0]
    assert r["quad"].tolist() == [-1, 0, 0, -1, -1, 2, 2, -1]
    assert r["pi"].tolist() == [0, 1, 2, 0, 0, 1, 2, 0]
    m = r["mismatch"]
    assert (m.point, m.kernel, m.walk) == (5, 2, 1)
    # totals 2, 4: in step; the second spline starts on its own quad
    p = _prog_of([_spline(0, 2, 0, 3), _spline(2, 1, 5, 2)], quads=[2.0, 4.0, 2.5], n=9)
    r = fm.check_program(p)
    assert r["quad"].tolist() == [-1, 0, 0, 1, -1, -1, 2, 2, -1] and r["mismatch"] is None
    # the gid: None at contour ends and on the last point of the insert
    p = _prog_of([_spline(0, 0, 0, 0, ends=True), _spline(0, 0, 2, 0)], n=4)
    b = fm.layout([p, p], geom_ids=[7, 9])
    r = fm.replay(b)
    assert r["gid"].tolist() == [7, 0, 7, 0, 9, 0, 9, 0] and r["contour"].tolist() == [0, 1, 0, 0] * 2


@pytest.mark.parametrize("broken", ["no_quad", "quad_outside_job", "points_overrun", "unsorted_totals", "kind"])
def test_model_rejects_broken_records(broken):
    if broken == "no_quad":
        p = _prog_of([_spline(0, 0, 0, 2)], n=4)
    elif broken == "quad_outside_job":
        pts = np.zeros(3, POINT_REC)
        pts["a"] = np.array([0, 5, 0], np.uint32).view(np.float32)
        p = _prog_of(points=pts, kinds=np.array([0, 2, 0], np.uint8), quads=[2.0], n=3)
    elif broken == "points_overrun":
        p = _prog_of([_spline(0, 1, 0, 2)], quads=[3.0], n=6)
    elif broken == "unsorted_totals":
        p = _prog_of([_spline(0, 2, 0, 3)], quads=[3.0, 2.5], n=5)
    else:
        p = _prog_of(points=np.zeros(2, POINT_REC), kinds=np.array([0, 7], np.uint8), n=2)
    with pytest.raises(fm.ModelError):
        fm.replay(fm.layout([p]))


def test_budget_reports_every_excess():
    assert fm.Budget(10, 10, 0).problems() == []
    assert len(fm.Budget(fm.POINT_CAP + 1, fm.SEGMENT_CAP + 1, 2).problems()) == 3
    with pytest.raises(AssertionError):
        fm.assert_preflight(fm.Budget(1, None, 1), "scene")
