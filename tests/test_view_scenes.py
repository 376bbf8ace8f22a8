"""The view scenes (tests/view_scenes.py) on the CPU, before any of them reaches a GPU: every
composed transform is one the oracle accepts, every scene reaches its target, and every in-limit
call fits the segment budget (the refusal scene's total is only counted)."""
import numpy as np
import pytest

import line_model as lm
import view_scenes as vs

MAX_VIEWS = lambda h: 0 if h == 0 or h > 32768 else 2046 // ((h + 15) // 16)  # noqa: E731  (forma_renderer_max_views)


def _oracle_segments(oracle_api, sc):
    """Segments of every view, from the oracle's line setup of the composed transforms."""
    comp, xf = vs.build(oracle_api, sc)
    r = oracle_api.Renderer(0)
    out = []
    for v in sc.views:
        vs.set_view(comp, xf, v)  # raises GeomPresTransformError if the oracle refuses a C
        out.append(int(r.rasterize_only(comp, sc.width, sc.height).size))
    return out


def test_compose_matches_float32_reference():
    rng = np.random.default_rng(3)
    for _ in range(200):
        v, t = rng.normal(size=6).astype(np.float32), rng.normal(size=6).astype(np.float32)
        c = vs.compose(v, t)
        # with exact products (float64) and one rounding per fma, as the formula is written
        f = lambda a, b, cc: np.float32(np.float64(a) * np.float64(b) + np.float64(cc))  # noqa: E731
        want = [f(v[0], t[0], np.float32(v[1] * t[2])), f(v[0], t[1], np.float32(v[1] * t[3])),
                f(v[2], t[0], np.float32(v[3] * t[2])), f(v[2], t[1], np.float32(v[3] * t[3])),
                f(v[0], t[4], f(v[1], t[5], v[4])), f(v[2], t[4], f(v[3], t[5], v[5]))]
        assert np.array_equal(np.float32(c), np.float32(want))
    assert vs.compose(vs.IDENTITY, None) == vs.IDENTITY


@pytest.mark.parametrize("name", vs.IN_LIMIT)
def test_views_fit_budget_and_oracle_accepts(oracle_api, name):
    sc = vs.SCENES[name]
    assert 1 <= len(sc.views) <= MAX_VIEWS(sc.height)
    for v in sc.views:
        assert np.all(np.isfinite(v))
    segs = _oracle_segments(oracle_api, sc)
    assert sum(segs) <= vs.SEGMENT_BUDGET, (name, sum(segs))
    assert sum(segs) > 0, name


def test_limit_scenes_are_at_the_limit():
    for name in vs.LIMIT_SCENES:
        sc = vs.SCENES[name]
        assert len(sc.views) == MAX_VIEWS(sc.height) and len(sc.views) * vs.rows(sc.height) >= 2016
    assert len(vs.SCENES["limit_h16"].views) * vs.rows(16) == 2046


@pytest.mark.parametrize("name", [n for n, s in vs.SCENES.items() if s.straddles])
def test_straddling_views_reach_both_edges(oracle_api, name):
    sc = vs.SCENES[name]
    both = 0
    for b, v in enumerate(sc.views):
        rec = vs.view_model(oracle_api, sc, v)
        above, below = vs.outside_rows(rec, sc.height)
        both += above > 0 and below > 0
        assert rec["counts"].status == lm.FORMA_OK
    assert both >= 3, name


def test_segment_limit_scene_is_over_only_together(oracle_api):
    sc = vs.SCENES["segment_limit"]
    totals = [int(vs.view_model(oracle_api, sc, v)["counts"].total) for v in sc.views]
    assert all(t < lm.SEGMENT_LIMIT for t in totals), totals
    assert sum(totals) >= lm.SEGMENT_LIMIT, totals


@pytest.mark.parametrize("name", ["far_compose", "far_compose_neg"])
def test_far_compose_views_depend_on_the_fma_nesting(name):
    sc = vs.SCENES[name]
    assert all(vs.nesting_matters(v, sc.specs[0].xf) for v in sc.views)


def test_far_points_views_depend_on_the_order_of_the_linear_terms(oracle_api):
    """Some of C.ux ... C.vy changes when its two products trade places, and so do the lines."""
    sc = vs.SCENES["far_points"]
    t = sc.specs[0].xf
    assert all(vs.linear_order_matters(v, t) for v in sc.views)
    _, _, inserts = vs.ls.build(oracle_api, sc.specs)
    x, y, ids = lm.point_buffer([(k, *p.segments()) for k, p in inserts])
    for v in sc.views:
        c = vs.compose(v, t)
        vux, vvx, vuy, vvy = (np.float32(a) for a in v[:4])
        tux, tvx, tuy, tvy = (np.float32(a) for a in t[:4])
        sw = [float(lm.fmaf(vvx, tuy, vux * tux)), float(lm.fmaf(vvx, tvy, vux * tvx)),
              float(lm.fmaf(vvy, tuy, vuy * tux)), float(lm.fmaf(vvy, tvy, vuy * tvx))] + c[4:]
        a = lm.replay(x, y, ids, [lm.LayerXf(s.order, c) for s in sc.specs], sc.width, sc.height, (0.0, float(sc.height)))
        b = lm.replay(x, y, ids, [lm.LayerXf(s.order, sw) for s in sc.specs], sc.width, sc.height, (0.0, float(sc.height)))
        assert a["keep"].any() and not np.array_equal(a["x0"], b["x0"])


def test_identity_rule_is_observable(oracle_api):
    """On inf_points, an identity applied as a transform keeps one more line than no transform."""
    sc = vs.SCENES["inf_points"]
    _, _, inserts = vs.ls.build(oracle_api, sc.specs)
    x, y, ids = lm.point_buffer([(k, *p.segments()) for k, p in inserts])
    totals = [lm.counts(lm.replay(x, y, ids, [lm.LayerXf(s.order, xf) for s in sc.specs], sc.width, sc.height,
                                  (0.0, float(sc.height)))["length"], len(x)).total for xf in (None, vs.IDENTITY)]
    assert totals[0] != totals[1], totals
