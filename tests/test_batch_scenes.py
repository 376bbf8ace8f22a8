"""The batch scenes (tests/batch_scenes.py) on the CPU, before any of them reaches a GPU: every
in-limit scene fits the frame and segment budgets, the limit scenes sit exactly at their
limit, and the order bases follow the slice rule."""
import numpy as np
import pytest

import batch_scenes as bs
import line_model as lm
import view_scenes as vs


def _counts(comps):
    return {id(c): bs.n_orders(c) for c in comps}


@pytest.mark.parametrize("name", [n for n in bs.IN_LIMIT if n != "orders_at_limit"])
def test_batches_fit_budget(oracle_api, name):
    sc = bs.SCENES[name]
    assert 1 <= len(sc.frames) <= bs.max_frames(sc.height)
    distinct, frames = bs.build(oracle_api, sc)
    r = oracle_api.Renderer(0)
    segs = [int(r.rasterize_only(c, sc.width, sc.height).size) for c in distinct]
    total = sum(segs[k] for k in sc.frames)
    assert 0 < total <= bs.SEGMENT_BUDGET, (name, total)
    assert bs.order_sum(frames, _counts(distinct)) <= bs.ORDER_FIELD


def test_limit_scenes_are_at_the_limit():
    for name in bs.LIMIT_SCENES:
        sc = bs.SCENES[name]
        assert len(sc.frames) == bs.max_frames(sc.height)
        assert (len(sc.frames) + 1) * bs.rows(sc.height) > 2046
    assert len(bs.SCENES["limit_h16"].frames) * bs.rows(16) == 2046
    assert bs.max_frames(16) == 2046 and bs.max_frames(1000) == 32


def test_order_limit_scenes(oracle_api):
    at, frames = bs.build(oracle_api, bs.SCENES["orders_at_limit"])
    assert bs.order_sum(frames, _counts(at)) == bs.ORDER_FIELD
    over, frames = bs.build(oracle_api, bs.SCENES["orders_over"])
    assert bs.order_sum(frames, _counts(over)) == bs.ORDER_FIELD + 1


def test_segment_limit_scene_is_over_only_together(oracle_api):
    sc = bs.SCENES["segment_limit"]
    assert sc.frames == [0, 0]
    # view_scenes' segment_limit is the same composition (64 x 64): its identity view is this frame.
    one = int(vs.view_model(oracle_api, vs.SCENES["segment_limit"], vs.IDENTITY)["counts"].total)
    assert one < lm.SEGMENT_LIMIT <= 2 * one, one


def test_order_bases_follow_the_slice_rule(oracle_api):
    distinct, frames = bs.build(oracle_api, bs.SCENES["repeats"])  # A, B, A, C, A
    a, b, c = (bs.n_orders(x) for x in distinct)
    assert bs.order_bases(frames, _counts(distinct)) == [0, a, 0, a + b, 0]
    distinct, frames = bs.build(oracle_api, bs.SCENES["degenerate"])  # covers, empty, disabled, sparse, radial, empty
    n = [bs.n_orders(x) for x in distinct]
    assert n[1] == 0 and n[3] == 1_000_001
    assert bs.order_bases(frames, _counts(distinct)) == [0, n[0], n[0], n[0] + n[2], n[0] + n[2] + n[3], n[0]]
    distinct, frames = bs.build(oracle_api, bs.SCENES["clip_leak"])
    # the Clip(1000) of the first composition reaches into the second one's slice if slices leaked
    assert bs.n_orders(distinct[0]) < 1 + 1000


def test_paris_tiles_cover_the_drawing():
    """Every tile gets paths, and together they hold every path that meets the drawing's frame."""
    p = bs._paris_paths()
    lo = np.minimum.reduceat(p.pts, p.pt_off[:-1], axis=0) * bs.PARIS_SCALE
    hi = np.maximum.reduceat(p.pts, p.pt_off[:-1], axis=0) * bs.PARIS_SCALE
    inside = (hi[:, 0] >= 0) & (lo[:, 0] <= 1920) & (hi[:, 1] >= 0) & (lo[:, 1] <= 1080)
    sizes = [len(bs.paris_tile_paths(k)) for k in range(16)]
    assert min(sizes) > 0
    assert sum(sizes) >= int(inside.sum())
