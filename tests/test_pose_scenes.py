"""The pose scenes on the CPU: every pose transform is one the composition could be set to, every
scene fits one call's limits (chunked over max_views), the spaceship poses are exactly
synth.spaceship_scene's animation, and the frames of a scene differ where they are meant to."""
import numpy as np
import pytest

import pose_scenes as ps
import synth
from forma_b200.binding import GeomPresTransformError

MAX_TILE_ROWS = 2046  # max_views(height) = 2046 // ceil(height / 16)


@pytest.mark.parametrize("name", list(ps.SCENES))
def test_pose_transforms_pass_set_transform(oracle_api, name):
    sc = ps.SCENES[name]
    if sc.transforms is None:
        return
    comp = oracle_api.Composition()
    layer = comp.get_mut_or_insert_default(0)
    rows = np.unique(sc.transforms.reshape(-1, 6).view(np.uint32), axis=0).view(np.float32)
    for t in rows:
        layer.set_transform([float(x) for x in t])  # raises GeomPresTransformError when refused


def test_a_scaling_pose_is_refused_by_the_oracle(oracle_api):
    layer = oracle_api.Composition().get_mut_or_insert_default(0)
    with pytest.raises(GeomPresTransformError):
        layer.set_transform([2.0, 0.0, 0.0, 2.0, 0.0, 0.0])


@pytest.mark.parametrize("name", list(ps.SCENES))
def test_scene_fits_the_call(name):
    sc = ps.SCENES[name]
    rows = (sc.height + 15) // 16
    per_call = MAX_TILE_ROWS // rows
    assert per_call >= 1
    assert sc.n_orders >= 1 and sc.first_order + sc.n_orders <= ps.LAYER_LIMIT
    if sc.transforms is not None and sc.visible is not None:
        assert sc.transforms.shape[:2] == sc.visible.shape
    if sc.transforms is not None:
        assert sc.transforms.dtype == np.float32 and sc.transforms.shape[2] == 6
    if name == "spaceship1080p":
        assert per_call == 30 and sc.n == 200  # 7 chunks: 6 x 30 + 20
    if name == "library_511x64":
        assert per_call == 511 and sc.n == 511  # one call at the limit


@pytest.mark.parametrize("name", [n for n in ps.LIGHT if not n.startswith("e2e_")] + ["e2e_clipping", "e2e_texture"])
def test_segments_within_budget(oracle_api, name):
    """Each pose frame of the light scenes stays far below the 2^30-segment limit, with room for
    every frame of one call (the oracle's segment count of the frame)."""
    sc = ps.SCENES[name]
    comp, orders = sc.build(oracle_api)
    r = oracle_api.Renderer(0)
    total = 0
    for b in range(sc.n):
        ps.set_pose(comp, sc, orders, b)
        buf = np.zeros(sc.width * sc.height * 4, np.uint8)
        total += r.render(comp, buf, sc.width, sc.height).n_segments
    assert 0 < total < (1 << 30) // 4


def _proxy_animate():
    """The transforms synth.spaceship_scene's animate(f) sets, recorded through a stand-in composition."""
    class _Rec:
        def __init__(self):
            self.xf = {}

        def get_mut_or_insert_default(self, order):
            return _Layer(self, order)

        def get(self, order):
            return _Layer(self, order)

    class _Layer:
        def __init__(self, rec, order):
            self.rec, self.order = rec, order

        def insert(self, path):
            return self

        def set_props(self, props):
            return self

        def set_transform(self, t):
            self.rec.xf[self.order] = list(t)
            return self

    class _Api:
        def PathBuilder(self):
            class _PB:
                def __getattr__(self, name):
                    return lambda *a: self
            return _PB()

    rec = _Rec()
    animate = synth.spaceship_scene(_Api(), rec, 400, 1920, 1080, 43)
    return rec, animate


def test_spaceship_poses_are_the_animation():
    sc = ps.SCENES["spaceship1080p"]
    rec, animate = _proxy_animate()
    for f in (0, 1, 57, 199):
        animate(f)
        want = np.asarray([rec.xf[o] for o in range(1, 402)], np.float32)
        assert np.array_equal(sc.transforms[f], want), f


@pytest.mark.parametrize("name", list(ps.SCENES))
def test_frames_differ_where_meant(name):
    sc = ps.SCENES[name]
    for a, b in sc.differ:
        same_t = sc.transforms is None or np.array_equal(sc.transforms[a].view(np.uint32), sc.transforms[b].view(np.uint32))
        same_v = sc.visible is None or np.array_equal(sc.visible[a], sc.visible[b])
        assert not (same_t and same_v), (name, a, b)


def test_scene_edges_are_reached():
    assert ps.SCENES["k1"].n_orders == 1
    top = ps.SCENES["window_top"]
    assert top.first_order + top.n_orders == ps.LAYER_LIMIT
    assert ps.SCENES["window_past_end"].first_order > 12  # the last attached order of its composition
    nf = ps.SCENES["nonfinite"].transforms
    assert np.isnan(nf).any() and np.isinf(nf).any()
    lib = ps.SCENES["library_511x64"]
    counts = lib.visible.sum(axis=1)
    assert counts.min() >= 1 and counts.max() < ps.LIBRARY_SHAPES
    assert ps.SCENES["paris_poses"].n_orders == ps.PARIS_LAYERS
