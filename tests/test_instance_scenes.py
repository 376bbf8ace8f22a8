"""The instance scenes (tests/instance_scenes.py) without a GPU: each is well formed for one call of
Renderer.render_instances_device, reaches the case it is there for, and its twins render on the
oracle and differ where the scene says they do."""
import numpy as np
import pytest

import instance_scenes as ins
from forma_b200.binding import RGBA, Color

CLEAR = Color(1.0, 1.0, 1.0, 0.0)


def _max_views(height):
    return 2046 // ((height + 15) // 16)


def _render(api, r, comp, sc):
    buf = np.zeros(sc.width * sc.height * 4, np.uint8)
    r.render(comp, buf, sc.width, sc.height, RGBA, CLEAR)
    return buf.reshape(sc.height, sc.width, 4)


@pytest.mark.parametrize("name", list(ins.SCENES))
def test_scene_is_well_formed(name):
    sc = ins.SCENES[name]
    assert sc.prototypes.dtype == np.uint32 and sc.prototypes.ndim == 2 and sc.m >= 1
    assert 1 <= sc.n <= _max_views(sc.height), "one call takes the whole scene"
    assert sc.n * sc.m <= ins.LAYER_LIMIT
    for t, width in ((sc.transforms, 6), (sc.colors, 4)):
        assert t is None or (t.dtype == np.float32 and t.shape == (sc.n, sc.m, width))
    orders = {p.order for p in sc.protos}
    assert len(orders) == len(sc.protos), "one spec per prototype order"
    used = {int(p) for p in sc.prototypes.ravel() if p != ins.NONE}
    assert used <= orders, "every prototype is a layer of the library"
    for a, b in sc.differ:
        assert 0 <= a < sc.n and 0 <= b < sc.n


def test_scenes_reach_their_cases():
    S = ins.SCENES
    rep = S["repeats"].prototypes
    assert any(len(set(row[row != ins.NONE])) < np.count_nonzero(row != ins.NONE) for row in rep), "a prototype repeated in a frame"
    assert np.any(rep == ins.NONE) and np.all(rep[3] == ins.NONE), "empty slots and an empty frame"
    assert list(rep[0, :2]) == list(rep[1, 1::-1]), "a pair of shapes in reversed orders"
    assert any(not p.enabled for p in S["repeats"].protos), "a disabled prototype"
    protos = {p.order: p for p in S["inserts"].protos}
    assert len(protos[5].paths) == 2 and protos[5].path_xf is not None, "two inserts with a path transform"
    assert protos[6].cleared and protos[6].paths, "a prototype cleared and drawn again"
    assert not protos[9].paths, "a prototype without geometry"
    fills = [p.props.func.draw.fill for p in S["styles"].protos]
    assert any(f.gradient is not None for f in fills) and any(f.texture is not None for f in fills)
    assert S["styles"].colors is None
    assert S["colors_blend"].colors is not None
    assert any(p.props.func.draw.blend_mode >= 12 for p in S["colors_blend"].protos), "a non-separable blend mode"
    clip = [p for p in S["clip_leak"].protos if p.props.func.clip is not None]
    assert clip and clip[0].props.func.clip > S["clip_leak"].m, "a clip range past the frame's slots"
    t = S["nonfinite"].transforms[..., 4:]
    assert np.isnan(t).any() and np.isinf(t).any()
    lib = S["library_511x64"]
    assert (lib.n, lib.m, lib.width, lib.height, len(lib.protos)) == (511, 8, 64, 64, 64)
    g = S["glyphs_1080p"]
    assert g.n == 1 and g.m >= 20000 and (g.width, g.height) == (1920, 1080) and 80 <= len(g.protos) <= 100


@pytest.mark.parametrize("name", ins.LIGHT)
def test_twins_render_and_differ(oracle_api, name):
    sc = ins.SCENES[name]
    r = oracle_api.Renderer(0)
    frames = [_render(oracle_api, r, ins.twin(oracle_api, sc, b), sc) for b in range(sc.n)]
    clear = np.array([255, 255, 255, 0], np.uint8)
    for b, f in enumerate(frames):
        empty = np.all(sc.prototypes[b] == ins.NONE)
        assert bool(np.all(f == clear)) == bool(empty), f"{name}: frame {b} drawn iff it has an instance"
    for a, b in sc.differ:
        assert not np.array_equal(frames[a], frames[b]), f"{name}: frames {a} and {b} should differ"


def test_library_is_invisible_on_its_own(oracle_api):
    """The disabled library draws nothing in an ordinary frame: what an instance frame shows comes
    from the instances alone."""
    sc = ins.SCENES["repeats"]
    r = oracle_api.Renderer(0)
    lib = ins.build_library(oracle_api, sc)
    f = _render(oracle_api, r, lib, sc)
    enabled = [p for p in sc.protos if p.enabled]
    assert enabled and sum(1 for p in sc.protos if not p.enabled) >= 5
    for p in sc.protos:
        if not p.enabled:
            lib.get(p.order).enable()
    g = _render(oracle_api, r, lib, sc)
    assert not np.array_equal(f, g)


def test_dead_inserts_would_show(oracle_api):
    """The cleared prototype's dead geometry covers pixels its live geometry does not: drawing it
    would change frame 0."""
    sc = ins.SCENES["inserts"]
    r = oracle_api.Renderer(0)
    want = _render(oracle_api, r, ins.twin(oracle_api, sc, 0), sc)
    protos = [ins.Proto(p.order, p.cleared + p.paths, p.path_xf, p.props, p.xf, p.enabled) for p in sc.protos]
    wrong = ins.InstanceScene(sc.name, protos, sc.width, sc.height, sc.prototypes)
    assert not np.array_equal(want, _render(oracle_api, r, ins.twin(oracle_api, wrong, 0), wrong))


def test_reversed_pair_overlaps(oracle_api):
    """Frames 0 and 1 of `repeats` draw the same hexagon and bar in the same places, stacked the
    other way round, so they differ only where the two overlap."""
    sc = ins.SCENES["repeats"]
    assert list(sc.transforms[0, 0]) == list(sc.transforms[1, 1]) and list(sc.transforms[0, 1]) == list(sc.transforms[1, 0])
    r = oracle_api.Renderer(0)
    f0, f1 = (_render(oracle_api, r, ins.twin(oracle_api, sc, b), sc) for b in (0, 1))
    differ = np.any(f0 != f1, axis=2)
    ys, xs = np.nonzero(differ)
    # hexagon of radius 11 at (30, 30), bar [-5, 5] x [-14, 14] at (34, 33): they overlap in [29, 39] x [19, 41]
    assert differ.any() and 28 <= xs.min() and xs.max() <= 40 and 18 <= ys.min() and ys.max() <= 42


def test_heavy_twins_render(oracle_api):
    """A few frames of the library scene and the glyph page render on the oracle and draw."""
    r = oracle_api.Renderer(0)
    for name, frames in (("library_511x64", (0, 1, 510)), ("glyphs_1080p", (0,))):
        sc = ins.SCENES[name]
        out = [_render(oracle_api, r, ins.twin(oracle_api, sc, b), sc) for b in frames]
        for f in out:
            assert np.count_nonzero(np.any(f != np.array([255, 255, 255, 0], np.uint8), axis=2)) > 0.05 * sc.width * sc.height
        if len(out) > 1:
            assert not np.array_equal(out[0], out[1])
