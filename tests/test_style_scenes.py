"""The style scenes (tests/style_scenes.py) without a GPU: every scene builds on the oracle, its
oracle f32 frame encodes to its oracle sRGB8 frame, and every condition it declares holds in
the path model built from the oracle's segments: each matrix cell reaches the path it was
built for with active and inactive f32x8 groups, every hostile value class reaches the fold,
fast, pair and generic paths, the gradient stack straddles the 32-entry groups with masked and
zero-coverage entries. A scene that stops reaching its path fails here, before it costs GPU
time. tests/test_gpu_styles.py then holds the device to the oracle's frames."""
import math

import numpy as np
import pytest

import oracle_linear
import style_scenes as ss
from forma_b200.binding import BGRA, RGB0, RGBA, FillRule

_MODELS = {}


@pytest.fixture(autouse=True)
def _setup(oracle_api):
    oracle_linear.attach(oracle_api)
    oracle_api.hooks.fo_set_recip_mode(0)


def model_of(oracle_api, name):
    """(PathModel, Built, StyleScene, oracle f32 frame) of scene `name`."""
    if name not in _MODELS:
        comp, built, sc = ss.build(oracle_api, name)
        frame = oracle_linear.render(oracle_api, comp, sc.width, sc.height, RGBA, sc.clear)
        r = oracle_api.Renderer(0)
        r.render(comp, np.zeros(sc.width * sc.height * 4, np.uint8), sc.width, sc.height, RGBA, sc.clear)
        _MODELS[name] = (ss.PathModel(r.segments(), sc.width, sc.height, built.layers), built, sc, frame)
    return _MODELS[name]


@pytest.mark.parametrize("name", list(ss.SCENES))
def test_scene_encodes_to_the_oracle(oracle_api, name):
    comp, _, sc = ss.build(oracle_api, name)
    orders = (RGBA, BGRA, RGB0) if sc.family in ("encoder", "defect", "hostile") else (RGBA,)
    for ch in orders:
        frame = oracle_linear.render(oracle_api, comp, sc.width, sc.height, ch, sc.clear)
        got = oracle_linear.encode(frame, ch)
        want = np.zeros(sc.width * sc.height * 4, np.uint8)
        oracle_api.Renderer(0).render(comp, want, sc.width, sc.height, ch, sc.clear)
        want = want.reshape(sc.height, sc.width, 4)
        if not np.array_equal(got, want):
            ys, xs = np.nonzero((got != want).any(axis=2))
            raise AssertionError(f"{name} {ch}: {len(ys)} pixels differ, first at x={xs[0]} y={ys[0]}: encoded "
                                 f"{got[ys[0], xs[0]]} from {frame[ys[0], xs[0]]}, sRGB8 oracle {want[ys[0], xs[0]]}")


@pytest.mark.parametrize("name", list(ss.SCENES))
def test_declared_conditions_hold(oracle_api, name):
    model, built, _, _ = model_of(oracle_api, name)
    fails = ss.check_expectations(model, built)
    assert not fails, f"{name}: {len(fails)} conditions fail, e.g. {fails[:5]}"


def test_matrix_reaches_every_cell_on_its_path(oracle_api):
    """10 fills x 16 modes x 4 clip states x 2 fill rules, each on the path it was built for."""
    seen = {}
    for name in [n for n, s in ss.SCENES.items() if s.family == "matrix"]:
        model, built, _, _ = model_of(oracle_api, name)
        for (layer, kind, mode, clip, rule, _), (lay2, tile, want, _, _) in zip(built.notes["cells"], built.expect):
            assert layer == lay2
            e = model.entry(tile, layer)
            seen[(kind, mode, clip, rule)] = e.path if e is not None else None
    assert len(seen) == len(ss.FILLS) * 16 * len(ss.CLIPS) * 2
    for (kind, mode, clip, rule), path in seen.items():
        want = "masked" if clip == "outside" else ss.expected_path(kind, mode)
        assert path == want, (kind, mode, clip, rule, path)
    for mode in range(12):  # e.g. every separable mode reaches the pair path with a 4-stop gradient
        assert seen[("lin4", mode, "none", FillRule.NonZero)] == "pair"
        assert seen[("lin5", mode, "none", FillRule.NonZero)] == "generic"


def test_every_hostile_class_reaches_every_path(oracle_api):
    reached = {cls: set() for cls in list(ss.HOSTILE) + ["alpha"]}
    nan_over_inactive = False
    for name in [n for n, s in ss.SCENES.items() if s.family in ("hostile", "fold", "defect")]:
        model, built, _, _ = model_of(oracle_api, name)
        for _, e in model.all_entries():
            props = built.layers[e.layer]
            for c in ss.layer_colors(props):
                for cls in ss.value_classes(c):
                    reached[cls].add(e.path)
                if e.path == "fast" and math.isnan(c.r) and e.active.any() and not e.active.all():
                    nan_over_inactive = True
    for cls, paths in reached.items():
        assert set(ss.PATHS) <= paths, f"class {cls} reaches only {sorted(paths)}"
    assert nan_over_inactive, "no tile has an inactive f32x8 group under a NaN solid Over layer"


def test_encoder_sweep_rows_fold_and_paint_the_same_colours(oracle_api):
    model, built, sc, frame = model_of(oracle_api, "encoder_sweep")
    srgb = oracle_linear.encode(frame, RGBA)
    for ty, _ in built.notes["solid_rows"]:
        rows = slice(16 * ty, 16 * ty + 16)
        assert (srgb[rows] == srgb[16 * ty, 0]).all(), f"tile row {ty}: folded and painted tiles encode differently"
    # the sweeps cross the sRGB knee and byte boundaries: many distinct bytes per row
    assert len(np.unique(srgb[0, :, 0])) > 4 and len(np.unique(srgb[16, :, 2])) > 150


def test_defect_scenes_keep_inactive_groups_in_the_oracle(oracle_api):
    """The reference leaves pixels without coverage in their f32x8 alone: the four active f32x8
    groups (columns 0-3 of rows 0-7) are blended, the other 224 of 256 pixels keep
    the clear colour (red 255, or the sign of a -0 clear)."""
    for name in ("defect_nan_r", "defect_inf_r", "defect_inf_a"):
        _, _, sc, frame = model_of(oracle_api, name)
        srgb = oracle_linear.encode(frame, RGBA)
        assert int((srgb[..., 0] == 255).sum()) == 224, name
    _, _, _, frame = model_of(oracle_api, "defect_neg_zero_clear")
    assert int(np.signbit(frame[..., 0]).sum()) == 224


def test_path_model_fold_tiles_are_one_colour(oracle_api):
    for name in [n for n, s in ss.SCENES.items() if s.family in ("fold", "encoder")]:
        model, _, _, frame = model_of(oracle_api, name)
        for (tx, ty), e in model.all_entries():
            if e.path == "fold":
                t = frame[16 * ty:16 * ty + 16, 16 * tx:16 * tx + 16].reshape(-1, 4)
                bits = t.view(np.uint32)
                same = (bits == bits[0]).all(axis=1) | (np.isnan(t) & np.isnan(t[0])).all(axis=1)
                assert same.all(), (name, tx, ty)
