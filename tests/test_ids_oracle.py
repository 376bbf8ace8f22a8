"""The oracle's ID frames (fo_renderer_render_ids, tests/oracle_ids.py), pinned without a GPU: against its own RGBA
frames, against a NumPy model built from its sorted segments, at hand-picked pixels of the clip
scenes, and on invalid arguments. tests/test_gpu_ids.py then holds the device to these IDs."""
import numpy as np
import pytest

import oracle_ids
import scenes
import synth
from forma_b200.binding import (ID_NONE, RGBA, BlendMode, Color, Fill, FillRule, FormaError, Func, Point, Props, Rect,
                                Style, unpack_segments)
from oracle import oracle

E2E_IDS = [n for n in scenes.E2E if n not in scenes.NON_SEPARABLE]


@pytest.fixture(autouse=True)
def _oracle_ids(oracle_api):
    oracle_ids.attach(oracle_api)


def sorted_segments(api, comp, w, h):
    """The oracle's sorted pixel segments of the frame (from an RGBA render)."""
    r = api.Renderer(0)
    r.render(comp, np.zeros(w * h * 4, np.uint8), w, h, RGBA, Color())
    return r.segments()


def ids_of(api, comp, w, h, min_coverage=0.0, crop=None, renderer=None):
    r = renderer if renderer is not None else api.Renderer(0)
    ids = np.zeros(w * h, np.uint32)
    r.render_ids(comp, ids, w, h, crop=crop, min_coverage=min_coverage)
    return ids.reshape(h, w)


def rgba_of(api, comp, w, h, clear):
    buf = np.zeros(w * h * 4, np.uint8)
    api.Renderer(0).render(comp, buf, w, h, RGBA, clear)
    return buf.reshape(h, w, 4)


def random_polygons(api, comp, n, w, h, seed, rule=None, opaque=False):
    """Clip-free polygons and stars with small windings; distinct colours. -> {order: Color}."""
    rng = synth.SplitMix64(seed)
    colors = {}
    for i in range(n):
        cx, cy = rng.uniform(-0.1 * w, 1.1 * w), rng.uniform(-0.1 * h, 1.1 * h)
        e = rng.uniform(3.0, 0.4 * min(w, h))
        pb = api.PathBuilder().move_to(Point(synth.f32(cx + e), synth.f32(cy)))
        for k in range(1, 3 + rng.randint(5)):
            pb.line_to(Point(synth.f32(cx + rng.uniform(-e, e)), synth.f32(cy + rng.uniform(-e, e))))
        col = Color(synth.f32((i * 37 % 101) / 100.0), synth.f32((i * 59 % 97) / 96.0), synth.f32(rng.uniform()),
                    1.0 if opaque else synth.f32(rng.uniform(0.1, 1.0)))
        fr = rule if rule is not None else (FillRule.EvenOdd if rng.randint(2) else FillRule.NonZero)
        blend = BlendMode.Over if opaque else rng.randint(12)
        comp.get_mut_or_insert_default(i).insert(pb.build()).set_props(
            Props(fill_rule=fr, func=Func.Draw(Style(fill=Fill.Solid(col), blend_mode=blend))))
        colors[i] = (col, fr)
    return colors


@pytest.mark.parametrize("name", E2E_IDS)
def test_no_id_means_clear_colour_e2e(oracle_api, name):
    comp = oracle_api.Composition()
    scenes.E2E[name](oracle_api, comp)
    ids = ids_of(oracle_api, comp, 64, 64)
    img = scenes.render_e2e(oracle_api, name)
    clear = oracle.to_srgb_bytes(oracle_api.hooks, [1.0, 1.0, 1.0, 0.0])
    none = ids == ID_NONE
    assert np.array_equal(img[none], np.broadcast_to(np.array(clear, np.uint8), img[none].shape))
    assert (~none).any() or name.startswith("solid_color")


def test_no_id_means_clear_colour_random_mixed(oracle_api):
    w, h = 200, 120
    comp = oracle_api.Composition()
    synth.random_mixed(oracle_api, comp, 150, w, h, 11)
    ids = ids_of(oracle_api, comp, w, h)
    img = rgba_of(oracle_api, comp, w, h, scenes.E2E_CLEAR)
    none = ids == ID_NONE
    assert none.any() and (~none).any()
    assert (img[none] == np.array([255, 255, 255, 0], np.uint8)).all()


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_full_top_layer_shows_its_colour(oracle_api, seed):
    w, h = 160, 96
    comp = oracle_api.Composition()
    colors = random_polygons(oracle_api, comp, 40, w, h, seed, opaque=True)
    lo = ids_of(oracle_api, comp, w, h, 0.0)
    hi = ids_of(oracle_api, comp, w, h, 511.0 / 512.0)
    img = rgba_of(oracle_api, comp, w, h, Color(1.0, 1.0, 1.0, 1.0)).astype(int)
    sure = (lo == hi) & (lo != ID_NONE)
    assert sure.sum() > 1000
    for layer in np.unique(lo[sure]):
        c, _ = colors[int(layer)]
        want = np.array(oracle.to_srgb_bytes(oracle_api.hooks, [c.r, c.g, c.b, c.a]))
        got = img[sure & (lo == layer)]
        assert np.abs(got - want).max() <= 1, (layer, got[:3], want)


def model_ids(segs, w, h, rules, min_coverage):
    """IDs of a clip-free scene from the sorted segments: each layer's doubled area per pixel is
    its cell areas plus 32 x the covers left of the pixel in its row (cumulative sums)."""
    s = unpack_segments(segs)
    x = s["tile_x"] * 16 + s["local_x"]
    y = s["tile_y"] * 16 + s["local_y"]
    out = np.full((h, w), ID_NONE, np.uint32)
    for layer in np.unique(s["layer_id"]):
        m = (s["layer_id"] == layer) & (y >= 0) & (y < h)
        xs, ys = x[m], y[m]
        area = np.zeros((h, w), np.int64)
        inside = xs < w
        np.add.at(area, (ys[inside & (xs >= 0)], xs[inside & (xs >= 0)]), s["double_area"][m][inside & (xs >= 0)])
        cov_col = np.zeros((h, w + 1), np.int64)
        np.add.at(cov_col, (ys, np.clip(xs + 1, 0, w)), s["cover"][m])
        da = area + 32 * np.cumsum(cov_col, axis=1)[:, :w]
        if rules[int(layer)] == FillRule.NonZero:
            cov = np.minimum(np.abs(da) / 512.0, 1.0)
        else:
            cov = (512 - np.abs((da & 1023) - 512)) / 512.0
        out[cov > min_coverage] = layer  # layers ascend: the last hit is the top-most
    return out


@pytest.mark.parametrize("rule", [FillRule.NonZero, FillRule.EvenOdd, None])
@pytest.mark.parametrize("min_coverage", [0.0, 0.25, 0.5])
def test_numpy_model_matches_oracle_ids(oracle_api, rule, min_coverage):
    w, h = 160, 96
    comp = oracle_api.Composition()
    colors = random_polygons(oracle_api, comp, 48, w, h, 5 + (rule or 0), rule=rule)
    ids = ids_of(oracle_api, comp, w, h, min_coverage)
    rules = {k: fr for k, (_, fr) in colors.items()}
    want = model_ids(sorted_segments(oracle_api, comp, w, h), w, h, rules, min_coverage)
    assert np.array_equal(ids, want), f"{int((ids != want).sum())} pixels differ"


def test_numpy_model_matches_oracle_ids_random_mixed(oracle_api):
    w, h = 200, 120
    comp = oracle_api.Composition()
    synth.random_mixed(oracle_api, comp, 120, w, h, 3)
    ids = ids_of(oracle_api, comp, w, h)
    # random_mixed draws its fill rules among its other choices: the model runs under both rules
    # and is held to the pixels where they agree.
    segs = sorted_segments(oracle_api, comp, w, h)
    layers = np.unique(unpack_segments(segs)["layer_id"])
    nz = model_ids(segs, w, h, {int(k): FillRule.NonZero for k in layers}, 0.0)
    eo = model_ids(segs, w, h, {int(k): FillRule.EvenOdd for k in layers}, 0.0)
    agree = nz == eo
    assert agree.mean() > 0.5
    assert np.array_equal(ids[agree], nz[agree])


@pytest.mark.parametrize("name,picks", [
    ("clipping", {(50, 12): 2, (12, 50): 0, (40, 24): 5, (24, 40): 4, (2, 2): ID_NONE}),
    ("clipping2", {(40, 24): 2, (50, 12): 0, (24, 40): 0, (2, 2): ID_NONE}),
])
def test_clip_scenes_at_picked_pixels(oracle_api, name, picks):
    comp = oracle_api.Composition()
    scenes.E2E[name](oracle_api, comp)
    ids = ids_of(oracle_api, comp, 64, 64)
    for (x, y), want in picks.items():
        assert ids[y, x] == want, (name, x, y, int(ids[y, x]))
    assert not np.isin(ids, [1]).any()  # a Func::Clip layer never hits
    if name == "clipping":
        assert not np.isin(ids, [6]).any()  # clipped, but outside the clip's range: never painted


@pytest.mark.parametrize("stride_delta,min_coverage", [(-4, 0.0), (2, 0.0), (0, -0.1), (0, 1.0), (0, float("nan"))])
def test_invalid_arguments_leave_the_buffer(oracle_api, stride_delta, min_coverage):
    w, h = 64, 64
    comp = oracle_api.Composition()
    scenes.E2E["clipping"](oracle_api, comp)
    stride = 4 * w + stride_delta
    ids = np.full((h * (4 * w + 8)) // 4, 0x12345678, np.uint32)
    with pytest.raises(FormaError):
        oracle_api.Renderer(0).render_ids(comp, ids, w, h, stride=stride, min_coverage=min_coverage)
    assert (ids == 0x12345678).all()


def test_crop_and_stride_write_only_the_tile_rectangle(oracle_api):
    w, h, pad = 100, 70, 12
    comp = oracle_api.Composition()
    synth.random_mixed(oracle_api, comp, 60, w, h, 4)
    full = ids_of(oracle_api, comp, w, h)
    stride = 4 * w + pad
    ids = np.full(h * stride // 4, 0xABABABAB, np.uint32)
    oracle_api.Renderer(0).render_ids(comp, ids, w, h, crop=Rect((20, 50), (17, 40)), stride=stride)
    grid = ids.reshape(h, stride // 4)
    inside = np.zeros(grid.shape, bool)
    inside[16:48, 16:64] = True
    assert np.array_equal(grid[inside].reshape(32, 48), full[16:48, 16:64])
    assert (grid[~inside] == 0xABABABAB).all()
