"""The clip walk of the oracle's masks, IDs and statistics held to an independent NumPy model
(tests/clip_model.py) bit for bit, on the clip scenes of tests/clip_scenes.py and on every e2e,
extreme and style scene with clips; and the invariants that tie masks to IDs: a layer is an ID only
where its mask exceeds the threshold, so visible <= pixels and visible_box lies inside box.
tests/test_gpu_clip_limits.py then holds the device to the same results."""
import numpy as np
import pytest

import clip_model
import clip_scenes as cs
import extremes
import oracle_ids
import oracle_masks
import oracle_stats
import scenes
import style_scenes as ss
from forma_b200.binding import ID_NONE, RGBA
from oracle import oracle

# Order 15 of nest_restart: the clipped layer the painter paints over x 2..12.5 with a fresh clip (clip 5 above the
# full opaque layer 3). Before the clip state restarted at layer 3, its mask was empty: area 0, pixels 0, visible 176.
NEST_RESTART_15 = dict(area=16 * 21 * (1 << 17), pixels=176, visible=176, box=[2, 0, 13, 16], visible_box=[2, 0, 13, 16])


@pytest.fixture(autouse=True)
def _attach(oracle_api):
    oracle_ids.attach(oracle_api)
    oracle_masks.attach(oracle_api)
    oracle_stats.attach(oracle_api)


def segments(api, comp, w, h):
    r = api.Renderer(0)
    r.render(comp, np.zeros(w * h * 4, np.uint8), w, h, RGBA, cs.CLEAR)
    return r.segments()


def windows(n, extra=()):
    return [(0, n)] + list(extra)


def oracle_ids_of(api, comp, w, h, t, crop=None):
    ids = np.zeros(w * h, np.uint32)
    api.Renderer(0).render_ids(comp, ids, w, h, crop=crop, min_coverage=t)
    return ids.reshape(h, w)


def check_scene(api, comp, props, w, h, n, extra_windows=(), thresholds=cs.THRESHOLDS, check=None):
    model = clip_model.Model(segments(api, comp, w, h), props, w, h)
    if check is not None:
        check(model)
    for first, k in windows(n, extra_windows):
        want = model.masks(first, k)
        got = oracle_masks.render(api, comp, w, h, first, k)
        bad = np.argwhere(got != want)
        assert not len(bad), f"masks [{first}, +{k}): {len(bad)} values differ, first {bad[0].tolist()}: " \
                             f"oracle {got[tuple(bad[0])]}, model {want[tuple(bad[0])]}"
    for t in thresholds:
        ids = model.ids(t)
        got = oracle_ids_of(api, comp, w, h, t)
        assert np.array_equal(got, ids), f"IDs at {t}: {int((got != ids).sum())} pixels differ"
        for o in np.unique(ids[ids != ID_NONE]):  # ID == o  =>  mask_o > t
            assert (model.masks(int(o), 1)[0][ids == o] > t).all(), f"order {o} is an ID where its mask is <= {t}"
        for first, k in windows(n, extra_windows):
            want = model.stats(first, k, t)
            got = oracle_stats.render(api, comp, w, h, first, k, t)
            assert not oracle_stats.diff(got, want), f"stats [{first}, +{k}) at {t}: {oracle_stats.diff(got, want)}"
            assert (want["visible"] <= want["pixels"]).all()
            vis = want["visible"] > 0
            assert (want["visible_box"][vis][:, :2] >= want["box"][vis][:, :2]).all()
            assert (want["visible_box"][vis][:, 2:] <= want["box"][vis][:, 2:]).all()
    return model


@pytest.mark.parametrize("name", sorted(cs.SCENES))
def test_clip_scenes(oracle_api, name):
    sc = cs.SCENES[name]
    comp = oracle_api.Composition()
    sc.build(oracle_api, comp)
    n = min(sc.n_orders(), 512)
    extra = [(f, k) for f, k in sc.windows]
    check_scene(oracle_api, comp, cs.props_of(sc), sc.width, sc.height, n, extra, check=sc.check)


def test_nest_restart_pins_the_painted_layer(oracle_api):
    sc = cs.SCENES["nest_restart"]
    comp = oracle_api.Composition()
    sc.build(oracle_api, comp)
    rec = oracle_stats.render(oracle_api, comp, 16, 16, 15, 1)[0]
    for k, v in NEST_RESTART_15.items():
        assert np.array_equal(rec[k], v), (k, rec[k], v)
    ids = oracle_ids_of(oracle_api, comp, 16, 16, 0.0)
    assert (ids[:, 2:13] == 15).all() and (ids[:, :2] == 3).all() and (ids[:, 13:] == 3).all()
    m = oracle_masks.render(oracle_api, comp, 16, 16, 15, 1)[0]
    assert (m[:, 2:12] == 1.0).all() and (m[:, 12] == 0.5).all() and (m[:, :2] == 0).all() and (m[:, 13:] == 0).all()


def _with_clips(props):
    return any(p.func.clip is not None or (p.func.draw is not None and p.func.draw.is_clipped) for p in props.values())


E2E_CLIP = [n for n in sorted(scenes.E2E) if _with_clips(cs.record(oracle.load(), scenes.E2E[n], 64)[1])]


@pytest.mark.parametrize("name", E2E_CLIP)
def test_e2e_scenes_with_clips(oracle_api, name):
    comp, props = cs.record(oracle_api, scenes.E2E[name], 64)
    check_scene(oracle_api, comp, props, 64, 64, max(props) + 1, thresholds=(0.0, 0.5))


def _small_with_clips(module):
    """The module's scenes of at most 2^17 pixels, without a crop, that have clip-ish layers."""
    api = oracle.load()
    return [(module, name) for name, sc in sorted(module.SCENES.items())
            if sc.width * sc.height <= 1 << 17 and getattr(sc, "crop", None) is None and _with_clips(cs.record(api, sc.build)[1])]


@pytest.mark.parametrize("module,name", _small_with_clips(extremes) + _small_with_clips(ss), ids=lambda v: getattr(v, "__name__", v))
def test_extreme_and_style_scenes_with_clips(oracle_api, module, name):
    sc = module.SCENES[name]
    comp, props = cs.record(oracle_api, sc.build)
    check_scene(oracle_api, comp, props, sc.width, sc.height, max(props) + 1, thresholds=(0.0, 0.5))
