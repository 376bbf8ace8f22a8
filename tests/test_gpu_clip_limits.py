"""The device's clip walk at its limits (tests/clip_scenes.py): masks (F32 and U8), ID frames and layer
statistics of every clip scene held to the oracle and to the NumPy model of tests/clip_model.py at
tolerance 0, as single frames (whole, cropped, with padded strides that take the scalar stores), as
views with a partial last tile row and as frames >= 1 of batches, in every table mode. A batch frame
of a scene whose clip range nearly wraps 32 bits is the scene's own single frame; one full layer over
7680 x 4320 has an area above 2^32; a sparse composition takes statistics for all 2^21 orders.

Every scene is built and checked on the CPU (its model reaches the edge it is named for, and equals
the oracle) before the device sees it."""
import numpy as np
import pytest

import clip_model
import clip_scenes as cs
import oracle_ids
import oracle_masks
import oracle_stats
from forma_b200.binding import RGBA, STATS_DTYPE, Color, Rect

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A
THRESHOLDS = (0.0, 0.25, cs.THRESHOLDS[2], 511.0 / 512.0)
# A filler composition that goes first in every batch, so that each scene is a frame >= 1 (order base 7).
FILLER = cs.Scene(64, 64, [cs.L(o, (2.0 * o, 3.0, 20.0 + 3 * o, 40.5), cs.draw(Color(0.1 * o, 0.5, 0.2, 0.75))) for o in range(7)],
                  lambda m: None)
# The scenes a batch with the filler can hold (the orders of a batch share one 2^21 field).
BATCHABLE = [n for n, sc in sorted(cs.SCENES.items()) if sc.n_orders() + FILLER.n_orders() <= 1 << 21]
RANGES = [n for n in sorted(cs.SCENES) if n.startswith("range_")]


@pytest.fixture(autouse=True)
def _attach(oracle_api):
    oracle_ids.attach(oracle_api)
    oracle_masks.attach(oracle_api)
    oracle_stats.attach(oracle_api)


def windows(sc):
    return [(0, min(sc.n_orders(), 512))] + list(sc.windows)


class Expected:
    """A scene built for the oracle and checked on the CPU: its model reaches the scene's edge and
    equals the oracle; `masks`, `ids` and `stats` are then the oracle's."""

    def __init__(self, oracle_api, sc):
        self.sc = sc
        w, h = sc.width, sc.height
        comp = oracle_api.Composition()
        sc.build(oracle_api, comp)
        r = oracle_api.Renderer(0)
        self.rgba = np.zeros(w * h * 4, np.uint8)
        r.render(comp, self.rgba, w, h, RGBA, cs.CLEAR)
        self.model = clip_model.Model(r.segments(), cs.props_of(sc), w, h)
        sc.check(self.model)
        self.comp, self.api = comp, oracle_api

    def masks(self, first, k, fmt="f32", crop=None):
        got = oracle_masks.render(self.api, self.comp, self.sc.width, self.sc.height, first, k, fmt, crop)
        if fmt == "f32" and crop is None:
            assert np.array_equal(got, self.model.masks(first, k))
        return got

    def ids(self, t, crop=None):
        w, h = self.sc.width, self.sc.height
        ids = np.zeros(w * h, np.uint32)
        self.api.Renderer(0).render_ids(self.comp, ids, w, h, crop=crop, min_coverage=t)
        ids = ids.reshape(h, w)
        if crop is None:
            assert np.array_equal(ids, self.model.ids(t))
        return ids

    def stats(self, first, k, t, crop=None):
        got = oracle_stats.render(self.api, self.comp, self.sc.width, self.sc.height, first, k, t, crop)
        if crop is None:
            assert not oracle_stats.diff(got, self.model.stats(first, k, t))
        return got


def device_comp(cuda_api, sc):
    comp = cuda_api.Composition()
    sc.build(cuda_api, comp)
    return comp


def _torch():
    import torch
    return torch


def dev_masks(r, comp, w, h, first, k, fmt, crop=None, stride=None, plane_stride=None):
    """The device's planes [k, h, w] from a sentinel-filled buffer, and whether nothing outside the
    crop's tile rectangle of each plane was written."""
    torch = _torch()
    bpp = 4 if fmt == "f32" else 1
    stride = bpp * w if stride is None else stride
    plane_stride = stride * h if plane_stride is None else plane_stride
    buf = torch.full((k * plane_stride + 64,), SENTINEL, dtype=torch.uint8, device="cuda:0")
    r.render_masks_device(comp, buf.data_ptr(), w, h, first, k, fmt, crop=crop, stride=stride, plane_stride=plane_stride)
    torch.cuda.synchronize()
    raw = buf.cpu().numpy()
    x0, x1, y0, y1 = oracle_stats.region(w, h, crop)
    out = np.zeros((k, h, w), np.float32 if fmt == "f32" else np.uint8)
    untouched = True
    for j in range(k):
        plane = raw[j * plane_stride:j * plane_stride + h * stride].reshape(h, stride)
        inside = np.zeros(plane.shape, bool)
        inside[y0:y1, bpp * x0:bpp * x1] = True
        out[j] = plane[:, :bpp * w].copy().view(out.dtype)
        untouched &= bool((plane[~inside] == SENTINEL).all())
    return out, untouched


def dev_ids(r, comp, w, h, t, crop=None):
    torch = _torch()
    ids = torch.full((h, w), -1, dtype=torch.int32, device="cuda:0")
    r.render_ids_device(comp, ids.data_ptr(), w, h, crop=crop, min_coverage=t)
    torch.cuda.synchronize()
    return ids.cpu().numpy().view(np.uint32)


def dev_stats(r, comp, w, h, first, k, t, crop=None):
    torch = _torch()
    rec = torch.full((k, 12), 0x5A5A5A5A, dtype=torch.int32, device="cuda:0")
    r.render_stats_device(comp, rec.data_ptr(), w, h, first, k, t, crop=crop)
    torch.cuda.synchronize()
    return rec.cpu().numpy().view(STATS_DTYPE)[:, 0]


def assert_equal(got, want, what):
    if got.dtype == np.float32:
        got, want = got.view(np.uint32), want.view(np.uint32)
    bad = np.argwhere(got != want)
    assert not len(bad), f"{what}: {len(bad)} values differ, first at {bad[0].tolist()}: got {got[tuple(bad[0])]}, " \
                         f"want {want[tuple(bad[0])]}"


def check_single(cuda_api, exp, crop=None, padded=False):
    sc = exp.sc
    w, h = sc.width, sc.height
    r = cuda_api.Renderer(0)
    comp = device_comp(cuda_api, sc)
    for first, k in windows(sc):
        for fmt in ("f32", "u8"):
            bpp = 4 if fmt == "f32" else 1
            stride = bpp * w + (4 if padded else 0) + (1 if padded and fmt == "u8" else 0)
            plane_stride = stride * h + (12 if padded else 0)
            got, untouched = dev_masks(r, comp, w, h, first, k, fmt, crop, stride, plane_stride)
            want = exp.masks(first, k, fmt, crop)
            x0, x1, y0, y1 = oracle_stats.region(w, h, crop)
            assert_equal(got[:, y0:y1, x0:x1], want[:, y0:y1, x0:x1], f"masks {fmt} [{first}, +{k}) crop {crop}")
            assert untouched, f"masks {fmt} [{first}, +{k}): bytes outside the planes' rectangle written"
    for t in THRESHOLDS:
        got = dev_ids(r, comp, w, h, t, crop)
        want = exp.ids(t, crop)
        x0, x1, y0, y1 = oracle_stats.region(w, h, crop)
        assert_equal(got[y0:y1, x0:x1], want[y0:y1, x0:x1], f"IDs at {t} crop {crop}")
        for first, k in windows(sc):
            assert_equal(dev_stats(r, comp, w, h, first, k, t, crop), exp.stats(first, k, t, crop), f"stats [{first}, +{k}) at {t}")


@pytest.mark.parametrize("name", sorted(cs.SCENES))
def test_single_frames(cuda_api, oracle_api, name):
    check_single(cuda_api, Expected(oracle_api, cs.SCENES[name]))


@pytest.mark.parametrize("name", ["nest_restart", "nest_inner_longer", "clip_full", "clip_even_odd_zero", "heavy_65_clips",
                                  "heavy_257_clips", "windows", "quarter", "edge_17x17"])
def test_crops_and_padded_strides(cuda_api, oracle_api, name):
    exp = Expected(oracle_api, cs.SCENES[name])
    w, h = exp.sc.width, exp.sc.height
    check_single(cuda_api, exp, padded=True)
    if w > 16 or h > 16:
        check_single(cuda_api, exp, crop=Rect((min(17, w - 1), w), (min(3, h - 1), h)), padded=True)


@pytest.mark.parametrize("name", ["edge_9x17", "edge_17x17", "edge_7x15", "nest_restart", "quarter", "clip_even_odd_zero"])
def test_views_with_partial_last_tile_row(cuda_api, oracle_api, name):
    """Identity views of a frame whose height is not a multiple of 16: every view is the single frame."""
    torch = _torch()
    sc = cs.SCENES[name]
    exp = Expected(oracle_api, sc)
    w, h, n = sc.width, sc.height + 1 if sc.height % 16 == 0 else sc.height, 3
    if h != sc.height:
        exp = Expected(oracle_api, cs.Scene(w, h, sc.layers, lambda m: None, sc.windows))
    comp = device_comp(cuda_api, sc)
    views = [[1.0, 0.0, 0.0, 1.0, 0.0, 0.0]] * n
    r = cuda_api.Renderer(0)
    k = min(sc.n_orders(), 512)
    for fmt in ("f32", "u8"):
        t = torch.zeros((n, k, h, w), dtype=torch.float32 if fmt == "f32" else torch.uint8, device="cuda:0")
        r.render_views_masks_device(comp, views, t.data_ptr(), w, h, 0, k, fmt)
        torch.cuda.synchronize()
        want = exp.masks(0, k, fmt)
        for v in range(n):
            assert_equal(t[v].cpu().numpy(), want, f"view {v} masks {fmt}")
    ids = torch.zeros((n, h, w), dtype=torch.int32, device="cuda:0")
    r.render_views_ids_device(comp, views, ids.data_ptr(), w, h, min_coverage=0.25)
    rec = torch.zeros((n, k, 12), dtype=torch.int32, device="cuda:0")
    r.render_views_stats_device(comp, views, rec.data_ptr(), w, h, 0, k, 0.25)
    torch.cuda.synchronize()
    for v in range(n):
        assert_equal(ids[v].cpu().numpy().view(np.uint32), exp.ids(0.25), f"view {v} IDs")
        assert_equal(rec[v].cpu().numpy().view(STATS_DTYPE)[:, 0], exp.stats(0, k, 0.25), f"view {v} stats")


def _batch(cuda_api, sc):
    filler, comp = device_comp(cuda_api, FILLER), device_comp(cuda_api, sc)
    return [filler, comp, filler, comp]


@pytest.mark.parametrize("name", BATCHABLE)
def test_batches_with_every_scene_after_frame_0(cuda_api, oracle_api, name):
    torch = _torch()
    sc = cs.SCENES[name]
    exp = Expected(oracle_api, sc)
    w, h = sc.width, sc.height
    frames = _batch(cuda_api, sc)
    n = len(frames)
    r = cuda_api.Renderer(0)
    for first, k in windows(sc):
        for fmt in ("f32", "u8"):
            t = torch.zeros((n, k, h, w), dtype=torch.float32 if fmt == "f32" else torch.uint8, device="cuda:0")
            r.render_batch_masks_device(frames, t.data_ptr(), w, h, first, k, fmt)
            torch.cuda.synchronize()
            want = exp.masks(first, k, fmt)
            for c in (1, 3):
                assert_equal(t[c].cpu().numpy(), want, f"frame {c} masks {fmt} [{first}, +{k})")
    for thr in THRESHOLDS:
        ids = torch.zeros((n, h, w), dtype=torch.int32, device="cuda:0")
        r.render_batch_ids_device(frames, ids.data_ptr(), w, h, min_coverage=thr)
        torch.cuda.synchronize()
        for c in (1, 3):
            assert_equal(ids[c].cpu().numpy().view(np.uint32), exp.ids(thr), f"frame {c} IDs at {thr}")
        for first, k in windows(sc):
            rec = torch.zeros((n, k, 12), dtype=torch.int32, device="cuda:0")
            r.render_batch_stats_device(frames, rec.data_ptr(), w, h, first, k, thr)
            torch.cuda.synchronize()
            for c in (1, 3):
                assert_equal(rec[c].cpu().numpy().view(STATS_DTYPE)[:, 0], exp.stats(first, k, thr), f"frame {c} stats at {thr}")


@pytest.mark.parametrize("name", RANGES)
def test_batch_clip_ranges_near_2_32(cuda_api, oracle_api, name):
    """Frame c of a batch paints what the single-frame call paints, whatever its order base does to
    order + clip_layers in 32 bits: RGBA, IDs, masks and statistics."""
    torch = _torch()
    sc = cs.SCENES[name]
    exp = Expected(oracle_api, sc)
    w, h = sc.width, sc.height
    frames = _batch(cuda_api, sc)
    n, comp = len(frames), frames[1]
    r = cuda_api.Renderer(0)
    single = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda:0")
    r.render_device(comp, single.data_ptr(), w, h, RGBA, cs.CLEAR)
    rgba = torch.zeros((n, h, w, 4), dtype=torch.uint8, device="cuda:0")
    r.render_batch_device(frames, rgba.data_ptr(), w, h, RGBA, cs.CLEAR)
    torch.cuda.synchronize()
    assert np.array_equal(single.cpu().numpy().ravel(), exp.rgba), "single frame RGBA != oracle"
    for c in (1, 3):
        assert torch.equal(rgba[c], single), f"frame {c} RGBA"
    ids = torch.zeros((n, h, w), dtype=torch.int32, device="cuda:0")
    r.render_batch_ids_device(frames, ids.data_ptr(), w, h)
    torch.cuda.synchronize()
    one = dev_ids(r, comp, w, h, 0.0)
    assert_equal(one, exp.ids(0.0), "single frame IDs")
    for c in (1, 3):
        assert_equal(ids[c].cpu().numpy().view(np.uint32), one, f"frame {c} IDs")
    for first, k in windows(sc):
        planes = torch.zeros((n, k, h, w), dtype=torch.float32, device="cuda:0")
        r.render_batch_masks_device(frames, planes.data_ptr(), w, h, first, k, "f32")
        rec = torch.zeros((n, k, 12), dtype=torch.int32, device="cuda:0")
        r.render_batch_stats_device(frames, rec.data_ptr(), w, h, first, k, 0.0)
        torch.cuda.synchronize()
        m1, _ = dev_masks(r, comp, w, h, first, k, "f32")
        s1 = dev_stats(r, comp, w, h, first, k, 0.0)
        assert_equal(m1, exp.masks(first, k), f"single frame masks [{first}, +{k})")
        assert_equal(s1, exp.stats(first, k, 0.0), f"single frame stats [{first}, +{k})")
        for c in (1, 3):
            assert_equal(planes[c].cpu().numpy(), m1, f"frame {c} masks [{first}, +{k})")
            assert_equal(rec[c].cpu().numpy().view(STATS_DTYPE)[:, 0], s1, f"frame {c} stats [{first}, +{k})")


OPTIONS = ("sync_free", "test_fast_shrink")


@pytest.fixture()
def restore_options(cuda_api):
    saved = {n: cuda_api.get_option(n) for n in OPTIONS}
    yield
    for n, v in saved.items():
        cuda_api.set_option(n, v)


@pytest.mark.parametrize("opts", [{"sync_free": 0}, {"sync_free": 1}, {"sync_free": 1, "test_fast_shrink": 1}])
def test_table_modes(cuda_api, oracle_api, restore_options, opts):
    for k, v in opts.items():
        cuda_api.set_option(k, v)
    for name in ("nest_restart", "heavy_257_clips", "clip_even_odd_zero", "range_u32_max_minus_1", "windows"):
        exp = Expected(oracle_api, cs.SCENES[name])
        for _ in range(2):  # the second frame of a renderer takes the sync-free tables
            check_single(cuda_api, exp)


def test_area_above_2_32(cuda_api):
    """One full layer over 7680 x 4320: area = pixels << 18 = 8697308774400, pixels = 33177600."""
    w, h = 7680, 4320
    sc = cs.Scene(w, h, [cs.L(0, (-10.0, -10.0, w + 10.0, h + 10.0), cs.draw(cs.RED))], lambda m: None)
    comp = device_comp(cuda_api, sc)
    rec = dev_stats(cuda_api.Renderer(0), comp, w, h, 0, 1, 0.0)[0]
    assert int(rec["area"]) == (w * h) << 18 == 8697308774400 and int(rec["pixels"]) == w * h == int(rec["visible"])
    assert rec["box"].tolist() == [0, 0, w, h] == rec["visible_box"].tolist()


def test_stats_for_every_order(cuda_api, oracle_api):
    """A sparse composition with layers at orders 0 and 2^21 - 1: records for K = 2^21 (96 MiB)."""
    k = 1 << 21
    sc = cs.Scene(48, 40, [cs.L(0, (3.0, 2.0, 40.5, 30.0), cs.draw(cs.RED)),
                           cs.L(cs.LAYER_LIMIT, (10.0, 5.0, 45.0, 37.25), cs.draw(cs.GREEN))], lambda m: None)
    exp = Expected(oracle_api, sc)
    comp = device_comp(cuda_api, sc)
    got = dev_stats(cuda_api.Renderer(0), comp, sc.width, sc.height, 0, k, 0.5)
    want = np.zeros(k, STATS_DTYPE)
    for o in (0, cs.LAYER_LIMIT):
        want[o] = exp.stats(o, 1, 0.5)[0]
    assert_equal(got, want, "2^21 records")
    assert got[0]["pixels"] > 0 and got[cs.LAYER_LIMIT]["visible"] > 0
