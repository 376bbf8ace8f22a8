"""Frames over a background on the device (forma_renderer_render{,_views,_batch}_over_device),
at tolerance 0: sRGB8 byte for byte, RGBA16F / RGBA32F bit for bit (a NaN is any NaN).

- Against the over oracle (tests/oracle_over.py) on random-byte, per-tile and smooth-gradient
  backgrounds in the three formats: the e2e, extreme and style scenes (all 16 blend modes, clips,
  gradients, textures, the defect_* / hostile_* scenes), random_mixed at 1080p with a crop and
  padded strides (every byte outside the crop's tiles untouched), and paris4k. RGBA16F frames are
  the oracle's f32 frame over the f16 background's values, rounded to half.
- The self-check: over a uniform background each call equals its twin with that pixel's decoded
  colour as clear colour, with the same counters, for every in-limit view and batch scene in direct
  and repacked layouts; float backgrounds holding NaN, +-inf, -0, subnormals, values above 1 and
  negative values against the twin with each as its clear colour.
- Every schedule option, and the sync-free redo (test_fast_shrink): its first attempt must not
  write, or the background would be gone before the redo.
- Refusals write nothing; a layer cache around an over frame is left as it was; the CLI's --over."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import batch_scenes as bs
import extremes
import oracle_over
import scenes
import style_scenes as ss
import synth
import view_scenes as vs
import workloads
from forma_b200.binding import BGRA, RGB0, RGB1, RGBA, Channel, Color, FormaError, Rect

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FORMATS = ("srgb8", "f16", "f32")
DTYPES = {"srgb8": np.uint8, "f16": np.float16, "f32": np.float32}
BPP = {"srgb8": 4, "f16": 8, "f32": 16}
SENTINEL = 0xA5
CLEAR = Color(1.0, 1.0, 1.0, 0.0)


@pytest.fixture(autouse=True)
def _recip_mode_0(oracle_api):
    oracle_api.hooks.fo_set_recip_mode(0)


# --- backgrounds -----------------------------------------------------------------------------------
def background(kind, h, w, fmt, seed=0):
    """[h, w, 4] of the format's dtype: random bytes / values, one random colour per 16 x 16 tile,
    or a smooth gradient; float values in [-0.25, 1.25] with alpha in [0, 1] and some alpha 1."""
    rng = np.random.default_rng(seed)
    if kind == "random":
        v = rng.random((h, w, 4))
    elif kind == "tiles":
        v = rng.random(((h + 15) // 16, (w + 15) // 16, 4)).repeat(16, 0).repeat(16, 1)[:h, :w]
    else:
        y, x = np.mgrid[0:h, 0:w]
        v = np.stack([x / max(w - 1, 1), y / max(h - 1, 1), (x + y) / max(w + h - 2, 1), 1.0 - x / max(w - 1, 1)], axis=2)
    if fmt == "srgb8":
        out = np.round(v * 255.0).astype(np.uint8)
        out[rng.random((h, w)) < 0.3, 3] = 255
        return out
    out = (v * 1.5 - 0.25).astype(np.float32)
    out[..., 3] = np.clip(v[..., 3], 0.0, 1.0)
    out[rng.random((h, w)) < 0.3, 3] = 1.0
    return out.astype(DTYPES[fmt])


def to_device(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def from_device(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy()


def assert_same(got, want, fmt, what):
    g, w = np.ascontiguousarray(got), np.ascontiguousarray(want, DTYPES[fmt])
    if fmt == "srgb8":
        bad = g != w
    else:
        bits = np.uint32 if fmt == "f32" else np.uint16
        bad = (g.view(bits) != w.view(bits)) & ~(np.isnan(g) & np.isnan(w))
    if bad.any():
        idx = tuple(int(i[0]) for i in np.nonzero(bad))
        raise AssertionError(f"{what} ({fmt}): {int(bad.sum())} values differ, first at {idx}: cuda {g[idx]!r} expected {w[idx]!r}")


def oracle_over_frame(ocomp, bg, fmt, channels=RGBA, crop=None):
    """The over oracle's frame over bg: sRGB8 as it is, float formats in f32 then rounded to the format."""
    frame = np.array(bg if fmt == "srgb8" else bg.astype(np.float32), order="C", copy=True)
    assert oracle_over.render(ocomp, frame, channels, crop) == 0
    return frame.astype(DTYPES[fmt])


def device_over(r, comp, bg, fmt, channels=RGBA, crop=None):
    t = to_device(bg)
    r.render_over_device(comp, t.data_ptr(), bg.shape[1], bg.shape[0], channels, crop, format=fmt)
    return from_device(t)


# --- against the oracle ------------------------------------------------------------------------------
KINDS = ("random", "tiles", "gradient")


def check_scene(cuda_api, comp, ocomp, w, h, crop, index, what):
    r = cuda_api.Renderer(0)
    for k, fmt in enumerate(FORMATS):
        kind = KINDS[(index + k) % 3]
        bg = background(kind, h, w, fmt, seed=index)
        assert_same(device_over(r, comp, bg, fmt, crop=crop), oracle_over_frame(ocomp, bg, fmt, crop=crop), fmt, f"{what} {kind}")


@pytest.mark.parametrize("name", list(scenes.E2E))
def test_e2e_scene(cuda_api, oracle_api, name):
    comps = []
    for api in (cuda_api, oracle_api):
        comps.append(api.Composition())
        scenes.E2E[name](api, comps[-1])
    check_scene(cuda_api, comps[0], comps[1], 64, 64, None, list(scenes.E2E).index(name), name)


@pytest.mark.parametrize("name", list(extremes.SCENES))
def test_extreme_scene(cuda_api, oracle_api, name):
    ocomp, _, sc = extremes.build(oracle_api, name)
    comp, _, _ = extremes.build(cuda_api, name)
    check_scene(cuda_api, comp, ocomp, sc.width, sc.height, sc.crop, list(extremes.SCENES).index(name), name)


@pytest.mark.parametrize("name", list(ss.SCENES))
def test_style_scene(cuda_api, oracle_api, name):
    ocomp, _, sc = ss.build(oracle_api, name)
    comp, _, _ = ss.build(cuda_api, name)
    check_scene(cuda_api, comp, ocomp, sc.width, sc.height, None, list(ss.SCENES).index(name), name)


@pytest.mark.parametrize("fmt", FORMATS)
def test_random_mixed_1080p_crop_and_padded_stride(cuda_api, oracle_api, fmt):
    """BGRA, a crop and a padded row stride: the crop's tile rectangle is the oracle's, every other
    byte of the buffer (padding included) is as it was."""
    import torch
    w, h, bpp = 1920, 1080, BPP[fmt]
    comp, ocomp = cuda_api.Composition(), oracle_api.Composition()
    synth.random_mixed(cuda_api, comp, 400, w, h, 7)
    synth.random_mixed(oracle_api, ocomp, 400, w, h, 7)
    crop = Rect((100, 1500), (37, 1000))
    bg = background("random", h, w, fmt, seed=3)
    want = oracle_over_frame(ocomp, bg, fmt, BGRA, crop)
    stride = bpp * w + 48
    raw = np.full(h * stride + 64, SENTINEL, np.uint8)
    for y in range(h):
        raw[y * stride:y * stride + bpp * w] = bg[y].reshape(-1).view(np.uint8)
    expect = raw.copy()
    for y in range(h):
        expect[y * stride:y * stride + bpp * w] = want[y].reshape(-1).view(np.uint8)
    t = torch.from_numpy(raw).to("cuda:0")
    cuda_api.Renderer(0).render_over_device(comp, t.data_ptr(), w, h, BGRA, crop, format=fmt, stride=stride)
    got = from_device(t)
    assert_same(rows_of(got, h, w, stride, fmt), rows_of(expect, h, w, stride, fmt), fmt, "1080p crop")
    pad = np.ones(got.size, bool)
    for y in range(h):
        pad[y * stride:y * stride + bpp * w] = False
    assert (got[pad] == SENTINEL).all(), "padding written"
    outside = np.ones((h, w), bool)
    outside[32:1008, 96:1504] = False  # the crop's tile rectangle
    assert_same(rows_of(got, h, w, stride, fmt)[outside], bg[outside], fmt, "outside the crop")


def rows_of(raw, h, w, stride, fmt):
    bpp = BPP[fmt]
    return np.stack([raw[y * stride:y * stride + bpp * w] for y in range(h)]).view(DTYPES[fmt]).reshape(h, w, 4)


@pytest.mark.parametrize("fmt", ["srgb8", "f32"])
def test_paris4k(cuda_api, oracle_api, fmt):
    comp, w, h = workloads.build_scene(cuda_api, "paris4k")
    ocomp, _, _ = workloads.build_scene(oracle_api, "paris4k")
    bg = background("tiles", h, w, fmt, seed=11)
    assert_same(device_over(cuda_api.Renderer(0), comp, bg, fmt), oracle_over_frame(ocomp, bg, fmt), fmt, "paris4k")


# --- the self-check: a uniform background is the twin's clear colour ---------------------------------
UNIFORM = {"srgb8": (90, 11, 200, 255), "f16": (0.25, -0.5, 1.5, 0.375), "f32": (0.1, 0.2, 0.3, 1.0)}


def uniform_clear(fmt, channels=RGBA):
    """(pixel in channel order, clear colour) of the uniform background of `fmt`."""
    rgba = UNIFORM[fmt]
    px = [rgba[int(c)] for c in channels]
    if fmt == "srgb8":
        return px, oracle_over.clear_of(px, channels)
    return px, Color(*[float(np.float32(np.float16(v) if fmt == "f16" else v)) for v in rgba])


class Stack:
    """A device buffer of n frames of `fmt` with the given strides: frames filled with `px`, every
    other byte SENTINEL."""

    def __init__(self, n, w, h, fmt, px, stride=None, frame_stride=None):
        import torch
        self.n, self.w, self.h, self.fmt, self.bpp = n, w, h, fmt, BPP[fmt]
        self.stride = self.bpp * w if stride is None else stride
        self.frame_stride = h * self.stride if frame_stride is None else frame_stride
        raw = np.full((n - 1) * self.frame_stride + h * self.stride + 64, SENTINEL, np.uint8)
        row = np.tile(np.asarray(px, DTYPES[fmt]), w).view(np.uint8)
        for b in range(n):
            for y in range(h):
                o = b * self.frame_stride + y * self.stride
                raw[o:o + self.bpp * w] = row
        self.t = torch.from_numpy(raw).to("cuda:0")
        self.ptr = self.t.data_ptr()

    def raw(self):
        return from_device(self.t)


@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("name", vs.IN_LIMIT)
def test_views_over_uniform_background_is_the_twin(cuda_api, name, padded):
    sc = vs.SCENES[name]
    comp, _ = vs.build(cuda_api, sc)
    n = len(sc.views)
    for k, fmt in enumerate(FORMATS):
        bpp = BPP[fmt]
        pad = dict(stride=bpp * sc.width + 16, frame_stride=(bpp * sc.width + 16) * sc.height + 32) if padded else {}
        px, clear = uniform_clear(fmt, RGBA if k % 2 == 0 else BGRA)
        ch = RGBA if k % 2 == 0 else BGRA
        over, twin = Stack(n, sc.width, sc.height, fmt, px, **pad), Stack(n, sc.width, sc.height, fmt, px, **pad)
        r = cuda_api.Renderer(0)
        r.render_views_over_device(comp, sc.views, over.ptr, sc.width, sc.height, ch, format=fmt, stride=over.stride,
                                   view_stride=over.frame_stride)
        c_over = r.counters()
        kw = dict(stride=twin.stride, view_stride=twin.frame_stride)
        if fmt == "srgb8":
            r.render_views_device(comp, sc.views, twin.ptr, sc.width, sc.height, ch, clear, **kw)
        else:
            r.render_views_linear_device(comp, sc.views, twin.ptr, sc.width, sc.height, ch, clear, format=fmt, **kw)
        check_counters(c_over, r.counters(), f"{name} {fmt}")
        assert_same(over.raw().view(np.uint8), twin.raw().view(np.uint8), "srgb8", f"{name} {fmt} padded {padded}")


@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("name", bs.IN_LIMIT)
def test_batch_over_uniform_background_is_the_twin(cuda_api, name, padded):
    sc = bs.SCENES[name]
    _, frames = bs.build(cuda_api, sc)
    n = len(frames)
    for k, fmt in enumerate(FORMATS):
        bpp = BPP[fmt]
        pad = dict(stride=bpp * sc.width + 16, frame_stride=(bpp * sc.width + 16) * sc.height + 16) if padded else {}
        ch = BGRA if k % 2 == 0 else RGBA
        px, clear = uniform_clear(fmt, ch)
        over, twin = Stack(n, sc.width, sc.height, fmt, px, **pad), Stack(n, sc.width, sc.height, fmt, px, **pad)
        r = cuda_api.Renderer(0)
        r.render_batch_over_device(frames, over.ptr, sc.width, sc.height, ch, format=fmt, stride=over.stride,
                                   frame_stride=over.frame_stride)
        c_over = r.counters()
        kw = dict(stride=twin.stride, frame_stride=twin.frame_stride)
        if fmt == "srgb8":
            r.render_batch_device(frames, twin.ptr, sc.width, sc.height, ch, clear, **kw)
        else:
            r.render_batch_linear_device(frames, twin.ptr, sc.width, sc.height, ch, clear, format=fmt, **kw)
        check_counters(c_over, r.counters(), f"{name} {fmt}")
        assert_same(over.raw().view(np.uint8), twin.raw().view(np.uint8), "srgb8", f"{name} {fmt} padded {padded}")


def check_counters(over, twin, what):
    """The counters of the frame (launches, bytes: totals since the renderer was made)."""
    for k in ("segments", "cells", "entries", "written_tiles"):
        assert over[k] == twin[k], (what, k, over[k], twin[k])


def test_single_frame_over_uniform_background_is_the_twin(cuda_api):
    import torch
    w, h = 640, 360
    comp = cuda_api.Composition()
    synth.random_mixed(cuda_api, comp, 300, w, h, 5)
    r = cuda_api.Renderer(0)
    for fmt in FORMATS:
        for ch in (RGBA, BGRA):
            px, clear = uniform_clear(fmt, ch)
            bg = np.ascontiguousarray(np.broadcast_to(np.asarray(px, DTYPES[fmt]), (h, w, 4)))
            got = device_over(r, comp, bg, fmt, ch)
            segs = r.counters()["segments"]
            t = to_device(bg)
            if fmt == "srgb8":
                r.render_device(comp, t.data_ptr(), w, h, ch, clear)
            else:
                r.render_linear_device(comp, t.data_ptr(), w, h, ch, clear, format=fmt)
            assert r.counters()["segments"] == segs
            assert_same(got, from_device(t), fmt, f"uniform {ch}")


# Float backgrounds with special values, each pixel its own (r, g, b, a).
SPECIAL = [(np.nan, 0.5, 0.25, 0.5), (np.inf, -np.inf, 0.5, 1.0), (-0.0, -0.0, -0.0, -0.0), (0.5, 0.5, 0.5, np.nan),
           (2.5, -1.0, 0.5, 1.0), (-0.5, 3.0, 1e-3, 0.25), (0.2, 0.3, 0.4, np.inf), (0.1, 0.1, 0.1, -0.5)]


@pytest.mark.parametrize("fmt", ["f32", "f16"])
def test_special_float_backgrounds_are_the_twin(cuda_api, fmt):
    w, h = 256, 160
    comp = cuda_api.Composition()
    synth.random_mixed(cuda_api, comp, 150, w, h, 13)
    r = cuda_api.Renderer(0)
    sub = np.float32(1e-40) if fmt == "f32" else np.float32(np.float16(3e-6))  # a subnormal of the format
    for px in SPECIAL + [(sub, -sub, 0.5, 1.0), (0.5, sub, sub, sub)]:
        v = np.asarray(px, np.float32).astype(DTYPES[fmt])
        bg = np.ascontiguousarray(np.broadcast_to(v, (h, w, 4)))
        got = device_over(r, comp, bg, fmt)
        t = to_device(np.zeros((h, w, 4), DTYPES[fmt]))
        r.render_linear_device(comp, t.data_ptr(), w, h, RGBA, Color(*[float(x) for x in v.astype(np.float32)]), format=fmt)
        assert_same(got, from_device(t), fmt, f"background {px}")


def test_channel_permutations_of_float_frames(cuda_api, oracle_api):
    """Float frames take any permutation of R, G, B, A, alpha first too."""
    w, h = 200, 120
    comp, ocomp = cuda_api.Composition(), oracle_api.Composition()
    synth.random_mixed(cuda_api, comp, 150, w, h, 11)
    synth.random_mixed(oracle_api, ocomp, 150, w, h, 11)
    ch = (Channel.Alpha, Channel.Blue, Channel.Red, Channel.Green)
    bg = background("random", h, w, "f32", seed=4)
    assert_same(device_over(cuda_api.Renderer(0), comp, bg, "f32", ch), oracle_over_frame(ocomp, bg, "f32", ch), "f32", "ABRG")


# --- schedule options and the sync-free redo -------------------------------------------------------------
OPTIONS = ("speculate", "band_copy", "copy_bands", "sort_full_key", "sort_big_log2", "test_gap_cap", "paint_lpt", "paint_wide",
           "paint_solid", "sort_scan_log2", "band_filter", "sync_free", "test_fast_shrink", "host_slices", "slice_bands",
           "slice_min_points", "slice_chain")
OW, OH = 1280, 720


@pytest.fixture()
def restore_options(cuda_api):
    saved = {n: cuda_api.get_option(n) for n in OPTIONS}
    yield
    for n, v in saved.items():
        cuda_api.set_option(n, v)


@pytest.fixture(scope="module")
def mixed_over(oracle_api):
    ocomp = oracle_api.Composition()
    synth.random_mixed(oracle_api, ocomp, 900, OW, OH, 31)
    bgs = {fmt: background("random", OH, OW, fmt, seed=21) for fmt in ("srgb8", "f32")}
    return bgs, {fmt: oracle_over_frame(ocomp, bgs[fmt], fmt) for fmt in bgs}


def _mixed(cuda_api):
    comp = cuda_api.Composition()
    synth.random_mixed(cuda_api, comp, 900, OW, OH, 31)
    return comp


@pytest.mark.parametrize("name,value", [("speculate", 0), ("band_copy", 0), ("copy_bands", 16), ("sort_full_key", 1),
                                        ("sort_big_log2", 10), ("sort_scan_log2", 10), ("paint_lpt", 0), ("paint_wide", 1),
                                        ("paint_solid", 0), ("band_filter", 0), ("sync_free", 0), ("host_slices", 2),
                                        ("slice_bands", 1), ("slice_min_points", 0), ("slice_chain", 0), ("test_gap_cap", 1)])
def test_option_does_not_change_the_frame(cuda_api, mixed_over, restore_options, name, value):
    bgs, want = mixed_over
    cuda_api.set_option(name, value)
    comp, r = _mixed(cuda_api), cuda_api.Renderer(0)
    for fmt in ("srgb8", "f32"):
        for frame in range(2):  # counted tables, then (by default) sync-free
            assert_same(device_over(r, comp, bgs[fmt], fmt), want[fmt], fmt, f"{name}={value} frame {frame + 1}")


def test_sync_free_redo_keeps_the_background(cuda_api, mixed_over, restore_options):
    """A sync-free frame whose counts outgrow their halved bounds is painted twice; its first
    attempt writes nothing, so the second paints over the background, not over a clear colour."""
    bgs, want = mixed_over
    cuda_api.set_option("sync_free", 1)
    cuda_api.set_option("test_fast_shrink", 1)
    comp, r = _mixed(cuda_api), cuda_api.Renderer(0)
    for fmt in ("srgb8", "f32"):
        device_over(r, comp, bgs[fmt], fmt)  # the bounds of the next frame
        assert_same(device_over(r, comp, bgs[fmt], fmt), want[fmt], fmt, "redone frame")
        assert r.counters()["tables_mode"] == 2, r.counters()


def test_sync_free_redo_of_a_repacked_stack(cuda_api, restore_options):
    """The same for a batch painted in scratch: the background is copied in again for the redo."""
    w, h = 200, 120  # not whole tile rows: repacked
    comps = []
    for seed in range(16):  # enough cells that the halved bounds of the second frame are too small
        comps.append(cuda_api.Composition())
        synth.random_mixed(cuda_api, comps[-1], 600, w, h, seed)
    r = cuda_api.Renderer(0)
    bg = np.stack([background(KINDS[k % 3], h, w, "srgb8", seed=k) for k in range(len(comps))])
    outs = []
    for shrink in (0, 1):
        cuda_api.set_option("sync_free", 1)
        cuda_api.set_option("test_fast_shrink", shrink)
        t = to_device(bg)
        r.render_batch_over_device(comps, t.data_ptr(), w, h)
        t = to_device(bg)
        r.render_batch_over_device(comps, t.data_ptr(), w, h)
        assert r.counters()["tables_mode"] == (2 if shrink else 1), r.counters()
        outs.append(from_device(t))
    assert np.array_equal(outs[0], outs[1]) and not np.array_equal(outs[0], bg)


# --- refusals, caches, the CLI -------------------------------------------------------------------------------
def test_refusals_write_nothing(cuda_api):
    import torch
    w, h, n = 64, 48, 3
    comp = cuda_api.Composition()
    scenes.E2E["clipping"](cuda_api, comp)
    r = cuda_api.Renderer(0)
    a = cuda_api
    t = torch.full((n * h * 16 * w + 256,), SENTINEL, dtype=torch.uint8, device="cuda:0")
    p = t.data_ptr()
    chans = lambda c: (C.c_uint32 * 4)(*c)
    rgba = chans(RGBA)
    views = (C.c_float * (6 * n))(*([1.0, 0.0, 0.0, 1.0, 0.0, 0.0] * n))
    comps = (C.c_void_p * n)(comp._h, comp._h, None)
    single = lambda ptr, stride, fmt, ch=rgba: a.renderer_render_over_device(r._h, comp._h, C.c_void_p(ptr), w, stride, h, ch, None,
                                                                             fmt, None)
    calls = {
        "null buffer": single(0, 4 * w, 0),
        "format 3": single(p, 16 * w, 3),
        "sRGB8 stride below 4 W": single(p, 4 * w - 4, 0),
        "f32 stride below 16 W": single(p, 16 * w - 4, 2),
        "sRGB8 stride not a multiple of 4": single(p, 4 * w + 2, 0),
        "f16 pointer not a multiple of 4": single(p + 2, 8 * w, 1),
        "sRGB8 pointer not a multiple of 4": single(p + 1, 4 * w, 0),
        "RGB1": single(p, 4 * w, 0, chans(RGB1)),
        "RGB0 f32": single(p, 16 * w, 2, chans(RGB0)),
        "repeated channel": single(p, 16 * w, 2, chans((0, 0, 1, 3))),
        "channel 9": single(p, 16 * w, 2, chans((0, 1, 2, 9))),
        "sRGB8 alpha first": single(p, 4 * w, 0, chans((3, 0, 1, 2))),
        "views n = 0": a.renderer_render_views_over_device(r._h, comp._h, views, 0, C.c_void_p(p), w, 4 * w, h, 4 * w * h, rgba, 0,
                                                           None),
        "views n too large": a.renderer_render_views_over_device(r._h, comp._h, views, r.max_views(h) + 1, C.c_void_p(p), w, 4 * w, h,
                                                                 4 * w * h, rgba, 0, None),
        "view stride short": a.renderer_render_views_over_device(r._h, comp._h, views, n, C.c_void_p(p), w, 16 * w, h, 16 * w * h - 4,
                                                                 rgba, 2, None),
        "view stride not a multiple of 4": a.renderer_render_views_over_device(r._h, comp._h, views, n, C.c_void_p(p), w, 4 * w, h,
                                                                               4 * w * h + 2, rgba, 0, None),
        "batch null entry": a.renderer_render_batch_over_device(r._h, comps, n, C.c_void_p(p), w, 8 * w, h, 8 * w * h, rgba, 1, None),
        "batch bad format": a.renderer_render_batch_over_device(r._h, comps, 2, C.c_void_p(p), w, 8 * w, h, 8 * w * h, rgba, 7, None),
    }
    for what, st in calls.items():
        assert st == 1, f"{what}: status {st}"
    torch.cuda.synchronize()
    assert bool(torch.all(t == SENTINEL)), "a refused call wrote"
    with pytest.raises(FormaError):
        r.render_over_device(comp, p, w, h, BGRA, format="srgb8", stride=4 * w - 4)
    with pytest.raises(ValueError):
        r.render_over_device(comp, p, w, h, format="rgba8")


def test_over_frame_leaves_the_layer_cache(cuda_api):
    """A cached sRGB8 frame, then an over frame, then a cached sRGB8 frame: the last one writes
    exactly the tiles (and bytes) it writes without the over frame in between."""
    w, h = 640, 360
    runs = []
    for with_over in (False, True):
        comp = cuda_api.Composition()
        synth.random_mixed(cuda_api, comp, 300, w, h, 5)
        r = cuda_api.Renderer(0)
        cache = r.create_buffer_layer_cache()
        buf = np.zeros(w * h * 4, np.uint8)
        r.render(comp, buf, w, h, RGBA, CLEAR, None, cache)
        comp.get(7).disable()
        if with_over:
            device_over(r, comp, background("tiles", h, w, "srgb8"), "srgb8", BGRA)
        r.render(comp, buf, w, h, RGBA, CLEAR, None, cache)
        runs.append((r.counters()["written_tiles"], buf.copy()))
        r.render(comp, buf, w, h, RGBA, CLEAR, None, cache)
        assert r.counters()["written_tiles"] == 0
    assert runs[0][0] == runs[1][0] and runs[0][0] > 0
    assert np.array_equal(runs[0][1], runs[1][1])


def test_cli_over(cuda_api, tmp_path):
    from forma_b200 import svg
    from forma_b200.render import read_image, write_ppm
    svg_path = os.path.join(ROOT, "tests", "golden", "paris30k_excerpt.svg")
    w, h = 400, 300
    photo = background("gradient", h, w, "srgb8")
    photo[..., 3] = 255
    src, out = tmp_path / "photo.ppm", tmp_path / "out.ppm"
    write_ppm(str(src), photo.reshape(-1), w, h)
    subprocess.check_call([sys.executable, "-m", "forma_b200.render", svg_path, str(out), "--over", str(src)], cwd=ROOT)
    got = read_image(str(out))
    comp = cuda_api.Composition()
    svg.compose(cuda_api, comp, svg.parse_svg(svg_path))
    want = device_over(cuda_api.Renderer(0), comp, read_image(str(src)), "srgb8")
    assert np.array_equal(got[..., :3], want[..., :3])
    assert not np.array_equal(want, photo)
