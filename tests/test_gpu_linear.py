"""Linear float frames on the device (paint_linear_kernel, paint_views_linear_kernel) against the
oracle's f32 frames (tests/oracle_linear.py), at tolerance 0: RGBA32F bit for bit, RGBA16F bit for
bit with the oracle's f32 after astype(float16); a NaN matches any NaN.

Covered: every e2e scene and every scene of tests/extremes.py in both formats; random_mixed at
1920 x 1080 in host and device memory with crops and padded strides (bytes outside the written
rectangle untouched); paris4k; the six reference channel orders, ZERO / ONE and the ALPHA -> ONE
upgrade; an HDR scene; the device f32 frame encoded with compute_srgb against render_device's
bytes; every in-limit view and batch scene in direct and repacked layouts, host and device; every
table mode and schedule option; refusals; layer caches around a float frame; the CLI's --linear."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import batch_scenes as bs
import extremes
import oracle_linear
import scenes
import synth
import view_scenes as vs
import workloads
from forma_b200.binding import BGR0, BGR1, BGRA, RGB0, RGB1, RGBA, Channel, Color, FormaError, Rect

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLEAR = Color(1.0, 1.0, 1.0, 0.0)
ORDERS = {"RGBA": RGBA, "BGRA": BGRA, "RGB0": RGB0, "BGR0": BGR0, "RGB1": RGB1, "BGR1": BGR1}
FORMATS = ["f32", "f16"]
DTYPES = {"f32": np.float32, "f16": np.float16}
BPP = {"f32": 16, "f16": 8}
CODES = {"f32": 2, "f16": 1}
SENTINEL = 0xA5


@pytest.fixture(autouse=True)
def _oracle_linear(oracle_api):
    oracle_linear.attach(oracle_api)


def torch_dtype(fmt):
    import torch
    return torch.float32 if fmt == "f32" else torch.float16


def assert_same(got, want32, fmt, what):
    """got (any shape ending in 4, the format's dtype) against the oracle's f32 values."""
    want = want32.astype(DTYPES[fmt])
    bits = np.uint32 if fmt == "f32" else np.uint16
    g, w = np.ascontiguousarray(got, DTYPES[fmt]), np.ascontiguousarray(want)
    bad = (g.view(bits) != w.view(bits)) & ~(np.isnan(g) & np.isnan(w))
    if bad.any():
        idx = tuple(int(i[0]) for i in np.nonzero(bad))
        raise AssertionError(f"{what} ({fmt}): {int(bad.sum())} values differ, first at {idx}: cuda {g[idx]!r} oracle {w[idx]!r} "
                             f"(f32 {want32[idx]!r})")


def host_frame(r, comp, w, h, fmt, channels=RGBA, clear=CLEAR, crop=None):
    out = np.zeros((h, w, 4), DTYPES[fmt])
    r.render_linear(comp, out, w, h, channels, clear, crop, format=fmt)
    return out


def device_frame(r, comp, w, h, fmt, channels=RGBA, clear=CLEAR, crop=None):
    import torch
    t = torch.zeros((h, w, 4), dtype=torch_dtype(fmt), device="cuda:0")
    r.render_linear_device(comp, t.data_ptr(), w, h, channels, clear, crop, format=fmt)
    torch.cuda.synchronize()
    return t.cpu().numpy()


def oracle_frame(oracle_api, comp, w, h, channels=RGBA, clear=CLEAR, crop=None):
    return oracle_linear.render(oracle_api, comp, w, h, channels, clear, crop)


# ---------------------------------------------------------------------------
# Single frames
# ---------------------------------------------------------------------------


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("name", list(scenes.E2E))
def test_e2e_scene(cuda_api, oracle_api, cuda_renderer, name, fmt):
    frames = []
    for api in (cuda_api, oracle_api):
        comp = api.Composition()
        scenes.E2E[name](api, comp)
        frames.append(host_frame(cuda_renderer, comp, 64, 64, fmt) if api is cuda_api else oracle_frame(api, comp, 64, 64))
    assert_same(frames[0], frames[1], fmt, name)


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("name", list(extremes.SCENES))
def test_extreme_scene(cuda_api, oracle_api, name, fmt):
    ocomp, _, sc = extremes.build(oracle_api, name)
    want = oracle_frame(oracle_api, ocomp, sc.width, sc.height, crop=sc.crop)
    comp, _, _ = extremes.build(cuda_api, name)
    r = cuda_api.Renderer(0)
    for frame in range(2):  # counted tables, then sync-free
        assert_same(host_frame(r, comp, sc.width, sc.height, fmt, crop=sc.crop), want, fmt, f"{name} frame {frame + 1}")
    assert r.counters()["tables_mode"] == 1


@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("fmt", FORMATS)
def test_random_mixed_1080p_crop_and_stride(cuda_api, oracle_api, fmt, where):
    import torch
    w, h, bpp = 1920, 1080, BPP[fmt]
    comps = {}
    for api in (cuda_api, oracle_api):
        comps[api] = api.Composition()
        synth.random_mixed(api, comps[api], 400, w, h, 7)
    r = cuda_api.Renderer(0)
    whole = oracle_frame(oracle_api, comps[oracle_api], w, h)
    got = (host_frame if where == "host" else device_frame)(r, comps[cuda_api], w, h, fmt)
    assert_same(got, whole, fmt, f"uncropped, {where}")
    crop = Rect((100, 1333), (37, 700))  # tiles 6..83 x 2..43: columns 96 ... 1343, rows 32 ... 703
    for pad in (64, 4):  # 16-byte rows (vector stores), then 4-byte rows (4-byte stores)
        stride = bpp * w + pad
        n = h * stride
        if where == "host":
            raw = np.full(n, SENTINEL, np.uint8)
            r.render_linear(comps[cuda_api], raw.view(DTYPES[fmt]), w, h, RGBA, CLEAR, crop, format=fmt, stride=stride)
        else:
            t = torch.full((n,), SENTINEL, dtype=torch.uint8, device="cuda:0")
            r.render_linear_device(comps[cuda_api], t.data_ptr(), w, h, RGBA, CLEAR, crop, format=fmt, stride=stride)
            torch.cuda.synchronize()
            raw = t.cpu().numpy()
        grid = raw.reshape(h, stride)
        inside = grid[32:704, 96 * bpp:1344 * bpp].copy().view(DTYPES[fmt]).reshape(672, 1248, 4)
        assert_same(inside, whole[32:704, 96:1344], fmt, f"crop, pad {pad}, {where}")
        mask = np.ones(grid.shape, bool)
        mask[32:704, 96 * bpp:1344 * bpp] = False
        assert (grid[mask] == SENTINEL).all(), f"pad {pad}, {where}: bytes outside the crop's tile rectangle written"


@pytest.mark.parametrize("fmt", FORMATS)
def test_paris4k(cuda_api, oracle_api, fmt):
    comp, w, h = workloads.build_scene(cuda_api, "paris4k")
    ocomp, _, _ = workloads.build_scene(oracle_api, "paris4k")
    assert_same(device_frame(cuda_api.Renderer(0), comp, w, h, fmt), oracle_frame(oracle_api, ocomp, w, h), fmt, "paris4k")


CHANNELS = dict(ORDERS, ZERO_ONE=(Channel.Zero, Channel.One, Channel.Alpha, Channel.Red),
                ALPHA_FIRST=(Channel.Alpha, Channel.Blue, Channel.Zero, Channel.Green))


@pytest.mark.parametrize("clear", [CLEAR, Color(0.25, 0.5, 0.75, 1.0)])
@pytest.mark.parametrize("order", list(CHANNELS))
def test_channel_orders(cuda_api, oracle_api, cuda_renderer, order, clear):
    w, h = 200, 120
    comp, ocomp = cuda_api.Composition(), oracle_api.Composition()
    synth.random_mixed(cuda_api, comp, 150, w, h, 11)
    synth.random_mixed(oracle_api, ocomp, 150, w, h, 11)
    ch = CHANNELS[order]
    want = oracle_frame(oracle_api, ocomp, w, h, ch, clear)
    for fmt in FORMATS:
        got = host_frame(cuda_renderer, comp, w, h, fmt, ch, clear)
        assert_same(got, want, fmt, f"{order}, clear alpha {clear.a}")
        for k, c in enumerate(ch):
            if c == Channel.Zero:
                assert (got[..., k] == 0.0).all()
            elif c == Channel.One or (c == Channel.Alpha and clear.a == 1.0):  # ALPHA -> ONE
                assert (got[..., k] == 1.0).all()


@pytest.mark.parametrize("fmt", FORMATS)
def test_hdr_values_come_back_unclamped(cuda_api, oracle_api, cuda_renderer, fmt):
    import torch
    w, h = oracle_linear.HDR_W, oracle_linear.HDR_H
    comp, ocomp = cuda_api.Composition(), oracle_api.Composition()
    oracle_linear.hdr_scene(cuda_api, comp)
    oracle_linear.hdr_scene(oracle_api, ocomp)
    want = oracle_frame(oracle_api, ocomp, w, h, RGBA, oracle_linear.HDR_CLEAR)
    got = device_frame(cuda_renderer, comp, w, h, fmt, RGBA, oracle_linear.HDR_CLEAR)
    assert_same(got, want, fmt, "hdr")
    s = oracle_linear.HDR_SOLID
    assert (got[:, :32] == np.array([s.r, s.g, s.b, 1.0], DTYPES[fmt])).all()
    t = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda:0")
    cuda_renderer.render_device(comp, t.data_ptr(), w, h, RGBA, oracle_linear.HDR_CLEAR)
    torch.cuda.synchronize()
    srgb = t.cpu().numpy().reshape(h, w, 4)
    saturated = (srgb[..., :3] == 255) | (srgb[..., :3] == 0)
    beyond = (got[..., :3] > 1.0) | (got[..., :3] < 0.0)
    assert beyond.sum() > 1000 and saturated[beyond].all()  # where the sRGB8 frame saturates


@pytest.mark.parametrize("scene", ["random_mixed", "paris4k"])
def test_encoded_f32_frame_is_the_srgb8_frame(cuda_api, scene):
    import torch
    if scene == "paris4k":
        comp, w, h = workloads.build_scene(cuda_api, scene)
    else:
        w, h = 1920, 1080
        comp = cuda_api.Composition()
        synth.random_mixed(cuda_api, comp, 400, w, h, 3)
    r = cuda_api.Renderer(0)
    for order, ch in ORDERS.items():
        for clear in (CLEAR, Color(0.1, 0.2, 0.3, 1.0)):
            frame = device_frame(r, comp, w, h, "f32", ch, clear)
            t = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda:0")
            r.render_device(comp, t.data_ptr(), w, h, ch, clear)
            torch.cuda.synchronize()
            want = t.cpu().numpy().reshape(h, w, 4)
            got = oracle_linear.encode(frame, ch)
            assert np.array_equal(got, want), f"{scene} {order} clear {clear}: {int((got != want).any(axis=2).sum())} pixels differ"


# ---------------------------------------------------------------------------
# Views and batches
# ---------------------------------------------------------------------------


class Target:
    """A sentinel-filled buffer (device or host) for a stack of n float frames."""

    def __init__(self, n, w, h, fmt, where, stride=None, frame_stride=None):
        import torch
        self.n, self.w, self.h, self.fmt, self.where, self.bpp = n, w, h, fmt, where, BPP[fmt]
        self.stride = self.bpp * w if stride is None else stride
        self.frame_stride = h * self.stride if frame_stride is None else frame_stride
        size = (n - 1) * self.frame_stride + h * self.stride + 64
        if where == "device":
            self.t = torch.full((size,), SENTINEL, dtype=torch.uint8, device="cuda:0")
            self.ptr = self.t.data_ptr()
        else:
            self.raw_host = np.full(size // self.bpp * self.bpp + self.bpp, SENTINEL, np.uint8)
            self.buf = self.raw_host.view(DTYPES[fmt])

    def raw(self):
        import torch
        if self.where == "host":
            return self.raw_host
        torch.cuda.synchronize()
        return self.t.cpu().numpy()

    def frames(self):
        raw, bpp = self.raw(), self.bpp
        out = np.empty((self.n, self.h, self.w * bpp), np.uint8)
        mask = np.ones(raw.size, bool)
        for b in range(self.n):
            for y in range(self.h):
                o = b * self.frame_stride + y * self.stride
                out[b, y] = raw[o:o + self.w * bpp]
                mask[o:o + self.w * bpp] = False
        assert (raw[mask] == SENTINEL).all(), "bytes outside the frames written"
        return out.view(DTYPES[self.fmt]).reshape(self.n, self.h, self.w, 4)


def render_views(r, comp, sc, tgt):
    kw = dict(channels=RGBA, clear_color=CLEAR, format=tgt.fmt, stride=tgt.stride, view_stride=tgt.frame_stride)
    if tgt.where == "device":
        r.render_views_linear_device(comp, sc.views, tgt.ptr, sc.width, sc.height, **kw)
    else:
        r.render_views_linear(comp, sc.views, tgt.buf, sc.width, sc.height, **kw)
    return tgt.frames()


def render_batch(r, frames, sc, tgt):
    kw = dict(channels=RGBA, clear_color=CLEAR, format=tgt.fmt, stride=tgt.stride, frame_stride=tgt.frame_stride)
    if tgt.where == "device":
        r.render_batch_linear_device(frames, tgt.ptr, sc.width, sc.height, **kw)
    else:
        r.render_batch_linear(frames, tgt.buf, sc.width, sc.height, **kw)
    return tgt.frames()


_ORACLE = {}


def oracle_views(oracle_api, name):
    if ("views", name) not in _ORACLE:
        sc = vs.SCENES[name]
        comp, xf = vs.build(oracle_api, sc)
        out = {}
        for v in sc.views:
            if tuple(v) not in out:
                vs.set_view(comp, xf, v)
                out[tuple(v)] = oracle_frame(oracle_api, comp, sc.width, sc.height)
        _ORACLE[("views", name)] = out
    return _ORACLE[("views", name)]


def oracle_batch(oracle_api, name):
    if ("batch", name) not in _ORACLE:
        sc = bs.SCENES[name]
        distinct, _ = bs.build(oracle_api, sc)
        _ORACLE[("batch", name)] = [oracle_frame(oracle_api, c, sc.width, sc.height) for c in distinct]
    return _ORACLE[("batch", name)]


# direct: the stacked frame is painted in the caller's buffer (device, whole tile rows, default
# strides) where the height allows; padded: repacked (device) or copied frame by frame (host).
LAYOUTS = [("device", False), ("device", True), ("host", False)]


@pytest.mark.parametrize("where,padded", LAYOUTS)
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("name", vs.IN_LIMIT)
def test_views(cuda_api, oracle_api, name, fmt, where, padded):
    sc = vs.SCENES[name]
    comp, _ = vs.build(cuda_api, sc)
    bpp = BPP[fmt]
    pad = dict(stride=bpp * sc.width + 4, frame_stride=(bpp * sc.width + 4) * sc.height + 36) if padded else {}
    got = render_views(cuda_api.Renderer(0), comp, sc, Target(len(sc.views), sc.width, sc.height, fmt, where, **pad))
    want = oracle_views(oracle_api, name)
    for b, v in enumerate(sc.views):
        assert_same(got[b], want[tuple(v)], fmt, f"{name} view {b}, {where}, padded {padded}")


@pytest.mark.parametrize("where,padded", LAYOUTS)
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("name", bs.IN_LIMIT)
def test_batch(cuda_api, oracle_api, name, fmt, where, padded):
    sc = bs.SCENES[name]
    _, frames = bs.build(cuda_api, sc)
    bpp = BPP[fmt]
    pad = dict(stride=bpp * sc.width + 16, frame_stride=(bpp * sc.width + 16) * sc.height + 16) if padded else {}
    got = render_batch(cuda_api.Renderer(0), frames, sc, Target(len(frames), sc.width, sc.height, fmt, where, **pad))
    want = oracle_batch(oracle_api, name)
    for c, k in enumerate(sc.frames):
        assert_same(got[c], want[k], fmt, f"{name} frame {c}, {where}, padded {padded}")


# ---------------------------------------------------------------------------
# Table modes and schedule options
# ---------------------------------------------------------------------------

OPTIONS = ("speculate", "band_copy", "copy_bands", "sort_full_key", "sort_big_log2", "test_gap_cap", "paint_lpt", "paint_wide",
           "sort_scan_log2", "band_filter", "sync_free", "test_fast_shrink", "host_slices", "slice_min_points")


@pytest.fixture()
def restore_options(cuda_api):
    saved = {n: cuda_api.get_option(n) for n in OPTIONS}
    yield
    for n, v in saved.items():
        cuda_api.set_option(n, v)


@pytest.fixture(scope="module")
def mixed_2000(oracle_api):
    w, h = 1920, 1080
    ocomp = oracle_api.Composition()
    synth.random_mixed(oracle_api, ocomp, 2000, w, h, 9)
    return w, h, oracle_frame(oracle_api, ocomp, w, h)


def _mixed_comp(cuda_api):
    comp = cuda_api.Composition()
    synth.random_mixed(cuda_api, comp, 2000, 1920, 1080, 9)
    return comp


def test_every_table_mode(cuda_api, mixed_2000, restore_options):
    w, h, want = mixed_2000
    comp, r = _mixed_comp(cuda_api), cuda_api.Renderer(0)
    for sync_free, shrink, mode in ((0, 0, 0), (1, 0, 1), (1, 1, 2)):
        cuda_api.set_option("sync_free", sync_free)
        cuda_api.set_option("test_fast_shrink", shrink)
        for fmt in FORMATS:
            assert_same(device_frame(r, comp, w, h, fmt), want, fmt, f"sync_free {sync_free} shrink {shrink}")
            assert r.counters()["tables_mode"] == mode, (sync_free, shrink, r.counters())
    cuda_api.set_option("sync_free", 0)
    cuda_api.set_option("test_fast_shrink", 0)
    c = r.counters()
    for delta in (-1, 0, 1):  # the speculative carry pass capped around the count
        cuda_api.set_option("test_gap_cap", c["entries"] - c["cells"] + delta)
        assert_same(host_frame(r, comp, w, h, "f32"), want, "f32", f"test_gap_cap count {delta:+d}")


@pytest.mark.parametrize("name,value", [("speculate", 0), ("band_copy", 0), ("copy_bands", 16), ("sort_full_key", 1),
                                        ("sort_big_log2", 10), ("sort_scan_log2", 10), ("paint_lpt", 0), ("paint_wide", 1),
                                        ("band_filter", 0), ("host_slices", 4), ("slice_min_points", 0)])
def test_option_does_not_change_the_values(cuda_api, mixed_2000, restore_options, name, value):
    w, h, want = mixed_2000
    cuda_api.set_option(name, value)
    comp, r = _mixed_comp(cuda_api), cuda_api.Renderer(0)
    for fmt in FORMATS:
        for frame in range(2):
            assert_same(host_frame(r, comp, w, h, fmt), want, fmt, f"{name}={value} host frame {frame + 1}")
        assert_same(device_frame(r, comp, w, h, fmt), want, fmt, f"{name}={value} device")
        crop = Rect((0, w), (300, 700))
        got = host_frame(r, comp, w, h, fmt, crop=crop)
        assert_same(got[288:704], want[288:704], fmt, f"{name}={value} band crop")


# ---------------------------------------------------------------------------
# Refusals, caches, the CLI
# ---------------------------------------------------------------------------


def test_refusals_write_nothing(cuda_api):
    import torch
    w, h, n = 64, 48, 3
    comp = cuda_api.Composition()
    scenes.E2E["clipping"](cuda_api, comp)
    r = cuda_api.Renderer(0)
    a = cuda_api
    t = torch.full((n * h * 16 * w + 256,), SENTINEL, dtype=torch.uint8, device="cuda:0")
    p = t.data_ptr()
    ch, cc = (C.c_uint32 * 4)(*RGBA), (C.c_float * 4)(1.0, 1.0, 1.0, 0.0)
    views = (C.c_float * (6 * n))(*([1.0, 0.0, 0.0, 1.0, 0.0, 0.0] * n))
    comps = (C.c_void_p * n)(comp._h, comp._h, None)
    single = lambda ptr, stride, fmt: a.renderer_render_linear_device(r._h, comp._h, C.c_void_p(ptr), w, stride, h, ch, cc, None, fmt,
                                                                     None)
    calls = {
        "null buffer": single(0, 16 * w, 2),
        "format 0": single(p, 16 * w, 0),
        "format 3": single(p, 16 * w, 3),
        "f32 stride below 16 W": single(p, 16 * w - 4, 2),
        "f16 stride below 8 W": single(p, 8 * w - 4, 1),
        "stride not a multiple of 4": single(p, 16 * w + 2, 2),
        "pointer not a multiple of 4": single(p + 2, 16 * w, 2),
        "views n = 0": a.renderer_render_views_linear_device(r._h, comp._h, views, 0, C.c_void_p(p), w, 16 * w, h, 16 * w * h, ch, cc,
                                                             2, None),
        "views n too large": a.renderer_render_views_linear_device(r._h, comp._h, views, r.max_views(h) + 1, C.c_void_p(p), w,
                                                                   16 * w, h, 16 * w * h, ch, cc, 2, None),
        "view stride short": a.renderer_render_views_linear_device(r._h, comp._h, views, n, C.c_void_p(p), w, 16 * w, h,
                                                                   16 * w * h - 4, ch, cc, 2, None),
        "view stride not a multiple of 4": a.renderer_render_views_linear_device(r._h, comp._h, views, n, C.c_void_p(p), w, 16 * w,
                                                                                 h, 16 * w * h + 2, ch, cc, 2, None),
        "batch null entry": a.renderer_render_batch_linear_device(r._h, comps, n, C.c_void_p(p), w, 8 * w, h, 8 * w * h, ch, cc, 1,
                                                                  None),
        "batch bad format": a.renderer_render_batch_linear_device(r._h, comps, 2, C.c_void_p(p), w, 8 * w, h, 8 * w * h, ch, cc, 7,
                                                                  None),
    }
    for what, st in calls.items():
        assert st == 1, f"{what}: status {st}"
    torch.cuda.synchronize()
    assert bool(torch.all(t == SENTINEL)), "a refused call wrote"
    host = np.full(h * 16 * w // 4, 7.0, np.float32)
    assert a.renderer_render_linear(r._h, comp._h, host.ctypes.data_as(C.c_void_p), w, 16 * w, h, ch, cc, None, 5, None) == 1
    assert (host == 7.0).all()
    with pytest.raises(FormaError):
        r.render_linear(comp, host, w, h, format="f32", stride=16 * w - 16)


def test_float_frame_leaves_the_layer_cache(cuda_api):
    """A cached sRGB8 frame, then a float frame, then a cached sRGB8 frame: the last one writes
    exactly the tiles (and bytes) it writes without the float frame in between."""
    w, h = 640, 360
    runs = []
    for with_float in (False, True):
        comp = cuda_api.Composition()
        synth.random_mixed(cuda_api, comp, 300, w, h, 5)
        r = cuda_api.Renderer(0)
        cache = r.create_buffer_layer_cache()
        buf = np.zeros(w * h * 4, np.uint8)
        r.render(comp, buf, w, h, RGBA, CLEAR, None, cache)
        layer = comp.get(7)
        assert layer is not None
        layer.disable()
        if with_float:
            host_frame(r, comp, w, h, "f16", BGRA, Color(0.0, 0.0, 0.0, 1.0))
        r.render(comp, buf, w, h, RGBA, CLEAR, None, cache)
        runs.append((r.counters()["written_tiles"], buf.copy()))
        r.render(comp, buf, w, h, RGBA, CLEAR, None, cache)
        assert r.counters()["written_tiles"] == 0
    assert runs[0][0] == runs[1][0] and runs[0][0] > 0
    assert np.array_equal(runs[0][1], runs[1][1])


def test_cli_linear(cuda_api, tmp_path):
    svg_path = os.path.join(ROOT, "tests", "golden", "paris30k_excerpt.svg")
    out, npy = tmp_path / "out.ppm", tmp_path / "linear.npy"
    subprocess.check_call([sys.executable, "-m", "forma_b200.render", svg_path, str(out), "--width", "400", "--height", "300",
                           "--linear", str(npy)], cwd=ROOT)
    got = np.load(npy)
    assert got.shape == (300, 400, 4) and got.dtype == np.float32
    from forma_b200 import svg
    comp = cuda_api.Composition()
    svg.compose(cuda_api, comp, svg.parse_svg(svg_path))
    want = host_frame(cuda_api.Renderer(0), comp, 400, 300, "f32", RGBA, Color(1.0, 1.0, 1.0, 1.0))
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert (got[..., 3] == 1.0).all() and (got[..., :3] < 1.0).any()
