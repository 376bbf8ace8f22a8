"""Layer coverage masks on the device (Renderer.render_masks*, forma_renderer_render_*masks*), held to
the mask oracle (tests/oracle_masks.py, pinned in tests/test_masks_oracle.py) at tolerance 0, in F32
and U8: the e2e, extreme and style scenes, random_mixed at 1080p with a crop and padded strides in
host and device memory, paris4k with a window of 64 orders, every in-limit view and batch scene with
padded planes and sentinel bytes, the combined calls (their RGBA bytes are the plain calls'), every
table mode including the sync-free redo, the schedule options, refusals, layer caches and the CLI."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import batch_scenes as bs
import extremes
import oracle_masks
import scenes
import style_scenes as ss
import synth
import view_scenes as vs
import workloads
from forma_b200.binding import RGBA, Color, Rect, _CMasks

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLEAR = Color(1.0, 1.0, 1.0, 0.0)
SENTINEL = 0xA5
DTYPES = {"f32": np.float32, "u8": np.uint8}
BPP = {"f32": 4, "u8": 1}


@pytest.fixture(autouse=True)
def _attach(oracle_api):
    oracle_masks.attach(oracle_api)


def n_orders(comp):
    return max(bs.n_orders(comp), 1)


class Planes:
    """A sentinel-filled device buffer holding n frames of K planes, plane (b, k) at
    (b K + k) plane_stride bytes from its base, `offset` bytes into the allocation."""

    def __init__(self, n, k, w, h, fmt, stride=None, plane_stride=None, offset=0):
        import torch
        self.n, self.k, self.w, self.h, self.fmt, self.bpp = n, k, w, h, fmt, BPP[fmt]
        self.stride = self.bpp * w if stride is None else stride
        self.plane_stride = h * self.stride if plane_stride is None else plane_stride
        self.offset = offset
        size = offset + (n * k - 1) * self.plane_stride + (h - 1) * self.stride + self.bpp * w + 64
        self.t = torch.full((size,), SENTINEL, dtype=torch.uint8, device="cuda:0")
        self.ptr = self.t.data_ptr() + offset

    def raw(self):
        import torch
        torch.cuda.synchronize()
        return self.t.cpu().numpy()

    def planes(self):
        """(n, K, h, w) values, and whether every byte outside the planes' pixels is the sentinel."""
        raw = self.raw()
        row = np.arange(self.bpp * self.w)
        idx = (self.offset + np.arange(self.n * self.k)[:, None, None] * self.plane_stride +
               np.arange(self.h)[None, :, None] * self.stride + row[None, None, :])
        inside = np.zeros(raw.size, bool)
        inside[idx.ravel()] = True
        out = raw[idx].copy().view(DTYPES[self.fmt]).reshape(self.n, self.k, self.h, self.w)
        return out, bool(np.all(raw[~inside] == SENTINEL))


def assert_planes(got, want, what):
    if got.dtype == np.float32:
        got, want = got.view(np.uint32), want.view(np.uint32)
    bad = got != want
    assert not bad.any(), f"{what}: {int(bad.sum())} values differ, first at {np.argwhere(bad)[0].tolist()}"


def device_masks(r, comp, w, h, first, k, fmt, crop=None, **kw):
    import torch
    t = torch.zeros((k, h, w), dtype=getattr(torch, "float32" if fmt == "f32" else "uint8"), device="cuda:0")
    r.render_masks_device(comp, t.data_ptr(), w, h, first, k, fmt, crop=crop, **kw)
    torch.cuda.synchronize()
    return t.cpu().numpy()


def both_formats(cuda_api, oracle_api, comp, ocomp, w, h, first, k, crop=None):
    r = cuda_api.Renderer(0)
    for fmt in ("f32", "u8"):
        want = oracle_masks.render(oracle_api, ocomp, w, h, first, k, fmt, crop)
        assert_planes(device_masks(r, comp, w, h, first, k, fmt, crop), want, f"device {fmt}")
        host = np.zeros((k, h, w), DTYPES[fmt])
        r.render_masks(comp, host, w, h, first, crop=crop)
        assert_planes(host, want, f"host {fmt}")


# --- scenes -----------------------------------------------------------------------------------------


@pytest.mark.parametrize("name", sorted(scenes.E2E))
def test_e2e(cuda_api, oracle_api, name):
    comp, ocomp = cuda_api.Composition(), oracle_api.Composition()
    scenes.E2E[name](cuda_api, comp)
    scenes.E2E[name](oracle_api, ocomp)
    both_formats(cuda_api, oracle_api, comp, ocomp, 64, 64, 0, n_orders(ocomp) + 1)


@pytest.mark.parametrize("name", sorted(extremes.SCENES))
def test_extremes(cuda_api, oracle_api, name):
    comp, _, sc = extremes.build(cuda_api, name)
    ocomp, _, _ = extremes.build(oracle_api, name)
    n = n_orders(ocomp)
    for first, k in ((0, min(n, 64)), (max(n - 5, 0), 8)):
        both_formats(cuda_api, oracle_api, comp, ocomp, sc.width, sc.height, first, k, sc.crop)


@pytest.mark.parametrize("name", sorted(ss.SCENES))
def test_styles(cuda_api, oracle_api, name):
    comp, _, sc = ss.build(cuda_api, name)
    ocomp, _, _ = ss.build(oracle_api, name)
    both_formats(cuda_api, oracle_api, comp, ocomp, sc.width, sc.height, 0, min(n_orders(ocomp), 96))


@pytest.mark.parametrize("fmt", ["f32", "u8"])
def test_random_mixed_1080p_crop_padded(cuda_api, oracle_api, fmt):
    w, h, k, first = 1920, 1080, 24, 300
    build = lambda api, comp: synth.random_mixed(api, comp, 900, w, h, 17)  # noqa: E731
    comp, ocomp = cuda_api.Composition(), oracle_api.Composition()
    build(cuda_api, comp)
    build(oracle_api, ocomp)
    crop = Rect((130, 1500), (70, 1010))
    want = oracle_masks.render(oracle_api, ocomp, w, h, first, k, fmt, crop)
    bpp = BPP[fmt]
    stride, plane_stride = bpp * w + 20, (bpp * w + 20) * h + 36
    r = cuda_api.Renderer(0)
    for offset in (0, 4):
        dev = Planes(1, k, w, h, fmt, stride, plane_stride, offset)
        r.render_masks_device(comp, dev.ptr, w, h, first, k, fmt, crop=crop, stride=stride, plane_stride=plane_stride)
        got, _ = dev.planes()
        raw = dev.raw()[dev.offset:]
        x0, x1, y0, y1 = 128, 1504, 64, 1024
        for j in range(k):
            plane = raw[j * plane_stride:j * plane_stride + h * stride].reshape(h, stride)
            inside = np.zeros(plane.shape, bool)
            inside[y0:y1, x0 * bpp:x1 * bpp] = True
            assert_planes(plane[inside].view(DTYPES[fmt]).reshape(y1 - y0, x1 - x0), want[j, y0:y1, x0:x1], f"plane {j}")
            assert (plane[~inside] == SENTINEL).all()
    host = np.full(k * plane_stride, SENTINEL, np.uint8)
    r.render_masks(comp, host.view(DTYPES[fmt]), w, h, first, n_orders=k, crop=crop, stride=stride, plane_stride=plane_stride)
    for j in range(k):
        plane = host[j * plane_stride:j * plane_stride + h * stride].reshape(h, stride)
        assert_planes(plane[64:1024, 128 * bpp:1504 * bpp].copy().view(DTYPES[fmt]), want[j, 64:1024, 128:1504], f"host plane {j}")
        assert (plane[:64] == SENTINEL).all() and (plane[:, :128 * bpp] == SENTINEL).all()


def test_paris4k_window(cuda_api, oracle_api):
    comp, w, h = workloads.build_scene(cuda_api, "paris4k")
    ocomp, _, _ = workloads.build_scene(oracle_api, "paris4k")
    r = cuda_api.Renderer(0)
    for first in (0, 20000):
        for fmt in ("f32", "u8"):
            want = oracle_masks.render(oracle_api, ocomp, w, h, first, 64, fmt)
            got = device_masks(r, comp, w, h, first, 64, fmt)
            assert_planes(got, want, f"paris4k [{first}, {first + 64}) {fmt}")
            assert got.any()


# --- views and batches --------------------------------------------------------------------------------


def _oracle_views(oracle_api, sc, first, k, fmt):
    comp, xf = vs.build(oracle_api, sc)
    out = []
    for v in sc.views:
        vs.set_view(comp, xf, v)
        out.append(oracle_masks.render(oracle_api, comp, sc.width, sc.height, first, k, fmt))
    return np.stack(out)


def _oracle_batch(oracle_api, sc, first, k, fmt):
    distinct, _ = bs.build(oracle_api, sc)
    per = [oracle_masks.render(oracle_api, c, sc.width, sc.height, first, k, fmt) for c in distinct]
    return np.stack([per[i] for i in sc.frames])


def _layouts(w, h, k, fmt):
    bpp = BPP[fmt]
    return [(None, None, 0), (bpp * w + 12, (bpp * w + 12) * h + 20, 4 if fmt == "f32" else 3)]


@pytest.mark.parametrize("fmt", ["f32", "u8"])
@pytest.mark.parametrize("name", vs.IN_LIMIT)
def test_views(cuda_api, oracle_api, name, fmt):
    sc = vs.SCENES[name]
    comp, _ = vs.build(cuda_api, sc)
    k = min(n_orders(comp) + 1, 40)
    want = _oracle_views(oracle_api, sc, 0, k, fmt)
    r = cuda_api.Renderer(0)
    for stride, plane_stride, offset in _layouts(sc.width, sc.height, k, fmt):
        dev = Planes(len(sc.views), k, sc.width, sc.height, fmt, stride, plane_stride, offset)
        r.render_views_masks_device(comp, sc.views, dev.ptr, sc.width, sc.height, 0, k, fmt, stride=dev.stride,
                                    plane_stride=dev.plane_stride)
        got, clean = dev.planes()
        assert_planes(got, want, name)
        assert clean, "bytes outside the planes were written"


@pytest.mark.parametrize("fmt", ["f32", "u8"])
@pytest.mark.parametrize("name", bs.IN_LIMIT)
def test_batches(cuda_api, oracle_api, name, fmt):
    sc = bs.SCENES[name]
    distinct, frames = bs.build(cuda_api, sc)
    k = min(max(n_orders(c) for c in distinct) + 1, 24)
    want = _oracle_batch(oracle_api, sc, 0, k, fmt)
    r = cuda_api.Renderer(0)
    for stride, plane_stride, offset in _layouts(sc.width, sc.height, k, fmt):
        dev = Planes(len(frames), k, sc.width, sc.height, fmt, stride, plane_stride, offset)
        r.render_batch_masks_device(frames, dev.ptr, sc.width, sc.height, 0, k, fmt, stride=dev.stride, plane_stride=dev.plane_stride)
        got, clean = dev.planes()
        assert_planes(got, want, name)
        assert clean, "bytes outside the planes were written"


# --- combined calls -----------------------------------------------------------------------------------


def _rgba(n, w, h):
    import torch
    return torch.full((n, h, w, 4), SENTINEL, dtype=torch.uint8, device="cuda:0")


def test_combined_single(cuda_api, oracle_api):
    import torch
    w, h = 300, 200
    comp, ocomp = cuda_api.Composition(), oracle_api.Composition()
    synth.random_mixed(cuda_api, comp, 150, w, h, 8)
    synth.random_mixed(oracle_api, ocomp, 150, w, h, 8)
    r = cuda_api.Renderer(0)
    crop = Rect((17, 250), (5, 190))
    for fmt in ("f32", "u8"):
        rgba, plain = _rgba(1, w, h), _rgba(1, w, h)
        got = device_masks(r, comp, w, h, 10, 30, fmt, crop=crop, rgba_ptr=rgba.data_ptr(), clear_color=CLEAR)
        r.render_device(comp, plain.data_ptr(), w, h, RGBA, CLEAR, crop=crop)
        torch.cuda.synchronize()
        assert torch.equal(rgba, plain)
        assert_planes(got, oracle_masks.render(oracle_api, ocomp, w, h, 10, 30, fmt, crop), fmt)


def test_combined_stacks(cuda_api, oracle_api):
    import torch
    r = cuda_api.Renderer(0)
    for name in ("straddle", "odd_h100"):
        sc = vs.SCENES[name]
        comp, _ = vs.build(cuda_api, sc)
        n, k = len(sc.views), n_orders(comp)
        dev, rgba, plain = Planes(n, k, sc.width, sc.height, "f32"), _rgba(n, sc.width, sc.height), _rgba(n, sc.width, sc.height)
        r.render_views_masks_device(comp, sc.views, dev.ptr, sc.width, sc.height, 0, k, "f32", rgba_ptr=rgba.data_ptr(),
                                    clear_color=CLEAR)
        r.render_views_device(comp, sc.views, plain.data_ptr(), sc.width, sc.height, RGBA, CLEAR)
        torch.cuda.synchronize()
        assert torch.equal(rgba, plain), name
        assert_planes(dev.planes()[0], _oracle_views(oracle_api, sc, 0, k, "f32"), name)
    for name in ("mixed_order", "repeats_h40"):
        sc = bs.SCENES[name]
        distinct, frames = bs.build(cuda_api, sc)
        n, k = len(frames), max(n_orders(c) for c in distinct)
        dev, rgba, plain = Planes(n, k, sc.width, sc.height, "u8"), _rgba(n, sc.width, sc.height), _rgba(n, sc.width, sc.height)
        r.render_batch_masks_device(frames, dev.ptr, sc.width, sc.height, 0, k, "u8", rgba_ptr=rgba.data_ptr(), clear_color=CLEAR)
        r.render_batch_device(frames, plain.data_ptr(), sc.width, sc.height, RGBA, CLEAR)
        torch.cuda.synchronize()
        assert torch.equal(rgba, plain), name
        assert_planes(dev.planes()[0], _oracle_batch(oracle_api, sc, 0, k, "u8"), name)


# --- table modes and schedule options -------------------------------------------------------------------

OPTIONS = ("speculate", "band_copy", "copy_bands", "sort_full_key", "sort_big_log2", "test_gap_cap", "paint_lpt", "paint_wide",
           "paint_solid", "sort_scan_log2", "band_filter", "sync_free", "test_fast_shrink", "host_slices", "slice_bands",
           "slice_min_points", "slice_chain", "sort_counts")


@pytest.fixture()
def restore_options(cuda_api):
    saved = {n: cuda_api.get_option(n) for n in OPTIONS}
    yield
    for n, v in saved.items():
        cuda_api.set_option(n, v)


@pytest.fixture(scope="module")
def mixed720(oracle_api):
    ocomp = oracle_api.Composition()
    synth.random_mixed(oracle_api, ocomp, 900, 1280, 720, 31)
    return {fmt: oracle_masks.render(oracle_api, ocomp, 1280, 720, 100, 48, fmt) for fmt in ("f32", "u8")}


@pytest.mark.parametrize("opts", [{"sync_free": 0}, {"sync_free": 1}, {"sync_free": 1, "test_fast_shrink": 1}])
def test_table_modes(cuda_api, mixed720, restore_options, opts):
    """Counted tables, sync-free tables, and halved bounds that send the frame through again: the
    redo repeats the zero fill and the mask kernel (its first attempt leaves every tile range empty)."""
    for k, v in opts.items():
        cuda_api.set_option(k, v)
    comp = cuda_api.Composition()
    synth.random_mixed(cuda_api, comp, 900, 1280, 720, 31)
    r = cuda_api.Renderer(0)
    for frame in range(3):
        for fmt in ("f32", "u8"):
            assert_planes(device_masks(r, comp, 1280, 720, 100, 48, fmt), mixed720[fmt], f"{opts} frame {frame} {fmt}")
    # Enough cells for halved bounds to fall short: 511 frames, twice; each frame's planes are those of
    # its composition rendered alone.
    sc = bs.SCENES["random_511"]
    distinct, frames = bs.build(cuda_api, sc)
    alone = [device_masks(r, c, sc.width, sc.height, 0, 6, "u8") for c in distinct]
    for _ in range(2):
        dev = Planes(len(frames), 6, sc.width, sc.height, "u8")
        r.render_batch_masks_device(frames, dev.ptr, sc.width, sc.height, 0, 6, "u8")
        got, clean = dev.planes()
        assert clean
        assert_planes(got, np.stack([alone[i] for i in sc.frames]), "random_511")


@pytest.mark.parametrize("name,value", [("speculate", 0), ("band_copy", 0), ("copy_bands", 16), ("sort_full_key", 1),
                                        ("sort_big_log2", 10), ("sort_scan_log2", 10), ("paint_lpt", 0), ("paint_wide", 1),
                                        ("paint_solid", 0), ("band_filter", 0), ("sync_free", 0), ("host_slices", 2),
                                        ("slice_bands", 1), ("slice_min_points", 0), ("slice_chain", 0), ("test_gap_cap", 1),
                                        ("sort_counts", 0)])
def test_option_does_not_change_the_masks(cuda_api, mixed720, restore_options, name, value):
    cuda_api.set_option(name, value)
    comp = cuda_api.Composition()
    synth.random_mixed(cuda_api, comp, 900, 1280, 720, 31)
    r = cuda_api.Renderer(0)
    for frame in range(2):
        for fmt in ("f32", "u8"):
            assert_planes(device_masks(r, comp, 1280, 720, 100, 48, fmt), mixed720[fmt], f"{name}={value} frame {frame} {fmt}")
        host = np.zeros((48, 720, 1280), np.float32)
        r.render_masks(comp, host, 1280, 720, 100)
        assert_planes(host, mixed720["f32"], f"{name}={value} host")


# --- refusals and caches ---------------------------------------------------------------------------------


def _raw_call(cuda_api, r, comp, m, w, h, rgba_ptr=None):
    ch, cc = (C.c_uint32 * 4)(*RGBA), (C.c_float * 4)(1.0, 1.0, 1.0, 0.0)
    return cuda_api.renderer_render_masks_device(r._h, comp._h, C.byref(m) if m is not None else None, w, h, None,
                                                 None if rgba_ptr is None else C.c_void_p(rgba_ptr), 4 * w, ch, cc, None)


def test_refusals_write_nothing(cuda_api):
    import torch
    w, h = 64, 64
    comp = cuda_api.Composition()
    scenes.E2E["clipping"](cuda_api, comp)
    r = cuda_api.Renderer(0)
    dev = Planes(1, 4, w, h, "f32")
    rgba = _rgba(1, w, h)
    good = dict(ptr=dev.ptr, first_order=0, n_orders=4, format=0, stride=4 * w, plane_stride=4 * w * h)
    cases = [dict(ptr=None), dict(n_orders=0), dict(first_order=(1 << 21) - 3), dict(format=2), dict(stride=4 * w - 4),
             dict(plane_stride=4 * w * h - 4), dict(stride=4 * w + 2, plane_stride=(4 * w + 2) * h), dict(ptr=dev.ptr + 2),
             dict(plane_stride=1 << 63)]  # 3 x 2^63: the stack of 4 planes overflows 64 bits
    for case in cases:
        args = {**good, **case}
        m = _CMasks(args["ptr"], args["first_order"], args["n_orders"], args["format"], args["stride"], args["plane_stride"])
        assert _raw_call(cuda_api, r, comp, m, w, h, rgba.data_ptr()) == 1, case
    assert _raw_call(cuda_api, r, comp, None, w, h, rgba.data_ptr()) == 1
    m = _CMasks(dev.ptr, 0, 4, 0, 4 * w, 4 * w * h)
    assert _raw_call(cuda_api, r, comp, m, 0, h) == 1
    assert _raw_call(cuda_api, r, comp, m, w, 1 << 20) == 1
    views = np.array([[1, 0, 0, 1, 0, 0]], np.float32)
    vp = views.ctypes.data_as(C.POINTER(C.c_float))
    for n in (0, 5000):  # no views, more than max_views(h)
        assert cuda_api.renderer_render_views_masks_device(r._h, comp._h, vp, n, C.byref(m), w, h, None, 0, 0, None, None, None) == 1
    comps = (C.c_void_p * 1)(None)
    assert cuda_api.renderer_render_batch_masks_device(r._h, comps, 1, C.byref(m), w, h, None, 0, 0, None, None, None) == 1
    torch.cuda.synchronize()
    assert bool(torch.all(dev.t == SENTINEL)) and bool(torch.all(rgba == SENTINEL))


def test_layer_cache_untouched(cuda_api, oracle_api):
    import torch
    w, h = 256, 160
    comp = cuda_api.Composition()
    synth.random_mixed(cuda_api, comp, 120, w, h, 12)
    r = cuda_api.Renderer(0)
    cache = r.create_buffer_layer_cache()
    a, b, c = _rgba(1, w, h), _rgba(1, w, h), _rgba(1, w, h)
    r.render_device(comp, a.data_ptr(), w, h, RGBA, CLEAR, layer_cache=cache)
    device_masks(r, comp, w, h, 0, 20, "f32")
    host = np.zeros((20, h, w), np.uint8)
    r.render_masks(comp, host, w, h, 0)
    b.copy_(a)
    r.render_device(comp, b.data_ptr(), w, h, RGBA, CLEAR, layer_cache=cache)  # nothing changed: the cache skips every tile
    r.render_device(comp, c.data_ptr(), w, h, RGBA, CLEAR)
    torch.cuda.synchronize()
    assert torch.equal(a, c) and torch.equal(b, c)


def test_cli_masks(cuda_api, tmp_path):
    from forma_b200 import svg
    svg_path = os.path.join(ROOT, "tests", "golden", "paris30k_excerpt.svg")
    out, masks = tmp_path / "out.ppm", tmp_path / "masks.npy"
    for u8 in (False, True):
        subprocess.check_call([sys.executable, "-m", "forma_b200.render", svg_path, str(out), "--width", "400", "--height", "300",
                               "--masks", str(masks), "--mask-orders", "3:40"] + (["--mask-u8"] if u8 else []), cwd=ROOT)
        got = np.load(masks)
        comp = cuda_api.Composition()
        svg.compose(cuda_api, comp, svg.parse_svg(svg_path))
        want = np.zeros((37, 300, 400), np.uint8 if u8 else np.float32)
        cuda_api.Renderer(0).render_masks(comp, want, 400, 300, 3)
        assert got.dtype == want.dtype and np.array_equal(got, want)
        assert got.any()
