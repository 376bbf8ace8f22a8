"""The oracle's linear float frames (fo_renderer_render_linear, tests/oracle_linear.py), pinned
without a GPU: encoded with compute_srgb they are libforma_oracle.so's sRGB8 frames (the
golden-pinned oracle) for every e2e golden scene, every scene of tests/extremes.py and a
random_mixed scene in the reference's six channel orders, both oracles with recip mode 0. Also
the binding of the six linear entry points (default strides and chunking with the library calls
replaced by recorders), their declarations in the header, and the oracle library, which has none
of them, still loading through the same binding. tests/test_gpu_linear.py then holds the device
to these frames."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import extremes
import oracle_linear
import scenes
import synth
from forma_b200 import binding
from forma_b200.binding import BGR0, BGR1, BGRA, RGB0, RGB1, RGBA, Color, Rect, Renderer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORDERS = {"RGBA": RGBA, "BGRA": BGRA, "RGB0": RGB0, "BGR0": BGR0, "RGB1": RGB1, "BGR1": BGR1}


@pytest.fixture(autouse=True)
def _recip_mode_0(oracle_api):
    oracle_api.hooks.fo_set_recip_mode(0)


def srgb_of(oracle_api, comp, w, h, channels, clear, crop=None):
    buf = np.zeros(w * h * 4, np.uint8)
    oracle_api.Renderer(0).render(comp, buf, w, h, channels, clear, crop)
    return buf.reshape(h, w, 4)


def assert_encodes_to(oracle_api, comp, w, h, channels, clear, crop=None, what=""):
    frame = oracle_linear.render(oracle_api, comp, w, h, channels, clear, crop)
    got, want = oracle_linear.encode(frame, channels), srgb_of(oracle_api, comp, w, h, channels, clear, crop)
    if not np.array_equal(got, want):
        ys, xs = np.nonzero((got != want).any(axis=2))
        raise AssertionError(f"{what}: {len(ys)} pixels differ, first at x={xs[0]} y={ys[0]}: encoded "
                             f"{got[ys[0], xs[0]]} from {frame[ys[0], xs[0]]}, sRGB8 oracle {want[ys[0], xs[0]]}")
    return frame


@pytest.mark.parametrize("order", list(ORDERS))
@pytest.mark.parametrize("name", list(scenes.E2E))
def test_e2e_scene_encodes_to_the_oracle(oracle_api, name, order):
    comp = oracle_api.Composition()
    scenes.E2E[name](oracle_api, comp)
    assert_encodes_to(oracle_api, comp, 64, 64, ORDERS[order], scenes.E2E_CLEAR, what=f"{name} {order}")


@pytest.mark.parametrize("name", list(extremes.SCENES))
def test_extreme_scene_encodes_to_the_oracle(oracle_api, name):
    comp, _, sc = extremes.build(oracle_api, name)
    for order, ch in ORDERS.items():
        assert_encodes_to(oracle_api, comp, sc.width, sc.height, ch, scenes.E2E_CLEAR, sc.crop, f"{name} {order}")


@pytest.mark.parametrize("clear", [Color(1.0, 1.0, 1.0, 0.0), Color(0.2, 0.4, 0.6, 1.0)])
def test_random_mixed_encodes_to_the_oracle(oracle_api, clear):
    w, h = 200, 120
    comp = oracle_api.Composition()
    synth.random_mixed(oracle_api, comp, 150, w, h, 11)
    for order, ch in ORDERS.items():
        frame = assert_encodes_to(oracle_api, comp, w, h, ch, clear, what=order)
        if clear.a == 1.0 and ch[3] != binding.Channel.Zero:
            assert (frame[:, :, 3] == 1.0).all()  # ALPHA became ONE, as for sRGB8 frames
    frame = oracle_linear.render(oracle_api, comp, w, h, RGBA, Color(1.0, 1.0, 1.0, 0.0), Rect((20, 50), (17, 40)))
    outside = np.ones((h, w), bool)
    outside[16:48, 16:64] = False
    assert (frame[outside] == 0.0).all() and (frame[~outside] != 0.0).any()  # only the crop's tile rectangle


def test_hdr_values_are_not_clamped(oracle_api):
    w, h = oracle_linear.HDR_W, oracle_linear.HDR_H
    comp = oracle_api.Composition()
    oracle_linear.hdr_scene(oracle_api, comp)
    frame = assert_encodes_to(oracle_api, comp, w, h, RGBA, oracle_linear.HDR_CLEAR, what="hdr")
    s, c = oracle_linear.HDR_SOLID, oracle_linear.HDR_CLEAR
    assert (frame[:, :32] == np.array([s.r, s.g, s.b, 1.0], np.float32)).all()
    assert (frame[:, 94:] == np.array([c.r, c.g, c.b, 1.0], np.float32)).all()  # alpha: ONE
    circle = frame[8:56, 44:90, :3]
    assert (circle > 1.0).any() and (circle < 0.0).any()


def test_invalid_arguments_are_refused(oracle_api):
    comp = oracle_api.Composition()
    scenes.E2E["clipping"](oracle_api, comp)
    oracle_linear.attach(oracle_api)
    buf = np.full((64, 65, 4), 7.0, np.float32)
    r = oracle_api.Renderer(0)
    for kw in ({"stride": 16 * 64 - 4}, {"stride": 16 * 64 + 2}):
        with pytest.raises(binding.FormaError):
            r.render_linear(comp, buf, 64, 64, RGBA, Color(), **kw)
    assert (buf == 7.0).all()


# --- the binding -------------------------------------------------------------------------------
W, H = 10, 7


class _Handle:
    def __init__(self, h):
        self._h = h


class _Recorder:
    """Stands in for an Api: the six entry points record their arguments and succeed."""

    def __init__(self, max_views):
        self.calls = []
        self._max_views = max_views
        for name in binding.LINEAR_SYMBOLS:
            setattr(self, name, self._entry(name))

    def _entry(self, name):
        def call(*args):
            self.calls.append((name, [a.value if isinstance(a, C.c_void_p) else a for a in args]))
            return 0
        return call

    def renderer_max_views(self, height):
        return self._max_views

    def renderer_free(self, h):
        pass

    def check(self, status, what):
        assert status == 0, what


def _renderer(max_views):
    r = object.__new__(Renderer)
    r._api, r._h = _Recorder(max_views), 77
    return r


@pytest.mark.parametrize("fmt,code,bpp", [("f32", 2, 16), ("f16", 1, 8)])
def test_single_frame_defaults(fmt, code, bpp):
    r = _renderer(4)
    dtype = np.float32 if fmt == "f32" else np.float16
    buf = np.zeros((H, W, 4), dtype)
    r.render_linear(_Handle(5), buf, W, H, format=fmt, timings=False)
    r.render_linear_device(_Handle(5), 1 << 20, W, H, BGRA, Color(0.0, 0.0, 0.0, 1.0), format=fmt, stride=bpp * W + 16,
                           timings=False)
    (n0, a), (n1, b) = r._api.calls
    assert (n0, n1) == ("renderer_render_linear", "renderer_render_linear_device")
    assert a[:6] == [77, 5, buf.ctypes.data, W, bpp * W, H] and a[8:] == [None, code, None]
    assert b[:6] == [77, 5, 1 << 20, W, bpp * W + 16, H] and list(b[6]) == list(BGRA) and b[9] == code
    with pytest.raises(AssertionError):  # the other dtype
        r.render_linear(_Handle(5), np.zeros((H, W, 4), np.float64), W, H, format=fmt)
    with pytest.raises(AssertionError):  # too small
        r.render_linear(_Handle(5), np.zeros((H, W - 1, 4), dtype), W, H, format=fmt)
    with pytest.raises(ValueError):
        r.render_linear(_Handle(5), buf, W, H, format="u8")


@pytest.mark.parametrize("fmt,code,bpp", [("f32", 2, 16), ("f16", 1, 8)])
def test_batch_device_defaults_and_chunks(fmt, code, bpp):
    r = _renderer(2)
    comps = [_Handle(100 + k) for k in range(5)]
    r.render_batch_linear_device(comps, 1 << 30, W, H, clear_color=Color(0.0, 0.0, 0.0, 1.0), format=fmt, timings=False)
    calls = r._api.calls
    assert [c[0] for c in calls] == ["renderer_render_batch_linear_device"] * 3
    for k, (_, a) in enumerate(calls):
        first, count = 2 * k, min(2, 5 - 2 * k)
        handle, arr, n, ptr, w, stride, h, frame_stride, ch, cc, f, t = a
        assert (handle, n, w, h, f, t) == (77, count, W, H, code, None)
        assert [arr[i] for i in range(count)] == [100 + first + i for i in range(count)]
        assert (stride, frame_stride) == (bpp * W, bpp * W * H)
        assert ptr == (1 << 30) + first * bpp * W * H
        assert list(ch) == list(RGBA) and list(cc) == [0.0, 0.0, 0.0, 1.0]


def test_views_host_and_device_strides_and_chunks():
    r = _renderer(2)
    views = [[1.0, 0.0, 0.0, 1.0, float(k), 0.0] for k in range(3)]
    buf = np.zeros((3, H, W, 4), np.float16)
    r.render_views_linear(_Handle(5), views, buf, W, H, format="f16", timings=False)
    (n0, a), (n1, b) = r._api.calls
    assert n0 == n1 == "renderer_render_views_linear"
    assert (a[3], b[3]) == (2, 1)
    assert [a[2][i] for i in range(12)] == sum(views[:2], []) and [b[2][i] for i in range(6)] == views[2]
    assert a[4:9] == [buf.ctypes.data, W, 8 * W, H, 8 * W * H] and a[11:] == [1, None]
    assert b[4] == buf.ctypes.data + 2 * 8 * W * H
    r = _renderer(8)
    r.render_views_linear_device(_Handle(5), views, 4096, W, H, stride=16 * W + 32, view_stride=(16 * W + 32) * H + 64,
                                 timings=False)
    (_, a), = r._api.calls
    assert a[4:9] == [4096, W, 16 * W + 32, H, (16 * W + 32) * H + 64] and a[11] == 2
    with pytest.raises(AssertionError):
        r.render_batch_linear([_Handle(1)] * 3, np.zeros((2, H, W, 4), np.float32), W, H)


def test_the_header_declares_the_six_entry_points():
    with open(os.path.join(ROOT, "include", "forma_b200.h")) as f:
        header = f.read()
    assert re.search(r"FORMA_PIXEL_RGBA16F = 1, FORMA_PIXEL_RGBA32F = 2", header)
    for name in binding.LINEAR_SYMBOLS:
        assert name in binding.SIGNATURES
        m = re.search(r"\bint forma_%s\(([^;]*)\);" % name, header)
        assert m, name
        params = [p for p in m.group(1).split(",") if p.strip()]
        assert len(params) == len(binding.SIGNATURES[name][1]), name


def test_the_oracle_loads_without_them():
    from oracle import oracle
    api = oracle.load()
    for name in binding.LINEAR_SYMBOLS:
        assert not hasattr(api, name)
    assert hasattr(api, "renderer_render")
