"""Views (Renderer.render_views / render_views_device) on the device, at tolerance 0.

Frame b of a call equals the oracle's ordinary frame of the scene with every layer's transform
set to C = V_b ∘ T (tests/view_scenes.py), for host and device buffers, frames painted in place
and repacked, padded strides, and buffers prefilled with a sentinel whose bytes outside the
views' pixels must survive. The sorted segments of a view are those of the single frame, moved
to the view's rows; the schedule switches, refusals, a layer-cache sequence around a views call
and the binding's chunking are covered too.
"""
import ctypes as C

import numpy as np
import pytest

import line_model as lm
import view_scenes as vs
from forma_b200.binding import RGBA, Color, FormaError

pytestmark = pytest.mark.gpu

CLEAR = Color(1.0, 1.0, 1.0, 0.0)
SENTINEL = 0xA5
FORMA_ERR_INVALID_ARGUMENT = 1
_ORACLE = {}


def _oracle_frames(oracle_api, name):
    """{view tuple: the oracle's frame (H, W, 4)} of every distinct view of scene `name`."""
    if name not in _ORACLE:
        sc = vs.SCENES[name]
        comp, xf = vs.build(oracle_api, sc)
        r = oracle_api.Renderer(0)
        out = {}
        for v in sc.views:
            key = tuple(v)
            if key in out:
                continue
            vs.set_view(comp, xf, v)
            buf = np.zeros(sc.width * sc.height * 4, np.uint8)
            r.render(comp, buf, sc.width, sc.height, RGBA, CLEAR)
            out[key] = buf.reshape(sc.height, sc.width, 4)
        _ORACLE[name] = out
    return _ORACLE[name]


def _views_device(r, comp, sc, stride=None, view_stride=None, views=None):
    """(frames (N, H, W, 4), the raw buffer) of render_views_device into a sentinel-filled tensor."""
    import torch
    views = sc.views if views is None else views
    w, h, n = sc.width, sc.height, len(views)
    stride = 4 * w if stride is None else stride
    view_stride = h * stride if view_stride is None else view_stride
    size = (n - 1) * view_stride + h * stride + 64
    t = torch.full((size,), SENTINEL, dtype=torch.uint8, device="cuda:0")
    r.render_views_device(comp, views, t.data_ptr(), w, h, RGBA, CLEAR, stride=stride, view_stride=view_stride)
    torch.cuda.synchronize()
    raw = t.cpu().numpy()
    return _unpack(raw, n, w, h, stride, view_stride), raw


def _unpack(raw, n, w, h, stride, view_stride):
    frames = np.empty((n, h, w, 4), np.uint8)
    for b in range(n):
        for y in range(h):
            o = b * view_stride + y * stride
            frames[b, y] = raw[o:o + 4 * w].reshape(w, 4)
    return frames


def _outside_untouched(raw, n, w, h, stride, view_stride):
    mask = np.ones(raw.size, bool)
    for b in range(n):
        for y in range(h):
            o = b * view_stride + y * stride
            mask[o:o + 4 * w] = False
    return bool(np.all(raw[mask] == SENTINEL))


def _check(frames, oracle_api, name, views=None):
    want = _oracle_frames(oracle_api, name)
    for b, v in enumerate(vs.SCENES[name].views if views is None else views):
        assert np.array_equal(frames[b], want[tuple(v)]), f"{name}: view {b} differs"


@pytest.mark.parametrize("name", vs.IN_LIMIT)
def test_device_views_match_oracle(cuda_api, oracle_api, name):
    sc = vs.SCENES[name]
    comp, _ = vs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    frames, raw = _views_device(r, comp, sc)
    _check(frames, oracle_api, name)
    assert _outside_untouched(raw, len(sc.views), sc.width, sc.height, 4 * sc.width, 4 * sc.width * sc.height)


@pytest.mark.parametrize("name", ["straddle", "odd_h100", "e2e_texture", "e2e_clipping", "extreme_crowd_64", "paris_tiles"])
def test_padded_views_match_oracle(cuda_api, oracle_api, name):
    """Row and view padding (the repack path on the device), and a host buffer."""
    sc = vs.SCENES[name]
    w, h, n = sc.width, sc.height, len(sc.views)
    stride, view_stride = 4 * w + 12, h * (4 * w + 12) + 20
    comp, _ = vs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    frames, raw = _views_device(r, comp, sc, stride, view_stride)
    _check(frames, oracle_api, name)
    assert _outside_untouched(raw, n, w, h, stride, view_stride)
    for s, vst in ((4 * w, 4 * w * h), (stride, view_stride)):
        host = np.full((n - 1) * vst + h * s + 64, SENTINEL, np.uint8)
        r.render_views(comp, sc.views, host, w, h, RGBA, CLEAR, stride=s, view_stride=vst)
        _check(_unpack(host, n, w, h, s, vst), oracle_api, name)
        assert _outside_untouched(host, n, w, h, s, vst)


@pytest.mark.parametrize("name", ["e2e_linear_gradient", "straddle", "extreme_dense_stars", "inf_points"])
def test_identity_view_equals_render_device(cuda_api, name):
    import torch
    sc = vs.SCENES[name]
    w, h = sc.width, sc.height
    comp, _ = vs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    t = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda:0")
    r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR)
    torch.cuda.synchronize()
    want, want_n = t.cpu().numpy(), r.counters()["segments"]
    frames, _ = _views_device(r, comp, sc, views=[vs.IDENTITY])
    assert np.array_equal(frames[0].reshape(-1), want)
    assert r.counters()["segments"] == want_n


def test_composition_formula_device_against_device(cuda_api):
    """A view over layers with transforms T equals render_device with each layer's transform set
    to the model's C (device against device)."""
    for name in ("straddle", "far_compose", "far_compose_neg", "far_points", "far_left"):
        _device_against_device(cuda_api, vs.SCENES[name])


def _device_against_device(cuda_api, sc):
    import torch
    w, h = sc.width, sc.height
    comp, _ = vs.build(cuda_api, sc)
    ref, xf = vs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    frames, _ = _views_device(r, comp, sc)
    for b, v in enumerate(sc.views):
        vs.set_view(ref, xf, v)
        t = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda:0")
        r.render_device(ref, t.data_ptr(), w, h, RGBA, CLEAR)
        torch.cuda.synchronize()
        assert np.array_equal(frames[b].reshape(-1), t.cpu().numpy()), f"{sc.name}: view {b}"


@pytest.mark.parametrize("name", ["straddle", "straddle_h100", "far_compose", "far_points", "far_left", "inf_points", "e2e_covers",
                                  "extreme_crowd_64"])
def test_view_segments_are_the_single_frames_moved(cuda_api, unsliced, name):
    import torch
    sc = vs.SCENES[name]
    w, h, rows = sc.width, sc.height, vs.rows(sc.height)
    comp, _ = vs.build(cuda_api, sc)
    ref, xf = vs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    _views_device(r, comp, sc)
    segs = np.sort(r.segments())
    ty = (segs >> np.uint64(53)).astype(np.int64)
    total = 0
    for b, v in enumerate(sc.views):
        vs.set_view(ref, xf, v)
        t = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda:0")
        r1 = cuda_api.Renderer(0)
        r1.render_device(ref, t.data_ptr(), w, h, RGBA, CLEAR)
        torch.cuda.synchronize()
        one = np.sort(r1.segments())
        total += one.size
        one_ty = (one >> np.uint64(53)).astype(np.int64)
        want = one[(one_ty >= 1) & (one_ty <= rows)]
        got = segs[(ty >= b * rows + 1) & (ty <= (b + 1) * rows)]
        got = got - np.uint64(b * rows) * np.uint64(1 << 53)
        assert np.array_equal(np.sort(got), np.sort(want)), f"{name}: view {b} segments differ"
    assert segs.size == total


@pytest.mark.parametrize("opts", [{"sync_free": 0}, {"sync_free": 1}, {"sync_free": 1, "test_fast_shrink": 1},
                                  {"speculate": 0}, {"speculate": 1}])
def test_schedules(cuda_api, oracle_api, opts):
    saved = {k: cuda_api.get_option(k) for k in opts}
    try:
        for k, v in opts.items():
            cuda_api.set_option(k, v)
        r = cuda_api.Renderer(0)
        for name in ("straddle", "e2e_texture", "straddle", "odd_h100"):  # single frames between batches, too
            sc = vs.SCENES[name]
            comp, _ = vs.build(cuda_api, sc)
            buf = np.zeros(sc.width * sc.height * 4, np.uint8)
            r.render(comp, buf, sc.width, sc.height, RGBA, CLEAR)
            frames, _ = _views_device(r, comp, sc)
            _check(frames, oracle_api, name)
    finally:
        for k, v in saved.items():
            cuda_api.set_option(k, v)


def _raw(cuda_api, r, comp, views, n, ptr, w, h, stride, view_stride, fn=None):
    v = np.ascontiguousarray(np.asarray(views, np.float32).reshape(-1, 6))
    ch = (C.c_uint32 * 4)(*RGBA)
    cc = (C.c_float * 4)(CLEAR.r, CLEAR.g, CLEAR.b, CLEAR.a)
    fn = cuda_api.renderer_render_views_device if fn is None else fn
    return fn(r._h, comp._h, v.ctypes.data_as(C.POINTER(C.c_float)), n, C.c_void_p(ptr), w, stride, h, view_stride, ch, cc, None)


def test_refusals_write_nothing(cuda_api, oracle_api):
    import torch
    sc = vs.SCENES["straddle"]
    w, h = sc.width, sc.height
    comp, _ = vs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    n_max = r.max_views(h)
    assert n_max == 2046 // vs.rows(h)
    t = torch.full(((n_max + 1) * w * h * 4,), SENTINEL, dtype=torch.uint8, device="cuda:0")
    good = [vs.IDENTITY] * (n_max + 1)
    cases = [
        ([[float("nan"), 0, 0, 1, 0, 0]], 1, 4 * w * h),
        ([[1, 0, 0, 1, float("inf"), 0]], 1, 4 * w * h),
        ([[2.0, 0, 0, 1, 0, 0]], 1, 4 * w * h),          # scales up
        ([vs.IDENTITY, [0.6, 0.9, 0.9, -0.6, 0, 0]], 2, 4 * w * h),  # second view scales up
        ([vs.IDENTITY], 0, 4 * w * h),                     # n = 0
        ([vs.IDENTITY] * 2, 2, (h - 1) * 4 * w + 4 * w - 1),  # views would overlap
        (good, n_max + 1, 4 * w * h),                      # one past the limit
    ]
    host = np.full((n_max + 1) * w * h * 4, SENTINEL, np.uint8)
    for views, n, vst in cases:
        st = _raw(cuda_api, r, comp, views, n, t.data_ptr(), w, h, 4 * w, vst)
        torch.cuda.synchronize()
        assert st == FORMA_ERR_INVALID_ARGUMENT, (views[:2], n, vst)
        assert bool(torch.all(t == SENTINEL)), (views[:2], n, vst)
        st = _raw(cuda_api, r, comp, views, n, host.ctypes.data, w, h, 4 * w, vst, cuda_api.renderer_render_views)
        assert st == FORMA_ERR_INVALID_ARGUMENT, ("host", views[:2], n, vst)
        assert np.all(host == SENTINEL), ("host", views[:2], n, vst)
    with pytest.raises(FormaError):
        r.render_views(comp, np.zeros((0, 6), np.float32), host, w, h, RGBA, CLEAR)
    assert np.all(host == SENTINEL)
    with pytest.raises(FormaError):
        r.render_views_device(comp, np.zeros((0, 6), np.float32), t.data_ptr(), w, h, RGBA, CLEAR)
    # at the limit it renders
    assert _raw(cuda_api, r, comp, good, n_max, t.data_ptr(), w, h, 4 * w, 4 * w * h) == 0


def test_segment_limit_is_refused_then_next_call_matches(cuda_api, oracle_api):
    import torch
    sc = vs.SCENES["segment_limit"]
    w, h = sc.width, sc.height
    comp, _ = vs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    t = torch.full((2 * w * h * 4,), SENTINEL, dtype=torch.uint8, device="cuda:0")
    st = _raw(cuda_api, r, comp, sc.views, 2, t.data_ptr(), w, h, 4 * w, 4 * w * h)
    torch.cuda.synchronize()
    assert st == lm.FORMA_ERR_CAPACITY
    assert bool(torch.all(t == SENTINEL))
    assert r.counters()["segments"] == 0
    ok = vs.SCENES["straddle"]
    comp2, _ = vs.build(cuda_api, ok)
    frames, _ = _views_device(r, comp2, ok)
    _check(frames, oracle_api, "straddle")


@pytest.mark.parametrize("name", vs.LIMIT_SCENES)
def test_at_the_limit(cuda_api, oracle_api, name):
    sc = vs.SCENES[name]
    comp, _ = vs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    assert len(sc.views) == r.max_views(sc.height)
    frames, _ = _views_device(r, comp, sc)
    _check(frames, oracle_api, name)


def test_layer_cache_sequence_around_views(cuda_api, oracle_api):
    """Cached RGBA frames before and after a views call equal the oracle's, frame by frame."""
    sc = vs.SCENES["straddle"]
    w, h = sc.width, sc.height
    outs = []
    for api in (cuda_api, oracle_api):
        comp, xf = vs.build(api, sc)
        r = api.Renderer(0)
        cache = r.create_buffer_layer_cache()
        seq = []
        buf = np.zeros(w * h * 4, np.uint8)
        r.render(comp, buf, w, h, RGBA, CLEAR, layer_cache=cache)
        seq.append(buf.copy())
        if api is cuda_api:
            frames, _ = _views_device(r, comp, sc)
            _check(frames, oracle_api, "straddle")
        r.render(comp, buf, w, h, RGBA, CLEAR, layer_cache=cache)
        seq.append(buf.copy())
        vs.set_view(comp, xf, sc.views[0])
        r.render(comp, buf, w, h, RGBA, CLEAR, layer_cache=cache)
        seq.append(buf.copy())
        outs.append(seq)
    for k, (a, b) in enumerate(zip(*outs)):
        assert np.array_equal(a, b), f"cached frame {k}"


def test_binding_chunks_like_single_views(cuda_api, monkeypatch):
    sc = vs.SCENES["e2e_radial_gradient"]
    w, h, n = sc.width, sc.height, len(sc.views)
    comp, _ = vs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    singles = np.stack([_views_device(r, comp, sc, views=[v])[0][0] for v in sc.views])
    monkeypatch.setattr(r, "max_views", lambda height: 3)
    chunked, _ = _views_device(r, comp, sc)
    assert np.array_equal(chunked, singles)
    host = np.zeros(n * w * h * 4, np.uint8)
    r.render_views(comp, sc.views, host, w, h, RGBA, CLEAR)
    assert np.array_equal(host.reshape(n, h, w, 4), singles)


def test_tensor_defaults(cuda_api, oracle_api):
    """A [N, H, W, 4] uint8 CUDA tensor's data_ptr() with the default strides."""
    import torch
    sc = vs.SCENES["odd_h100"]
    comp, _ = vs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    t = torch.zeros((len(sc.views), sc.height, sc.width, 4), dtype=torch.uint8, device="cuda:0")
    r.render_views_device(comp, sc.views, t.data_ptr(), sc.width, sc.height, RGBA, CLEAR)
    torch.cuda.synchronize()
    _check(t.cpu().numpy(), oracle_api, "odd_h100")
    assert r.lines()["orders"].size == 0
