"""Batches (Renderer.render_batch / render_batch_device) on the device, at tolerance 0.

Frame c of a call equals the oracle's ordinary frame of its composition (tests/batch_scenes.py),
for host and device buffers, frames painted in place and repacked, padded strides and gaps
between frames, and buffers prefilled with a sentinel whose bytes outside the frames' pixels must
survive. The sorted segments of a frame are those of its single frame, moved to the frame's rows
and its composition's order slice. Schedule switches, changes between batches, refusals, a
layer-cache sequence around a batch and the binding's chunking are covered too.
"""
import ctypes as C
import gc

import numpy as np
import pytest

import batch_scenes as bs
import line_model as lm
import scenes
from forma_b200.binding import RGBA, Color, FormaError, OrderError

pytestmark = pytest.mark.gpu

CLEAR = Color(1.0, 1.0, 1.0, 0.0)
SENTINEL = 0xA5
FORMA_ERR_INVALID_ARGUMENT = 1
FORMA_ERR_ORDER_LIMIT = 2
BATCH_FRAME_BYTES = 64  # BatchFrame, one per frame, then one u32 per frame + 1 (kernels.h)


def _oracle_frame(oracle_api, comp, w, h):
    r = oracle_api.Renderer(0)
    buf = np.zeros(w * h * 4, np.uint8)
    r.render(comp, buf, w, h, RGBA, CLEAR)
    return buf.reshape(h, w, 4)


_ORACLE = {}


def _oracle_frames(oracle_api, name):
    """The oracle's frame of every distinct composition of scene `name`."""
    if name not in _ORACLE:
        sc = bs.SCENES[name]
        distinct, _ = bs.build(oracle_api, sc)
        _ORACLE[name] = [_oracle_frame(oracle_api, c, sc.width, sc.height) for c in distinct]
    return _ORACLE[name]


def _unpack(raw, n, w, h, stride, frame_stride):
    frames = np.empty((n, h, w, 4), np.uint8)
    for c in range(n):
        for y in range(h):
            o = c * frame_stride + y * stride
            frames[c, y] = raw[o:o + 4 * w].reshape(w, 4)
    return frames


def _outside_untouched(raw, n, w, h, stride, frame_stride):
    mask = np.ones(raw.size, bool)
    for c in range(n):
        for y in range(h):
            o = c * frame_stride + y * stride
            mask[o:o + 4 * w] = False
    return bool(np.all(raw[mask] == SENTINEL))


def _batch_device(r, frames, w, h, stride=None, frame_stride=None):
    """(frames (N, H, W, 4), the raw buffer) of render_batch_device into a sentinel-filled tensor."""
    import torch
    n = len(frames)
    stride = 4 * w if stride is None else stride
    frame_stride = h * stride if frame_stride is None else frame_stride
    t = torch.full(((n - 1) * frame_stride + h * stride + 64,), SENTINEL, dtype=torch.uint8, device="cuda:0")
    r.render_batch_device(frames, t.data_ptr(), w, h, RGBA, CLEAR, stride=stride, frame_stride=frame_stride)
    torch.cuda.synchronize()
    raw = t.cpu().numpy()
    return _unpack(raw, n, w, h, stride, frame_stride), raw


def _check(got, oracle_api, name):
    want = _oracle_frames(oracle_api, name)
    for c, k in enumerate(bs.SCENES[name].frames):
        assert np.array_equal(got[c], want[k]), f"{name}: frame {c} (composition {k}) differs"


@pytest.mark.parametrize("name", bs.IN_LIMIT)
def test_device_batch_matches_oracle(cuda_api, oracle_api, name):
    sc = bs.SCENES[name]
    _, frames = bs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    got, raw = _batch_device(r, frames, sc.width, sc.height)
    _check(got, oracle_api, name)
    assert _outside_untouched(raw, len(frames), sc.width, sc.height, 4 * sc.width, 4 * sc.width * sc.height)


@pytest.mark.parametrize("name", ["e2e_all", "repeats_h40", "odd_h37", "odd_h1", "degenerate", "paris_tiles"])
def test_padded_batches_match_oracle(cuda_api, oracle_api, name):
    """Row padding and gaps between frames (the repack path on the device), and host buffers."""
    sc = bs.SCENES[name]
    w, h = sc.width, sc.height
    _, frames = bs.build(cuda_api, sc)
    n = len(frames)
    stride, frame_stride = 4 * w + 12, h * (4 * w + 12) + 20
    r = cuda_api.Renderer(0)
    got, raw = _batch_device(r, frames, w, h, stride, frame_stride)
    _check(got, oracle_api, name)
    assert _outside_untouched(raw, n, w, h, stride, frame_stride)
    for s, fst in ((4 * w, 4 * w * h), (stride, frame_stride)):
        host = np.full((n - 1) * fst + h * s + 64, SENTINEL, np.uint8)
        r.render_batch(frames, host, w, h, RGBA, CLEAR, stride=s, frame_stride=fst)
        _check(_unpack(host, n, w, h, s, fst), oracle_api, name)
        assert _outside_untouched(host, n, w, h, s, fst)


@pytest.mark.parametrize("name", ["e2e_all", "mixed_order", "clip_leak", "degenerate"])
def test_batch_equals_render_device(cuda_api, name):
    import torch
    sc = bs.SCENES[name]
    w, h = sc.width, sc.height
    distinct, frames = bs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    got, _ = _batch_device(r, frames, w, h)
    for c, comp in enumerate(frames):
        t = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda:0")
        r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR)
        torch.cuda.synchronize()
        assert np.array_equal(got[c].reshape(-1), t.cpu().numpy()), f"{name}: frame {c}"


LAYER_MASK = np.uint64(((1 << 21) - 1) << 20)


@pytest.mark.parametrize("name", ["repeats", "clip_leak", "mixed_order", "e2e_all", "odd_h37"])
def test_batch_segments_are_the_single_frames_moved(cuda_api, name):
    import torch
    sc = bs.SCENES[name]
    w, h, rows = sc.width, sc.height, bs.rows(sc.height)
    distinct, frames = bs.build(cuda_api, sc)
    bases = bs.order_bases(frames, {id(c): bs.n_orders(c) for c in distinct})
    r = cuda_api.Renderer(0)
    _batch_device(r, frames, w, h)
    segs = r.segments()
    ty = (segs >> np.uint64(53)).astype(np.int64)
    total = 0
    for c, comp in enumerate(frames):
        r1 = cuda_api.Renderer(0)
        t = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda:0")
        r1.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR)
        torch.cuda.synchronize()
        one = r1.segments()
        total += one.size
        one_ty = (one >> np.uint64(53)).astype(np.int64)
        want = one[(one_ty >= 1) & (one_ty <= rows)]
        got = segs[(ty >= c * rows + 1) & (ty <= (c + 1) * rows)]
        layer = (got & LAYER_MASK) - np.uint64(bases[c] << 20)
        got = (got & ~LAYER_MASK) - np.uint64(c * rows) * np.uint64(1 << 53) + layer
        assert np.array_equal(np.sort(got), np.sort(want)), f"{name}: frame {c} segments differ"
    assert segs.size == total


@pytest.mark.parametrize("opts", [{"sync_free": 0}, {"sync_free": 1}, {"sync_free": 1, "test_fast_shrink": 1},
                                  {"sort_full_key": 1}, {"sort_full_key": 0, "speculate": 0}, {"paint_wide": 1},
                                  {"paint_lpt": 0}])
def test_schedules(cuda_api, oracle_api, opts):
    saved = {k: cuda_api.get_option(k) for k in opts}
    try:
        for k, v in opts.items():
            cuda_api.set_option(k, v)
        r = cuda_api.Renderer(0)
        for name in ("mixed_order", "repeats", "e2e_all", "mixed_order"):  # single frames between batches, too
            sc = bs.SCENES[name]
            distinct, frames = bs.build(cuda_api, sc)
            buf = np.zeros(sc.width * sc.height * 4, np.uint8)
            r.render(distinct[0], buf, sc.width, sc.height, RGBA, CLEAR)
            got, _ = _batch_device(r, frames, sc.width, sc.height)
            _check(got, oracle_api, name)
    finally:
        for k, v in saved.items():
            cuda_api.set_option(k, v)


def test_changes_between_batches(cuda_api, oracle_api):
    """Props, a new insert, a removal with compaction and a freed composition replaced by a new one
    between batches; a repeated batch of unchanged compositions uploads its line-setup records only."""
    import torch
    w, h = 64, 64
    r = cuda_api.Renderer(0)

    def both(build):
        out = []
        for api in (cuda_api, oracle_api):
            out.append(build(api))
        return out

    def run(pairs):
        comps = [p[0] for p in pairs]
        got, _ = _batch_device(r, comps, w, h)
        for c, (_, ref) in enumerate(pairs):
            assert np.array_equal(got[c], _oracle_frame(oracle_api, ref, w, h)), f"frame {c}"

    a = both(bs._e2e("clipping"))
    b = both(bs._e2e("linear_gradient"))
    c = both(bs._random(7))
    run([a, b, c, a])
    # (a composition's first frame marks its device tables stale again when it makes its geometry
    # resident, as for single frames: the second call uploads them once more)
    run([a, b, c, a])
    before = r.counters()["h2d_bytes"]
    run([a, b, c, a])
    assert r.counters()["h2d_bytes"] - before == 4 * BATCH_FRAME_BYTES + 5 * 4
    # props
    for comp in a:
        comp.get(0).set_props(scenes.solid(Color(0.2, 0.7, 0.3, 0.9)))
    run([a, b, c, a])
    # a new insert
    for api, comp in zip((cuda_api, oracle_api), b):
        comp.get_mut_or_insert_default(7).insert(scenes.custom_circle(api, 20.0, 20.0, 15.0)).set_props(
            scenes.solid(Color(0.9, 0.9, 0.1, 0.5)))
    run([b, a, c])
    # removal of most layers' geometry (compaction at the next upload)
    for comp in c:
        for o in range(0, 20):
            if comp.get(o) is not None:
                comp.get(o).clear()
    run([c, a, b])
    # a freed composition, replaced by a new one built the same number of times
    del a
    gc.collect()
    d = both(bs._e2e("texture"))
    run([d, b, c, d])
    t = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda:0")
    r.render_device(d[0], t.data_ptr(), w, h, RGBA, CLEAR)
    torch.cuda.synchronize()
    assert np.array_equal(t.cpu().numpy().reshape(h, w, 4), _oracle_frame(oracle_api, d[1], w, h))


def _raw(cuda_api, r, comps, n, ptr, w, h, stride, frame_stride, fn=None):
    arr = (C.c_void_p * max(len(comps), 1))(*[None if c is None else c._h for c in comps])
    ch = (C.c_uint32 * 4)(*RGBA)
    cc = (C.c_float * 4)(CLEAR.r, CLEAR.g, CLEAR.b, CLEAR.a)
    fn = cuda_api.renderer_render_batch_device if fn is None else fn
    return fn(r._h, arr, n, C.c_void_p(ptr), w, stride, h, frame_stride, ch, cc, None)


def test_refusals_write_nothing(cuda_api, oracle_api):
    import torch
    w, h = 64, 40
    sc = bs.SCENES["repeats_h40"]
    distinct, frames = bs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    n_max = r.max_views(h)
    assert n_max == bs.max_frames(h)
    t = torch.full(((n_max + 1) * w * h * 4,), SENTINEL, dtype=torch.uint8, device="cuda:0")
    host = np.full((n_max + 1) * w * h * 4, SENTINEL, np.uint8)
    over, over_frames = bs.build(cuda_api, bs.SCENES["orders_over"])
    cases = [
        (frames[:1], 0, 4 * w * h, FORMA_ERR_INVALID_ARGUMENT),                       # n = 0
        ([frames[0]] * (n_max + 1), n_max + 1, 4 * w * h, FORMA_ERR_INVALID_ARGUMENT),  # one past the limit
        ([frames[0], None], 2, 4 * w * h, FORMA_ERR_INVALID_ARGUMENT),                 # a null entry
        (frames[:2], 2, (h - 1) * 4 * w + 4 * w - 1, FORMA_ERR_INVALID_ARGUMENT),       # frames would overlap
        (over_frames, 2, 4 * w * h, FORMA_ERR_ORDER_LIMIT),                            # 2^21 + 1 orders
    ]
    for comps, n, fst, want in cases:
        st = _raw(cuda_api, r, comps, n, t.data_ptr(), w, h, 4 * w, fst)
        torch.cuda.synchronize()
        assert st == want, (n, fst, st)
        assert bool(torch.all(t == SENTINEL)), (n, fst)
        st = _raw(cuda_api, r, comps, n, host.ctypes.data, w, h, 4 * w, fst, cuda_api.renderer_render_batch)
        assert st == want, ("host", n, fst, st)
        assert np.all(host == SENTINEL), ("host", n, fst)
    ch = (C.c_uint32 * 4)(*RGBA)
    cc = (C.c_float * 4)(CLEAR.r, CLEAR.g, CLEAR.b, CLEAR.a)
    assert cuda_api.renderer_render_batch_device(r._h, None, 1, C.c_void_p(t.data_ptr()), w, 4 * w, h, 4 * w * h, ch, cc,
                                                 None) == FORMA_ERR_INVALID_ARGUMENT
    bad_ch = (C.c_uint32 * 4)(0, 1, 2, 9)
    arr = (C.c_void_p * 1)(frames[0]._h)
    assert cuda_api.renderer_render_batch_device(r._h, arr, 1, C.c_void_p(t.data_ptr()), w, 4 * w, h, 4 * w * h, bad_ch, cc,
                                                 None) == FORMA_ERR_INVALID_ARGUMENT
    torch.cuda.synchronize()
    assert bool(torch.all(t == SENTINEL))
    with pytest.raises(OrderError):
        r.render_batch_device(over_frames, t.data_ptr(), w, h, RGBA, CLEAR)
    with pytest.raises(FormaError):
        r.render_batch(frames[:0], host, w, h, RGBA, CLEAR)
    assert np.all(host == SENTINEL)
    # at the limit it renders, and the next call is right
    assert _raw(cuda_api, r, [frames[0]] * n_max, n_max, t.data_ptr(), w, h, 4 * w, 4 * w * h) == 0
    got, _ = _batch_device(r, frames, w, h)
    _check(got, oracle_api, "repeats_h40")


def test_segment_limit_is_refused_then_next_call_matches(cuda_api, oracle_api):
    import torch
    sc = bs.SCENES["segment_limit"]
    w, h = sc.width, sc.height
    _, frames = bs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    t = torch.full((2 * w * h * 4,), SENTINEL, dtype=torch.uint8, device="cuda:0")
    st = _raw(cuda_api, r, frames, 2, t.data_ptr(), w, h, 4 * w, 4 * w * h)
    torch.cuda.synchronize()
    assert st == lm.FORMA_ERR_CAPACITY
    assert bool(torch.all(t == SENTINEL))
    assert r.counters()["segments"] == 0
    _, ok = bs.build(cuda_api, bs.SCENES["repeats"])
    got, _ = _batch_device(r, ok, 64, 64)
    _check(got, oracle_api, "repeats")


def test_layer_cache_sequence_around_batch(cuda_api, oracle_api):
    """Cached RGBA frames before and after a batch equal the oracle's, frame by frame."""
    w, h = 64, 64
    outs = []
    for api in (cuda_api, oracle_api):
        distinct, frames = bs.build(api, bs.SCENES["repeats"])
        comp = distinct[0]
        r = api.Renderer(0)
        cache = r.create_buffer_layer_cache()
        seq = []
        buf = np.zeros(w * h * 4, np.uint8)
        r.render(comp, buf, w, h, RGBA, CLEAR, layer_cache=cache)
        seq.append(buf.copy())
        if api is cuda_api:
            got, _ = _batch_device(r, frames, w, h)
            _check(got, oracle_api, "repeats")
        r.render(comp, buf, w, h, RGBA, CLEAR, layer_cache=cache)
        seq.append(buf.copy())
        comp.get(0).set_props(scenes.solid(Color(0.3, 0.3, 0.8, 0.7)))
        r.render(comp, buf, w, h, RGBA, CLEAR, layer_cache=cache)
        seq.append(buf.copy())
        outs.append(seq)
    for k, (a, b) in enumerate(zip(*outs)):
        assert np.array_equal(a, b), f"cached frame {k}"


def test_binding_chunks_like_single_frames(cuda_api, monkeypatch):
    sc = bs.SCENES["repeats"]
    w, h = sc.width, sc.height
    _, frames = bs.build(cuda_api, sc)
    n = len(frames)
    r = cuda_api.Renderer(0)
    singles = np.stack([_batch_device(r, [c], w, h)[0][0] for c in frames])
    monkeypatch.setattr(r, "max_views", lambda height: 2)
    chunked, _ = _batch_device(r, frames, w, h)
    assert np.array_equal(chunked, singles)
    host = np.zeros(n * w * h * 4, np.uint8)
    r.render_batch(frames, host, w, h, RGBA, CLEAR)
    assert np.array_equal(host.reshape(n, h, w, 4), singles)


def test_tensor_defaults(cuda_api, oracle_api):
    """A [N, H, W, 4] uint8 CUDA tensor's data_ptr() with the default strides; no line records after."""
    import torch
    sc = bs.SCENES["odd_h37"]
    _, frames = bs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    t = torch.zeros((len(frames), sc.height, sc.width, 4), dtype=torch.uint8, device="cuda:0")
    timings = r.render_batch_device(frames, t.data_ptr(), sc.width, sc.height, RGBA, CLEAR)
    torch.cuda.synchronize()
    _check(t.cpu().numpy(), oracle_api, "odd_h37")
    assert r.lines()["orders"].size == 0
    assert timings is not None
