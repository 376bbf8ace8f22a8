"""ID frames of views and batches (Renderer.render_views_ids* / render_batch_ids*) on the device,
at tolerance 0.

ID frame b of a views call equals the oracle's ID frame of the scene with every layer's transform
set to C = V_b ∘ T (tests/view_scenes.py); ID frame c of a batch equals the oracle's ID frame of
comps[c] alone (tests/batch_scenes.py), in the composition's own orders. Covered: every in-limit
scene of both files at two coverage thresholds, padded and misaligned layouts with the bytes
outside the frames untouched, the combined RGBA + ID call in every direct / repacked pairing, the
host variants, every table mode, refusals, and layer caches around an ID stack.
"""
import ctypes as C

import numpy as np
import pytest

import batch_scenes as bs
import oracle_ids
import scenes
import view_scenes as vs
from forma_b200.binding import ID_NONE, RGBA, Color, FormaError, OrderError

pytestmark = pytest.mark.gpu

CLEAR = Color(1.0, 1.0, 1.0, 0.0)
SENTINEL = 0xA5
FORMA_ERR_INVALID_ARGUMENT = 1
FORMA_ERR_ORDER_LIMIT = 2
FAR_LEFT = -(2.0 ** 20)  # views translated this far: render_ids_device of the single frame is not the reference


@pytest.fixture(autouse=True)
def _oracle_ids(oracle_api):
    oracle_ids.attach(oracle_api)


def _oracle_id_frame(oracle_api, comp, w, h, min_coverage):
    ids = np.zeros(w * h, np.uint32)
    oracle_api.Renderer(0).render_ids(comp, ids, w, h, min_coverage=min_coverage)
    return ids.reshape(h, w)


_ORACLE = {}


def _oracle_view_ids(oracle_api, name, min_coverage=0.0):
    """{view tuple: the oracle's ID frame (H, W)} of every distinct view of view scene `name`."""
    key = ("views", name, min_coverage)
    if key not in _ORACLE:
        sc = vs.SCENES[name]
        comp, xf = vs.build(oracle_api, sc)
        out = {}
        for v in sc.views:
            if tuple(v) not in out:
                vs.set_view(comp, xf, v)
                out[tuple(v)] = _oracle_id_frame(oracle_api, comp, sc.width, sc.height, min_coverage)
        _ORACLE[key] = out
    return _ORACLE[key]


def _oracle_batch_ids(oracle_api, name, min_coverage=0.0):
    """The oracle's ID frame of every distinct composition of batch scene `name`."""
    key = ("batch", name, min_coverage)
    if key not in _ORACLE:
        sc = bs.SCENES[name]
        distinct, _ = bs.build(oracle_api, sc)
        _ORACLE[key] = [_oracle_id_frame(oracle_api, c, sc.width, sc.height, min_coverage) for c in distinct]
    return _ORACLE[key]


def _check_views(got, oracle_api, name, min_coverage=0.0):
    want = _oracle_view_ids(oracle_api, name, min_coverage)
    for b, v in enumerate(vs.SCENES[name].views):
        assert np.array_equal(got[b], want[tuple(v)]), f"{name}: ID frame of view {b} differs"


def _check_batch(got, oracle_api, name, min_coverage=0.0):
    want = _oracle_batch_ids(oracle_api, name, min_coverage)
    for c, k in enumerate(bs.SCENES[name].frames):
        assert np.array_equal(got[c], want[k]), f"{name}: ID frame {c} (composition {k}) differs"


def _unpack(raw, n, w, h, stride, frame_stride, dtype=np.uint32):
    """Frames (n, h, w[, 4]) out of the bytes `raw`."""
    frames = np.empty((n, h, 4 * w), np.uint8)
    for b in range(n):
        for y in range(h):
            o = b * frame_stride + y * stride
            frames[b, y] = raw[o:o + 4 * w]
    return frames.view(np.uint32).reshape(n, h, w) if dtype == np.uint32 else frames.reshape(n, h, w, 4)


def _outside_untouched(raw, n, w, h, stride, frame_stride):
    mask = np.ones(raw.size, bool)
    for b in range(n):
        for y in range(h):
            o = b * frame_stride + y * stride
            mask[o:o + 4 * w] = False
    return bool(np.all(raw[mask] == SENTINEL))


class Target:
    """A sentinel-filled device buffer for a stack of n frames, its base `offset` bytes past the
    allocation (which is aligned to 256 bytes and more)."""

    def __init__(self, n, w, h, stride=None, frame_stride=None, offset=0):
        import torch
        self.n, self.w, self.h = n, w, h
        self.stride = 4 * w if stride is None else stride
        self.frame_stride = h * self.stride if frame_stride is None else frame_stride
        self.offset = offset
        self.t = torch.full((offset + (n - 1) * self.frame_stride + h * self.stride + 64,), SENTINEL, dtype=torch.uint8,
                            device="cuda:0")
        self.ptr = self.t.data_ptr() + offset

    def raw(self):
        import torch
        torch.cuda.synchronize()
        return self.t.cpu().numpy()[self.offset:]

    def frames(self, dtype=np.uint32):
        return _unpack(self.raw(), self.n, self.w, self.h, self.stride, self.frame_stride, dtype)

    def untouched_outside(self):
        whole = self.t.cpu().numpy()
        return bool(np.all(whole[:self.offset] == SENTINEL)) and _outside_untouched(self.raw(), self.n, self.w, self.h, self.stride,
                                                                                  self.frame_stride)

    def all_sentinel(self):
        import torch
        torch.cuda.synchronize()
        return bool(torch.all(self.t == SENTINEL))


def _views_ids(r, comp, sc, ids, rgba=None, min_coverage=0.0):
    r.render_views_ids_device(comp, sc.views, ids.ptr, sc.width, sc.height, rgba_ptr=rgba.ptr if rgba else None, channels=RGBA,
                              clear_color=CLEAR, stride=rgba.stride if rgba else None, view_stride=rgba.frame_stride if rgba else None,
                              ids_stride=ids.stride, ids_view_stride=ids.frame_stride, min_coverage=min_coverage)
    return ids.frames()


def _batch_ids(r, frames, sc, ids, rgba=None, min_coverage=0.0):
    r.render_batch_ids_device(frames, ids.ptr, sc.width, sc.height, rgba_ptr=rgba.ptr if rgba else None, channels=RGBA,
                              clear_color=CLEAR, stride=rgba.stride if rgba else None, frame_stride=rgba.frame_stride if rgba else None,
                              ids_stride=ids.stride, ids_frame_stride=ids.frame_stride, min_coverage=min_coverage)
    return ids.frames()


# ---------------------------------------------------------------------------
# Every in-limit scene against the oracle
# ---------------------------------------------------------------------------


@pytest.mark.parametrize("min_coverage", [0.0, 0.5])
@pytest.mark.parametrize("name", vs.IN_LIMIT)
def test_view_ids_match_oracle(cuda_api, oracle_api, name, min_coverage):
    sc = vs.SCENES[name]
    comp, _ = vs.build(cuda_api, sc)
    ids = Target(len(sc.views), sc.width, sc.height)
    got = _views_ids(cuda_api.Renderer(0), comp, sc, ids, min_coverage=min_coverage)
    _check_views(got, oracle_api, name, min_coverage)
    assert ids.untouched_outside()


@pytest.mark.parametrize("min_coverage", [0.0, 0.5])
@pytest.mark.parametrize("name", bs.IN_LIMIT)
def test_batch_ids_match_oracle(cuda_api, oracle_api, name, min_coverage):
    sc = bs.SCENES[name]
    _, frames = bs.build(cuda_api, sc)
    ids = Target(len(frames), sc.width, sc.height)
    got = _batch_ids(cuda_api.Renderer(0), frames, sc, ids, min_coverage=min_coverage)
    _check_batch(got, oracle_api, name, min_coverage)
    assert ids.untouched_outside()


def test_batch_ids_are_each_compositions_own_orders(cuda_api, oracle_api):
    """Compositions that all use orders from 0 up: every frame after the first would hold
    base + order without the rebase."""
    w, h = 64, 64
    builders = [bs._low_orders, bs._e2e("covers"), bs._low_orders, bs._e2e("clipping"), bs._out_of_order]
    sc = bs.BatchScene("own_orders", builders, w, h, [0, 1, 2, 3, 4, 2, 0])
    distinct, frames = bs.build(cuda_api, sc)
    ref, _ = bs.build(oracle_api, sc)
    ids = Target(len(frames), w, h)
    got = _batch_ids(cuda_api.Renderer(0), frames, sc, ids)
    tops = [bs.n_orders(c) for c in distinct]
    assert sum(tops[:-1]) > max(tops)  # the later slices lie beyond every composition's own orders
    for c, k in enumerate(sc.frames):
        assert np.array_equal(got[c], _oracle_id_frame(oracle_api, ref[k], w, h, 0.0)), f"frame {c}"
        hit = got[c][got[c] != ID_NONE]
        assert hit.size and int(hit.max()) < tops[k], f"frame {c}: IDs outside the composition's orders"


# ---------------------------------------------------------------------------
# Layouts: padding, misaligned bases, host buffers
# ---------------------------------------------------------------------------


@pytest.mark.parametrize("name", ["odd_h100", "odd_h1", "straddle", "e2e_clipping"])
def test_padded_view_ids(cuda_api, oracle_api, name):
    sc = vs.SCENES[name]
    w, h, n = sc.width, sc.height, len(sc.views)
    comp, _ = vs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    stride, frame_stride = 4 * w + 12, h * (4 * w + 12) + 20
    for offset, s, fs in ((0, stride, frame_stride), (4, stride, frame_stride), (4, 4 * w, 4 * w * h), (12, 4 * w + 4, h * (4 * w + 4))):
        ids = Target(n, w, h, s, fs, offset)
        _check_views(_views_ids(r, comp, sc, ids), oracle_api, name)
        assert ids.untouched_outside(), (offset, s, fs)
    for s, fs in ((4 * w, 4 * w * h), (stride, frame_stride)):
        host = np.full(((n - 1) * fs + h * s + 64) // 4, SENTINEL * 0x01010101, np.uint32)
        r.render_views_ids(comp, sc.views, host, w, h, ids_stride=s, ids_view_stride=fs)
        _check_views(_unpack(host.view(np.uint8), n, w, h, s, fs), oracle_api, name)
        assert _outside_untouched(host.view(np.uint8), n, w, h, s, fs)


@pytest.mark.parametrize("name", ["odd_h37", "odd_h1", "repeats_h40", "clip_leak"])
def test_padded_batch_ids(cuda_api, oracle_api, name):
    sc = bs.SCENES[name]
    w, h = sc.width, sc.height
    _, frames = bs.build(cuda_api, sc)
    n = len(frames)
    r = cuda_api.Renderer(0)
    stride, frame_stride = 4 * w + 12, h * (4 * w + 12) + 20
    for offset, s, fs in ((0, stride, frame_stride), (4, stride, frame_stride), (4, 4 * w, 4 * w * h), (12, 4 * w + 4, h * (4 * w + 4))):
        ids = Target(n, w, h, s, fs, offset)
        _check_batch(_batch_ids(r, frames, sc, ids), oracle_api, name)
        assert ids.untouched_outside(), (offset, s, fs)
    for s, fs in ((4 * w, 4 * w * h), (stride, frame_stride)):
        host = np.full(((n - 1) * fs + h * s + 64) // 4, SENTINEL * 0x01010101, np.uint32)
        r.render_batch_ids(frames, host, w, h, ids_stride=s, ids_frame_stride=fs)
        _check_batch(_unpack(host.view(np.uint8), n, w, h, s, fs), oracle_api, name)
        assert _outside_untouched(host.view(np.uint8), n, w, h, s, fs)


# ---------------------------------------------------------------------------
# RGBA + IDs from one pass
# ---------------------------------------------------------------------------

PAD = (12, 20)  # row padding, bytes between frames: the repacked layout


def _layout(w, h, direct):
    return (None, None) if direct else (4 * w + PAD[0], h * (4 * w + PAD[0]) + PAD[1])


@pytest.mark.parametrize("ids_direct", [True, False])
@pytest.mark.parametrize("rgba_direct", [True, False])
@pytest.mark.parametrize("kind", ["views", "batch"])
def test_rgba_with_ids_equals_the_separate_calls(cuda_api, kind, rgba_direct, ids_direct):
    """64 x 64 frames: contiguous stacks are painted in place, padded ones through the scratch."""
    if kind == "views":
        sc = vs.SCENES["e2e_texture"]
        comp, _ = vs.build(cuda_api, sc)
        n = len(sc.views)
    else:
        sc = bs.SCENES["e2e_all"]
        _, frames = bs.build(cuda_api, sc)
        n = len(frames)
    w, h = sc.width, sc.height
    r = cuda_api.Renderer(0)
    want_rgba, want_ids = Target(n, w, h), Target(n, w, h)
    if kind == "views":
        r.render_views_device(comp, sc.views, want_rgba.ptr, w, h, RGBA, CLEAR)
        _views_ids(r, comp, sc, want_ids)
    else:
        r.render_batch_device(frames, want_rgba.ptr, w, h, RGBA, CLEAR)
        _batch_ids(r, frames, sc, want_ids)
    assert (want_ids.frames() != ID_NONE).any()
    for attempt in range(2):  # counted tables, then sync-free
        rgba, ids = Target(n, w, h, *_layout(w, h, rgba_direct)), Target(n, w, h, *_layout(w, h, ids_direct))
        got = _views_ids(r, comp, sc, ids, rgba) if kind == "views" else _batch_ids(r, frames, sc, ids, rgba)
        assert np.array_equal(got, want_ids.frames()), f"IDs differ from the IDs-only call ({attempt})"
        assert np.array_equal(rgba.frames(np.uint8), want_rgba.frames(np.uint8)), f"RGBA differs from the RGBA call ({attempt})"
        assert rgba.untouched_outside() and ids.untouched_outside()


# ---------------------------------------------------------------------------
# A stacked frame is the single frame's ID frame
# ---------------------------------------------------------------------------


def _single_ids(r, comp, w, h):
    import torch
    t = torch.zeros(w * h, dtype=torch.int32, device="cuda:0")
    r.render_ids_device(comp, t.data_ptr(), w, h)
    torch.cuda.synchronize()
    return t.cpu().numpy().view(np.uint32).reshape(h, w)


@pytest.mark.parametrize("name", ["straddle", "far_compose", "extreme_crowd_64", "e2e_clipping2", "odd_h100"])
def test_view_ids_equal_render_ids_device(cuda_api, name):
    sc = vs.SCENES[name]
    w, h = sc.width, sc.height
    comp, _ = vs.build(cuda_api, sc)
    ref, xf = vs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    got = _views_ids(r, comp, sc, Target(len(sc.views), w, h))
    for b, v in enumerate(sc.views):
        if v[4] == FAR_LEFT:
            continue
        vs.set_view(ref, xf, v)
        assert np.array_equal(got[b], _single_ids(r, ref, w, h)), f"{name}: view {b}"


@pytest.mark.parametrize("name", ["e2e_all", "mixed_order", "clip_leak", "degenerate", "odd_h37"])
def test_batch_ids_equal_render_ids_device(cuda_api, name):
    sc = bs.SCENES[name]
    w, h = sc.width, sc.height
    _, frames = bs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    got = _batch_ids(r, frames, sc, Target(len(frames), w, h))
    for c, comp in enumerate(frames):
        assert np.array_equal(got[c], _single_ids(r, comp, w, h)), f"{name}: frame {c}"


# ---------------------------------------------------------------------------
# Table modes
# ---------------------------------------------------------------------------


@pytest.mark.parametrize("opts,mode", [({"sync_free": 0}, 0), ({"sync_free": 1}, 1), ({"sync_free": 1, "test_fast_shrink": 1}, 2)])
def test_table_modes(cuda_api, oracle_api, opts, mode):
    """Counted tables, sync-free tables, and halved bounds that send the frame through again:
    the paint step (paint kernel, then ID kernel) and both outputs are repeated."""
    saved = {k: cuda_api.get_option(k) for k in ("sync_free", "test_fast_shrink")}
    try:
        for k, v in opts.items():
            cuda_api.set_option(k, v)
        r = cuda_api.Renderer(0)
        for name in ("straddle", "odd_h100"):
            sc = vs.SCENES[name]
            comp, _ = vs.build(cuda_api, sc)
            buf = np.zeros(sc.width * sc.height * 4, np.uint8)
            r.render(comp, buf, sc.width, sc.height, RGBA, CLEAR)  # a frame before: bounds for the sync-free tables
            n = len(sc.views)
            for rgba in (None, Target(n, sc.width, sc.height), Target(n, sc.width, sc.height, *_layout(sc.width, sc.height, False))):
                _check_views(_views_ids(r, comp, sc, Target(n, sc.width, sc.height), rgba), oracle_api, name)
                if rgba is not None:
                    want = Target(n, sc.width, sc.height)
                    r.render_views_device(comp, sc.views, want.ptr, sc.width, sc.height, RGBA, CLEAR)
                    assert np.array_equal(rgba.frames(np.uint8), want.frames(np.uint8)), name
        for name in ("mixed_order", "repeats_h40"):
            sc = bs.SCENES[name]
            distinct, frames = bs.build(cuda_api, sc)
            buf = np.zeros(sc.width * sc.height * 4, np.uint8)
            r.render(distinct[0], buf, sc.width, sc.height, RGBA, CLEAR)
            n = len(frames)
            for rgba in (None, Target(n, sc.width, sc.height), Target(n, sc.width, sc.height, *_layout(sc.width, sc.height, False))):
                _check_batch(_batch_ids(r, frames, sc, Target(n, sc.width, sc.height), rgba), oracle_api, name)
                if rgba is not None:
                    want = Target(n, sc.width, sc.height)
                    r.render_batch_device(frames, want.ptr, sc.width, sc.height, RGBA, CLEAR)
                    assert np.array_equal(rgba.frames(np.uint8), want.frames(np.uint8)), name
        # Enough cells for the halved bounds to fall short: 511 frames painted in place, twice.
        sc = bs.SCENES["random_511"]
        _, frames = bs.build(cuda_api, sc)
        n = len(frames)
        for attempt in range(2):
            rgba, want = Target(n, sc.width, sc.height), Target(n, sc.width, sc.height)
            _check_batch(_batch_ids(r, frames, sc, Target(n, sc.width, sc.height), rgba), oracle_api, "random_511")
            assert r.counters()["tables_mode"] == (mode if attempt else min(2 * mode, 2))
            r.render_batch_device(frames, want.ptr, sc.width, sc.height, RGBA, CLEAR)
            assert np.array_equal(rgba.frames(np.uint8), want.frames(np.uint8))
    finally:
        for k, v in saved.items():
            cuda_api.set_option(k, v)


# ---------------------------------------------------------------------------
# Refusals
# ---------------------------------------------------------------------------


def _raw_views(cuda_api, r, comp, views, n, rgba_ptr, ids_ptr, w, h, ids_stride, ids_view_stride, min_coverage, host=False):
    v = np.ascontiguousarray(np.asarray(views, np.float32).reshape(-1, 6))
    vp = v.ctypes.data_as(C.POINTER(C.c_float))
    if host:
        return cuda_api.renderer_render_views_ids(r._h, comp._h, vp, n, C.c_void_p(ids_ptr), w, ids_stride, h, ids_view_stride,
                                                  min_coverage, None)
    ch = (C.c_uint32 * 4)(*RGBA)
    cc = (C.c_float * 4)(CLEAR.r, CLEAR.g, CLEAR.b, CLEAR.a)
    return cuda_api.renderer_render_views_ids_device(r._h, comp._h, vp, n, C.c_void_p(rgba_ptr), w, 4 * w, h, 4 * w * h, ch, cc,
                                                     C.c_void_p(ids_ptr), ids_stride, ids_view_stride, min_coverage, None)


def _raw_batch(cuda_api, r, comps, n, rgba_ptr, ids_ptr, w, h, ids_stride, ids_frame_stride, min_coverage, host=False):
    arr = (C.c_void_p * max(len(comps), 1))(*[None if c is None else c._h for c in comps])
    if host:
        return cuda_api.renderer_render_batch_ids(r._h, arr, n, C.c_void_p(ids_ptr), w, ids_stride, h, ids_frame_stride, min_coverage,
                                                  None)
    ch = (C.c_uint32 * 4)(*RGBA)
    cc = (C.c_float * 4)(CLEAR.r, CLEAR.g, CLEAR.b, CLEAR.a)
    return cuda_api.renderer_render_batch_ids_device(r._h, arr, n, C.c_void_p(rgba_ptr), w, 4 * w, h, 4 * w * h, ch, cc,
                                                     C.c_void_p(ids_ptr), ids_stride, ids_frame_stride, min_coverage, None)


def test_refusals_write_nothing(cuda_api, oracle_api):
    w, h = 64, 40
    vsc = vs.SCENES["straddle"]
    assert (vsc.width, vsc.height) == (w, h)
    comp, _ = vs.build(cuda_api, vsc)
    bsc = bs.SCENES["repeats_h40"]
    _, frames = bs.build(cuda_api, bsc)
    _, over_frames = bs.build(cuda_api, bs.SCENES["orders_over"])
    r = cuda_api.Renderer(0)
    n_max = r.max_views(h)
    rgba, ids = Target(n_max + 1, w, h), Target(n_max + 1, w, h)
    host = np.full((n_max + 1) * w * h, SENTINEL * 0x01010101, np.uint32)
    fs = 4 * w * h
    nan = float("nan")
    # (n, ids_stride, ids frame stride, min_coverage)
    layouts = [(2, 4 * w, fs, nan), (2, 4 * w, fs, 1.0), (2, 4 * w, fs, -0.25), (2, 4 * w, fs, float("inf")),
               (2, 4 * w + 2, fs + 2 * h, 0.0),        # ids_stride not a multiple of 4
               (2, 4 * w - 4, fs, 0.0),                # ids_stride short of a row
               (2, 4 * w, fs - 4, 0.0),                # frames would overlap
               (2, 4 * w, fs + 2, 0.0),                # frame stride not a multiple of 4
               (0, 4 * w, fs, 0.0), (n_max + 1, 4 * w, fs, 0.0)]
    views = [vs.IDENTITY] * (n_max + 1)
    comps = [frames[0]] * (n_max + 1)

    def nothing_written(what):
        assert rgba.all_sentinel() and ids.all_sentinel(), what
        assert np.all(host == SENTINEL * 0x01010101), what

    for n, s, f, mc in layouts:
        for rgba_ptr in (rgba.ptr, None):
            st = _raw_views(cuda_api, r, comp, views[:max(n, 1)], n, rgba_ptr, ids.ptr, w, h, s, f, mc)
            assert st == FORMA_ERR_INVALID_ARGUMENT, ("views", n, s, f, mc, st)
            st = _raw_batch(cuda_api, r, comps[:max(n, 1)], n, rgba_ptr, ids.ptr, w, h, s, f, mc)
            assert st == FORMA_ERR_INVALID_ARGUMENT, ("batch", n, s, f, mc, st)
        assert _raw_views(cuda_api, r, comp, views[:max(n, 1)], n, None, host.ctypes.data, w, h, s, f, mc, True) == FORMA_ERR_INVALID_ARGUMENT
        assert _raw_batch(cuda_api, r, comps[:max(n, 1)], n, None, host.ctypes.data, w, h, s, f, mc, True) == FORMA_ERR_INVALID_ARGUMENT
        nothing_written((n, s, f, mc))
    # a view that scales up, a null batch entry, the order-sum limit, a null ID buffer
    for host_call, ptr in ((False, ids.ptr), (True, host.ctypes.data)):
        rp = None if host_call else rgba.ptr
        assert _raw_views(cuda_api, r, comp, [vs.IDENTITY, [2.0, 0, 0, 1, 0, 0]], 2, rp, ptr, w, h, 4 * w, fs, 0.0,
                          host_call) == FORMA_ERR_INVALID_ARGUMENT
        assert _raw_batch(cuda_api, r, [frames[0], None], 2, rp, ptr, w, h, 4 * w, fs, 0.0, host_call) == FORMA_ERR_INVALID_ARGUMENT
        assert _raw_batch(cuda_api, r, over_frames, 2, rp, ptr, w, h, 4 * w, fs, 0.0, host_call) == FORMA_ERR_ORDER_LIMIT
        assert _raw_views(cuda_api, r, comp, [vs.IDENTITY], 1, rp, None, w, h, 4 * w, fs, 0.0, host_call) == FORMA_ERR_INVALID_ARGUMENT
        assert _raw_batch(cuda_api, r, frames[:1], 1, rp, None, w, h, 4 * w, fs, 0.0, host_call) == FORMA_ERR_INVALID_ARGUMENT
        nothing_written(("arguments", host_call))
    with pytest.raises(OrderError):
        r.render_batch_ids_device(over_frames, ids.ptr, w, h, rgba_ptr=rgba.ptr)
    with pytest.raises(FormaError):
        r.render_views_ids_device(comp, vsc.views, ids.ptr, w, h, min_coverage=1.0)
    with pytest.raises(FormaError):
        r.render_batch_ids(frames[:0], host, w, h)
    nothing_written("binding")
    # at the limit it renders, and the next calls are right
    assert _raw_batch(cuda_api, r, comps[:n_max], n_max, rgba.ptr, ids.ptr, w, h, 4 * w, fs, 0.0) == 0
    _check_batch(_batch_ids(r, frames, bsc, Target(len(frames), w, h)), oracle_api, "repeats_h40")
    _check_views(_views_ids(r, comp, vsc, Target(len(vsc.views), w, h)), oracle_api, "straddle")


# ---------------------------------------------------------------------------
# Layer caches
# ---------------------------------------------------------------------------


def test_id_stacks_between_cached_frames(cuda_api, oracle_api):
    """ID stacks (views and a batch, with and without RGBA) between two cached RGBA frames: the
    second cached frame and the tiles it writes are what they are without the stacks."""
    sc = bs.SCENES["repeats"]
    w, h = sc.width, sc.height
    runs = []
    for with_stacks in (False, True):
        distinct, frames = bs.build(cuda_api, sc)
        comp = distinct[0]
        r = cuda_api.Renderer(0)
        cache = r.create_buffer_layer_cache()
        buf = np.zeros(w * h * 4, np.uint8)
        seq, written = [], []

        def cached():
            r.render(comp, buf, w, h, RGBA, CLEAR, layer_cache=cache)
            seq.append(buf.copy())
            written.append(r.counters()["written_tiles"])
        cached()
        if with_stacks:
            n = len(frames)
            _check_batch(_batch_ids(r, frames, sc, Target(n, w, h)), oracle_api, "repeats")
            _check_batch(_batch_ids(r, frames, sc, Target(n, w, h), Target(n, w, h)), oracle_api, "repeats")
            views = vs.e2e_views(64)[:3]
            vsc = vs.ViewScene("around_cache", None, w, h, views)
            r.render_views_ids_device(comp, views, Target(3, w, h).ptr, w, h)
            _views_ids(r, comp, vsc, Target(3, w, h), Target(3, w, h))
        cached()
        comp.get(0).set_props(scenes.solid(Color(0.3, 0.3, 0.8, 0.7)))
        cached()
        runs.append((seq, written))
    (plain, plain_written), (stacked, stacked_written) = runs
    assert plain_written == stacked_written and plain_written[1] == 0
    for k, (a, b) in enumerate(zip(plain, stacked)):
        assert np.array_equal(a, b), f"cached frame {k}"
    # and the oracle agrees with the sequence
    distinct, _ = bs.build(oracle_api, sc)
    r = oracle_api.Renderer(0)
    cache = r.create_buffer_layer_cache()
    buf = np.zeros(w * h * 4, np.uint8)
    for k in range(3):
        if k == 2:
            distinct[0].get(0).set_props(scenes.solid(Color(0.3, 0.3, 0.8, 0.7)))
        r.render(distinct[0], buf, w, h, RGBA, CLEAR, layer_cache=cache)
        assert np.array_equal(buf, stacked[k]), f"cached frame {k} against the oracle"


# ---------------------------------------------------------------------------
# The binding
# ---------------------------------------------------------------------------


def test_binding_chunks_like_single_frames(cuda_api, monkeypatch):
    import torch
    sc = bs.SCENES["repeats"]
    w, h = sc.width, sc.height
    _, frames = bs.build(cuda_api, sc)
    n = len(frames)
    r = cuda_api.Renderer(0)
    want_ids, want_rgba = Target(n, w, h), Target(n, w, h)
    _batch_ids(r, frames, sc, want_ids, want_rgba)
    monkeypatch.setattr(r, "max_views", lambda height: 2)
    ids = torch.zeros((n, h, w), dtype=torch.int32, device="cuda:0")
    rgba = torch.zeros((n, h, w, 4), dtype=torch.uint8, device="cuda:0")
    assert r.render_batch_ids_device(frames, ids.data_ptr(), w, h, rgba_ptr=rgba.data_ptr(), clear_color=CLEAR) is not None
    torch.cuda.synchronize()
    assert np.array_equal(ids.cpu().numpy().view(np.uint32), want_ids.frames())
    assert np.array_equal(rgba.cpu().numpy(), want_rgba.frames(np.uint8))
    host = np.zeros((n, h, w), np.uint32)
    r.render_batch_ids(frames, host, w, h)
    assert np.array_equal(host, want_ids.frames())
    views = vs.e2e_views(64)[:5]
    whole = np.zeros((5, h, w), np.uint32)
    monkeypatch.undo()
    r.render_views_ids(frames[0], views, whole, w, h)
    monkeypatch.setattr(r, "max_views", lambda height: 2)
    vids = torch.zeros((5, h, w), dtype=torch.int32, device="cuda:0")
    r.render_views_ids_device(frames[0], views, vids.data_ptr(), w, h)
    torch.cuda.synchronize()
    assert np.array_equal(vids.cpu().numpy().view(np.uint32), whole)
    assert r.lines()["orders"].size == 0
