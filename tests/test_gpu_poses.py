"""Poses (Renderer.render_poses and its ID, mask and statistics twins) on the device, at tolerance 0.

Frame b of a call equals the oracle's ordinary frame of the scene put into pose b
(tests/pose_scenes.py: set_pose), and render_device of the composition put into that pose, for
host and device buffers, frames painted in place and repacked, padded strides, and buffers
prefilled with a sentinel whose bytes outside the frames' pixels must survive. The sorted segments
of frame b are the single frame's moved to its rows. IDs, masks and statistics equal the
single-frame calls; the call leaves the composition as it was; the schedule switches and the
refusals are covered too.
"""
import ctypes as C

import numpy as np
import pytest

import pose_scenes as ps
from forma_b200 import binding
from forma_b200.binding import RGBA, Color, FormaError, Poses

pytestmark = pytest.mark.gpu

CLEAR = Color(1.0, 1.0, 1.0, 0.0)
SENTINEL = 0xA5
FORMA_ERR_INVALID_ARGUMENT = 1
_ORACLE = {}


def _oracle_frames(oracle_api, name, frames=None):
    """{b: the oracle's frame (H, W, 4) of pose b} for the frames asked for (all by default)."""
    sc = ps.SCENES[name]
    frames = range(sc.n) if frames is None else frames
    cache = _ORACLE.setdefault(name, {})
    todo = [b for b in frames if b not in cache]
    if todo:
        comp, orders = sc.build(oracle_api)
        r = oracle_api.Renderer(0)
        for b in todo:
            ps.set_pose(comp, sc, orders, b)
            buf = np.zeros(sc.width * sc.height * 4, np.uint8)
            r.render(comp, buf, sc.width, sc.height, RGBA, CLEAR)
            cache[b] = buf.reshape(sc.height, sc.width, 4)
    return cache


def _twin_frames(cuda_api, name, frames=None):
    """{b: render_device (H, W, 4) of a second composition put into pose b}."""
    import torch
    sc = ps.SCENES[name]
    comp, orders = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    out = {}
    t = torch.zeros(sc.width * sc.height * 4, dtype=torch.uint8, device="cuda:0")
    for b in (range(sc.n) if frames is None else frames):
        ps.set_pose(comp, sc, orders, b)
        r.render_device(comp, t.data_ptr(), sc.width, sc.height, RGBA, CLEAR)
        torch.cuda.synchronize()
        out[b] = t.cpu().numpy().reshape(sc.height, sc.width, 4)
    return out


def _unpack(raw, n, w, h, stride, view_stride, bpp=4):
    frames = np.empty((n, h, w * bpp), np.uint8)
    for b in range(n):
        for y in range(h):
            o = b * view_stride + y * stride
            frames[b, y] = raw[o:o + bpp * w]
    return frames.reshape(n, h, w, bpp) if bpp == 4 else frames


def _outside_untouched(raw, n, w, h, stride, view_stride, bpp=4):
    mask = np.ones(raw.size, bool)
    for b in range(n):
        for y in range(h):
            o = b * view_stride + y * stride
            mask[o:o + bpp * w] = False
    return bool(np.all(raw[mask] == SENTINEL))


def _poses_device(r, comp, sc, stride=None, view_stride=None):
    """(frames (N, H, W, 4), the raw buffer) of render_poses_device into a sentinel-filled tensor."""
    import torch
    w, h, n = sc.width, sc.height, sc.n
    stride = 4 * w if stride is None else stride
    view_stride = h * stride if view_stride is None else view_stride
    t = torch.full(((n - 1) * view_stride + h * stride + 64,), SENTINEL, dtype=torch.uint8, device="cuda:0")
    r.render_poses_device(comp, ps.poses(binding, sc), t.data_ptr(), w, h, RGBA, CLEAR, stride=stride, view_stride=view_stride)
    torch.cuda.synchronize()
    raw = t.cpu().numpy()
    return _unpack(raw, n, w, h, stride, view_stride), raw


def _check(frames, want, name):
    for b, f in want.items():
        assert np.array_equal(frames[b], f), f"{name}: pose {b} differs"


@pytest.mark.parametrize("name", ps.LIGHT)
def test_poses_match_oracle_and_render_device(cuda_api, oracle_api, name):
    sc = ps.SCENES[name]
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    frames, raw = _poses_device(r, comp, sc)
    _check(frames, _oracle_frames(oracle_api, name), name)
    _check(frames, _twin_frames(cuda_api, name), name)
    assert _outside_untouched(raw, sc.n, sc.width, sc.height, 4 * sc.width, 4 * sc.width * sc.height)


@pytest.mark.parametrize("name", ps.HEAVY)
def test_workload_poses(cuda_api, oracle_api, name):
    """spaceship1080p (200 frames, chunks of 30), paris with 50 620 translated layers, the shape
    library (511 frames in one call): every frame against render_device, a spread against the oracle."""
    sc = ps.SCENES[name]
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    frames, raw = _poses_device(r, comp, sc)
    assert _outside_untouched(raw, sc.n, sc.width, sc.height, 4 * sc.width, 4 * sc.width * sc.height)
    _check(frames, _twin_frames(cuda_api, name), name)
    spread = sorted({0, 1, sc.n // 2, sc.n - 1} | set(range(0, sc.n, max(sc.n // 8, 1))))
    _check(frames, _oracle_frames(oracle_api, name, spread), name)


@pytest.mark.parametrize("name", ["nonfinite", "e2e_texture", "e2e_clipping", "clip_hidden", "window_gaps", "show_hide"])
def test_padded_and_host_poses(cuda_api, oracle_api, name):
    """Row and frame padding (the repack path on the device), and host buffers."""
    sc = ps.SCENES[name]
    w, h, n = sc.width, sc.height, sc.n
    stride, view_stride = 4 * w + 12, h * (4 * w + 12) + 20
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    want = _oracle_frames(oracle_api, name)
    frames, raw = _poses_device(r, comp, sc, stride, view_stride)
    _check(frames, want, name)
    assert _outside_untouched(raw, n, w, h, stride, view_stride)
    for s, vst in ((4 * w, 4 * w * h), (stride, view_stride)):
        host = np.full((n - 1) * vst + h * s + 64, SENTINEL, np.uint8)
        r.render_poses(comp, ps.poses(binding, sc), host, w, h, RGBA, CLEAR, stride=s, view_stride=vst)
        _check(_unpack(host, n, w, h, s, vst), want, name)
        assert _outside_untouched(host, n, w, h, s, vst)


@pytest.mark.parametrize("name", ["nonfinite", "inf_points", "e2e_covers", "show_hide", "window_top", "clip_moved"])
def test_pose_segments_are_the_single_frames_moved(cuda_api, unsliced, name):
    import torch
    sc = ps.SCENES[name]
    w, h, rows = sc.width, sc.height, (sc.height + 15) // 16
    comp, _ = sc.build(cuda_api)
    ref, orders = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    _poses_device(r, comp, sc)
    segs = np.sort(r.segments())
    ty = (segs >> np.uint64(53)).astype(np.int64)
    for b in range(sc.n):
        ps.set_pose(ref, sc, orders, b)
        t = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda:0")
        r1 = cuda_api.Renderer(0)
        r1.render_device(ref, t.data_ptr(), w, h, RGBA, CLEAR)
        torch.cuda.synchronize()
        one = np.sort(r1.segments())
        one_ty = (one >> np.uint64(53)).astype(np.int64)
        want = one[(one_ty >= 1) & (one_ty <= rows)]
        got = segs[(ty >= b * rows + 1) & (ty <= (b + 1) * rows)] - np.uint64(b * rows) * np.uint64(1 << 53)
        assert np.array_equal(np.sort(got), np.sort(want)), f"{name}: pose {b} segments differ"


@pytest.mark.parametrize("name", ["e2e_clipping", "clip_hidden", "clip_moved", "clip2_both", "show_hide", "window_gaps", "e2e_texture",
                                  "nonfinite", "library_511x64"])
def test_ids_masks_stats_equal_single_frames(cuda_api, name):
    """IDs at two thresholds, F32 and U8 masks and statistics of every pose equal the single-frame
    calls on the composition put into that pose; the RGBA stack of each pass equals render_poses_device."""
    import torch
    sc = ps.SCENES[name]
    w, h, n = sc.width, sc.height, sc.n
    comp, orders = sc.build(cuda_api)
    ref, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    p = ps.poses(binding, sc)
    rgba_want, _ = _poses_device(r, comp, sc)
    first, K = (0, 8) if not orders else (max(orders[0] - 1, 0), min(orders[-1] + 2, ps.LAYER_LIMIT) - max(orders[0] - 1, 0))
    K = min(K, 66)
    dev = "cuda:0"
    rgba = torch.zeros((n, h, w, 4), dtype=torch.uint8, device=dev)
    ids = {mc: torch.zeros((n, h, w), dtype=torch.int32, device=dev) for mc in (0.0, 0.5)}
    for mc, t in ids.items():
        rgba.zero_()
        r.render_poses_ids_device(comp, p, t.data_ptr(), w, h, rgba_ptr=rgba.data_ptr(), channels=RGBA, clear_color=CLEAR,
                                  min_coverage=mc)
        torch.cuda.synchronize()
        assert np.array_equal(rgba.cpu().numpy(), rgba_want), f"{name}: RGBA with IDs"
    host_ids = np.zeros((n, h, w), np.uint32)
    r.render_poses_ids(comp, p, host_ids, w, h, min_coverage=0.5)
    masks = {}
    for fmt, dt in (("f32", torch.float32), ("u8", torch.uint8)):
        masks[fmt] = torch.zeros((n, K, h, w), dtype=dt, device=dev)
        rgba.zero_()
        r.render_poses_masks_device(comp, p, masks[fmt].data_ptr(), w, h, first, K, format=fmt, rgba_ptr=rgba.data_ptr(),
                                    clear_color=CLEAR)
        torch.cuda.synchronize()
        assert np.array_equal(rgba.cpu().numpy(), rgba_want), f"{name}: RGBA with masks"
    stats = torch.zeros((n, K, 12), dtype=torch.int32, device=dev)
    rgba.zero_()
    r.render_poses_stats_device(comp, p, stats.data_ptr(), w, h, first, K, min_coverage=0.25, rgba_ptr=rgba.data_ptr(),
                                clear_color=CLEAR)
    torch.cuda.synchronize()
    assert np.array_equal(rgba.cpu().numpy(), rgba_want), f"{name}: RGBA with statistics"
    got = {k: v.cpu().numpy() for k, v in ids.items()}
    got_m = {k: v.cpu().numpy() for k, v in masks.items()}
    got_s = stats.cpu().numpy()
    r1 = cuda_api.Renderer(0)
    one_ids = torch.zeros((h, w), dtype=torch.int32, device=dev)
    one_m = {"f32": torch.zeros((K, h, w), dtype=torch.float32, device=dev), "u8": torch.zeros((K, h, w), dtype=torch.uint8, device=dev)}
    one_s = torch.zeros((K, 12), dtype=torch.int32, device=dev)
    for b in range(n):
        ps.set_pose(ref, sc, orders, b)
        for mc in ids:
            r1.render_ids_device(ref, one_ids.data_ptr(), w, h, min_coverage=mc)
            torch.cuda.synchronize()
            assert np.array_equal(got[mc][b], one_ids.cpu().numpy()), f"{name}: pose {b} IDs at {mc}"
        assert np.array_equal(host_ids[b], got[0.5][b].view(np.uint32)), f"{name}: pose {b} host IDs"
        for fmt, t in one_m.items():
            r1.render_masks_device(ref, t.data_ptr(), w, h, first, K, format=fmt)
            torch.cuda.synchronize()
            assert np.array_equal(got_m[fmt][b], t.cpu().numpy()), f"{name}: pose {b} {fmt} masks"
        r1.render_stats_device(ref, one_s.data_ptr(), w, h, first, K, min_coverage=0.25)
        torch.cuda.synchronize()
        assert np.array_equal(got_s[b], one_s.cpu().numpy()), f"{name}: pose {b} statistics"


def _state(comp, orders):
    return [(o, comp.get(o).is_enabled()) for o in orders]


@pytest.mark.parametrize("name", ["show_hide", "window_gaps", "e2e_clipping", "library_511x64"])
def test_call_leaves_the_composition(cuda_api, name):
    """Enabled states read back unchanged, the frame rendered afterwards is the one before (so are
    the layer transforms), and the ordinary render right after the call uploads nothing."""
    import torch
    sc = ps.SCENES[name]
    w, h = sc.width, sc.height
    comp, orders = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    t = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda:0")
    h2d = lambda: r.counters()["h2d_bytes"]  # noqa: E731
    for _ in range(2):
        r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR)
    b0 = h2d()
    r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR)  # what an ordinary render uploads with nothing changed
    torch.cuda.synchronize()
    idle, before, state = h2d() - b0, t.cpu().numpy(), _state(comp, orders)
    _poses_device(r, comp, sc)
    assert _state(comp, orders) == state
    t.zero_()
    b1 = h2d()
    r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR)
    torch.cuda.synchronize()
    assert h2d() - b1 <= idle, "the render after a poses call uploaded"
    assert np.array_equal(t.cpu().numpy(), before)


def test_layer_cache_sequence_with_a_poses_call(cuda_api):
    """A cached sequence with a poses call in the middle gives the bytes and written-tile counts of
    the same sequence without it."""
    sc = ps.SCENES["window_gaps"]
    w, h = sc.width, sc.height
    runs = []
    for with_poses in (False, True):
        comp, orders = sc.build(cuda_api)
        r = cuda_api.Renderer(0)
        cache = r.create_buffer_layer_cache()
        seq, written = [], []
        buf = np.zeros(w * h * 4, np.uint8)
        for step in range(4):
            if step == 2:
                ps.set_pose(comp, sc, orders, 1)
            r.render(comp, buf, w, h, RGBA, CLEAR, layer_cache=cache)
            seq.append(buf.copy())
            written.append(r.counters()["written_tiles"])
            if step == 0 and with_poses:
                _poses_device(r, comp, sc)
        runs.append((seq, written))
    (a, wa), (b, wb) = runs
    assert wa == wb
    for k, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x, y), f"cached frame {k}"


@pytest.mark.parametrize("opts", [{"sync_free": 0}, {"sync_free": 1}, {"sync_free": 1, "test_fast_shrink": 1}, {"speculate": 0},
                                  {"speculate": 1}, {"sort_full_key": 0}, {"sort_full_key": 1}, {"sort_counts": 0},
                                  {"sort_counts": 1}, {"paint_solid": 0}, {"paint_solid": 1}, {"paint_lpt": 0}, {"paint_lpt": 1}])
def test_switches(cuda_api, oracle_api, opts):
    saved = {k: cuda_api.get_option(k) for k in opts}
    try:
        for k, v in opts.items():
            cuda_api.set_option(k, v)
        r = cuda_api.Renderer(0)
        for name in ("show_hide", "e2e_texture", "clip_hidden", "window_gaps", "show_hide"):  # single frames between, too
            sc = ps.SCENES[name]
            comp, _ = sc.build(cuda_api)
            buf = np.zeros(sc.width * sc.height * 4, np.uint8)
            r.render(comp, buf, sc.width, sc.height, RGBA, CLEAR)
            frames, _ = _poses_device(r, comp, sc)
            _check(frames, _oracle_frames(oracle_api, name), name)
    finally:
        for k, v in saved.items():
            cuda_api.set_option(k, v)


def test_refusals_write_nothing(cuda_api):
    import torch
    sc = ps.SCENES["show_hide"]
    w, h = sc.width, sc.height
    comp, orders = sc.build(cuda_api)
    state = _state(comp, orders)
    r = cuda_api.Renderer(0)
    n_max = r.max_views(h)
    t = torch.full(((n_max + 1) * w * h * 4,), SENTINEL, dtype=torch.uint8, device="cuda:0")
    ids = torch.full(((n_max + 1) * w * h,), -1, dtype=torch.int32, device="cuda:0")
    host = np.full((n_max + 1) * w * h * 4, SENTINEL, np.uint8)
    ch = (C.c_uint32 * 4)(*RGBA)
    cc = (C.c_float * 4)(CLEAR.r, CLEAR.g, CLEAR.b, CLEAR.a)
    ident = np.tile(np.asarray(ps.IDENTITY, np.float32), (n_max + 1, 4, 1))
    scale = ident.copy()
    scale[1, 2] = [2.0, 0.0, 0.0, 1.0, 0.0, 0.0]
    vis = np.ones((n_max + 1, 4), np.uint8)

    def desc(first, k, tr, vi):
        return binding._CPoses(first, k, None if tr is None else tr.ctypes.data, None if vi is None else vi.ctypes.data)

    cases = [
        ("null poses", None, 2, 4 * w * h),
        ("no tables", desc(0, 4, None, None), 2, 4 * w * h),
        ("K = 0", desc(0, 0, ident, vis), 2, 4 * w * h),
        ("past 2^21", desc(ps.LAYER_LIMIT - 3, 4, ident, vis), 2, 4 * w * h),
        ("scales up", desc(0, 4, scale, vis), 3, 4 * w * h),
        ("n = 0", desc(0, 4, ident, vis), 0, 4 * w * h),
        ("overlap", desc(0, 4, ident, vis), 2, (h - 1) * 4 * w + 4 * w - 1),
        ("past max_views", desc(0, 4, ident, vis), n_max + 1, 4 * w * h),
    ]
    for what, d, n, vst in cases:
        dp = None if d is None else C.byref(d)
        st = cuda_api.renderer_render_poses_device(r._h, comp._h, dp, n, C.c_void_p(t.data_ptr()), w, 4 * w, h, vst, ch, cc, None)
        assert st == FORMA_ERR_INVALID_ARGUMENT, what
        st = cuda_api.renderer_render_poses(r._h, comp._h, dp, n, C.c_void_p(host.ctypes.data), w, 4 * w, h, vst, ch, cc, None)
        assert st == FORMA_ERR_INVALID_ARGUMENT, ("host", what)
        st = cuda_api.renderer_render_poses_ids_device(r._h, comp._h, dp, n, C.c_void_p(t.data_ptr()), w, 4 * w, h, vst, ch, cc,
                                                       C.c_void_p(ids.data_ptr()), 4 * w, vst, 0.0, None)
        assert st == FORMA_ERR_INVALID_ARGUMENT, ("ids", what)
        m = binding._CMasks(ids.data_ptr(), 0, 2, 0, 4 * w, vst)
        st = cuda_api.renderer_render_poses_masks_device(r._h, comp._h, dp, n, C.byref(m), w, h, C.c_void_p(t.data_ptr()), 4 * w, vst,
                                                         ch, cc, None)
        assert st == FORMA_ERR_INVALID_ARGUMENT, ("masks", what)
        s = binding._CStats(ids.data_ptr(), 0, 2, 0.0)
        st = cuda_api.renderer_render_poses_stats_device(r._h, comp._h, dp, n, C.byref(s), w, h, C.c_void_p(t.data_ptr()), 4 * w, vst,
                                                         ch, cc, None)
        assert st == FORMA_ERR_INVALID_ARGUMENT, ("stats", what)
        torch.cuda.synchronize()
        assert bool(torch.all(t == SENTINEL)) and bool(torch.all(ids == -1)), what
        assert np.all(host == SENTINEL), what
        assert _state(comp, orders) == state, what
    d = desc(0, 4, scale, vis)
    cuda_api.renderer_render_poses_device(r._h, comp._h, C.byref(d), 3, C.c_void_p(t.data_ptr()), w, 4 * w, h, 4 * w * h, ch, cc, None)
    msg = cuda_api.last_error().decode()
    assert "frame 1" in msg and "order 2" in msg, msg
    with pytest.raises(ValueError):
        Poses(0)
    # at the limit it renders
    d = desc(0, 4, ident, vis)
    assert cuda_api.renderer_render_poses_device(r._h, comp._h, C.byref(d), n_max, C.c_void_p(t.data_ptr()), w, 4 * w, h, 4 * w * h,
                                                 ch, cc, None) == 0
    with pytest.raises(FormaError):
        r.render_poses_device(comp, Poses(0, np.tile(np.asarray([[[2.0, 0, 0, 1, 0, 0]]], np.float32), (1, 4, 1))), t.data_ptr(), w, h)


def test_tensor_defaults_and_chunks(cuda_api, oracle_api, monkeypatch):
    """A [N, H, W, 4] uint8 CUDA tensor with the default strides, chunked by the binding."""
    import torch
    name = "transform_only"
    sc = ps.SCENES[name]
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    monkeypatch.setattr(r, "max_views", lambda height: 2)
    t = torch.zeros((sc.n, sc.height, sc.width, 4), dtype=torch.uint8, device="cuda:0")
    r.render_poses_device(comp, ps.poses(binding, sc), t.data_ptr(), sc.width, sc.height, RGBA, CLEAR)
    torch.cuda.synchronize()
    _check(t.cpu().numpy(), _oracle_frames(oracle_api, name), name)
    assert r.lines()["orders"].size == 0
