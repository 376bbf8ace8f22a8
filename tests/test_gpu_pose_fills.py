"""Pose fills (Poses with colours) on the device, at tolerance 0, in every frame format.

Frame b of a call equals the oracle's frame of the scene put into frame b's state
(tests/pose_fill_scenes.py: set_pose_fill): sRGB8 byte for byte, RGBA32F bit for bit (a NaN
matches any NaN), RGBA16F as the oracle's f32 rounded to half, and over a different background
per frame in all three formats. It also equals the single-frame call (render_device,
render_linear_device, render_over_device) on a binding composition after the same edits, and
so do its IDs, masks and statistics. Host and device buffers, padded strides, chunking, the
composition left unchanged, the schedule switches and the refusals are covered too.
"""
import ctypes as C

import numpy as np
import pytest

import oracle_linear
import oracle_over
import pose_fill_scenes as pfs
from forma_b200 import binding
from forma_b200.binding import RGBA, Color, Poses

pytestmark = pytest.mark.gpu

CLEAR = Color(1.0, 1.0, 1.0, 0.0)
SENTINEL = 0xA5
FORMA_ERR_INVALID_ARGUMENT = 1
FORMA_ERR_CAPACITY = 5
DTYPES = {"srgb8": np.uint8, "f16": np.float16, "f32": np.float32}
BPP = {"srgb8": 4, "f16": 8, "f32": 16}
_ORACLE = {}


@pytest.fixture(autouse=True)
def _oracle_modes(oracle_api):
    oracle_linear.attach(oracle_api)
    oracle_api.hooks.fo_set_recip_mode(0)


def _torch_dtype(fmt):
    import torch
    return {"srgb8": torch.uint8, "f16": torch.float16, "f32": torch.float32}[fmt]


def assert_same(got, want, fmt, what):
    """got against want (the format's values; a float32 `want` is rounded to the format first)."""
    w = np.ascontiguousarray(np.asarray(want).astype(DTYPES[fmt]))
    g = np.ascontiguousarray(got, DTYPES[fmt])
    if fmt == "srgb8":
        bad = g != w
    else:
        bits = np.uint32 if fmt == "f32" else np.uint16
        bad = (g.view(bits) != w.view(bits)) & ~(np.isnan(g) & np.isnan(w))
    if bad.any():
        idx = tuple(int(i[0]) for i in np.nonzero(bad))
        raise AssertionError(f"{what} ({fmt}): {int(bad.sum())} values differ, first at {idx}: cuda {g[idx]!r} expected {w[idx]!r}")


def backgrounds(sc, fmt, seed=0):
    """[n, h, w, 4] of the format's dtype, a different background per frame: random values per 8 x 8
    block, float values in [-0.25, 1.25] with alpha in [0, 1], a third of the alphas exactly 1."""
    rng = np.random.default_rng(seed)
    n, h, w = sc.n, sc.height, sc.width
    v = rng.random((n, (h + 7) // 8, (w + 7) // 8, 4)).repeat(8, 1).repeat(8, 2)[:, :h, :w]
    if fmt == "srgb8":
        out = np.round(v * 255.0).astype(np.uint8)
        out[rng.random((n, h, w)) < 0.3, 3] = 255
        return out
    out = (v * 1.5 - 0.25).astype(np.float32)
    out[..., 3] = np.clip(v[..., 3], 0.0, 1.0)
    out[rng.random((n, h, w)) < 0.3, 3] = 1.0
    return out.astype(DTYPES[fmt])


def _oracle_frames(oracle_api, name, kind="srgb8", frames=None, bgs=None):
    """{b: the oracle's frame (H, W, 4) of frame b}: kind "srgb8" (uint8), "f32" (the linear float32
    frame) or "over" (over bgs[b], uint8 or float32; not cached)."""
    sc = pfs.SCENES[name]
    frames = range(sc.n) if frames is None else frames
    cache = {} if kind == "over" else _ORACLE.setdefault((name, kind), {})
    todo = [b for b in frames if b not in cache]
    if todo:
        comp, orders = sc.build(oracle_api)
        r = oracle_api.Renderer(0)
        for b in todo:
            pfs.set_pose_fill(comp, sc, orders, b)
            if kind == "srgb8":
                buf = np.zeros(sc.width * sc.height * 4, np.uint8)
                r.render(comp, buf, sc.width, sc.height, RGBA, CLEAR)
                cache[b] = buf.reshape(sc.height, sc.width, 4)
            elif kind == "f32":
                cache[b] = oracle_linear.render(oracle_api, comp, sc.width, sc.height, RGBA, CLEAR)
            else:
                f = np.array(bgs[b] if bgs.dtype == np.uint8 else bgs[b].astype(np.float32), order="C", copy=True)
                assert oracle_over.render(comp, f, RGBA) == 0
                cache[b] = f
    return {b: cache[b] for b in frames}


def _twin_frames(cuda_api, name, fmt="srgb8", frames=None, bgs=None):
    """{b: the single-frame call's frame (H, W, 4) of a binding composition put into frame b's state}:
    render_device (srgb8), render_linear_device (f16 / f32), or render_over_device over bgs[b]."""
    import torch
    sc = pfs.SCENES[name]
    comp, orders = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    out = {}
    for b in (range(sc.n) if frames is None else frames):
        pfs.set_pose_fill(comp, sc, orders, b)
        if bgs is not None:
            t = torch.from_numpy(np.ascontiguousarray(bgs[b])).to("cuda:0")
            r.render_over_device(comp, t.data_ptr(), sc.width, sc.height, RGBA, format=fmt)
        else:
            t = torch.zeros((sc.height, sc.width, 4), dtype=_torch_dtype(fmt), device="cuda:0")
            if fmt == "srgb8":
                r.render_device(comp, t.data_ptr(), sc.width, sc.height, RGBA, CLEAR)
            else:
                r.render_linear_device(comp, t.data_ptr(), sc.width, sc.height, RGBA, CLEAR, format=fmt)
        torch.cuda.synchronize()
        out[b] = t.cpu().numpy()
    return out


def _unpack(raw, n, w, h, stride, view_stride, bpp):
    frames = np.empty((n, h, w * bpp), np.uint8)
    for b in range(n):
        for y in range(h):
            o = b * view_stride + y * stride
            frames[b, y] = raw[o:o + bpp * w]
    return frames


def _outside_untouched(raw, n, w, h, stride, view_stride, bpp):
    mask = np.ones(raw.size, bool)
    for b in range(n):
        for y in range(h):
            o = b * view_stride + y * stride
            mask[o:o + bpp * w] = False
    return bool(np.all(raw[mask] == SENTINEL))


def _poses_device(r, comp, sc, fmt="srgb8", stride=None, view_stride=None, poses=None):
    """(frames (N, H, W, 4) of the format's dtype, raw bytes) of render_poses_device (srgb8) or
    render_poses_linear_device into a sentinel-filled buffer."""
    import torch
    w, h, n, bpp = sc.width, sc.height, sc.n, BPP[fmt]
    stride = bpp * w if stride is None else stride
    view_stride = h * stride if view_stride is None else view_stride
    t = torch.full(((n - 1) * view_stride + h * stride + 64,), SENTINEL, dtype=torch.uint8, device="cuda:0")
    p = pfs.poses(sc) if poses is None else poses
    if fmt == "srgb8":
        r.render_poses_device(comp, p, t.data_ptr(), w, h, RGBA, CLEAR, stride=stride, view_stride=view_stride)
    else:
        r.render_poses_linear_device(comp, p, t.data_ptr(), w, h, RGBA, CLEAR, format=fmt, stride=stride, view_stride=view_stride)
    torch.cuda.synchronize()
    raw = t.cpu().numpy()
    frames = _unpack(raw, n, w, h, stride, view_stride, bpp).view(DTYPES[fmt]).reshape(n, h, w, 4)
    assert _outside_untouched(raw, n, w, h, stride, view_stride, bpp)
    return frames, raw


def _poses_over(r, comp, sc, bgs, fmt, stride=None, view_stride=None):
    """The frames of render_poses_over_device over `bgs`, in a buffer with the given strides."""
    import torch
    w, h, n, bpp = sc.width, sc.height, sc.n, BPP[fmt]
    stride = bpp * w if stride is None else stride
    view_stride = h * stride if view_stride is None else view_stride
    raw = np.full((n - 1) * view_stride + h * stride + 64, SENTINEL, np.uint8)
    for b in range(n):
        for y in range(h):
            o = b * view_stride + y * stride
            raw[o:o + bpp * w] = bgs[b, y].view(np.uint8).reshape(-1)
    t = torch.from_numpy(raw).to("cuda:0")
    r.render_poses_over_device(comp, pfs.poses(sc), t.data_ptr(), w, h, RGBA, format=fmt, stride=stride, view_stride=view_stride)
    torch.cuda.synchronize()
    raw = t.cpu().numpy()
    assert _outside_untouched(raw, n, w, h, stride, view_stride, bpp)
    return _unpack(raw, n, w, h, stride, view_stride, bpp).view(DTYPES[fmt]).reshape(n, h, w, 4)


def _check(frames, want, fmt, name):
    for b, f in want.items():
        assert_same(frames[b], f, fmt, f"{name}: frame {b}")


@pytest.mark.parametrize("name", pfs.LIGHT)
def test_fills_match_oracle_and_single_frames(cuda_api, oracle_api, name):
    """sRGB8 and RGBA32F frames against the oracle and the single-frame calls."""
    sc = pfs.SCENES[name]
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    for fmt, kind in (("srgb8", "srgb8"), ("f32", "f32")):
        frames, _ = _poses_device(r, comp, sc, fmt)
        _check(frames, _oracle_frames(oracle_api, name, kind), fmt, name)
        _check(frames, _twin_frames(cuda_api, name, fmt), fmt, name)


@pytest.mark.parametrize("name", ["e2e_texture", "e2e_blend_modes__Luminosity", "blend_top_Hue", "clip_ignored", "alpha_edges",
                                  "nonfinite_colors", "window_gaps_filled"])
def test_half_host_and_padded(cuda_api, oracle_api, name):
    """RGBA16F with padded rows and frames (the repack path), and host buffers in all formats."""
    sc = pfs.SCENES[name]
    w, h, n = sc.width, sc.height, sc.n
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    want32 = _oracle_frames(oracle_api, name, "f32")
    for fmt in ("f16", "f32"):
        stride = BPP[fmt] * w + 16
        frames, _ = _poses_device(r, comp, sc, fmt, stride, h * stride + 32)
        _check(frames, want32, fmt, name)
        host = np.zeros((n, h, w, 4), DTYPES[fmt])
        r.render_poses_linear(comp, pfs.poses(sc), host, w, h, RGBA, CLEAR, format=fmt)
        _check(host, want32, fmt, name)
    for s, vst in ((4 * w, 4 * w * h), (4 * w + 12, h * (4 * w + 12) + 20)):
        host = np.full((n - 1) * vst + h * s + 64, SENTINEL, np.uint8)
        r.render_poses(comp, pfs.poses(sc), host, w, h, RGBA, CLEAR, stride=s, view_stride=vst)
        _check(_unpack(host, n, w, h, s, vst, 4).reshape(n, h, w, 4), _oracle_frames(oracle_api, name), "srgb8", name)
        assert _outside_untouched(host, n, w, h, s, vst, 4)


@pytest.mark.parametrize("fmt", ["srgb8", "f16", "f32"])
@pytest.mark.parametrize("name", ["e2e_linear_gradient", "e2e_blend_modes__Saturation", "blend_top_Color", "clip_ignored", "alpha_flips",
                                  "alpha_edges", "nonfinite_colors", "clip2_both_filled", "fill_window_top"])
def test_over_frames(cuda_api, oracle_api, name, fmt):
    """Over a different background per frame, in place and through padded strides."""
    sc = pfs.SCENES[name]
    bgs = backgrounds(sc, fmt, seed=len(name))
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    want = _oracle_frames(oracle_api, name, "over", bgs=bgs)
    twin = _twin_frames(cuda_api, name, fmt, bgs=bgs)
    bpp = BPP[fmt]
    for stride, vst in ((None, None), (bpp * sc.width + 16, sc.height * (bpp * sc.width + 16) + 48)):
        frames = _poses_over(r, comp, sc, bgs, fmt, stride, vst)
        _check(frames, want, fmt, f"{name} over")
        _check(frames, twin, fmt, f"{name} over, single frames")


@pytest.mark.parametrize("name", pfs.HEAVY)
def test_workload_fills(cuda_api, oracle_api, name):
    """The 200 spaceship frames (chunks), the 511 library frames and paris with all 50 620 layers
    recoloured: every sRGB8 frame against render_device, a spread against the oracle; RGBA32F of the
    library and paris against the single-frame call."""
    sc = pfs.SCENES[name]
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    frames, _ = _poses_device(r, comp, sc)
    _check(frames, _twin_frames(cuda_api, name), "srgb8", name)
    spread = sorted({0, 1, sc.n // 2, sc.n - 1} | set(range(0, sc.n, max(sc.n // 8, 1))))
    _check(frames, _oracle_frames(oracle_api, name, "srgb8", spread), "srgb8", name)
    if name != "spaceship_filled":
        frames, _ = _poses_device(r, comp, sc, "f32")
        _check(frames, _twin_frames(cuda_api, name, "f32", spread), "f32", name)


@pytest.mark.parametrize("name", ["alpha_flips", "alpha_edges", "nonfinite_colors", "clip_ignored", "e2e_clipping", "blend_top_Luminosity",
                                  "window_gaps_filled", "library_filled"])
def test_ids_masks_stats_equal_single_frames(cuda_api, name):
    """IDs at two thresholds, F32 and U8 masks and statistics of every frame equal the single-frame
    calls after the same edits (an alpha flip moves the first layer the walks start from); the
    RGBA stack of each pass equals render_poses_device."""
    import torch
    sc = pfs.SCENES[name]
    w, h, n = sc.width, sc.height, sc.n
    comp, orders = sc.build(cuda_api)
    ref, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    p = pfs.poses(sc)
    rgba_want, _ = _poses_device(r, comp, sc)
    first, K = max(orders[0] - 1, 0), min(orders[-1] + 2 - max(orders[0] - 1, 0), 66)
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
        pfs.set_pose_fill(ref, sc, orders, b)
        for mc in ids:
            r1.render_ids_device(ref, one_ids.data_ptr(), w, h, min_coverage=mc)
            torch.cuda.synchronize()
            assert np.array_equal(got[mc][b], one_ids.cpu().numpy()), f"{name}: frame {b} IDs at {mc}"
        assert np.array_equal(host_ids[b], got[0.5][b].view(np.uint32)), f"{name}: frame {b} host IDs"
        for fmt, t in one_m.items():
            r1.render_masks_device(ref, t.data_ptr(), w, h, first, K, format=fmt)
            torch.cuda.synchronize()
            assert np.array_equal(got_m[fmt][b], t.cpu().numpy()), f"{name}: frame {b} {fmt} masks"
        r1.render_stats_device(ref, one_s.data_ptr(), w, h, first, K, min_coverage=0.25)
        torch.cuda.synchronize()
        assert np.array_equal(got_s[b], one_s.cpu().numpy()), f"{name}: frame {b} statistics"


@pytest.mark.parametrize("name", ["alpha_flips", "e2e_texture", "window_gaps_filled", "library_filled"])
def test_call_leaves_the_composition(cuda_api, name):
    """The frame rendered afterwards is the one before, and the ordinary render right after the call
    uploads nothing: the props, the tables version and the unchanged bits are as they were."""
    import torch
    sc = pfs.SCENES[name]
    w, h = sc.width, sc.height
    comp, orders = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    t = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda:0")
    h2d = lambda: r.counters()["h2d_bytes"]  # noqa: E731
    for _ in range(2):
        r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR)
    b0 = h2d()
    r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR)
    torch.cuda.synchronize()
    idle, before = h2d() - b0, t.cpu().numpy()
    b1 = h2d()
    _poses_device(r, comp, sc)
    assert h2d() - b1 >= sc.n * sc.n_orders * 16, "the colours were not uploaded"
    t.zero_()
    b2 = h2d()
    r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR)
    torch.cuda.synchronize()
    assert h2d() - b2 <= idle, "the render after a pose-fill call uploaded"
    assert np.array_equal(t.cpu().numpy(), before)
    written = []
    for with_call in (False, True):  # a cached sequence gives the same written tiles with the call in it
        comp, _ = sc.build(cuda_api)
        r = cuda_api.Renderer(0)
        cache = r.create_buffer_layer_cache()
        buf = np.zeros(w * h * 4, np.uint8)
        r.render(comp, buf, w, h, RGBA, CLEAR, layer_cache=cache)
        if with_call:
            _poses_device(r, comp, sc)
        r.render(comp, buf, w, h, RGBA, CLEAR, layer_cache=cache)
        written.append((r.counters()["written_tiles"], buf.copy()))
    assert written[0][0] == written[1][0] and np.array_equal(written[0][1], written[1][1])


@pytest.mark.parametrize("opts", [{"sync_free": 0}, {"sync_free": 1}, {"sync_free": 1, "test_fast_shrink": 1}, {"speculate": 0},
                                  {"speculate": 1}, {"paint_solid": 0}, {"paint_solid": 1}, {"paint_lpt": 0}])
def test_switches(cuda_api, oracle_api, opts):
    """Every schedule gives the oracle's bytes, with single frames and pose calls without colours between."""
    saved = {k: cuda_api.get_option(k) for k in opts}
    try:
        for k, v in opts.items():
            cuda_api.set_option(k, v)
        r = cuda_api.Renderer(0)
        for name in ("alpha_flips", "e2e_texture", "fill_window_gaps", "clip_ignored", "alpha_flips", "library_filled"):
            sc = pfs.SCENES[name]
            comp, _ = sc.build(cuda_api)
            buf = np.zeros(sc.width * sc.height * 4, np.uint8)
            r.render(comp, buf, sc.width, sc.height, RGBA, CLEAR)
            frames, _ = _poses_device(r, comp, sc)
            _check(frames, _oracle_frames(oracle_api, name), "srgb8", name)
            frames, _ = _poses_device(r, comp, sc, "f32")
            _check(frames, _oracle_frames(oracle_api, name, "f32"), "f32", name)
            if sc.transforms is not None:  # the same call without colours renders the poses alone
                _poses_device(r, comp, sc, poses=Poses(sc.first_order, sc.transforms, sc.visible))
    finally:
        for k, v in saved.items():
            cuda_api.set_option(k, v)


def test_refusals_write_nothing(cuda_api):
    """No table at all (FORMA_ERR_INVALID_ARGUMENT), and more pose fills than the 2^31 style slots
    hold (FORMA_ERR_CAPACITY, refused before the colours are read: the table passed is far smaller
    than n K 4 floats), in every RGBA pose call: nothing is written."""
    import torch
    sc = pfs.SCENES["alpha_flips"]
    w = sc.width
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    ch = (C.c_uint32 * 4)(*RGBA)
    cc = (C.c_float * 4)(CLEAR.r, CLEAR.g, CLEAR.b, CLEAR.a)
    colors = np.ones((4, 9, 4), np.float32)
    n_big = r.max_views(16)
    assert n_big * (1 << 21) >= 1 << 31
    cases = [("no tables", binding._CPoses(0, 9, None, None, None), 2, sc.height, FORMA_ERR_INVALID_ARGUMENT),
             ("style slots", binding._CPoses(0, 1 << 21, None, None, colors.ctypes.data), n_big, 16, FORMA_ERR_CAPACITY)]
    api, vp = cuda_api, C.c_void_p
    for what, d, n, h, want in cases:
        dev = torch.full((n * h * 16 * w,), SENTINEL, dtype=torch.uint8, device="cuda:0")
        host = np.full(n * h * 16 * w, SENTINEL, np.uint8)
        s4, s16 = 4 * w, 16 * w
        calls = [
            ("device", lambda: api.renderer_render_poses_device(r._h, comp._h, C.byref(d), n, vp(dev.data_ptr()), w, s4, h, h * s4,
                                                                ch, cc, None)),
            ("host", lambda: api.renderer_render_poses(r._h, comp._h, C.byref(d), n, vp(host.ctypes.data), w, s4, h, h * s4, ch, cc,
                                                       None)),
            ("linear device", lambda: api.renderer_render_poses_linear_device(r._h, comp._h, C.byref(d), n, vp(dev.data_ptr()), w, s16, h,
                                                                              h * s16, ch, cc, 2, None)),
            ("linear host", lambda: api.renderer_render_poses_linear(r._h, comp._h, C.byref(d), n, vp(host.ctypes.data), w, s16, h,
                                                                     h * s16, ch, cc, 2, None)),
            ("over device", lambda: api.renderer_render_poses_over_device(r._h, comp._h, C.byref(d), n, vp(dev.data_ptr()), w, s4, h,
                                                                          h * s4, ch, 0, None)),
        ]
        for call_name, call in calls:
            st = call()
            assert st == want, (what, call_name, st, api.last_error())
            if want == FORMA_ERR_CAPACITY:
                assert "2^31" in api.last_error().decode(), (what, call_name)
        torch.cuda.synchronize()
        assert bool(torch.all(dev == SENTINEL)) and np.all(host == SENTINEL), what
    with pytest.raises(ValueError):
        Poses(0)
    # After the refusals the renderer still renders.
    frames, _ = _poses_device(r, comp, sc)
    _check(frames, _twin_frames(cuda_api, "alpha_flips"), "srgb8", "after the refusals")


def test_tensor_defaults_and_chunks(cuda_api, oracle_api, monkeypatch):
    """[N, H, W, 4] CUDA tensors with the default strides, chunked by the binding, in the float and
    over calls: every chunk takes its own frames' colours."""
    import torch
    name = "window_gaps_filled"
    sc = pfs.SCENES[name]
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    monkeypatch.setattr(r, "max_views", lambda height: 2)
    t = torch.zeros((sc.n, sc.height, sc.width, 4), dtype=torch.float32, device="cuda:0")
    r.render_poses_linear_device(comp, pfs.poses(sc), t.data_ptr(), sc.width, sc.height, RGBA, CLEAR)
    torch.cuda.synchronize()
    _check(t.cpu().numpy(), _oracle_frames(oracle_api, name, "f32"), "f32", name)
    bgs = backgrounds(sc, "srgb8", 3)
    t = torch.from_numpy(bgs.copy()).to("cuda:0")
    r.render_poses_over_device(comp, pfs.poses(sc), t.data_ptr(), sc.width, sc.height)
    torch.cuda.synchronize()
    _check(t.cpu().numpy(), _oracle_frames(oracle_api, name, "over", bgs=bgs), "srgb8", name)
