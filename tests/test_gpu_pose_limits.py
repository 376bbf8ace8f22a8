"""Poses at their limits on the device (tests/pose_limit_scenes.py, each scene proven on the CPU by
tests/test_pose_limit_scenes.py first), at tolerance 0.

Frame b of every call equals the oracle's frame of the composition put into pose b, and
render_device's (but for the frames whose lines all lie more than 2^19 px left of the frame, where
the header says render_device differs); its sorted segments are the single frame's moved by
b rows; bytes outside the frames keep a sentinel. Device tables give the bytes of host tables,
chunked at max_views with odd K; IDs, masks and statistics equal the single-frame calls; pose
fills equal the oracle in sRGB8 and RGBA32F bit for bit; the full stacks hold under the schedule
switches. The segment-limit scenes are refused with FORMA_ERR_CAPACITY by every pose call, with
every byte and the composition untouched, and the next call on the same renderer is right.
"""
import numpy as np
import pytest

import oracle_linear
import pose_fill_scenes as pfs
import pose_limit_scenes as pls
from forma_b200 import binding
from forma_b200.binding import RGBA, Color, FormaError

pytestmark = pytest.mark.gpu

CLEAR = Color(1.0, 1.0, 1.0, 0.0)
SENTINEL = 0xA5
DEV = "cuda:0"
_ORACLE = {}


@pytest.fixture(autouse=True)
def _oracle_modes(oracle_api):
    oracle_linear.attach(oracle_api)
    oracle_api.hooks.fo_set_recip_mode(0)


def _spread(n):
    """Every frame of a short call; the ends, the middle and every eighth of a long one."""
    return list(range(n)) if n <= 40 else sorted({0, 1, n // 2, n - 2, n - 1} | set(range(0, n, n // 8)))


def _oracle_frames(oracle_api, name, frames, kind="srgb8"):
    sc = pls.SCENES[name]
    cache = _ORACLE.setdefault((name, kind), {})
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
            else:
                cache[b] = oracle_linear.render(oracle_api, comp, sc.width, sc.height, RGBA, CLEAR)
    return {b: cache[b] for b in frames}


def _single_frames(cuda_api, sc, frames, fmt="srgb8"):
    """{b: render_device (or render_linear_device) of a second composition put into pose b}."""
    import torch
    comp, orders = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    out = {}
    for b in frames:
        pfs.set_pose_fill(comp, sc, orders, b)
        if fmt == "srgb8":
            t = torch.zeros((sc.height, sc.width, 4), dtype=torch.uint8, device=DEV)
            r.render_device(comp, t.data_ptr(), sc.width, sc.height, RGBA, CLEAR)
        else:
            t = torch.zeros((sc.height, sc.width, 4), dtype=torch.float32, device=DEV)
            r.render_linear_device(comp, t.data_ptr(), sc.width, sc.height, RGBA, CLEAR, format=fmt)
        torch.cuda.synchronize()
        out[b] = t.cpu().numpy()
    return out


def _poses(sc, device=False):
    """The scene's Poses, with numpy tables or with torch CUDA tables."""
    import torch
    tables = [sc.transforms, sc.visible, sc.colors]
    if device:
        tables = [None if t is None else torch.from_numpy(np.ascontiguousarray(t)).to(DEV) for t in tables]
    return binding.Poses(sc.first_order, *tables)


def _unpack(raw, n, w, h, stride, view_stride, bpp=4):
    frames = np.empty((n, h, w * bpp), np.uint8)
    for b in range(n):
        for y in range(h):
            o = b * view_stride + y * stride
            frames[b, y] = raw[o:o + bpp * w]
    return frames


def _outside_untouched(raw, n, w, h, stride, view_stride, bpp=4):
    mask = np.ones(raw.size, bool)
    for b in range(n):
        for y in range(h):
            o = b * view_stride + y * stride
            mask[o:o + bpp * w] = False
    return bool(np.all(raw[mask] == SENTINEL))


def _strides(sc, padded, bpp=4):
    stride = bpp * sc.width + (12 if padded else 0)
    return stride, sc.height * stride + (20 if padded else 0)


def _poses_device(r, comp, sc, padded=False, poses=None, fmt="srgb8"):
    """(frames [n, h, w, 4] of the format, raw bytes) of render_poses{,_linear}_device into a
    sentinel-filled buffer."""
    import torch
    bpp = 4 if fmt == "srgb8" else 16
    stride, view_stride = _strides(sc, padded, bpp)
    n, w, h = sc.n, sc.width, sc.height
    t = torch.full(((n - 1) * view_stride + h * stride + 64,), SENTINEL, dtype=torch.uint8, device=DEV)
    p = _poses(sc) if poses is None else poses
    if fmt == "srgb8":
        r.render_poses_device(comp, p, t.data_ptr(), w, h, RGBA, CLEAR, stride=stride, view_stride=view_stride)
    else:
        r.render_poses_linear_device(comp, p, t.data_ptr(), w, h, RGBA, CLEAR, format=fmt, stride=stride, view_stride=view_stride)
    torch.cuda.synchronize()
    raw = t.cpu().numpy()
    assert _outside_untouched(raw, n, w, h, stride, view_stride, bpp), sc.name
    frames = _unpack(raw, n, w, h, stride, view_stride, bpp).view(np.uint8 if fmt == "srgb8" else np.float32).reshape(n, h, w, 4)
    return frames, raw


def _same(got, want, what):
    if got.dtype == np.float32:
        bad = (got.view(np.uint32) != want.view(np.uint32)) & ~(np.isnan(got) & np.isnan(want))
    else:
        bad = got != want
    assert not bad.any(), f"{what}: {int(bad.sum())} values differ, first at {tuple(int(i[0]) for i in np.nonzero(bad))}"


# Frames painted in place (height a multiple of 16, dense frames) and repacked (padded strides).
PADDED = set(pls.ODD) | {"far_left", "far_up", "window_from_1", "window_odd_k", "lines_edges", "crowded_nan_blends"}


@pytest.mark.parametrize("name", pls.IN_LIMIT)
def test_frames_match_oracle_and_render_device(cuda_api, oracle_api, name):
    sc = pls.SCENES[name]
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    frames, _ = _poses_device(r, comp, sc, padded=name in PADDED)
    for b, f in _oracle_frames(oracle_api, name, range(sc.n)).items():
        _same(frames[b], f, f"{name}: frame {b} against the oracle")
    near = [b for b in _spread(sc.n) if b not in sc.far]
    for b, f in _single_frames(cuda_api, sc, near).items():
        _same(frames[b], f, f"{name}: frame {b} against render_device")


@pytest.mark.parametrize("name", ["limit_h17", "limit_h1", "odd_h37", "far_up", "far_left", "far_translations", "window_from_1",
                                  "out_of_order", "lines_translations_own", "lines_rotations", "crowded_crowd_129"])
def test_segments_are_the_single_frames_moved(cuda_api, unsliced, name):
    import torch
    sc = pls.SCENES[name]
    w, h, rows = sc.width, sc.height, sc.rows
    comp, _ = sc.build(cuda_api)
    ref, orders = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    _poses_device(r, comp, sc)
    segs = np.sort(r.segments())
    ty = (segs >> np.uint64(53)).astype(np.int64)
    assert int(ty.max(initial=0)) <= sc.n * rows
    frames, total = _spread(sc.n), 0
    r1 = cuda_api.Renderer(0)
    t = torch.zeros(w * h * 4, dtype=torch.uint8, device=DEV)
    for b in frames:
        pfs.set_pose_fill(ref, sc, orders, b)
        r1.render_device(ref, t.data_ptr(), w, h, RGBA, CLEAR)
        torch.cuda.synchronize()
        one = np.sort(r1.segments())
        total += one.size
        one_ty = (one >> np.uint64(53)).astype(np.int64)
        want = one[(one_ty >= 1) & (one_ty <= rows)]
        got = segs[(ty >= b * rows + 1) & (ty <= (b + 1) * rows)] - np.uint64(b * rows) * np.uint64(1 << 53)
        assert np.array_equal(np.sort(got), np.sort(want)), f"{name}: frame {b} segments differ"
    if len(frames) == sc.n:
        assert segs.size == total, name  # rows outside a frame are dropped to stacked row 0, not lost


@pytest.mark.parametrize("name", ["window_odd_k", "window_k2p16", "window_2p21", "limit_h17", "far_translations", "crowded_crowd_1000"])
def test_device_tables_equal_host_tables(cuda_api, name):
    """The same bytes from torch CUDA tables as from numpy tables, chunked by the binding at
    max_views(height): with odd K a chunk's visibility bytes start at an odd address."""
    sc = pls.SCENES[name]
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    _, host = _poses_device(r, comp, sc)
    _, dev = _poses_device(r, comp, sc, poses=_poses(sc, device=True))
    assert np.array_equal(host, dev), name
    if name == "window_odd_k":
        assert sc.n > r.max_views(sc.height) and sc.n_orders % 2 == 1


@pytest.mark.parametrize("name", ["limit_h1000", "odd_h37", "window_from_1", "far_up", "out_of_order", "crowded_crowd_129",
                                  "crowded_nan_blends"])
def test_ids_masks_stats_equal_single_frames(cuda_api, name):
    """IDs, F32 masks and statistics of every pose equal the single-frame calls on the composition
    put into that pose; the RGBA frames of each pass equal render_poses_device's."""
    import torch
    sc = pls.SCENES[name]
    w, h, n = sc.width, sc.height, sc.n
    comp, orders = sc.build(cuda_api)
    ref, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    p = _poses(sc)
    rgba_want, _ = _poses_device(r, comp, sc)
    first, K = 0, min(orders[-1] + 1, 66)
    rgba = torch.zeros((n, h, w, 4), dtype=torch.uint8, device=DEV)
    ids = torch.zeros((n, h, w), dtype=torch.int32, device=DEV)
    r.render_poses_ids_device(comp, p, ids.data_ptr(), w, h, rgba_ptr=rgba.data_ptr(), channels=RGBA, clear_color=CLEAR,
                              min_coverage=0.5)
    torch.cuda.synchronize()
    assert np.array_equal(rgba.cpu().numpy(), rgba_want), f"{name}: RGBA with IDs"
    masks = torch.zeros((n, K, h, w), dtype=torch.float32, device=DEV)
    r.render_poses_masks_device(comp, p, masks.data_ptr(), w, h, first, K, format="f32")
    stats = torch.zeros((n, K, 12), dtype=torch.int32, device=DEV)
    r.render_poses_stats_device(comp, p, stats.data_ptr(), w, h, first, K, min_coverage=0.25)
    torch.cuda.synchronize()
    got_i, got_m, got_s = ids.cpu().numpy(), masks.cpu().numpy(), stats.cpu().numpy()
    r1 = cuda_api.Renderer(0)
    one_i = torch.zeros((h, w), dtype=torch.int32, device=DEV)
    one_m = torch.zeros((K, h, w), dtype=torch.float32, device=DEV)
    one_s = torch.zeros((K, 12), dtype=torch.int32, device=DEV)
    for b in _spread(n):
        pfs.set_pose_fill(ref, sc, orders, b)
        r1.render_ids_device(ref, one_i.data_ptr(), w, h, min_coverage=0.5)
        r1.render_masks_device(ref, one_m.data_ptr(), w, h, first, K, format="f32")
        r1.render_stats_device(ref, one_s.data_ptr(), w, h, first, K, min_coverage=0.25)
        torch.cuda.synchronize()
        assert np.array_equal(got_i[b], one_i.cpu().numpy()), f"{name}: frame {b} IDs"
        _same(got_m[b], one_m.cpu().numpy(), f"{name}: frame {b} masks")
        assert np.array_equal(got_s[b], one_s.cpu().numpy()), f"{name}: frame {b} statistics"


@pytest.mark.parametrize("name", [n for n in pls.IN_LIMIT if n.startswith("crowded_")] + ["window_k2p16"])
def test_pose_fills_bit_for_bit(cuda_api, oracle_api, name):
    """RGBA32F frames against the oracle's linear frames after set_pose_fill, bit for bit, and
    against render_linear_device (sRGB8 is the first test's)."""
    sc = pls.SCENES[name]
    assert sc.colors is not None
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    frames, _ = _poses_device(r, comp, sc, padded=True, fmt="f32")
    frames_at = _spread(sc.n)
    for b, f in _oracle_frames(oracle_api, name, frames_at, kind="f32").items():
        _same(frames[b], np.asarray(f, np.float32), f"{name}: frame {b} RGBA32F against the oracle")
    for b, f in _single_frames(cuda_api, sc, frames_at, fmt="f32").items():
        _same(frames[b], f, f"{name}: frame {b} RGBA32F against render_linear_device")


SWITCHES = [{"sync_free": 0}, {"sync_free": 1}, {"sync_free": 1, "test_fast_shrink": 1}, {"sort_full_key": 0}, {"sort_full_key": 1},
            {"sort_counts": 0}, {"sort_counts": 1}, {"paint_solid": 0}, {"paint_solid": 1}, {"pdl": 0}, {"pdl": 1}]


@pytest.mark.parametrize("opts", SWITCHES, ids=lambda o: ",".join(f"{k}={v}" for k, v in o.items()))
def test_full_stacks_under_switches(cuda_api, oracle_api, opts):
    saved = {k: cuda_api.get_option(k) for k in opts}
    try:
        for k, v in opts.items():
            cuda_api.set_option(k, v)
        r = cuda_api.Renderer(0)
        for name in ("limit_h17", "odd_h37", "limit_h16", "limit_h1000", "limit_h17"):  # a smaller call between the full ones
            sc = pls.SCENES[name]
            comp, _ = sc.build(cuda_api)
            frames, _ = _poses_device(r, comp, sc)
            for b, f in _oracle_frames(oracle_api, name, range(sc.n)).items():
                _same(frames[b], f, f"{name} {opts}: frame {b}")
    finally:
        for k, v in saved.items():
            cuda_api.set_option(k, v)


def _state(comp, orders):
    return [(o, comp.get(o).is_enabled()) for o in orders]


@pytest.mark.parametrize("name", pls.OVER_LIMIT)
def test_segment_limit_refused_by_every_pose_call(cuda_api, oracle_api, name):
    """FORMA_ERR_CAPACITY from every pose call, every byte of every buffer still the sentinel, every
    layer's state unchanged, `segments` 0; then the next call on the renderer is right. (The
    composition's own frame is not rendered: it has 0.6 * 2^30 segments.)"""
    import torch
    sc = pls.SCENES[name]
    w, h, n = sc.width, sc.height, sc.n
    comp, orders = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    state = _state(comp, orders)
    colors = pfs.random_colors(n, sc.n_orders, 5)
    p, p_fill = _poses(sc), binding.Poses(sc.first_order, sc.transforms, sc.visible, colors)
    dev = torch.full((n * w * h * 16 + 64,), SENTINEL, dtype=torch.uint8, device=DEV)
    aux = torch.full((n * w * h * 16 + 64,), SENTINEL, dtype=torch.uint8, device=DEV)
    host = np.full(n * w * h * 4 + 64, SENTINEL, np.uint8)
    host_ids = np.full((n, h, w), 0xA5A5A5A5, np.uint32)
    calls = {
        "rgba": lambda: r.render_poses_device(comp, p, dev.data_ptr(), w, h, RGBA, CLEAR),
        "host": lambda: r.render_poses(comp, p, host, w, h, RGBA, CLEAR),
        "ids": lambda: r.render_poses_ids_device(comp, p, aux.data_ptr(), w, h, rgba_ptr=dev.data_ptr(), channels=RGBA,
                                                 clear_color=CLEAR),
        "host ids": lambda: r.render_poses_ids(comp, p, host_ids, w, h),
        "masks": lambda: r.render_poses_masks_device(comp, p, aux.data_ptr(), w, h, 0, sc.n_orders, format="f32",
                                                     rgba_ptr=dev.data_ptr(), clear_color=CLEAR),
        "stats": lambda: r.render_poses_stats_device(comp, p, aux.data_ptr(), w, h, 0, sc.n_orders, rgba_ptr=dev.data_ptr(),
                                                     clear_color=CLEAR),
        "fills": lambda: r.render_poses_device(comp, p_fill, dev.data_ptr(), w, h, RGBA, CLEAR),
        "linear": lambda: r.render_poses_linear_device(comp, p_fill, dev.data_ptr(), w, h, RGBA, CLEAR, format="f32"),
        "over": lambda: r.render_poses_over_device(comp, p, dev.data_ptr(), w, h, RGBA, format="srgb8"),
    }
    for what, call in calls.items():
        with pytest.raises(FormaError, match="status 5 "):
            call()
        torch.cuda.synchronize()
        assert bool(torch.all(dev == SENTINEL)) and bool(torch.all(aux == SENTINEL)), (name, what)
        assert np.all(host == SENTINEL) and np.all(host_ids == 0xA5A5A5A5), (name, what)
        assert r.counters()["segments"] == 0, (name, what)
        assert _state(comp, orders) == state, (name, what)
    ok = pls.SCENES["odd_h37"]
    comp2, _ = ok.build(cuda_api)
    frames, _ = _poses_device(r, comp2, ok)
    for b, f in _oracle_frames(oracle_api, "odd_h37", range(ok.n)).items():
        _same(frames[b], f, f"after {name}: frame {b}")
