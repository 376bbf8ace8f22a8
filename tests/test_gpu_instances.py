"""Instance scenes (Renderer.render_instances_device and its ID, mask and statistics twins) on the
device, at tolerance 0.

Frame b of a call equals the oracle's frame of T_b (tests/instance_scenes.py: twin) and
render_device of T_b. The call's sorted segments are the twins' painted-row segments moved to
frame b's rows and layer slice; IDs, masks and statistics equal the single-frame calls on T_b;
CUDA tables in every host / device mix give the bytes of host tables; the library is unchanged
afterwards; every refusal writes nothing; the layer-field and frame-count limits hold at their
edges; and the sync-free redo gives the same frames.
"""
import ctypes as C

import numpy as np
import pytest

import instance_scenes as ins
from forma_b200 import binding
from forma_b200.binding import RGBA, Color, FormaError, Instances, OrderError

pytestmark = pytest.mark.gpu

CLEAR = Color(1.0, 1.0, 1.0, 0.0)
SENTINEL = 0xA5
INVALID, ORDER, CAPACITY = 1, 2, 5
_ORACLE = {}


def _oracle_frames(oracle_api, name):
    """[the oracle's frame (H, W, 4) of T_b for every b]."""
    if name not in _ORACLE:
        sc = ins.SCENES[name]
        r = oracle_api.Renderer(0)
        out = []
        for b in range(sc.n):
            buf = np.zeros(sc.width * sc.height * 4, np.uint8)
            r.render(ins.twin(oracle_api, sc, b), buf, sc.width, sc.height, RGBA, CLEAR)
            out.append(buf.reshape(sc.height, sc.width, 4))
        _ORACLE[name] = np.stack(out)
    return _ORACLE[name]


def _instances_device(r, comp, sc, inst=None):
    """The frames (N, H, W, 4) of render_instances_device into a sentinel-filled tensor."""
    import torch
    t = torch.full((sc.n, sc.height, sc.width, 4), SENTINEL, dtype=torch.uint8, device="cuda:0")
    r.render_instances_device(comp, inst or ins.instances(binding, sc), t.data_ptr(), sc.width, sc.height, RGBA, CLEAR)
    torch.cuda.synchronize()
    return t.cpu().numpy()


@pytest.mark.parametrize("name", list(ins.SCENES))
def test_frames_match_oracle_and_render_device(cuda_api, oracle_api, name):
    import torch
    sc = ins.SCENES[name]
    comp = ins.build_library(cuda_api, sc)
    r = cuda_api.Renderer(0)
    got = _instances_device(r, comp, sc)
    want = _oracle_frames(oracle_api, name)
    bad = [b for b in range(sc.n) if not np.array_equal(got[b], want[b])]
    assert not bad, f"{name}: frames {bad[:8]} differ from the oracle"
    r1 = cuda_api.Renderer(0)
    t = torch.zeros((sc.height, sc.width, 4), dtype=torch.uint8, device="cuda:0")
    for b in range(sc.n):
        r1.render_device(ins.twin(cuda_api, sc, b), t.data_ptr(), sc.width, sc.height, RGBA, CLEAR)
        torch.cuda.synchronize()
        assert np.array_equal(got[b], t.cpu().numpy()), f"{name}: frame {b} differs from render_device of its twin"


@pytest.mark.parametrize("name", ins.LIGHT + ["library_511x64"])
def test_segments_are_the_twins_moved(cuda_api, unsliced, name):
    import torch
    sc = ins.SCENES[name]
    w, h, rows, M = sc.width, sc.height, (sc.height + 15) // 16, sc.m
    comp = ins.build_library(cuda_api, sc)
    r = cuda_api.Renderer(0)
    _instances_device(r, comp, sc)
    segs = np.sort(r.segments())
    ty = (segs >> np.uint64(53)).astype(np.int64)
    r1 = cuda_api.Renderer(0)
    t = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda:0")
    for b in range(sc.n):
        r1.render_device(ins.twin(cuda_api, sc, b), t.data_ptr(), w, h, RGBA, CLEAR)
        torch.cuda.synchronize()
        one = np.sort(r1.segments())
        one_ty = (one >> np.uint64(53)).astype(np.int64)
        want = one[(one_ty >= 1) & (one_ty <= rows)]
        got = segs[(ty >= b * rows + 1) & (ty <= (b + 1) * rows)]
        got = got - np.uint64(b * rows) * np.uint64(1 << 53) - np.uint64(b * M) * np.uint64(1 << 20)
        assert np.array_equal(np.sort(got), np.sort(want)), f"{name}: frame {b} segments differ"


@pytest.mark.parametrize("name", ["repeats", "inserts", "styles", "colors_blend", "clip_leak", "nonfinite", "library_511x64"])
def test_ids_masks_stats_equal_single_frames(cuda_api, name):
    """IDs at two thresholds, F32 and U8 masks and statistics of the slots equal the single-frame
    calls on each twin; the RGBA stack of each pass equals render_instances_device."""
    import torch
    sc = ins.SCENES[name]
    w, h, n, K = sc.width, sc.height, sc.n, sc.m + 1
    comp = ins.build_library(cuda_api, sc)
    r = cuda_api.Renderer(0)
    inst = ins.instances(binding, sc)
    rgba_want = _instances_device(r, comp, sc)
    dev = "cuda:0"
    rgba = torch.zeros((n, h, w, 4), dtype=torch.uint8, device=dev)
    ids = {mc: torch.zeros((n, h, w), dtype=torch.int32, device=dev) for mc in (0.0, 0.5)}
    for mc, t in ids.items():
        rgba.zero_()
        r.render_instances_ids_device(comp, inst, t.data_ptr(), w, h, rgba_ptr=rgba.data_ptr(), clear_color=CLEAR, min_coverage=mc)
        torch.cuda.synchronize()
        assert np.array_equal(rgba.cpu().numpy(), rgba_want), f"{name}: RGBA with IDs"
    only_ids = torch.zeros((n, h, w), dtype=torch.int32, device=dev)
    r.render_instances_ids_device(comp, inst, only_ids.data_ptr(), w, h, min_coverage=0.5)
    torch.cuda.synchronize()
    assert torch.equal(only_ids, ids[0.5]), f"{name}: IDs alone"
    masks = {}
    for fmt, dt in (("f32", torch.float32), ("u8", torch.uint8)):
        masks[fmt] = torch.zeros((n, K, h, w), dtype=dt, device=dev)
        rgba.zero_()
        r.render_instances_masks_device(comp, inst, masks[fmt].data_ptr(), w, h, 0, K, format=fmt, rgba_ptr=rgba.data_ptr(),
                                        clear_color=CLEAR)
        torch.cuda.synchronize()
        assert np.array_equal(rgba.cpu().numpy(), rgba_want), f"{name}: RGBA with masks"
    stats = torch.zeros((n, K, 12), dtype=torch.int32, device=dev)
    rgba.zero_()
    r.render_instances_stats_device(comp, inst, stats.data_ptr(), w, h, 0, K, min_coverage=0.25, rgba_ptr=rgba.data_ptr(),
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
        ref = ins.twin(cuda_api, sc, b)
        for mc in ids:
            r1.render_ids_device(ref, one_ids.data_ptr(), w, h, min_coverage=mc)
            torch.cuda.synchronize()
            assert np.array_equal(got[mc][b], one_ids.cpu().numpy()), f"{name}: frame {b} IDs at {mc}"
        for fmt, t in one_m.items():
            r1.render_masks_device(ref, t.data_ptr(), w, h, 0, K, format=fmt)
            torch.cuda.synchronize()
            assert np.array_equal(got_m[fmt][b], t.cpu().numpy()), f"{name}: frame {b} {fmt} masks"
        r1.render_stats_device(ref, one_s.data_ptr(), w, h, 0, K, min_coverage=0.25)
        torch.cuda.synchronize()
        assert np.array_equal(got_s[b], one_s.cpu().numpy()), f"{name}: frame {b} statistics"


@pytest.mark.parametrize("name", ["colors_blend", "library_511x64"])
def test_cuda_tables_in_every_mix(cuda_api, name):
    """Each of the three tables in host or device memory (int32 prototypes with -1 for empty slots
    on the device): the bytes of the all-host call."""
    import itertools

    import torch
    sc = ins.SCENES[name]
    comp = ins.build_library(cuda_api, sc)
    r = cuda_api.Renderer(0)
    want = _instances_device(r, comp, sc)
    dev = {"p": torch.from_numpy(sc.prototypes.view(np.int32).copy()).cuda(), "t": torch.from_numpy(sc.transforms).cuda(),
           "c": torch.from_numpy(sc.colors).cuda()}
    for mix in itertools.product((False, True), repeat=3):
        if not any(mix):
            continue
        p, t, c = (dev[k] if on else host for k, on, host in zip("ptc", mix, (sc.prototypes, sc.transforms, sc.colors)))
        got = _instances_device(r, comp, sc, Instances(p, t, c))
        assert np.array_equal(got, want), f"{name}: device tables {mix}"


def _state(comp, sc):
    return [(p.order, comp.get(p.order).is_enabled()) for p in sc.protos]


@pytest.mark.parametrize("name", ["repeats", "inserts", "library_511x64"])
def test_call_leaves_the_library(cuda_api, name):
    """Enabled states read back unchanged, the library's own frame is the one before, and the
    ordinary render right after the call uploads nothing."""
    import torch
    sc = ins.SCENES[name]
    w, h = sc.width, sc.height
    comp = ins.build_library(cuda_api, sc)
    r = cuda_api.Renderer(0)
    t = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda:0")
    h2d = lambda: r.counters()["h2d_bytes"]  # noqa: E731
    for _ in range(2):
        r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR)
    b0 = h2d()
    r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR)
    torch.cuda.synchronize()
    idle, before, state = h2d() - b0, t.cpu().numpy(), _state(comp, sc)
    _instances_device(r, comp, sc)
    assert _state(comp, sc) == state
    t.zero_()
    b1 = h2d()
    r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR)
    torch.cuda.synchronize()
    assert h2d() - b1 <= idle, "the render after an instance call uploaded"
    assert np.array_equal(t.cpu().numpy(), before)


@pytest.mark.parametrize("opts", [{"sync_free": 1, "test_fast_shrink": 1}, {"sync_free": 0}, {"sort_full_key": 1}, {"sort_counts": 0},
                                  {"speculate": 0}, {"paint_solid": 0}])
def test_switches_and_the_sync_free_redo(cuda_api, oracle_api, opts):
    """The frames under every schedule switch; with halved sync-free bounds the second call's
    tables are redone, with the same frames."""
    saved = {k: cuda_api.get_option(k) for k in opts}
    try:
        for k, v in opts.items():
            cuda_api.set_option(k, v)
        r = cuda_api.Renderer(0)
        for name in ("repeats", "colors_blend", "library_511x64", "clip_leak", "library_511x64"):
            sc = ins.SCENES[name]
            got = _instances_device(r, ins.build_library(cuda_api, sc), sc)
            assert np.array_equal(got, _oracle_frames(oracle_api, name)), f"{name} under {opts}"
            if opts.get("test_fast_shrink") and name == "library_511x64":
                assert r.counters()["tables_mode"] in (1, 2)
        if opts.get("test_fast_shrink"):
            assert r.counters()["tables_mode"] == 2, "the halved bounds force the redo"
    finally:
        for k, v in saved.items():
            cuda_api.set_option(k, v)


def _desc(m, protos, tr=None, co=None):
    return binding._CInstances(m, protos, tr, co)


def test_refusals_write_nothing(cuda_api):
    import torch
    sc = ins.SCENES["repeats"]
    w, h, M = sc.width, sc.height, sc.m
    comp = ins.build_library(cuda_api, sc)
    state = _state(comp, sc)
    r = cuda_api.Renderer(0)
    n_max = r.max_views(h)
    api = cuda_api
    t = torch.full(((n_max + 1) * w * h * 4,), SENTINEL, dtype=torch.uint8, device="cuda:0")
    ids = torch.full(((n_max + 1) * w * h,), -1, dtype=torch.int32, device="cuda:0")
    stats = torch.full(((n_max + 1) * (M + 1) * 12,), -1, dtype=torch.int32, device="cuda:0")
    ch = (C.c_uint32 * 4)(*RGBA)
    cc = (C.c_float * 4)(CLEAR.r, CLEAR.g, CLEAR.b, CLEAR.a)
    P = np.tile(sc.prototypes[:1], (n_max + 1, 1))
    ident = np.tile(np.asarray(ins.IDENTITY, np.float32), (n_max + 1, M, 1))
    scale = ident.copy()
    scale[1, 2] = [2.0, 0.0, 0.0, 1.0, 0.0, 0.0]
    unknown = P.copy()
    unknown[1, 3] = 5  # no layer at order 5
    d_scale = torch.from_numpy(scale).cuda()
    d_unknown = torch.from_numpy(unknown.view(np.int32)).cuda()
    d_ident = torch.from_numpy(ident).cuda()
    d_colors = torch.zeros((n_max + 1) * M * 4 + 1, dtype=torch.float32, device="cuda:0")
    big = np.zeros((1, (1 << 21) + 1), np.uint32)

    cases = [
        ("null descriptor", None, 2, INVALID, None),
        ("null prototypes", _desc(M, None), 2, INVALID, None),
        ("M = 0", _desc(0, P.ctypes.data), 2, INVALID, None),
        ("no layer at an order", _desc(M, unknown.ctypes.data), 2, INVALID, "frame 1, slot 3: no layer is attached at order 5"),
        ("no layer at an order (device)", _desc(M, d_unknown.data_ptr()), 2, INVALID, "frame 1, slot 3"),
        ("scaling transform", _desc(M, P.ctypes.data, scale.ctypes.data), 2, INVALID, "frame 1, slot 2"),
        ("scaling transform (device)", _desc(M, P.ctypes.data, d_scale.data_ptr()), 2, INVALID, "frame 1, slot 2"),
        ("misaligned device transforms", _desc(M, P.ctypes.data, d_ident.data_ptr() + 2), 2, INVALID, "aligned"),
        ("misaligned device colours", _desc(M, P.ctypes.data, None, d_colors.data_ptr() + 2), 2, INVALID, "aligned"),
        ("n = 0", _desc(M, P.ctypes.data), 0, INVALID, None),
        ("n > max_views", _desc(M, P.ctypes.data), n_max + 1, INVALID, None),
        ("n M > 2^21", _desc((1 << 21) + 1, big.ctypes.data), 1, ORDER, None),
    ]
    for what, d, n, code, msg in cases:
        ptr = C.byref(d) if d is not None else None
        st = api.renderer_render_instances_device(r._h, comp._h, ptr, n, C.c_void_p(t.data_ptr()), w, 4 * w, h, 4 * w * h, ch, cc, None)
        assert st == code, f"{what}: status {st}"
        if msg:
            assert msg in api.last_error().decode(), f"{what}: {api.last_error().decode()}"
        st = api.renderer_render_instances_ids_device(r._h, comp._h, ptr, n, C.c_void_p(t.data_ptr()), w, 4 * w, h, 4 * w * h, ch, cc,
                                                      C.c_void_p(ids.data_ptr()), 4 * w, 4 * w * h, 0.0, None)
        assert st == code, f"{what} (IDs): status {st}"
        s = binding._CStats(stats.data_ptr(), 0, M + 1, 0.0)
        st = api.renderer_render_instances_stats_device(r._h, comp._h, ptr, n, C.byref(s), w, h, None, 4 * w, 4 * w * h, ch, cc, None)
        assert st == code, f"{what} (statistics): status {st}"
        torch.cuda.synchronize()
        assert bool((t == SENTINEL).all()) and bool((ids == -1).all()) and bool((stats == -1).all()), f"{what}: a buffer was written"
        assert _state(comp, sc) == state
    with pytest.raises(OrderError):
        r.render_instances_device(comp, Instances(big), t.data_ptr(), w, h)


def test_segment_limit_is_refused(cuda_api):
    """2^21 instances of a long slanted bar in one 1920 x 1080 frame: more than 2^30 pixel segments,
    refused with FORMA_ERR_CAPACITY before anything is written."""
    import torch
    bar = [(0.0, 0.0), (1900.0, 1000.0), (1900.0, 1003.0), (0.0, 3.0)]
    sc = ins.InstanceScene("bars", [ins.Proto(0, [bar])], 1920, 1080, np.zeros((1, 1 << 21), np.uint32))
    comp = ins.build_library(cuda_api, sc)
    r = cuda_api.Renderer(0)
    t = torch.full((1080, 1920, 4), SENTINEL, dtype=torch.uint8, device="cuda:0")
    with pytest.raises(FormaError, match="status 5"):
        r.render_instances_device(comp, ins.instances(binding, sc), t.data_ptr(), 1920, 1080)
    torch.cuda.synchronize()
    assert bool((t == SENTINEL).all())


def test_layer_field_edge(cuda_api, oracle_api):
    """n M = 2^21 is accepted (2 frames of 2^20 slots, a few of them filled, at the top of the
    field too); one slot more per frame is refused."""
    import torch
    sc0 = ins.SCENES["repeats"]
    M = 1 << 20
    P = np.full((2, M), ins.NONE, np.uint32)
    P[0, [0, 5, M - 1]] = [2, 3, 1]
    P[1, [7, M - 2, M - 1]] = [3, 2, 0]
    T = np.tile(np.asarray(ins.move(30, 30), np.float32), (2, M, 1))
    T[0, 5] = ins.move(36, 34)
    T[1, M - 1] = ins.move(20, 24)
    sc = ins.InstanceScene("edge", sc0.protos, 64, 64, P, T)
    comp = ins.build_library(cuda_api, sc)
    r = cuda_api.Renderer(0)
    got = _instances_device(r, comp, sc)
    orc = oracle_api.Renderer(0)
    for b in range(2):
        small = ins.InstanceScene("edge_b", sc0.protos, 64, 64, P[b:b + 1][:, P[b] != ins.NONE], T[b:b + 1][:, P[b] != ins.NONE])
        buf = np.zeros(64 * 64 * 4, np.uint8)
        orc.render(ins.twin(oracle_api, small, 0), buf, 64, 64, RGBA, CLEAR)  # the same stacking order, fewer empty slots
        assert np.array_equal(got[b], buf.reshape(64, 64, 4)), f"frame {b} at the top of the layer field"
    ids = torch.zeros((2, 64, 64), dtype=torch.int32, device="cuda:0")
    r.render_instances_ids_device(comp, ins.instances(binding, sc), ids.data_ptr(), 64, 64)
    torch.cuda.synchronize()
    assert set(np.unique(ids[1].cpu().numpy()).tolist()) <= {7, M - 2, M - 1, -1} and M - 1 in ids[1].cpu().numpy()
    d = _desc(M + 1, np.zeros((2, M + 1), np.uint32).ctypes.data)
    t = torch.full((2 * 64 * 64 * 4,), SENTINEL, dtype=torch.uint8, device="cuda:0")
    ch = (C.c_uint32 * 4)(*RGBA)
    cc = (C.c_float * 4)(CLEAR.r, CLEAR.g, CLEAR.b, CLEAR.a)
    assert cuda_api.renderer_render_instances_device(r._h, comp._h, C.byref(d), 2, C.c_void_p(t.data_ptr()), 64, 256, 64, 256 * 64, ch,
                                                     cc, None) == ORDER
    torch.cuda.synchronize()
    assert bool((t == SENTINEL).all())


def test_max_views_and_chunks(cuda_api, oracle_api):
    """n = max_views(16) = 2046 frames in one call, and 600 frames of 64 rows (max_views 511)
    chunked by the binding, each frame its twin's."""
    import torch
    protos = ins.SCENES["repeats"].protos
    rng = np.random.default_rng(3)
    r = cuda_api.Renderer(0)
    orc = oracle_api.Renderer(0)
    for n, h in ((2046, 16), (600, 64)):
        assert n == r.max_views(h) or n > r.max_views(h)
        P = rng.choice([0, 1, 2, 3, 4, 7, ins.NONE], (n, 3)).astype(np.uint32)
        T = np.zeros((n, 3, 6), np.float32)
        T[:] = ins.move(0, 0)
        T[..., 4] = rng.uniform(0, 48, (n, 3))
        T[..., 5] = rng.uniform(0, h, (n, 3))
        sc = ins.InstanceScene("many", protos, 48, h, P, T)
        got = _instances_device(r, ins.build_library(cuda_api, sc), sc)
        for b in list(range(0, n, 97)) + [n - 1]:
            buf = np.zeros(48 * h * 4, np.uint8)
            orc.render(ins.twin(oracle_api, sc, b), buf, 48, h, RGBA, CLEAR)
            assert np.array_equal(got[b], buf.reshape(h, 48, 4)), f"{n} frames of {h} rows: frame {b}"
