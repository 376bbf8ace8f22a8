"""Pose tables in device memory: the same tables as torch CUDA tensors and as numpy arrays give the
same bytes, bit for bit in the float formats, in all nine pose calls (sRGB8 host and device
frames, IDs on both sides, F32 and U8 masks, statistics, RGBA16F and RGBA32F, and frames over
per-frame backgrounds), on every light scene of tests/pose_scenes.py and tests/pose_fill_scenes.py
and on the heavy workloads. Also: every mix of host and device tables, device transforms that
scale up (refused like host ones, with nothing written and the renderer fine afterwards), the
scaling threshold and NaN components, misaligned and foreign tables, tables written on the
renderer's stream just before the call, the bytes that cross PCIe, and the composition left as
it was.
"""
import itertools

import numpy as np
import pytest

import oracle_linear
import pose_fill_scenes as pfs
import pose_scenes as ps
from forma_b200.binding import RGBA, Color, FormaError, Poses

pytestmark = pytest.mark.gpu

CLEAR = Color(1.0, 1.0, 1.0, 0.0)
SENTINEL = 0xA5
DEV = "cuda:0"
SCENES = {**{f"poses/{n}": ps.SCENES[n] for n in ps.SCENES}, **{f"fills/{n}": pfs.SCENES[n] for n in pfs.SCENES}}
LIGHT = [f"poses/{n}" for n in ps.LIGHT] + [f"fills/{n}" for n in pfs.LIGHT]
HEAVY = [f"poses/{n}" for n in ps.HEAVY] + [f"fills/{n}" for n in pfs.HEAVY]
_ORACLE = {}


def _colors(sc):
    return getattr(sc, "colors", None)


def _set_state(comp, sc, orders, b):
    if isinstance(sc, pfs.FillScene):
        pfs.set_pose_fill(comp, sc, orders, b)
    else:
        ps.set_pose(comp, sc, orders, b)


def _poses(sc, on_device="tvc", n=None):
    """The scene's Poses, with the tables named by on_device (t, v, c) as CUDA tensors; n frames
    (the scene's tables repeated) when given."""
    import torch
    tables = []
    for key, t in zip("tvc", (sc.transforms, sc.visible, _colors(sc))):
        if t is not None and n is not None:
            t = np.ascontiguousarray(np.resize(t, (n,) + t.shape[1:]))
        if t is not None and key in on_device:
            t = torch.from_numpy(np.ascontiguousarray(t)).to(DEV)
        tables.append(t)
    return Poses(sc.first_order, *tables)


def _window(orders):
    first = max(orders[0] - 1, 0) if orders else 0
    k = max(min(min(orders[-1] + 2, 1 << 21) - first, 66), 1) if orders else 1
    return first, k


def _backgrounds(sc, seed=0):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (sc.n, sc.height, sc.width, 4), dtype=np.uint8)


def _outputs(r, comp, sc, orders, p):
    """{name: bytes} of the nine pose calls with Poses p."""
    import torch
    w, h, n = sc.width, sc.height, sc.n
    first, k = _window(orders)
    out = {}

    def dev():
        return torch.full((n, h, w, 4), SENTINEL, dtype=torch.uint8, device=DEV)

    rgba = dev()
    r.render_poses_device(comp, p, rgba.data_ptr(), w, h, RGBA, CLEAR)
    out["device"] = rgba
    host = np.full((n, h, w, 4), SENTINEL, np.uint8)
    r.render_poses(comp, p, host, w, h, RGBA, CLEAR)
    out["host"] = host
    rgba2, ids = dev(), torch.full((n, h, w), -1, dtype=torch.int32, device=DEV)
    r.render_poses_ids_device(comp, p, ids.data_ptr(), w, h, rgba_ptr=rgba2.data_ptr(), channels=RGBA, clear_color=CLEAR,
                              min_coverage=0.25)
    out["ids device"], out["ids rgba"] = ids, rgba2
    host_ids = np.full((n, h, w), 7, np.uint32)
    r.render_poses_ids(comp, p, host_ids, w, h, min_coverage=0.5)
    out["ids host"] = host_ids
    for fmt, dt in (("f32", torch.float32), ("u8", torch.uint8)):
        m = torch.full((n, k, h, w), 3, dtype=dt, device=DEV)
        r.render_poses_masks_device(comp, p, m.data_ptr(), w, h, first, k, format=fmt)
        out[f"masks {fmt}"] = m
    stats = torch.full((n, k, 12), -1, dtype=torch.int32, device=DEV)
    r.render_poses_stats_device(comp, p, stats.data_ptr(), w, h, first, k, min_coverage=0.25)
    out["stats"] = stats
    f16 = torch.full((n, h, w, 4), 2.0, dtype=torch.float16, device=DEV)
    r.render_poses_linear_device(comp, p, f16.data_ptr(), w, h, RGBA, CLEAR, format="f16")
    out["f16 device"] = f16
    f32 = np.full((n, h, w, 4), 2.0, np.float32)
    r.render_poses_linear(comp, p, f32, w, h, RGBA, CLEAR, format="f32")
    out["f32 host"] = f32
    over = torch.from_numpy(_backgrounds(sc, len(sc.name))).to(DEV)
    r.render_poses_over_device(comp, p, over.data_ptr(), w, h, RGBA)
    out["over"] = over
    torch.cuda.synchronize()
    return {key: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v).view(np.uint8) for key, v in out.items()}


def _assert_same(got, want, what):
    for key in want:
        if not np.array_equal(got[key], want[key]):
            bad = np.nonzero(got[key] != want[key])
            raise AssertionError(f"{what}: {key} differs at {len(bad[0])} bytes, first {tuple(int(i[0]) for i in bad)}")


def _device_frames(r, comp, sc, p, n=None):
    import torch
    n = sc.n if n is None else n
    t = torch.full((n, sc.height, sc.width, 4), SENTINEL, dtype=torch.uint8, device=DEV)
    r.render_poses_device(comp, p, t.data_ptr(), sc.width, sc.height, RGBA, CLEAR)
    torch.cuda.synchronize()
    return t.cpu().numpy()


def _oracle_frames(oracle_api, key, frames=None):
    sc = SCENES[key]
    frames = range(sc.n) if frames is None else frames
    cache = _ORACLE.setdefault(key, {})
    todo = [b for b in frames if b not in cache]
    if todo:
        comp, orders = sc.build(oracle_api)
        r = oracle_api.Renderer(0)
        for b in todo:
            _set_state(comp, sc, orders, b)
            buf = np.zeros(sc.width * sc.height * 4, np.uint8)
            r.render(comp, buf, sc.width, sc.height, RGBA, CLEAR)
            cache[b] = buf.reshape(sc.height, sc.width, 4)
    return {b: cache[b] for b in frames}


def _still(oracle_api, key):
    """The oracle's frame of the scene's composition as built."""
    sc = SCENES[key]
    comp, _ = sc.build(oracle_api)
    buf = np.zeros(sc.width * sc.height * 4, np.uint8)
    oracle_api.Renderer(0).render(comp, buf, sc.width, sc.height, RGBA, CLEAR)
    return buf.reshape(sc.height, sc.width, 4)


def _check_oracle(frames, want, what):
    for b, f in want.items():
        assert np.array_equal(frames[b], f), f"{what}: frame {b} differs from the oracle"


@pytest.fixture(autouse=True)
def _oracle_modes(oracle_api):
    oracle_linear.attach(oracle_api)
    oracle_api.hooks.fo_set_recip_mode(0)


@pytest.mark.parametrize("key", LIGHT)
def test_device_tables_match_host_tables(cuda_api, key):
    sc = SCENES[key]
    comp, orders = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    want = _outputs(r, comp, sc, orders, _poses(sc, ""))
    got = _outputs(r, comp, sc, orders, _poses(sc, "tvc"))
    _assert_same(got, want, key)


@pytest.mark.parametrize("key", ["poses/e2e_texture", "poses/window_gaps", "poses/show_hide_bits", "fills/alpha_flips",
                                 "fills/window_gaps_filled"])
def test_device_tables_match_the_oracle(cuda_api, oracle_api, key):
    sc = SCENES[key]
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    _check_oracle(_device_frames(r, comp, sc, _poses(sc)), _oracle_frames(oracle_api, key), key)


@pytest.mark.parametrize("key", HEAVY)
def test_workloads(cuda_api, oracle_api, key):
    """One call each with host and with device tables: the same frames; a few against the oracle."""
    sc = SCENES[key]
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    frames = _device_frames(r, comp, sc, _poses(sc))
    assert np.array_equal(frames, _device_frames(r, comp, sc, _poses(sc, ""))), key
    _check_oracle(frames, _oracle_frames(oracle_api, key, sorted({0, sc.n // 2, sc.n - 1})), key)


def _all_tables_scene():
    return next(k for k in LIGHT if all(t is not None for t in (SCENES[k].transforms, SCENES[k].visible, _colors(SCENES[k]))))


def test_every_mix_of_host_and_device_tables(cuda_api):
    key = _all_tables_scene()
    sc = SCENES[key]
    comp, orders = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    want = _outputs(r, comp, sc, orders, _poses(sc, ""))
    mixes = ["".join(m) for k in (1, 2, 3) for m in itertools.combinations("tvc", k)]
    assert len(mixes) == 7
    for mix in mixes:
        _assert_same(_outputs(r, comp, sc, orders, _poses(sc, mix)), want, f"{key}, device tables {mix}")


def test_bool_visibility_and_any_byte_offset(cuda_api):
    """Visibility as a torch bool tensor, and as uint8 rows starting at an odd byte."""
    import torch
    key = _all_tables_scene()
    sc = SCENES[key]
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    want = _device_frames(r, comp, sc, _poses(sc, ""))
    vis = torch.from_numpy(sc.visible.astype(bool)).to(DEV)
    got = _device_frames(r, comp, sc, Poses(sc.first_order, sc.transforms, vis, _colors(sc)))
    assert np.array_equal(got, want)
    backing = torch.zeros(sc.visible.size + 1, dtype=torch.uint8, device=DEV)
    backing[1:] = torch.from_numpy(sc.visible.reshape(-1)).to(DEV)
    odd = backing[1:].view(sc.visible.shape)
    assert odd.data_ptr() % 2 == 1
    got = _device_frames(r, comp, sc, Poses(sc.first_order, sc.transforms, odd, _colors(sc)))
    assert np.array_equal(got, want)


def _refusal_scene():
    return next(k for k in ps.LIGHT if ps.SCENES[k].transforms is not None and ps.SCENES[k].n >= 2)


def _nine_calls(r, comp, sc, p, bufs, orders):
    """The nine pose calls into the sentinel buffers `bufs`; each must raise FormaError."""
    w, h = sc.width, sc.height
    first, k = _window(orders)
    calls = [
        lambda: r.render_poses_device(comp, p, bufs["rgba"].data_ptr(), w, h, RGBA, CLEAR),
        lambda: r.render_poses(comp, p, bufs["host"], w, h, RGBA, CLEAR),
        lambda: r.render_poses_ids_device(comp, p, bufs["ids"].data_ptr(), w, h, rgba_ptr=bufs["rgba"].data_ptr(), channels=RGBA,
                                          clear_color=CLEAR),
        lambda: r.render_poses_ids(comp, p, bufs["host_ids"], w, h),
        lambda: r.render_poses_masks_device(comp, p, bufs["masks"].data_ptr(), w, h, first, k, format="u8"),
        lambda: r.render_poses_stats_device(comp, p, bufs["stats"].data_ptr(), w, h, first, k),
        lambda: r.render_poses_linear_device(comp, p, bufs["f32"].data_ptr(), w, h, RGBA, CLEAR, format="f32"),
        lambda: r.render_poses_linear(comp, p, bufs["host_f32"], w, h, RGBA, CLEAR, format="f32"),
        lambda: r.render_poses_over_device(comp, p, bufs["rgba"].data_ptr(), w, h, RGBA),
    ]
    return calls


@pytest.mark.parametrize("opts", [{"sync_free": 0, "sort_counts": 1}, {"sync_free": 1, "sort_counts": 1}])
def test_a_device_transform_that_scales_up_is_refused(cuda_api, oracle_api, opts):
    import torch
    key = "poses/" + _refusal_scene()
    sc = SCENES[key]
    saved = {k: cuda_api.get_option(k) for k in opts}
    try:
        for k, v in opts.items():
            cuda_api.set_option(k, v)
        comp, orders = sc.build(cuda_api)
        r = cuda_api.Renderer(0)
        w, h, n, K = sc.width, sc.height, sc.n, sc.n_orders
        still = torch.zeros((h, w, 4), dtype=torch.uint8, device=DEV)
        r.render_device(comp, still.data_ptr(), w, h, RGBA, CLEAR)  # the sync-free bounds of an ordinary frame
        enabled = {o: comp.get(o).is_enabled() for o in orders}
        b, kk = n - 1, K // 2
        xf = sc.transforms.copy()
        xf[b, kk] = [2.0, 0.0, 0.0, 2.0, 0.0, 0.0]
        p = Poses(sc.first_order, torch.from_numpy(xf).to(DEV), sc.visible)
        first, km = _window(orders)
        bufs = {"rgba": torch.full((n, h, w, 4), SENTINEL, dtype=torch.uint8, device=DEV),
                "host": np.full((n, h, w, 4), SENTINEL, np.uint8),
                "ids": torch.full((n, h, w), -7, dtype=torch.int32, device=DEV),
                "host_ids": np.full((n, h, w), 7, np.uint32),
                "masks": torch.full((n, km, h, w), SENTINEL, dtype=torch.uint8, device=DEV),
                "stats": torch.full((n, km, 12), -7, dtype=torch.int32, device=DEV),
                "f32": torch.full((n, h, w, 4), 3.0, dtype=torch.float32, device=DEV),
                "host_f32": np.full((n, h, w, 4), 3.0, np.float32)}
        before = {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v).copy() for k, v in bufs.items()}
        for call in _nine_calls(r, comp, sc, p, bufs, orders):
            with pytest.raises(FormaError, match="status 1 ") as e:
                call()
            assert f"frame {b}," in str(e.value) and f"order {sc.first_order + kk}:" in str(e.value), str(e.value)
        torch.cuda.synchronize()
        for k, v in bufs.items():
            assert np.array_equal(v.cpu().numpy() if isinstance(v, torch.Tensor) else v, before[k]), f"{k} was written"
        assert {o: comp.get(o).is_enabled() for o in orders} == enabled
        # The next poses call and the next ordinary frame are right.
        _check_oracle(_device_frames(r, comp, sc, _poses(sc)), _oracle_frames(oracle_api, key), f"{key} after the refusals")
        still.zero_()
        r.render_device(comp, still.data_ptr(), w, h, RGBA, CLEAR)
        torch.cuda.synchronize()
        assert np.array_equal(still.cpu().numpy(), _still(oracle_api, key)), "render_device after the refusals"
    finally:
        for k, v in saved.items():
            cuda_api.set_option(k, v)


def _threshold_cases():
    """(ux, vx, uy, vy) around the bounds of geom_pres_ok: ux^2 + uy^2 <= 1 + 2^-20 and
    vx^2 + vy^2 <= 1 + 2^-19, in f32 with each operation rounded; and NaN and infinite components."""
    f = np.float32
    max_x, max_y = f(1.0) + f(2.0 ** -20), f(1.0) + f(2.0 ** -19)
    cases = []
    for bound, col in ((max_x, 0), (max_y, 1)):
        u = f(np.sqrt(np.float64(bound)))
        for step in range(-3, 4):
            v = u
            for _ in range(abs(step)):
                v = np.nextafter(v, f(np.inf) if step > 0 else f(0), dtype=f)
            m = [f(1), f(0), f(0), f(1)]
            if col == 0:
                m[0] = v  # ux
            else:
                m[3] = v  # vy
            cases.append(m)
        # the sum at exactly the bound and one ulp above, over two components
        for a in (f(0.75), f(0.5)):
            b = f(np.sqrt(np.float64(bound - a * a)))
            for _ in range(3):
                s = f(a * a) + f(b * b)
                if s < bound:
                    b = np.nextafter(b, f(2), dtype=f)
                elif s > bound:
                    b = np.nextafter(b, f(0), dtype=f)
            for bb in (b, np.nextafter(b, f(2), dtype=f)):
                cases.append([a, f(0), bb, f(1)] if col == 0 else [f(1), a, f(0), bb])
    for k in range(4):
        for v in (f(np.nan), f(np.inf), f(-np.inf)):
            m = [f(1), f(0), f(0), f(1)]
            m[k] = v
            cases.append(m)
    return cases


def _model_ok(ux, vx, uy, vy):
    f = np.float32
    with np.errstate(invalid="ignore", over="ignore"):
        return not (f(ux * ux) + f(uy * uy) > f(1) + f(2.0 ** -20)) and not (f(vx * vx) + f(vy * vy) > f(1) + f(2.0 ** -19))


def test_threshold_and_nan_agree_with_host_tables(cuda_api):
    import torch
    key = "poses/" + _refusal_scene()
    sc = SCENES[key]
    comp, orders = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    t = torch.zeros((1, sc.height, sc.width, 4), dtype=torch.uint8, device=DEV)
    cases = _threshold_cases()
    outcomes = {True: 0, False: 0}
    for ux, vx, uy, vy in cases:
        xf = np.tile(np.array(ps.IDENTITY, np.float32), (1, sc.n_orders, 1))
        xf[0, sc.n_orders - 1, :4] = [ux, vx, uy, vy]
        xf[0, sc.n_orders - 1, 4:] = [0.5, np.nan if np.isnan(ux) else 0.25]
        got = []
        for table in (xf, torch.from_numpy(xf).to(DEV)):
            try:
                r.render_poses_device(comp, Poses(sc.first_order, table), t.data_ptr(), sc.width, sc.height, RGBA, CLEAR)
                torch.cuda.synchronize()
                got.append((True, t.cpu().numpy().copy()))
            except FormaError as e:
                got.append((False, str(e)))
        assert got[0][0] == got[1][0] == _model_ok(ux, vx, uy, vy), (ux, vx, uy, vy, got[0][0], got[1][0])
        if got[0][0]:
            assert np.array_equal(got[0][1], got[1][1]), (ux, vx, uy, vy)
        else:
            assert got[0][1] == got[1][1]
        outcomes[got[0][0]] += 1
    assert outcomes[True] >= 8 and outcomes[False] >= 8, outcomes


def test_misaligned_device_tables_are_refused(cuda_api):
    """Transforms or colours 2 bytes off a 4-byte boundary (inside a tensor that holds them whole)
    are refused by the host before anything is launched."""
    import torch
    key = _all_tables_scene()
    sc = SCENES[key]
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    t = torch.full((sc.n, sc.height, sc.width, 4), SENTINEL, dtype=torch.uint8, device=DEV)
    for which, table in (("transforms", sc.transforms), ("colors", sc.colors)):
        raw = np.ascontiguousarray(table).view(np.uint8).reshape(-1)
        backing = torch.zeros(raw.size + 4, dtype=torch.uint8, device=DEV)
        backing[2:2 + raw.size] = torch.from_numpy(raw).to(DEV)
        ptr = backing.data_ptr() + 2
        assert ptr % 4 == 2

        class Shifted:
            __cuda_array_interface__ = dict(shape=table.shape, typestr="<f4", data=(ptr, False), strides=None, version=3)
        tables = dict(transforms=sc.transforms, visible=sc.visible, colors=sc.colors)
        tables[which] = Shifted()
        launches = r.counters()["launches"]
        with pytest.raises(FormaError, match="aligned"):
            r.render_poses_device(comp, Poses(sc.first_order, **tables), t.data_ptr(), sc.width, sc.height, RGBA, CLEAR)
        assert r.counters()["launches"] == launches, which
    torch.cuda.synchronize()
    assert bool(torch.all(t == SENTINEL))


def test_a_table_on_another_device_is_refused(cuda_api):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    key = _all_tables_scene()
    sc = SCENES[key]
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    t = torch.full((sc.n, sc.height, sc.width, 4), SENTINEL, dtype=torch.uint8, device=DEV)
    with pytest.raises(FormaError, match="device 1.*device 0"):
        r.render_poses_device(comp, Poses(sc.first_order, torch.from_numpy(sc.transforms).to("cuda:1")), t.data_ptr(),
                              sc.width, sc.height, RGBA, CLEAR)
    torch.cuda.synchronize()
    assert bool(torch.all(t == SENTINEL))


def test_tables_written_on_the_renderers_stream(cuda_api):
    """The renderer's stream is a torch side stream; the tables are written there (behind a delay)
    just before the call, without a synchronisation: the call reads them in stream order."""
    import torch
    key = _all_tables_scene()
    sc = SCENES[key]
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    want = _device_frames(r, comp, sc, _poses(sc, ""))
    src = [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in (sc.transforms, sc.visible, sc.colors)]
    torch.cuda.synchronize()
    side = torch.cuda.Stream(device=DEV)
    r2 = cuda_api.Renderer(0)
    r2.set_stream(side.cuda_stream)
    with torch.cuda.stream(side):
        dst = [torch.zeros_like(a) for a in src]
        out = torch.zeros((sc.n, sc.height, sc.width, 4), dtype=torch.uint8, device=DEV)
        torch.cuda._sleep(20_000_000)
        for d, s in zip(dst, src):
            d.copy_(s)
        r2.render_poses_device(comp, Poses(sc.first_order, *dst), out.data_ptr(), sc.width, sc.height, RGBA, CLEAR)
    side.synchronize()
    assert np.array_equal(out.cpu().numpy(), want)


def test_bytes_over_pcie(cuda_api):
    """Device tables: the same upload for 1 and max_views frames, the window's 32 K bytes and a
    little more. Host tables: 24 n K for transforms, n K for visibility, 32 K for the window,
    16 n K for colours."""
    import torch
    key = _all_tables_scene()
    sc = SCENES[key]
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    w, h, K = sc.width, sc.height, sc.n_orders
    big = r.max_views(h)
    out = torch.zeros((big, h, w, 4), dtype=torch.uint8, device=DEV)
    for _ in range(2):
        r.render_device(comp, out.data_ptr(), w, h, RGBA, CLEAR)
    b0 = r.counters()["h2d_bytes"]
    r.render_device(comp, out.data_ptr(), w, h, RGBA, CLEAR)
    idle = r.counters()["h2d_bytes"] - b0

    def h2d(p):
        before = r.counters()["h2d_bytes"]
        r.render_poses_device(comp, p, out.data_ptr(), w, h, RGBA, CLEAR)
        return r.counters()["h2d_bytes"] - before - idle

    h2d(_poses(sc, "tvc", 1))  # every buffer of the call at its size
    h2d(_poses(sc, "tvc", big))
    one, many = h2d(_poses(sc, "tvc", 1)), h2d(_poses(sc, "tvc", big))
    assert one == many and 32 * K <= one <= 32 * K + 256, (one, many, K)
    for n in (1, 3, big):
        for mix, extra in (("", 41 * n * K), ("v", 40 * n * K), ("c", 25 * n * K), ("t", 17 * n * K), ("vc", 24 * n * K)):
            assert h2d(_poses(sc, mix, n)) == one + extra, (n, mix)
    torch.cuda.synchronize()


def test_the_call_leaves_the_composition(cuda_api):
    import torch
    key = _all_tables_scene()
    sc = SCENES[key]
    w, h = sc.width, sc.height
    comp, _ = sc.build(cuda_api)
    r = cuda_api.Renderer(0)
    t = torch.zeros(w * h * 4, dtype=torch.uint8, device=DEV)
    for _ in range(2):
        r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR)
    b0 = r.counters()["h2d_bytes"]
    r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR)
    torch.cuda.synchronize()
    idle, before = r.counters()["h2d_bytes"] - b0, t.cpu().numpy()
    _device_frames(r, comp, sc, _poses(sc))
    t.zero_()
    b1 = r.counters()["h2d_bytes"]
    r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR)
    torch.cuda.synchronize()
    assert r.counters()["h2d_bytes"] - b1 <= idle, "the render after a device-table call uploaded"
    assert np.array_equal(t.cpu().numpy(), before)


@pytest.mark.parametrize("opts", [{"sync_free": 0}, {"sync_free": 1}, {"sync_free": 1, "test_fast_shrink": 1}, {"speculate": 0},
                                  {"speculate": 1}, {"paint_solid": 0}, {"paint_solid": 1}, {"paint_lpt": 0}])
def test_switches(cuda_api, oracle_api, opts):
    """Every schedule gives the oracle's bytes with device tables, single frames between."""
    saved = {k: cuda_api.get_option(k) for k in opts}
    try:
        for k, v in opts.items():
            cuda_api.set_option(k, v)
        r = cuda_api.Renderer(0)
        for key in ("fills/alpha_flips", "poses/" + _refusal_scene(), _all_tables_scene(), "fills/library_filled"):
            sc = SCENES[key]
            comp, _ = sc.build(cuda_api)
            buf = np.zeros(sc.width * sc.height * 4, np.uint8)
            r.render(comp, buf, sc.width, sc.height, RGBA, CLEAR)
            frames = _device_frames(r, comp, sc, _poses(sc))
            spread = sorted({0, sc.n // 2, sc.n - 1})
            _check_oracle(frames, _oracle_frames(oracle_api, key, spread), key)
    finally:
        for k, v in saved.items():
            cuda_api.set_option(k, v)
