"""Layer statistics on the device (Renderer.render_stats*, forma_renderer_render_*stats*), held to the
stats oracle (tests/oracle_stats.py, pinned in tests/test_stats_oracle.py) with integer equality: the
e2e, extreme and style scenes, random_mixed at 1080p with a crop, paris4k with all of its orders,
every in-limit view and batch scene, the combined calls (their RGBA bytes are the plain calls'), the
device's own masks and ID frame, every table mode including the sync-free redo, the schedule
options, repeated calls, refusals, layer caches and the CLI."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import batch_scenes as bs
import extremes
import oracle_stats
import scenes
import style_scenes as ss
import synth
import view_scenes as vs
import workloads
from forma_b200.binding import ID_NONE, RGBA, STATS_DTYPE, Color, Rect, _CStats, split_stats

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLEAR = Color(1.0, 1.0, 1.0, 0.0)
SENTINEL = 0x5A5A5A5A


@pytest.fixture(autouse=True)
def _attach(oracle_api):
    oracle_stats.attach(oracle_api)


def n_orders(comp):
    return max(bs.n_orders(comp), 1)


def records(n, k):
    """A sentinel-filled [n, k, 12] int32 CUDA tensor."""
    import torch
    return torch.full((n, k, 12), SENTINEL, dtype=torch.int32, device="cuda:0")


def as_records(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy().view(STATS_DTYPE)[..., 0]


def assert_records(got, want, what):
    assert got.shape == want.shape, what
    bad = np.argwhere(got != want)
    assert not len(bad), f"{what}: {len(bad)} records differ, first at {bad[0].tolist()}: got {got[tuple(bad[0])]}, " \
                         f"want {want[tuple(bad[0])]}"


def device_stats(r, comp, w, h, first, k, min_coverage=0.0, crop=None, **kw):
    t = records(1, k)
    r.render_stats_device(comp, t.data_ptr(), w, h, first, k, min_coverage, crop=crop, **kw)
    return as_records(t)[0]


def both(cuda_api, oracle_api, comp, ocomp, w, h, first, k, min_coverage=0.0, crop=None):
    want = oracle_stats.render(oracle_api, ocomp, w, h, first, k, min_coverage, crop)
    r = cuda_api.Renderer(0)
    assert_records(device_stats(r, comp, w, h, first, k, min_coverage, crop), want, "device")
    assert_records(r.render_stats(comp, w, h, first, k, min_coverage, crop), want, "host")
    return want


# --- scenes -----------------------------------------------------------------------------------------


@pytest.mark.parametrize("threshold", [0.0, 0.5])
@pytest.mark.parametrize("name", sorted(scenes.E2E))
def test_e2e(cuda_api, oracle_api, name, threshold):
    comp, ocomp = cuda_api.Composition(), oracle_api.Composition()
    scenes.E2E[name](cuda_api, comp)
    scenes.E2E[name](oracle_api, ocomp)
    both(cuda_api, oracle_api, comp, ocomp, 64, 64, 0, n_orders(ocomp) + 1, threshold)


@pytest.mark.parametrize("name", sorted(extremes.SCENES))
def test_extremes(cuda_api, oracle_api, name):
    comp, _, sc = extremes.build(cuda_api, name)
    ocomp, _, _ = extremes.build(oracle_api, name)
    n = n_orders(ocomp)
    both(cuda_api, oracle_api, comp, ocomp, sc.width, sc.height, 0, n + 1, 0.0, sc.crop)
    both(cuda_api, oracle_api, comp, ocomp, sc.width, sc.height, max(n - 5, 0), 8, 0.5, sc.crop)


@pytest.mark.parametrize("name", sorted(ss.SCENES))
def test_styles(cuda_api, oracle_api, name):
    comp, _, sc = ss.build(cuda_api, name)
    ocomp, _, _ = ss.build(oracle_api, name)
    both(cuda_api, oracle_api, comp, ocomp, sc.width, sc.height, 0, n_orders(ocomp), 0.5)


def test_random_mixed_1080p_crop(cuda_api, oracle_api):
    w, h = 1920, 1080
    build = lambda api, comp: synth.random_mixed(api, comp, 900, w, h, 17)  # noqa: E731
    comp, ocomp = cuda_api.Composition(), oracle_api.Composition()
    build(cuda_api, comp)
    build(oracle_api, ocomp)
    for crop in (None, Rect((130, 1500), (70, 1010))):
        for threshold in (0.0, 0.5, 0.998):
            want = both(cuda_api, oracle_api, comp, ocomp, w, h, 0, 901, threshold, crop)
            assert want["visible"].any() and want["pixels"].any()
        both(cuda_api, oracle_api, comp, ocomp, w, h, 300, 24, 0.0, crop)


@pytest.mark.parametrize("threshold", [0.0, 0.5])
def test_paris4k_all_orders(cuda_api, oracle_api, threshold):
    comp, w, h = workloads.build_scene(cuda_api, "paris4k")
    ocomp, _, _ = workloads.build_scene(oracle_api, "paris4k")
    n = n_orders(ocomp)
    assert n >= 50000
    want = both(cuda_api, oracle_api, comp, ocomp, w, h, 0, n, threshold)
    assert (want["visible"] > 0).sum() > 1000


# --- views and batches --------------------------------------------------------------------------------


def _oracle_views(oracle_api, sc, first, k, min_coverage):
    comp, xf = vs.build(oracle_api, sc)
    out = []
    for v in sc.views:
        vs.set_view(comp, xf, v)
        out.append(oracle_stats.render(oracle_api, comp, sc.width, sc.height, first, k, min_coverage))
    return np.stack(out)


def _oracle_batch(oracle_api, sc, first, k, min_coverage):
    distinct, _ = bs.build(oracle_api, sc)
    per = [oracle_stats.render(oracle_api, c, sc.width, sc.height, first, k, min_coverage) for c in distinct]
    return np.stack([per[i] for i in sc.frames])


@pytest.mark.parametrize("name", vs.IN_LIMIT)
def test_views(cuda_api, oracle_api, name):
    sc = vs.SCENES[name]
    comp, _ = vs.build(cuda_api, sc)
    k = n_orders(comp) + 1
    r = cuda_api.Renderer(0)
    for threshold in (0.0, 0.5):
        t = records(len(sc.views), k)
        r.render_views_stats_device(comp, sc.views, t.data_ptr(), sc.width, sc.height, 0, k, threshold)
        assert_records(as_records(t), _oracle_views(oracle_api, sc, 0, k, threshold), f"{name} {threshold}")


@pytest.mark.parametrize("name", bs.IN_LIMIT)
def test_batches(cuda_api, oracle_api, name):
    sc = bs.SCENES[name]
    distinct, frames = bs.build(cuda_api, sc)
    k = max(n_orders(c) for c in distinct) + 1
    r = cuda_api.Renderer(0)
    for threshold in (0.0, 0.5):
        t = records(len(frames), k)
        r.render_batch_stats_device(frames, t.data_ptr(), sc.width, sc.height, 0, k, threshold)
        assert_records(as_records(t), _oracle_batch(oracle_api, sc, 0, k, threshold), f"{name} {threshold}")
    if name == "orders_at_limit":  # a window ending at the top order, and one past every order
        for first in (k - 8, k + 3):
            t = records(len(frames), 8)
            r.render_batch_stats_device(frames, t.data_ptr(), sc.width, sc.height, first, 8)
            assert_records(as_records(t), _oracle_batch(oracle_api, sc, first, 8, 0.0), f"{name} [{first}, +8)")


# --- combined calls -----------------------------------------------------------------------------------


def _rgba(n, w, h):
    import torch
    return torch.full((n, h, w, 4), 0xA5, dtype=torch.uint8, device="cuda:0")


def test_combined_single(cuda_api, oracle_api):
    import torch
    w, h = 300, 200
    comp, ocomp = cuda_api.Composition(), oracle_api.Composition()
    synth.random_mixed(cuda_api, comp, 150, w, h, 8)
    synth.random_mixed(oracle_api, ocomp, 150, w, h, 8)
    r = cuda_api.Renderer(0)
    for crop in (None, Rect((17, 250), (5, 190))):
        rgba, plain = _rgba(1, w, h), _rgba(1, w, h)
        got = device_stats(r, comp, w, h, 0, 151, 0.25, crop, rgba_ptr=rgba.data_ptr(), clear_color=CLEAR)
        r.render_device(comp, plain.data_ptr(), w, h, RGBA, CLEAR, crop=crop)
        torch.cuda.synchronize()
        assert torch.equal(rgba, plain)
        assert_records(got, oracle_stats.render(oracle_api, ocomp, w, h, 0, 151, 0.25, crop), str(crop))


def test_combined_stacks(cuda_api, oracle_api):
    import torch
    r = cuda_api.Renderer(0)
    for name in ("straddle", "odd_h100"):
        sc = vs.SCENES[name]
        comp, _ = vs.build(cuda_api, sc)
        n, k = len(sc.views), n_orders(comp)
        t, rgba, plain = records(n, k), _rgba(n, sc.width, sc.height), _rgba(n, sc.width, sc.height)
        r.render_views_stats_device(comp, sc.views, t.data_ptr(), sc.width, sc.height, 0, k, rgba_ptr=rgba.data_ptr(),
                                    clear_color=CLEAR)
        r.render_views_device(comp, sc.views, plain.data_ptr(), sc.width, sc.height, RGBA, CLEAR)
        torch.cuda.synchronize()
        assert torch.equal(rgba, plain), name
        assert_records(as_records(t), _oracle_views(oracle_api, sc, 0, k, 0.0), name)
    for name in ("mixed_order", "repeats_h40"):
        sc = bs.SCENES[name]
        distinct, frames = bs.build(cuda_api, sc)
        n, k = len(frames), max(n_orders(c) for c in distinct)
        t, rgba, plain = records(n, k), _rgba(n, sc.width, sc.height), _rgba(n, sc.width, sc.height)
        r.render_batch_stats_device(frames, t.data_ptr(), sc.width, sc.height, 0, k, 0.5, rgba_ptr=rgba.data_ptr(),
                                    clear_color=CLEAR)
        r.render_batch_device(frames, plain.data_ptr(), sc.width, sc.height, RGBA, CLEAR)
        torch.cuda.synchronize()
        assert torch.equal(rgba, plain), name
        assert_records(as_records(t), _oracle_batch(oracle_api, sc, 0, k, 0.5), name)


def test_the_devices_own_masks_and_ids(cuda_api):
    """The records are a reduction of the device's own F32 masks and ID frame of the same arguments."""
    import torch
    w, h = 700, 390
    comp = cuda_api.Composition()
    synth.random_mixed(cuda_api, comp, 300, w, h, 23)
    r = cuda_api.Renderer(0)
    for first, k, threshold, crop in ((0, 64, 0.0, None), (100, 48, 0.5, Rect((40, 650), (20, 300))), (250, 60, 0.998, None)):
        planes = torch.zeros((k, h, w), dtype=torch.float32, device="cuda:0")
        r.render_masks_device(comp, planes.data_ptr(), w, h, first, k, "f32", crop=crop)
        ids = np.full(w * h, ID_NONE, np.uint32)
        r.render_ids(comp, ids, w, h, crop=crop, min_coverage=threshold)
        torch.cuda.synchronize()
        want = oracle_stats.reduce(planes.cpu().numpy(), ids.reshape(h, w), first, threshold, oracle_stats.region(w, h, crop))
        t = records(1, k)
        r.render_stats_device(comp, t.data_ptr(), w, h, first, k, threshold, crop=crop)
        assert_records(as_records(t)[0], want, f"[{first}, +{k}) at {threshold}")
        f = split_stats(t[0])
        assert torch.equal(f["pixels"].cpu(), torch.from_numpy(want["pixels"].astype(np.int64)))
        assert torch.equal(f["area"].cpu(), torch.from_numpy(want["area"].astype(np.int64)))


# --- table modes, schedule options, repeated calls ------------------------------------------------------

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
    oracle_stats.attach(oracle_api)
    ocomp = oracle_api.Composition()
    synth.random_mixed(oracle_api, ocomp, 900, 1280, 720, 31)
    return oracle_stats.render(oracle_api, ocomp, 1280, 720, 0, 901, 0.5)


@pytest.mark.parametrize("opts", [{"sync_free": 0}, {"sync_free": 1}, {"sync_free": 1, "test_fast_shrink": 1}])
def test_table_modes(cuda_api, mixed720, restore_options, opts):
    """Counted tables, sync-free tables, and halved bounds that send the frame through again: the
    redo repeats the records' initialisation, so nothing is counted twice."""
    for k, v in opts.items():
        cuda_api.set_option(k, v)
    comp = cuda_api.Composition()
    synth.random_mixed(cuda_api, comp, 900, 1280, 720, 31)
    r = cuda_api.Renderer(0)
    for frame in range(3):
        assert_records(device_stats(r, comp, 1280, 720, 0, 901, 0.5), mixed720, f"{opts} frame {frame}")
        assert_records(r.render_stats(comp, 1280, 720, 0, 901, 0.5), mixed720, f"{opts} frame {frame} host")
    # Enough cells for halved bounds to fall short: 511 frames, twice; each frame's records are those of
    # its composition alone.
    sc = bs.SCENES["random_511"]
    distinct, frames = bs.build(cuda_api, sc)
    k = max(n_orders(c) for c in distinct)
    alone = [device_stats(r, c, sc.width, sc.height, 0, k) for c in distinct]
    for _ in range(2):
        t = records(len(frames), k)
        r.render_batch_stats_device(frames, t.data_ptr(), sc.width, sc.height, 0, k)
        assert_records(as_records(t), np.stack([alone[i] for i in sc.frames]), "random_511")


@pytest.mark.parametrize("name,value", [("speculate", 0), ("band_copy", 0), ("copy_bands", 16), ("sort_full_key", 1),
                                        ("sort_big_log2", 10), ("sort_scan_log2", 10), ("paint_lpt", 0), ("paint_wide", 1),
                                        ("paint_solid", 0), ("band_filter", 0), ("sync_free", 0), ("host_slices", 2),
                                        ("slice_bands", 1), ("slice_min_points", 0), ("slice_chain", 0), ("test_gap_cap", 1),
                                        ("sort_counts", 0)])
def test_option_does_not_change_the_records(cuda_api, mixed720, restore_options, name, value):
    cuda_api.set_option(name, value)
    comp = cuda_api.Composition()
    synth.random_mixed(cuda_api, comp, 900, 1280, 720, 31)
    r = cuda_api.Renderer(0)
    for frame in range(2):
        assert_records(device_stats(r, comp, 1280, 720, 0, 901, 0.5), mixed720, f"{name}={value} frame {frame}")
        assert_records(r.render_stats(comp, 1280, 720, 0, 901, 0.5), mixed720, f"{name}={value} host")


def test_repeated_calls_are_bit_identical(cuda_api):
    import torch
    comp, w, h = workloads.build_scene(cuda_api, "paris4k")
    n = n_orders(comp)
    r = cuda_api.Renderer(0)
    a, b = records(1, n), records(1, n)
    r.render_stats_device(comp, a.data_ptr(), w, h, 0, n)
    r.render_stats_device(comp, b.data_ptr(), w, h, 0, n)
    torch.cuda.synchronize()
    assert torch.equal(a, b)


# --- refusals and caches ---------------------------------------------------------------------------------


def _raw_call(cuda_api, r, comp, s, w, h, rgba_ptr=None):
    ch, cc = (C.c_uint32 * 4)(*RGBA), (C.c_float * 4)(1.0, 1.0, 1.0, 0.0)
    return cuda_api.renderer_render_stats_device(r._h, comp._h, C.byref(s) if s is not None else None, w, h, None,
                                                 None if rgba_ptr is None else C.c_void_p(rgba_ptr), 4 * w, ch, cc, None)


def test_refusals_write_nothing(cuda_api):
    import torch
    w, h = 64, 64
    comp = cuda_api.Composition()
    scenes.E2E["clipping"](cuda_api, comp)
    r = cuda_api.Renderer(0)
    t = records(1, 4)
    rgba = _rgba(1, w, h)
    good = dict(ptr=t.data_ptr(), first_order=0, n_orders=4, min_coverage=0.0)
    cases = [dict(ptr=None), dict(ptr=t.data_ptr() + 4), dict(n_orders=0), dict(first_order=(1 << 21) - 3),
             dict(min_coverage=float("nan")), dict(min_coverage=float("inf")), dict(min_coverage=-0.5), dict(min_coverage=1.0)]
    for case in cases:
        args = {**good, **case}
        s = _CStats(args["ptr"], args["first_order"], args["n_orders"], args["min_coverage"])
        assert _raw_call(cuda_api, r, comp, s, w, h, rgba.data_ptr()) == 1, case
    assert _raw_call(cuda_api, r, comp, None, w, h, rgba.data_ptr()) == 1
    s = _CStats(t.data_ptr(), 0, 4, 0.0)
    assert _raw_call(cuda_api, r, comp, s, 0, h) == 1
    assert _raw_call(cuda_api, r, comp, s, w, 1 << 20) == 1
    views = np.array([[1, 0, 0, 1, 0, 0]], np.float32)
    vp = views.ctypes.data_as(C.POINTER(C.c_float))
    for n in (0, 5000):  # no views, more than max_views(h)
        assert cuda_api.renderer_render_views_stats_device(r._h, comp._h, vp, n, C.byref(s), w, h, None, 0, 0, None, None, None) == 1
    comps = (C.c_void_p * 1)(None)
    assert cuda_api.renderer_render_batch_stats_device(r._h, comps, 1, C.byref(s), w, h, None, 0, 0, None, None, None) == 1
    torch.cuda.synchronize()
    assert bool(torch.all(t == SENTINEL)) and bool(torch.all(rgba == 0xA5))


def test_layer_cache_untouched(cuda_api):
    import torch
    w, h = 256, 160
    comp = cuda_api.Composition()
    synth.random_mixed(cuda_api, comp, 120, w, h, 12)
    r = cuda_api.Renderer(0)
    cache = r.create_buffer_layer_cache()
    a, b, c = _rgba(1, w, h), _rgba(1, w, h), _rgba(1, w, h)
    r.render_device(comp, a.data_ptr(), w, h, RGBA, CLEAR, layer_cache=cache)
    device_stats(r, comp, w, h, 0, 20)
    r.render_stats(comp, w, h, 0, 20, 0.5)
    b.copy_(a)
    r.render_device(comp, b.data_ptr(), w, h, RGBA, CLEAR, layer_cache=cache)  # nothing changed: the cache skips every tile
    r.render_device(comp, c.data_ptr(), w, h, RGBA, CLEAR)
    torch.cuda.synchronize()
    assert torch.equal(a, c) and torch.equal(b, c)


def test_cli_stats(cuda_api, tmp_path):
    from forma_b200 import svg
    svg_path = os.path.join(ROOT, "tests", "golden", "paris30k_excerpt.svg")
    out, path = tmp_path / "out.ppm", tmp_path / "stats.npz"
    comp = cuda_api.Composition()
    svg.compose(cuda_api, comp, svg.parse_svg(svg_path))
    n = n_orders(comp)
    for extra, first, k, threshold in (([], 0, n, 0.0), (["--stats-orders", "3:40", "--stats-min-coverage", "0.5"], 3, 37, 0.5)):
        subprocess.check_call([sys.executable, "-m", "forma_b200.render", svg_path, str(out), "--width", "400", "--height", "300",
                               "--stats", str(path)] + extra, cwd=ROOT)
        got = np.load(path)
        want = cuda_api.Renderer(0).render_stats(comp, 400, 300, first, k, threshold)
        assert int(got["first_order"]) == first
        for name in ("area", "pixels", "visible", "box", "visible_box"):
            assert np.array_equal(got[name], want[name]), name
        assert got["visible"].any()
