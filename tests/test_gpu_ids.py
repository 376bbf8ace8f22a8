"""ID frames on the device (paint_ids_kernel) against the oracle's ID frames, at tolerance 0:
the e2e scenes, random_mixed with crops and padded strides in host and device memory, every
scene of tests/extremes.py, paris4k and cubics100k at full size; the combined RGBA + ID call
against the two separate calls; both table modes and the sync-free redo; layer caches around
an ID frame; and the CLI's --ids."""
import os
import subprocess
import sys

import numpy as np
import pytest

import extremes
import oracle_ids
import scenes
import synth
import workloads
from forma_b200.binding import ID_NONE, RGBA, Color, Rect

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLEAR = Color(1.0, 1.0, 1.0, 0.0)


@pytest.fixture(autouse=True)
def _oracle_ids(oracle_api):
    oracle_ids.attach(oracle_api)


def host_ids(api, comp, w, h, renderer=None, **kw):
    r = renderer if renderer is not None else api.Renderer(0)
    ids = np.zeros(w * h, np.uint32)
    r.render_ids(comp, ids, w, h, **kw)
    return ids.reshape(h, w)


def device_ids(r, comp, w, h, **kw):
    import torch
    t = torch.zeros(w * h, dtype=torch.int32, device="cuda:0")
    r.render_ids_device(comp, t.data_ptr(), w, h, **kw)
    torch.cuda.synchronize()
    return t.cpu().numpy().view(np.uint32).reshape(h, w)


def assert_same(got, want, what):
    if np.array_equal(got, want):
        return
    ys, xs = np.nonzero(got != want)
    raise AssertionError(f"{what}: {len(ys)} pixels differ, first at x={xs[0]} y={ys[0]}: "
                         f"cuda {int(got[ys[0], xs[0]]):#x} oracle {int(want[ys[0], xs[0]]):#x}")


@pytest.mark.parametrize("min_coverage", [0.0, 0.5])
@pytest.mark.parametrize("name", list(scenes.E2E))
def test_e2e_scene_ids(cuda_api, oracle_api, cuda_renderer, name, min_coverage):
    got, want = [], []
    for api, out in ((cuda_api, got), (oracle_api, want)):
        comp = api.Composition()
        scenes.E2E[name](api, comp)
        out.append(host_ids(api, comp, 64, 64, cuda_renderer if api is cuda_api else None, min_coverage=min_coverage))
    assert_same(got[0], want[0], name)


@pytest.mark.parametrize("where", ["host", "device"])
def test_random_mixed_1080p_crop_and_stride(cuda_api, oracle_api, where):
    import torch
    w, h = 1920, 1080
    comps = {}
    for api in (cuda_api, oracle_api):
        comps[api] = api.Composition()
        synth.random_mixed(api, comps[api], 400, w, h, 7)
    want = host_ids(oracle_api, comps[oracle_api], w, h)
    r = cuda_api.Renderer(0)
    assert_same(host_ids(cuda_api, comps[cuda_api], w, h, r) if where == "host" else device_ids(r, comps[cuda_api], w, h),
                want, f"uncropped, {where}")
    crop = Rect((100, 1333), (37, 700))  # tiles 6..83 x 2..43
    for pad in (64, 4):  # 16-byte rows (vector stores), then 4-byte rows (scalar stores)
        stride = 4 * w + pad
        n = h * stride // 4
        if where == "host":
            buf = np.full(n, 0xDEADBEEF, np.uint32)
            r.render_ids(comps[cuda_api], buf, w, h, crop=crop, stride=stride, min_coverage=0.25)
        else:
            t = torch.full((n,), -559038737, dtype=torch.int32, device="cuda:0")
            r.render_ids_device(comps[cuda_api], t.data_ptr(), w, h, crop=crop, stride=stride, min_coverage=0.25)
            torch.cuda.synchronize()
            buf = t.cpu().numpy().view(np.uint32)
        ref = np.full(n, 0xDEADBEEF, np.uint32)
        oracle_api.Renderer(0).render_ids(comps[oracle_api], ref, w, h, crop=crop, stride=stride, min_coverage=0.25)
        assert_same(buf.reshape(h, stride // 4), ref.reshape(h, stride // 4), f"crop, pad {pad}, {where}")
        grid = buf.reshape(h, stride // 4)
        assert (grid[:32] == 0xDEADBEEF).all() and (grid[:, w:] == 0xDEADBEEF).all()


@pytest.fixture(scope="module")
def extreme_ids(oracle_api):
    memo = {}

    def get(name):
        if name not in memo:
            comp, built, sc = extremes.build(oracle_api, name)
            memo.clear()
            memo[name] = host_ids(oracle_api, comp, sc.width, sc.height, crop=sc.crop)
        return memo[name]
    return get


@pytest.mark.parametrize("name", list(extremes.SCENES))
def test_extreme_scene_ids(cuda_api, extreme_ids, name):
    comp, built, sc = extremes.build(cuda_api, name)
    r = cuda_api.Renderer(0)
    want = extreme_ids(name)
    for frame in range(2):  # counted tables, then sync-free
        got = np.zeros((sc.height, sc.width), np.uint32)
        r.render_ids(comp, got.reshape(-1), sc.width, sc.height, crop=sc.crop)
        assert_same(got, want, f"{name} frame {frame + 1}")
    assert r.counters()["tables_mode"] == 1


@pytest.mark.parametrize("name", ["paris4k", "cubics100k"])
def test_workload_ids_full_size(cuda_api, oracle_api, name):
    comp, w, h = workloads.build_scene(cuda_api, name)
    ocomp, _, _ = workloads.build_scene(oracle_api, name)
    assert_same(host_ids(cuda_api, comp, w, h), host_ids(oracle_api, ocomp, w, h), name)


@pytest.mark.parametrize("name", [n for n, s in extremes.SCENES.items() if "crowd" in s.tags] + ["paris4k"])
def test_rgba_with_ids_equals_the_separate_calls(cuda_api, name):
    import torch
    if name == "paris4k":
        comp, w, h = workloads.build_scene(cuda_api, name)
        crop = None
    else:
        comp, _, sc = extremes.build(cuda_api, name)
        w, h, crop = sc.width, sc.height, sc.crop
    r = cuda_api.Renderer(0)
    rgba = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda:0")
    r.render_device(comp, rgba.data_ptr(), w, h, RGBA, CLEAR, crop)
    ids = device_ids(r, comp, w, h, crop=crop)
    want_rgba = rgba.cpu().numpy()
    for frame in range(2):
        rgba2 = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda:0")
        ids2 = torch.zeros(w * h, dtype=torch.int32, device="cuda:0")
        r.render_device_with_ids(comp, rgba2.data_ptr(), ids2.data_ptr(), w, h, RGBA, CLEAR, crop)
        torch.cuda.synchronize()
        assert np.array_equal(rgba2.cpu().numpy(), want_rgba), f"{name}: RGBA frame differs from render_device's"
        assert_same(ids2.cpu().numpy().view(np.uint32).reshape(h, w), ids, f"{name} frame {frame + 1}")


@pytest.fixture()
def options_restored(cuda_api):
    saved = {k: cuda_api.get_option(k) for k in ("sync_free", "test_fast_shrink")}
    yield
    for k, v in saved.items():
        cuda_api.set_option(k, v)


def test_ids_in_every_table_mode(cuda_api, oracle_api, options_restored):
    w, h = 1920, 1080
    comp, ocomp = cuda_api.Composition(), oracle_api.Composition()
    synth.random_mixed(cuda_api, comp, 2000, w, h, 9)
    synth.random_mixed(oracle_api, ocomp, 2000, w, h, 9)
    want = host_ids(oracle_api, ocomp, w, h)
    r = cuda_api.Renderer(0)
    for sync_free, shrink, mode in ((0, 0, 0), (1, 0, 1), (1, 1, 2)):
        cuda_api.set_option("sync_free", sync_free)
        cuda_api.set_option("test_fast_shrink", shrink)
        assert_same(device_ids(r, comp, w, h), want, f"sync_free {sync_free} shrink {shrink}")
        c = r.counters()
        assert c["tables_mode"] == mode, (sync_free, shrink, c)
        assert c["segments"] > 0 and c["cells"] > 0 and c["entries"] >= c["cells"]


def test_ids_between_cached_frames(cuda_api, oracle_api):
    w, h = 640, 360
    sides = []
    for api in (cuda_api, oracle_api):
        comp = api.Composition()
        synth.random_mixed(api, comp, 300, w, h, 5)
        r = api.Renderer(0)
        sides.append((api, comp, r, r.create_buffer_layer_cache()))
    bufs = [np.zeros(w * h * 4, np.uint8) for _ in sides]
    for (api, comp, r, cache), buf in zip(sides, bufs):
        r.render(comp, buf, w, h, RGBA, CLEAR, None, cache)
    assert np.array_equal(bufs[0], bufs[1])
    ids = [host_ids(api, comp, w, h, r) for api, comp, r, cache in sides]
    assert_same(ids[0], ids[1], "IDs between cached frames")
    for (api, comp, r, cache), buf in zip(sides, bufs):
        r.render(comp, buf, w, h, RGBA, CLEAR, None, cache)
    assert sides[0][2].counters()["written_tiles"] == 0
    assert np.array_equal(bufs[0], bufs[1])


def test_cli_ids(cuda_api, tmp_path):
    svg_path = os.path.join(ROOT, "tests", "golden", "paris30k_excerpt.svg")
    out, npy = tmp_path / "out.ppm", tmp_path / "ids.npy"
    subprocess.check_call([sys.executable, "-m", "forma_b200.render", svg_path, str(out), "--width", "400", "--height", "300",
                           "--ids", str(npy)], cwd=ROOT)
    got = np.load(npy)
    assert got.shape == (300, 400) and got.dtype == np.uint32
    from forma_b200 import svg
    comp = cuda_api.Composition()
    svg.compose(cuda_api, comp, svg.parse_svg(svg_path))
    want = host_ids(cuda_api, comp, 400, 300)
    assert np.array_equal(got, want)
    assert (got != ID_NONE).any()
