"""Chained launches (option pdl) change when a kernel's CTAs start, never what they compute: every
frame kind rendered with pdl 0 and pdl 1 is byte for byte the same, with the same launch count, on
paris@4K, 100k cubics and a mixed synthetic scene. Also covered: a sync-free frame forced through
its redo, and frames alternating between two compositions of very different size."""
import numpy as np
import pytest

import synth
from forma_b200.binding import RGBA, Color, Poses
from workloads import build_scene

pytestmark = pytest.mark.gpu

CLEAR = Color(1.0, 1.0, 1.0, 0.0)
SCENES = ("paris4k", "cubics100k", "mixed")
KINDS = ("single", "host", "views", "batch", "poses", "ids", "masks", "stats", "over", "linear", "cache")


def _build(api, name):
    if name == "mixed":
        comp = api.Composition()
        synth.random_mixed(api, comp, 900, 1280, 720, 31)
        return comp, 1280, 720
    return build_scene(api, name)


@pytest.fixture(scope="module")
def scenes(cuda_api):
    return {}


@pytest.fixture()
def restore_pdl(cuda_api):
    saved = {n: cuda_api.get_option(n) for n in ("pdl", "test_fast_shrink", "sync_free")}
    yield
    for n, v in saved.items():
        cuda_api.set_option(n, v)


def _scene(cuda_api, scenes, name):
    """The scene, its geometry made resident by two frames of a renderer of its own, so that the
    launch counts of both arms exclude the composition's one-time uploads."""
    if name not in scenes:
        import torch
        comp, w, h = _build(cuda_api, name)
        r = cuda_api.Renderer(0)
        t = torch.zeros(h * w * 4, dtype=torch.uint8, device="cuda:0")
        for _ in range(2):
            r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR, timings=False)
        torch.cuda.synchronize()
        scenes[name] = (comp, w, h)
    return scenes[name]


def _frames(api, kind, comp, w, h):
    """Two frames of `kind` from a fresh renderer (the second one sync-free where the kind allows it):
    the bytes of both and the launches they took."""
    import torch
    r = api.Renderer(0)
    dev = torch.device("cuda", 0)
    out, launches = [], []
    cache = r.create_buffer_layer_cache() if kind == "cache" else None
    vw, vh = min(w, 960), min(h, 540)  # stacked kinds: frames of at most 960 x 540
    views = np.array([[1, 0, 0, 1, 0, 0], [1, 0, 0, 1, -vw * 0.5, -vh * 0.25], [1, 0, 0, 1, -vw, -vh * 0.5]], np.float32)
    for step in range(2):
        c0 = r.counters()["launches"]
        if kind == "host":
            buf = np.zeros(w * h * 4, np.uint8)
            r.render(comp, buf, w, h, RGBA, CLEAR, timings=False)
            out.append(buf.tobytes())
        else:
            if kind in ("single", "cache"):
                t = torch.zeros(h * w * 4, dtype=torch.uint8, device=dev)
                if kind == "cache" and step == 1:  # a cached frame rewrites only the tiles that changed: none here
                    t[:] = torch.as_tensor(np.frombuffer(out[0], np.uint8).copy(), device=dev)
                r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR, None, cache, timings=False)
            elif kind == "views":
                t = torch.zeros(len(views) * vh * vw * 4, dtype=torch.uint8, device=dev)
                r.render_views_device(comp, views, t.data_ptr(), vw, vh, RGBA, CLEAR, timings=False)
            elif kind == "batch":
                t = torch.zeros(3 * vh * vw * 4, dtype=torch.uint8, device=dev)
                r.render_batch_device([comp, comp, comp], t.data_ptr(), vw, vh, RGBA, CLEAR, timings=False)
            elif kind == "poses":
                k = 8
                xf = np.tile(np.array([1, 0, 0, 1, 0, 0], np.float32), (2, k, 1))
                xf[1, :, 4] = 13.0
                vis = np.ones((2, k), np.uint8)
                vis[0, ::3] = 0
                t = torch.zeros(2 * vh * vw * 4, dtype=torch.uint8, device=dev)
                r.render_poses_device(comp, Poses(0, xf, vis), t.data_ptr(), vw, vh, RGBA, CLEAR, timings=False)
            elif kind == "ids":
                t = torch.zeros(h * w, dtype=torch.int32, device=dev)
                r.render_ids_device(comp, t.data_ptr(), w, h, timings=False)
            elif kind == "masks":
                t = torch.zeros(4 * vh * vw, dtype=torch.float32, device=dev)
                r.render_masks_device(comp, t.data_ptr(), vw, vh, 0, 4, timings=False)
            elif kind == "stats":
                t = torch.zeros(64 * 12, dtype=torch.int32, device=dev)
                r.render_stats_device(comp, t.data_ptr(), w, h, 0, 64, timings=False)
            elif kind == "over":
                g = torch.Generator(device="cpu").manual_seed(5)
                t = torch.randint(0, 256, (h * w * 4,), dtype=torch.uint8, generator=g).to(dev)
                r.render_over_device(comp, t.data_ptr(), w, h, timings=False)
            elif kind == "linear":
                t = torch.zeros(h * w * 4, dtype=torch.float16, device=dev)
                r.render_linear_device(comp, t.data_ptr(), w, h, RGBA, CLEAR, format="f16", timings=False)
            torch.cuda.synchronize()
            out.append(t.cpu().numpy().tobytes())
        launches.append(r.counters()["launches"] - c0)
    return out, launches


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("scene", SCENES)
def test_chained_launches_keep_every_frame(cuda_api, scenes, restore_pdl, scene, kind):
    comp, w, h = _scene(cuda_api, scenes, scene)
    got = {}
    for pdl in (0, 1):
        cuda_api.set_option("pdl", pdl)
        got[pdl] = _frames(cuda_api, kind, comp, w, h)
    (plain, n0), (chained, n1) = got[0], got[1]
    for step in range(2):
        assert plain[step] == chained[step], f"{scene} {kind}: frame {step} differs between pdl 0 and pdl 1"
    assert n0 == n1, f"{scene} {kind}: launches {n0} with pdl 0, {n1} with pdl 1"


@pytest.mark.parametrize("scene", SCENES)
def test_sync_free_redo_with_chained_launches(cuda_api, scenes, restore_pdl, scene):
    """test_fast_shrink halves the sync-free bounds: the first attempt's tables overflow, and the
    frame is redone with counted tables. Chained, it must still equal the plain frame."""
    comp, w, h = _scene(cuda_api, scenes, scene)
    cuda_api.set_option("pdl", 0)
    plain, _ = _frames(cuda_api, "single", comp, w, h)
    cuda_api.set_option("pdl", 1)
    cuda_api.set_option("test_fast_shrink", 1)
    import torch
    r = cuda_api.Renderer(0)
    for step in range(3):
        t = torch.zeros(h * w * 4, dtype=torch.uint8, device="cuda:0")
        r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR, timings=False)
        torch.cuda.synchronize()
        assert t.cpu().numpy().tobytes() == plain[min(step, 1)], f"{scene}: frame {step} differs"
    if scene != "mixed":
        assert r.counters()["tables_mode"] == 2, "the last frame was not redone"


def test_alternating_compositions_with_chained_launches(cuda_api, restore_pdl):
    """A large and a small composition in turn on one renderer: every sync-free frame starts from the
    other composition's bounds (too large, then too small)."""
    import torch
    big, bw, bh = _build(cuda_api, "cubics100k")
    small = cuda_api.Composition()
    synth.random_mixed(cuda_api, small, 60, bw, bh, 9)
    frames = {}
    for pdl in (0, 1):
        cuda_api.set_option("pdl", pdl)
        r = cuda_api.Renderer(0)
        seq = []
        for step in range(6):
            comp = big if step % 2 == 0 else small
            t = torch.zeros(bh * bw * 4, dtype=torch.uint8, device="cuda:0")
            r.render_device(comp, t.data_ptr(), bw, bh, RGBA, CLEAR, timings=False)
            torch.cuda.synchronize()
            seq.append(t.cpu().numpy().tobytes())
        frames[pdl] = seq
    for step in range(6):
        assert frames[0][step] == frames[1][step], f"frame {step} differs between pdl 0 and pdl 1"
    assert frames[1][0] == frames[1][2] == frames[1][4] and frames[1][1] == frames[1][3] == frames[1][5]
