"""Single device frames on the sync_free_sort path (DESIGN.md section 3, "Host/device overlap"):
the segment sort, the painter tables and the paint are launched over the previous frame's segment
count and sort plan, without reading the count back. Every comparison is at tolerance 0 against
the same frames with the count read back (sync_free_sort 0), on a renderer of its own:

- frames, sorted segments, row costs and counters() over consecutive frames, with pdl 0 and 1,
  on paris@4K, cubics100k, a crop band, a mixed-style scene and linear and over frames;
- the redo: a bound forced just below, at and just above the count (test_sort_bound), scenes that
  grow and shrink, and a scene whose tile columns outgrow the previous frame's plan;
- the refusal: a frame over 2^30 segments after an in-limit one is refused with the read-back
  path's message and leaves the caller's buffer as it was; the next frame is right.
"""
import numpy as np
import pytest

import line_scenes as ls
import synth
from forma_b200.binding import RGBA, Color, FormaError, Rect
from workloads import build_scene

pytestmark = pytest.mark.gpu

CLEAR = Color(1.0, 1.0, 1.0, 0.0)
NAMES = ("sync_free_sort", "test_sort_bound", "pdl", "sort_big_log2", "sort_scan_log2", "sync_free")


@pytest.fixture()
def opts(cuda_api):
    saved = {n: cuda_api.get_option(n) for n in NAMES}

    def set_(**kw):
        for k, v in kw.items():
            cuda_api.set_option(k, v)
    yield set_
    for n, v in saved.items():
        cuda_api.set_option(n, v)


def _torch():
    import torch
    return torch


class Pair:
    """The same frames on two renderers: `ref` with the count read back, `dev` on the bounds. Each
    draws its own compositions (residency is per device: a shared one would be uploaded once)."""

    def __init__(self, api, opts):
        self.api, self.opts = api, opts
        self.ref, self.dev = api.Renderer(0), api.Renderer(0)

    def frame(self, comps, w, h, draw=None, nbytes=None, fill=0):
        torch = _torch()
        out = []
        for mode, r, comp in ((0, self.ref, comps[0]), (1, self.dev, comps[1])):
            self.opts(sync_free_sort=mode)
            t = torch.full((nbytes or w * h * 4,), fill, dtype=torch.uint8, device="cuda:0")
            (draw or (lambda r, comp, ptr: r.render_device(comp, ptr, w, h, RGBA, CLEAR)))(r, comp, t.data_ptr())
            torch.cuda.synchronize()
            out.append(t.cpu().numpy())
        return out

    def same(self, what, got, want):
        assert np.array_equal(got, want), f"{what}: the frame on bounds differs from the read-back frame"
        assert np.array_equal(self.dev.segments(), self.ref.segments()), f"{what}: sorted segments differ"
        assert np.array_equal(self.dev.row_costs(), self.ref.row_costs()), f"{what}: row costs differ"
        assert self.dev.sort_bounds() == self.ref.sort_bounds(), what


def _mixed(api, w, h):
    comp = api.Composition()
    synth.random_mixed(api, comp, 900, w, h, 31)
    return comp


@pytest.mark.parametrize("pdl", [0, 1])
@pytest.mark.parametrize("scene", ["paris4k", "cubics100k", "paris4k_band", "mixed", "linear", "over"])
def test_frames_on_bounds_equal_the_read_back_frames(cuda_api, opts, scene, pdl):
    opts(pdl=pdl, sort_big_log2=12, sort_scan_log2=12)
    p = Pair(cuda_api, opts)
    draw, nbytes = None, None
    if scene in ("paris4k", "cubics100k", "paris4k_band"):
        comps = [build_scene(cuda_api, scene.replace("_band", "")) for _ in range(2)]
        w, h = comps[0][1], comps[0][2]
        comps = [c[0] for c in comps]
        if scene == "paris4k_band":  # the rows one GPU of four paints (the multi-GPU bench's crop)
            crop = Rect((0, w), (544, 1088))
            draw = lambda r, comp, ptr: r.render_device(comp, ptr, w, h, RGBA, CLEAR, crop)
    else:
        w, h = 1280, 720
        comps = [_mixed(cuda_api, w, h) for _ in range(2)]
        if scene == "linear":
            draw, nbytes = (lambda r, comp, ptr: r.render_linear_device(comp, ptr, w, h, RGBA, CLEAR, format="f16")), w * h * 8
        elif scene == "over":
            draw = lambda r, comp, ptr: r.render_over_device(comp, ptr, w, h, RGBA)
    for k in range(4):
        want, got = p.frame(comps, w, h, draw, nbytes, fill=77)
        p.same(f"{scene} frame {k}", got, want)
        assert p.ref.sort_mode() == 0
        assert p.dev.sort_mode() == (1 if k else 0), (scene, k)  # frame 0 has no previous count
        assert p.dev.counters() == p.ref.counters(), (scene, k)
        assert p.dev.stage_times().keys() == p.ref.stage_times().keys()
        assert p.dev.kernel_times().keys() == p.ref.kernel_times().keys()
        assert {k: v["launches"] for k, v in p.dev.kernel_times().items()} == \
            {k: v["launches"] for k, v in p.ref.kernel_times().items()}


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_a_bound_just_below_at_and_above_the_count(cuda_api, opts, delta):
    """test_sort_bound puts the bound at n - 1, n and n + 1: the count lands above it (redone,
    sort_mode 2), on it and below it (sort_mode 1). The frame is the read-back path's each time."""
    opts(sort_big_log2=12, sort_scan_log2=12)
    w, h = 1280, 720
    comps = [_mixed(cuda_api, w, h) for _ in range(2)]
    p = Pair(cuda_api, opts)
    want, got = p.frame(comps, w, h)
    n = p.ref.counters()["segments"]
    assert n > 20000
    opts(test_sort_bound=n + delta)
    for k in range(2):
        want, got = p.frame(comps, w, h, fill=5)
        p.same(f"bound n{delta:+d}", got, want)
        assert p.dev.sort_mode() == (2 if delta < 0 else 1), (delta, k)
        assert p.dev.counters()["segments"] == n


def test_scenes_that_grow_shrink_and_move(cuda_api, opts):
    """One pair of renderers, scenes of very different sizes and extents one after the other: a
    count far above the bound, one far below the floor of the bounds' sort, and tile columns
    beyond the previous frame's plan are all redone; the rest stay on the bounds."""
    opts(sort_big_log2=12, sort_scan_log2=12)
    w, h = 4096, 720

    def two(n, width, seed):
        out = []
        for _ in range(2):
            c = cuda_api.Composition()
            synth.random_mixed(cuda_api, c, n, width, h, seed)
            out.append(c)
        return out
    small, large, left = two(200, w, 3), two(3000, w, 4), two(3000, 900, 5)  # `left`: tile columns below 128
    p = Pair(cuda_api, opts)
    seq = [(large, None), (large, 1), (small, None), (large, 2), (large, 1), (left, 2), (left, 1), (large, 2), (large, 1)]
    for k, (comps, mode) in enumerate(seq):
        want, got = p.frame(comps, w, h, fill=k)
        p.same(f"step {k}", got, want)
        if mode is not None:
            assert p.dev.sort_mode() == mode, (k, p.dev.sort_mode(), p.dev.counters())


def test_an_over_limit_frame_is_refused_and_writes_nothing(cuda_api, opts):
    torch = _torch()
    opts(sort_big_log2=12, sort_scan_log2=12)
    name = ls.OVER_LIMIT[0]
    sc = ls.SCENES[name]
    w, h = ls.W, ls.H
    rs = {}
    for mode in (0, 1):
        opts(sync_free_sort=mode)
        comp = cuda_api.Composition()
        synth.random_mixed(cuda_api, comp, 100, w, h, 9)  # (orders 0..99, inserted in order)
        r = cuda_api.Renderer(0)
        t = torch.zeros(h * w * 4, dtype=torch.uint8, device="cuda:0")
        for _ in range(3):
            r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR)
        torch.cuda.synchronize()
        assert r.sort_mode() == mode
        layer = comp.get_mut_or_insert_default(1000)  # (still in layer order: the sort plan stays)
        for spec in sc.layers:
            for pts in spec.paths:
                layer.insert(ls.build_path(cuda_api, pts))
            if spec.xf is not None:
                layer.set_transform(spec.xf)
        t.fill_(0xA5)
        with pytest.raises(FormaError):
            r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR)
        torch.cuda.synchronize()
        assert bool((t == 0xA5).all()), f"sync_free_sort {mode}: a refused frame wrote to the buffer"
        assert r.sort_mode() == mode  # (the frame was attempted on the bounds)
        assert r.counters()["segments"] == 0 and r.segments().size == 0 and r.row_costs().size == 0
        rs[mode] = (cuda_api.last_error().decode(), comp, r)
    assert rs[1][0] == rs[0][0] and "exceed" in rs[1][0]
    # Back in limit: the next frames equal the read-back path's.
    for mode in (0, 1):
        rs[mode][1].get(1000).disable()
    for k in range(2):
        frames = []
        for mode in (0, 1):
            opts(sync_free_sort=mode)
            t = torch.zeros(h * w * 4, dtype=torch.uint8, device="cuda:0")
            rs[mode][2].render_device(rs[mode][1], t.data_ptr(), w, h, RGBA, CLEAR)
            torch.cuda.synchronize()
            frames.append(t.cpu().numpy())
        assert np.array_equal(frames[0], frames[1]), f"frame {k} after the refusal"
