"""The segment sort's per-tile digit counts from the kernels that write its keys (option sort_counts):
the emit pass counts pass 0 (ahead of the count read-back with the previous frame's digit, or after
it with the plan's own), every downsweep the pass after it, and an upsweep pass 0 when neither
applies.

- Counts: the counts every pass was given equal a NumPy bincount per 4096-key tile of that pass's
  input keys (the emitted segments, stably sorted by the digits of the passes before it).
- Speculation outcomes, asserted through Renderer.sort_counts()["source"]: first frame, plan
  unchanged, plan changed (sort_full_key, a larger extent), no speculation, segments beyond
  the speculative capacity, a frame below the reduce-then-scan threshold, 1-, 2- and >= 3-pass plans,
  a sync-free tables redo and two renderers on one device.
- Results: the sorted segments and the frames equal those with sort_counts 0, for single frames,
  views and batches, and the oracle's.
- Launches: a sync-free frame launches the table chain around the rasterizer and a sort of 3
  launches per pass: chunk totals (from the producers' tile counts), tile scan and downsweep, or with
  sort_counts 0 upsweep, tile scan and downsweep.
"""
import numpy as np
import pytest
import torch

import synth
import workloads
from forma_b200.binding import RGBA, Color

CLEAR = Color(1.0, 1.0, 1.0, 0.0)
TILE = 4096
WIDE = {"sort_big_log2": 10, "sort_scan_log2": 10}  # reduce-then-scan passes from 1024 keys on
NAMES = ("sort_counts", "sort_big_log2", "sort_scan_log2", "sort_full_key", "speculate", "sync_free", "test_fast_shrink",
         "host_slices")


@pytest.fixture()
def opts(cuda_api):
    saved = {n: cuda_api.get_option(n) for n in NAMES}
    cuda_api.set_option("host_slices", 1)

    def setter(**kw):
        for k, v in kw.items():
            cuda_api.set_option(k, v)

    yield setter
    for n, v in saved.items():
        cuda_api.set_option(n, v)


def _plan(api, r):
    b = r.sort_bounds()
    raw = api.sort_plan(0, [b["layer"], b["tile_x"], b["tile_y"]])
    specs = []
    for p in range(raw[0]):
        d = raw[2 + 10 * p: 12 + 10 * p]
        specs.append([(d[k], d[3 + k], d[6 + k]) for k in range(3)])
    return specs


def _digits(keys, spec):
    v = np.zeros(keys.size, np.uint64)
    for shift, width, lsh in spec:
        if width:
            v |= ((keys >> np.uint64(shift)) & np.uint64((1 << width) - 1)) << np.uint64(lsh)
    return v.astype(np.int64)


def _expected_counts(keys, specs):
    """[passes, tiles, 256]: per pass, the digit counts per 4096-key tile of its input."""
    tiles = (keys.size + TILE - 1) // TILE
    out = np.zeros((len(specs), tiles, 256), np.uint32)
    cur = keys
    for p, spec in enumerate(specs):
        d = _digits(cur, spec)
        t = np.arange(cur.size) // TILE
        out[p] = np.bincount(t * 256 + d, minlength=tiles * 256).reshape(tiles, 256)
        cur = cur[np.argsort(d, kind="stable")]
    return out, cur


def _frame(r, comp, w, h, crop=None):
    fb = torch.zeros(h * w * 4, dtype=torch.uint8, device="cuda:0")
    r.render_device(comp, fb.data_ptr(), w, h, RGBA, CLEAR, crop=crop)
    torch.cuda.synchronize()
    return fb.cpu().numpy()


def _check_counts(api, r, comp, w, h):
    """The kept counts of the last frame against the emitted segments' (rasterize_only re-runs line
    setup for the same frame; the segments are the same), and the sorted output."""
    sc = r.sort_counts()
    assert sc["source"] != "none"
    specs = _plan(api, r)
    sorted_keys = r.segments()
    emitted = r.rasterize_only(comp, w, h)
    exp, final = _expected_counts(emitted, specs)
    assert sc["counts"].shape == exp.shape
    for p in range(len(specs)):
        assert np.array_equal(sc["counts"][p], exp[p]), f"pass {p} ({sc['source']})"
    assert np.array_equal(sorted_keys, final)
    return sc


def _scene(api, n_layers, w, h, seed):
    comp = api.Composition()
    synth.random_mixed(api, comp, n_layers, w, h, seed)
    return comp


@pytest.mark.gpu
def test_speculation_outcomes_and_counts(cuda_api, opts):
    opts(sort_counts=1, speculate=1, **WIDE)
    w, h = 640, 360
    comp = _scene(cuda_api, 300, w, h, 11)
    r = cuda_api.Renderer(0)
    r.sort_counts(keep=1)
    seen = []

    def frame(**kw):
        img = _frame(r, comp, w, h, **kw)
        sc = _check_counts(cuda_api, r, comp, w, h)
        seen.append(sc["source"])
        # rasterize_only ran line setup again: the next frame sees its digit as the previous one
        return img, sc["source"]

    _, s = frame()
    assert s in ("emit", "upsweep")  # first frame: nothing to speculate with
    _, s = frame()
    assert s == "speculative_emit"  # plan unchanged
    opts(sort_full_key=1)  # the layer digits join the plan: pass 0 is the layer digit now
    _, s = frame()
    assert s == "upsweep"
    _, s = frame()
    assert s == "speculative_emit"
    opts(sort_full_key=0)
    _, s = frame()
    assert s == "upsweep"
    opts(speculate=0)
    _, s = frame()
    assert s == "emit"
    opts(speculate=1)
    big = _scene(cuda_api, 3000, w, h, 12)  # more segments than the speculative capacity
    r.render_device(big, torch.zeros(h * w * 4, dtype=torch.uint8, device="cuda:0").data_ptr(), w, h, RGBA, CLEAR)
    torch.cuda.synchronize()
    sc = _check_counts(cuda_api, r, big, w, h)
    assert sc["source"] == "emit"
    opts(sort_scan_log2=30)  # below the reduce-then-scan threshold: no tile counts
    _frame(r, comp, w, h)
    assert r.sort_counts()["source"] == "none"
    opts(sort_scan_log2=10)
    _frame(r, comp, w, h)
    assert r.sort_counts()["source"] == "upsweep"  # the frame before had no tile counts


@pytest.mark.gpu
def test_plan_changes_with_extent(cuda_api, opts):
    """A larger frame gives tile_x another bit (pass 0 changes): the speculative counts are taken
    only when pass 0's digit is unchanged."""
    opts(sort_counts=1, **WIDE)
    comp = _scene(cuda_api, 400, 1280, 720, 21)
    r = cuda_api.Renderer(0)
    r.sort_counts(keep=1)
    ref = cuda_api.Renderer(0)
    sources = []
    for w, h in [(640, 360), (640, 360), (1280, 720), (1280, 720), (4000, 720)]:
        img = _frame(r, comp, w, h)
        sources.append(_check_counts(cuda_api, r, comp, w, h)["source"])
        opts(sort_counts=0)
        assert np.array_equal(_frame(ref, comp, w, h), img)
        opts(sort_counts=1)
    # 640 x 360: 6 + 5 key bits, 1280 x 720: 7 + 6 (pass 0 changes), 4000 x 720: 8 + 6, split 7 + 7
    # (pass 0 is the low 7 tile_x bits again: the speculative counts are taken)
    assert sources[1] == sources[3] == sources[4] == "speculative_emit", sources
    assert "speculative_emit" not in (sources[0], sources[2]), sources


@pytest.mark.gpu
@pytest.mark.parametrize("full_key,wh", [(0, (640, 360)), (1, (640, 360)), (0, (7680, 4320)), (1, (7680, 4320))],
                         ids=["2pass", "full_key", "8k", "8k_full_key"])
def test_pass_counts_of_every_plan_shape(cuda_api, opts, full_key, wh):
    """1-pass to >= 3-pass plans (odd and even): every pass's counts, the segments and the frames
    with and without tile counts."""
    opts(sort_counts=1, sort_full_key=full_key, **WIDE)
    w, h = wh
    comp = _scene(cuda_api, 600, w, h, 31)
    r = cuda_api.Renderer(0)
    r.sort_counts(keep=1)
    for _ in range(2):
        img = _frame(r, comp, w, h)
        sc = _check_counts(cuda_api, r, comp, w, h)
    passes = sc["passes"]
    assert passes >= (3 if full_key and w > 4000 else 1)
    img = _frame(r, comp, w, h)  # (rasterize_only left the unsorted segments behind)
    segs = r.segments()
    opts(sort_counts=0)
    r0 = cuda_api.Renderer(0)
    img0 = _frame(r0, comp, w, h)
    assert r0.sort_counts()["source"] == "none"
    assert np.array_equal(r0.segments(), segs)
    assert np.array_equal(img0, img)


@pytest.mark.gpu
@pytest.mark.parametrize("n_layers", [30, 60, 120, 250])
def test_small_plans_and_tile_edges(cuda_api, opts, n_layers):
    """Key counts around the 4096-key tiles (a partial last tile of every size class) and 1-pass
    plans (a frame of a single tile column)."""
    opts(sort_counts=1, **WIDE)
    for w, h in [(16, 256), (256, 256), (333, 97)]:  # 1 pass (7 bits), 2 passes
        comp = _scene(cuda_api, n_layers, w, h, n_layers + w)
        r = cuda_api.Renderer(0)
        r.sort_counts(keep=1)
        for _ in range(2):
            _frame(r, comp, w, h)
            if r.counters()["segments"] >= 1024:
                _check_counts(cuda_api, r, comp, w, h)


@pytest.mark.gpu
def test_two_renderers_and_tables_redo(cuda_api, opts):
    """Two renderers on one device speculate each with its own previous frame; a frame whose
    sync-free tables are redone keeps its sorted segments."""
    opts(sort_counts=1, **WIDE)
    # (scene A is large enough for halved sync-free bounds to be too small: test_fast_shrink redoes its tables)
    a_scene, b_scene = _scene(cuda_api, 2000, 1920, 1080, 41), _scene(cuda_api, 200, 1600, 900, 42)
    ra, rb = cuda_api.Renderer(0), cuda_api.Renderer(0)
    ra.sort_counts(keep=1)
    rb.sort_counts(keep=1)
    for _ in range(3):
        ia = _frame(ra, a_scene, 1920, 1080)
        ib = _frame(rb, b_scene, 1600, 900)
    assert ra.sort_counts()["source"] == "speculative_emit" and rb.sort_counts()["source"] == "speculative_emit"
    _check_counts(cuda_api, ra, a_scene, 1920, 1080)
    _check_counts(cuda_api, rb, b_scene, 1600, 900)
    opts(test_fast_shrink=1)
    redo = _frame(ra, a_scene, 1920, 1080)
    assert ra.counters()["tables_mode"] == 2
    assert np.array_equal(redo, ia)
    opts(test_fast_shrink=0, sort_counts=0)
    r0 = cuda_api.Renderer(0)
    assert np.array_equal(_frame(r0, b_scene, 1600, 900), ib)


@pytest.mark.gpu
def test_views_and_batches_match_without_counts(cuda_api, opts):
    """Views and batches take the same counts (emit of the views / batch kernels): segments and
    frames equal those of sort_counts 0."""
    opts(**WIDE)
    w, h = 480, 272
    comps = [_scene(cuda_api, 150 + 50 * k, w, h, 51 + k) for k in range(3)]
    views = np.array([[1, 0, 0, 1, 0, 0], [1, 0, 0, 1, -40, 12], [0.5, 0, 0, 0.5, 100, 60]], np.float32)
    out = {}
    for v in (1, 0):
        opts(sort_counts=v)
        r = cuda_api.Renderer(0)
        res = []
        for _ in range(3):
            fb = torch.zeros(3 * h * w * 4, dtype=torch.uint8, device="cuda:0")
            r.render_views_device(comps[0], views, fb.data_ptr(), w, h, RGBA, CLEAR)
            torch.cuda.synchronize()
            res.append((fb.cpu().numpy(), r.segments(), r.sort_counts()["source"]))
            fb = torch.zeros(3 * h * w * 4, dtype=torch.uint8, device="cuda:0")
            r.render_batch_device(comps, fb.data_ptr(), w, h, RGBA, CLEAR)
            torch.cuda.synchronize()
            res.append((fb.cpu().numpy(), r.segments(), r.sort_counts()["source"]))
        out[v] = res
    for (f1, s1, src1), (f0, s0, src0) in zip(out[1], out[0]):
        assert src0 == "none" and src1 != "none"
        assert np.array_equal(s1, s0)
        assert np.array_equal(f1, f0)


@pytest.mark.gpu
@pytest.mark.parametrize("workload", ["paris4k", "cubics100k"])
def test_workload_counts_and_segments(cuda_api, opts, workload):
    opts(sort_counts=1)
    comp, w, h = workloads.build_scene(cuda_api, workload)
    r = cuda_api.Renderer(0)
    r.sort_counts(keep=1)
    for _ in range(2):
        img = _frame(r, comp, w, h)
    sc = _check_counts(cuda_api, r, comp, w, h)
    assert sc["source"] == "speculative_emit"
    img = _frame(r, comp, w, h)  # (rasterize_only left the unsorted segments behind)
    segs = r.segments()
    opts(sort_counts=0)
    r0 = cuda_api.Renderer(0)
    assert np.array_equal(_frame(r0, comp, w, h), img)
    assert np.array_equal(r0.segments(), segs)


def _passes(bits: int) -> int:
    return (bits + 7) // 8


VIEWS = np.array([[1, 0, 0, 1, 0, 0], [1, 0, 0, 1, -40, 12], [0.5, 0, 0, 0.5, 100, 60]], np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("sort_counts", [1, 0])
@pytest.mark.parametrize("kind,h,after_tables", [
    ("render_device", 360, 1),
    ("render_ids_device", 360, 1),
    ("render_device_with_ids", 360, 2),  # paint + ID kernel
    ("render_views_device", 352, 1),     # whole tile rows: the views are painted in place
    ("render_views_device", 360, 2),     # paint into the framebuffer + repack
], ids=["rgba", "ids", "rgba_with_ids", "views_in_place", "views_repacked"])
def test_sync_free_frame_launches_the_table_chain(cuda_api, opts, kind, h, after_tables, sort_counts):
    """Segment sort forced onto its reduce-then-scan passes: a resident composition's sync-free
    frame rasterizes with 3 launches (line count, block-sum scan, emit), sorts with 3 launches per
    pass (chunk totals of the tile counts the emit pass and the downsweeps counted, or an upsweep
    with sort_counts 0; tile scan; downsweep), and launches 2 + carry passes + 1 + gap passes + 1
    table kernels and `after_tables` kernels after them."""
    w, layers = 640, 300
    opts(sort_counts=sort_counts, sync_free=1, **WIDE)
    comp = _scene(cuda_api, layers, w, h, 5)
    r = cuda_api.Renderer(0)
    n_views = len(VIEWS) if kind == "render_views_device" else 1
    dev = torch.zeros(n_views * w * h * 4, dtype=torch.uint8, device="cuda:0")
    ids = torch.zeros(w * h, dtype=torch.int32, device="cuda:0")
    render = {
        "render_device": lambda: r.render_device(comp, dev.data_ptr(), w, h, RGBA, CLEAR),
        "render_ids_device": lambda: r.render_ids_device(comp, ids.data_ptr(), w, h),
        "render_device_with_ids": lambda: r.render_device_with_ids(comp, dev.data_ptr(), ids.data_ptr(), w, h, RGBA, CLEAR),
        "render_views_device": lambda: r.render_views_device(comp, VIEWS, dev.data_ptr(), w, h, RGBA, CLEAR),
    }[kind]
    for _ in range(2):
        render()
        torch.cuda.synchronize()
    before = r.counters()["launches"]
    render()
    torch.cuda.synchronize()
    c = r.counters()
    assert c["tables_mode"] == 1
    assert r.sort_counts()["source"] == ("speculative_emit" if sort_counts else "none")
    frame = c["launches"] - before
    sort_passes = r.kernel_times()["radix_downsweep"]["launches"]
    assert sort_passes > 0
    raster = 3
    tiles_x, tiles_y = (w + 15) // 16, n_views * ((h + 15) // 16)
    carry = _passes(int(layers - 1).bit_length())
    gap = _passes(int(tiles_x).bit_length() + int(tiles_y).bit_length())
    tables = 2 + carry + 1 + gap + 1
    assert frame == raster + 3 * sort_passes + tables + after_tables, (frame, raster, sort_passes, tables)
