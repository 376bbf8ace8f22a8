"""The painter tables' kernel chain: cells (+ the carry sort's digit counts), the carry sort, the
carry pass (carry-ins, carry-only entries + the gap sort's digit counts), the gap sort and the
merge (entries, tile ranges, heavy-tile lists).

- Launch pin: a sync-free frame launches exactly that chain, 2 + carry passes + 1 + gap passes
  + 1 kernels, around the rasterizer, the segment sort and the kernels of its kind: RGBA, ID,
  RGBA + ID and view frames (painted in place or repacked).
- Carry groups across the carry pass's CTA tiles (1024 cells): a 32768 px wide frame whose
  (tile_y, layer) groups hold up to 2048 cells, start exactly on CTA tiles, and whose running
  cover empties and refills along the row under both fill rules; cropped inside the groups
  (cells right of the crop reach no painted tile and sort under a sentinel key). Frames
  equal the oracle's and the cell / entry counts equal tests/tables_model.py with the tables
  built from read-back counts (mode 0), sync-free (1) and sync-free but redone (2).
- A scene without carry-only entries: the gap sort sees no key.
"""
import numpy as np
import pytest
import torch

import extremes
import flatten_model as fm
import synth
import tables_model as tm
from extremes import polyline, rect_points, solid
from forma_b200.binding import RGBA, Color, FillRule, Rect

CLEAR = Color(1.0, 1.0, 1.0, 0.0)
CARRY_CTA = 1024  # cells per CTA tile of the carry pass


@pytest.fixture()
def tables_options(cuda_api):
    names = ("sync_free", "test_fast_shrink", "host_slices", "sort_big_log2", "sort_scan_log2")
    saved = {n: cuda_api.get_option(n) for n in names}
    cuda_api.set_option("host_slices", 1)
    yield
    for n, v in saved.items():
        cuda_api.set_option(n, v)


def _passes(bits: int) -> int:
    return (bits + 7) // 8


VIEWS = np.array([[1, 0, 0, 1, 0, 0], [1, 0, 0, 1, -40, 12], [0.5, 0, 0, 0.5, 100, 60]], np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,h,after_tables", [
    ("render_device", 360, 1),
    ("render_ids_device", 360, 1),
    ("render_device_with_ids", 360, 2),  # paint + ID kernel
    ("render_views_device", 352, 1),     # whole tile rows: the views are painted in place
    ("render_views_device", 360, 2),     # paint into the framebuffer + repack
], ids=["rgba", "ids", "rgba_with_ids", "views_in_place", "views_repacked"])
def test_sync_free_frame_launches_the_table_chain(cuda_api, tables_options, kind, h, after_tables):
    """Segment sort forced onto its reduce-then-scan passes (3 launches per pass, counted by
    kernel_times), so that everything but the tables is known: the resident composition's
    frame rasterizes with 3 launches (line count, block-sum scan, emit) and launches
    `after_tables` kernels after the tables, for every frame kind."""
    w, layers = 640, 300
    cuda_api.set_option("sort_big_log2", 10)
    cuda_api.set_option("sort_scan_log2", 10)
    comp = cuda_api.Composition()
    synth.random_mixed(cuda_api, comp, layers, w, h, 5)
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
    for _ in range(2):  # frame 1: counts read back; frame 2 has the previous counts as bounds
        render()
        torch.cuda.synchronize()
    before = r.counters()["launches"]
    render()
    torch.cuda.synchronize()
    c = r.counters()
    assert c["tables_mode"] == 1
    frame = c["launches"] - before
    sort_passes = r.kernel_times()["radix_downsweep"]["launches"]
    assert sort_passes > 0
    raster = 3
    assert c["segments"] > 2048  # more than one CTA tile of the cells pass: both cells kernels run
    tiles_x, tiles_y = (w + 15) // 16, n_views * ((h + 15) // 16)  # views: one frame of stacked views
    carry = _passes(int(layers - 1).bit_length())
    gap = _passes(int(tiles_x).bit_length() + int(tiles_y).bit_length())
    tables = 2 + carry + 1 + gap + 1
    if n_views == 1:
        assert tables == 8
    assert frame == raster + 3 * sort_passes + tables + after_tables, (frame, raster, sort_passes, tables)


# ---------------------------------------------------------------------------
# Carry groups across CTA tiles
# ---------------------------------------------------------------------------
WIDE_W, WIDE_H = 32768, 48  # 2048 x 3 tiles


def zigzag_band(x0: float, x1: float, y_lo: float, y_hi: float) -> np.ndarray:
    """A closed band from x0 to x1 whose top edge zig-zags every 8 px (segments in every tile
    it crosses) and whose bottom edge is straight."""
    xs = np.arange(x0, x1, 8.0, dtype=np.float32)
    top = np.stack([xs, np.where(np.arange(xs.size) % 2 == 0, y_lo, y_lo + 4.0)], 1)
    return np.concatenate([top, np.array([[x1, y_lo], [x1, y_hi], [x0, y_hi]], np.float32)]).astype(np.float32)


def rect_run(y0: float, y1: float) -> np.ndarray:
    """Rectangles along the row, each drawn twice (the copy shifted right by half its width):
    winding 1, 2, 1 inside, 0 between them. Widths 0.5 ... 4.5 tiles, gaps 1.5 or 2.5 tiles."""
    out, x, i = [], 5.25, 0
    widths, gaps = (8.0, 24.0, 40.0, 72.0), (24.0, 40.0)
    while True:
        wd = widths[i % 4]
        if x + 1.5 * wd >= WIDE_W - 4:
            break
        out.append(rect_points(x, y0, x + wd, y1))
        out.append(rect_points(x + wd / 2, y0, x + 1.5 * wd, y1))
        x += 1.5 * wd + gaps[i % 2]
        i += 1
    return np.concatenate(out)


def wide_groups(api, comp):
    rules = {}

    def layer(order, rule, alpha):
        rules[order] = rule
        lay = comp.get_mut_or_insert_default(order)
        lay.set_props(solid(Color(0.9, 0.1 + 0.1 * order, 0.3, alpha), rule))
        return lay

    # Layer 0: groups of exactly 1024 and 2048 cells: the next group starts on a CTA tile.
    l0 = layer(0, FillRule.NonZero, 0.6)
    l0.insert(polyline(api, zigzag_band(1.0, CARRY_CTA * 16 - 1.0, 2.0, 12.0)))
    l0.insert(polyline(api, zigzag_band(1.0, 2 * CARRY_CTA * 16 - 1.0, 18.0, 28.0)))
    # Layer 1: one group of 2048 cells (segments in every tile of row 1) across three CTA tiles.
    layer(1, FillRule.EvenOdd, 0.7).insert(polyline(api, zigzag_band(1.0, WIDE_W - 1.0, 19.0, 29.0)))
    # Layers 2 / 3: covers that empty and refill along row 2, under both rules.
    run = rect_run(34.5, 45.5)
    layer(2, FillRule.NonZero, 0.5).insert(polyline(api, run, contour_len=4))
    layer(3, FillRule.EvenOdd, 0.8).insert(polyline(api, run, contour_len=4))
    # Layers 4 / 5: a band in every row across the whole width (enough cells that the halved
    # bounds of test_fast_shrink fall short of the counts).
    for order, rule in ((4, FillRule.NonZero), (5, FillRule.EvenOdd)):
        lay = layer(order, rule, 0.4)
        for row in range(3):
            lay.insert(polyline(api, zigzag_band(3.0, WIDE_W - 3.0, 16.0 * row + 1.0, 16.0 * row + 14.0)))
    return extremes.Built(rules)


WIDE_CROPS = {
    "whole": None,
    "inside_groups": Rect((2008, 24000), (0, WIDE_H)),  # starts in tile 125, ends in tile 1500
    "left_part": Rect((0, 14000), (0, WIDE_H)),  # every group starts inside, most end outside
}


@pytest.fixture(scope="module")
def wide(oracle_api, oracle_renderer):
    comp = oracle_api.Composition()
    built = wide_groups(oracle_api, comp)
    fm.assert_preflight(fm.preflight(0, oracle_renderer, comp, WIDE_W, WIDE_H), "wide_groups")
    memo = {}

    def get(crop_name):
        if crop_name not in memo:
            crop = WIDE_CROPS[crop_name]
            r = oracle_api.Renderer(0)
            buf = np.zeros(WIDE_W * WIDE_H * 4, np.uint8)
            r.render(comp, buf, WIDE_W, WIDE_H, RGBA, CLEAR, crop)
            memo[crop_name] = (buf, tm.table_counts(r.segments(), WIDE_W, WIDE_H, built.rules, crop))
        return memo[crop_name]
    return get


def test_wide_groups_reach_their_targets(oracle_api, oracle_renderer, wide):
    """The scene does what the tests below rely on (checked on the CPU)."""
    _, tc = wide("whole")
    assert tc.cells > 6000  # test_fast_shrink: (cells * 1.25 + 4096) / 2 < cells
    assert tc.entries > tc.cells
    comp = oracle_api.Composition()
    wide_groups(oracle_api, comp)
    r = oracle_api.Renderer(0)
    r.render(comp, np.zeros(WIDE_W * WIDE_H * 4, np.uint8), WIDE_W, WIDE_H, RGBA, CLEAR)
    keys = r.segments() >> np.uint64(20)
    heads = np.ones(keys.size, bool)
    heads[1:] = keys[1:] != keys[:-1]
    ck = keys[heads]
    ty, tx, layer = (ck >> np.uint64(33)).astype(np.int64) - 1, ((ck >> np.uint64(21)) & np.uint64(0xFFF)).astype(np.int64) - 1, \
        (ck & np.uint64(0x1FFFFF)).astype(np.int64)
    order = np.lexsort((tx, ty, layer))  # carry order
    g = np.stack([layer[order], ty[order]], 1)
    starts = np.flatnonzero(np.r_[True, np.any(g[1:] != g[:-1], axis=1)])
    sizes = np.diff(np.r_[starts, g.shape[0]])
    assert sizes.max() >= 2 * CARRY_CTA
    assert (starts[1:] % CARRY_CTA == 0).sum() >= 2, "groups that start on a CTA tile of the carry pass"
    assert starts[1] == CARRY_CTA and starts[2] == 3 * CARRY_CTA


@pytest.mark.gpu
@pytest.mark.parametrize("crop_name", list(WIDE_CROPS))
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_carry_groups_across_cta_tiles(cuda_api, wide, tables_options, crop_name, mode):
    want, tc = wide(crop_name)
    crop = WIDE_CROPS[crop_name]
    comp = cuda_api.Composition()
    wide_groups(cuda_api, comp)
    r = cuda_api.Renderer(0)
    frames = 1 if mode == 0 else 2
    for f in range(frames):
        if mode == 2 and f == 1:
            cuda_api.set_option("test_fast_shrink", 1)
        buf = np.zeros(WIDE_W * WIDE_H * 4, np.uint8)
        r.render(comp, buf, WIDE_W, WIDE_H, RGBA, CLEAR, crop)
    c = r.counters()
    assert c["tables_mode"] == mode
    assert (c["cells"], c["entries"]) == (tc.cells, tc.entries)
    if not np.array_equal(buf, want):
        d = np.abs(buf.reshape(WIDE_H, WIDE_W, 4).astype(int) - want.reshape(WIDE_H, WIDE_W, 4).astype(int)).max(axis=2)
        ys, xs = np.nonzero(d)
        raise AssertionError(f"{len(ys)} pixels differ from the oracle, first at x={xs[0]} y={ys[0]} "
                             f"(tile {xs[0] // 16}, {ys[0] // 16})")


def stars_only(api, comp):
    """Closed pixel stars: every cell's cover sums to zero, so no tile carries a cover on."""
    rules = {}
    for i in range(40):
        rule = FillRule.EvenOdd if i % 2 else FillRule.NonZero
        comp.get_mut_or_insert_default(i).insert(polyline(api, extremes.star_points(16 * i + 3, 5 + (i % 3) * 16, 97))).set_props(
            solid(Color(0.2, 0.5, 0.1 + 0.02 * i, 0.9), rule))
        rules[i] = rule
    return extremes.Built(rules)


@pytest.mark.gpu
def test_scene_without_carry_only_entries(cuda_api, oracle_api, tables_options):
    w, h = 704, 48
    comp = oracle_api.Composition()
    built = stars_only(oracle_api, comp)
    ro = oracle_api.Renderer(0)
    want = np.zeros(w * h * 4, np.uint8)
    ro.render(comp, want, w, h, RGBA, CLEAR)
    tc = tm.table_counts(ro.segments(), w, h, built.rules)
    assert tc.entries == tc.cells
    comp = cuda_api.Composition()
    stars_only(cuda_api, comp)
    r = cuda_api.Renderer(0)
    modes = []
    for _ in range(3):
        buf = np.zeros(w * h * 4, np.uint8)
        r.render(comp, buf, w, h, RGBA, CLEAR)
        c = r.counters()
        modes.append(c["tables_mode"])
        assert (c["cells"], c["entries"]) == (tc.cells, tc.entries)
        assert np.array_equal(buf, want)
    assert modes == [0, 1, 1]
