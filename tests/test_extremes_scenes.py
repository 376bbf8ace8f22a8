"""CPU checks of the extreme scenes (tests/extremes.py) and of the painter-table model
(tests/tables_model.py).

Every scene must reach the condition it was built for, computed from the oracle's sorted
segments: a change in the path code that collapses a scene (see the spline-merge pitfall in
extremes.py) fails here instead of leaving the GPU tests without their purpose. The model is
pinned on hand-made segment lists with known answers."""
import numpy as np
import pytest

import extremes
import synth
import tables_model as tm
from forma_b200.binding import RGBA, BlendMode, Color, FillRule, Rect

CLEAR = Color(1.0, 1.0, 1.0, 0.0)
CTA = 2048          # segments per CTA tile of the cells pass (kernels_tables.cu: kCellTile)
FOLD = 2016         # segments per fold of the painter's packed cells (kernels_painter.cu: kPackedSegLimit)


_cache = {}


def oracle_scene(oracle_api, name):
    """(sorted segments, frame, Built, Extreme, TableCounts) of scene `name` from the oracle."""
    if name not in _cache:
        comp, built, sc = extremes.build(oracle_api, name)
        r = oracle_api.Renderer(0)
        buf = np.zeros(sc.width * sc.height * 4, np.uint8)
        t = r.render(comp, buf, sc.width, sc.height, RGBA, CLEAR, sc.crop)
        segs = r.segments()
        assert segs.size == t.n_segments
        _cache[name] = (segs, buf, built, sc, tm.table_counts(segs, sc.width, sc.height, built.rules, sc.crop))
    return _cache[name]


# --- the scenes reach their targets -----------------------------------------------------------
def test_dense_stars_give_cells_of_exactly_the_star_sizes(oracle_api):
    segs, buf, built, sc, tc = oracle_scene(oracle_api, "dense_stars")
    sizes = sorted(tc.cell_sizes.tolist())
    for n in extremes.STAR_SIZES:
        assert sizes.count(n) >= 2, f"no two cells of {n} segments (one per fill rule): {sizes}"
    assert tc.cell_sizes.max() > 2 * FOLD
    assert (tc.cell_sizes > CTA).sum() >= 8
    # one pixel sums a doubled area far beyond i16
    assert np.abs(tm.pixel_areas(segs)).max() > 32767
    # the stars' cells sit in the tiles of the translucent layer, which reaches them as a carry
    assert tc.gaps > 0
    assert buf.reshape(-1, 4)[:, 3].any()


def test_cell_boundaries_start_and_end_on_cta_tiles(oracle_api):
    segs, _, _, _, tc = oracle_scene(oracle_api, "cell_boundaries")
    assert tc.cell_sizes.tolist() == list(extremes.BOUNDARY_CELLS)
    starts, ends = tc.cell_starts, tc.cell_starts + tc.cell_sizes
    assert any(s % CTA == 0 and s > 0 for s in starts), "no cell starts on a CTA tile boundary"
    assert any(e % CTA == 0 and e < segs.size for e in ends), "no cell ends on a CTA tile boundary"
    spans = (ends - 1) // CTA - starts // CTA + 1
    assert spans.max() >= 3, "no cell spans three CTA tiles"
    tiles_with_head = set((starts // CTA).tolist())
    n_tiles = (segs.size + CTA - 1) // CTA
    assert set(range(n_tiles)) - tiles_with_head, "every CTA tile holds a cell head"


def test_sawtooth_entry_overflows_i16_covers_without_the_fold(oracle_api):
    segs, _, _, _, tc = oracle_scene(oracle_api, "sawtooth")
    assert tc.cell_sizes.max() > 20000
    d = tm.decode(segs)
    pix = (segs >> np.uint64(12)).astype(np.uint64)
    _, inv = np.unique(pix, return_inverse=True)
    cover = np.bincount(inv.ravel(), weights=d["cover"].astype(np.float64))
    assert np.abs(cover).max() > 32767, "no pixel sums a cover beyond i16"


@pytest.mark.parametrize("name", [n for n, s in extremes.SCENES.items() if "winding" in s.tags])
def test_deep_winding_rows_wrap_at_i8(oracle_api, name):
    segs, _, built, sc, tc = oracle_scene(oracle_api, name)
    rc = tc.row_covers[tc.row_covers != 0]
    assert np.any(rc % 256 == 0), "no row cover that is a nonzero multiple of 256"
    assert np.any(rc % 256 == 128), "no row cover = 128 (mod 256)"
    # K = 16: the fully covered rows of the carry wrap to 0, the half-covered top row to -128
    k16 = tc.row_covers[(tc.cell_keys[:, 2] == 1 + extremes.WINDINGS.index(16)) & (tc.cell_keys[:, 1] == 1)]
    assert np.any(k16 == 256) or np.any(k16 == -256) or "mixed" in name
    assert np.any(np.abs(k16) % 256 == 128) or "mixed" in name
    if "crop" in sc.tags:
        tx_lo = tm.tile_crop(sc.width, sc.height, sc.crop)[0]
        assert tx_lo > 1
        left = tc.cell_keys[:, 1] < tx_lo
        assert left.any()
        assert np.any(tc.gap_keys[:, 1] == tx_lo), "no carry reaches the crop's first column"


def test_crowds_fill_every_heavy_class_and_cross_entry_groups(oracle_api):
    classes, crossing, carry_clips, counts = set(), 0, 0, []
    for n in extremes.CROWDS:
        name = f"crowd_{n}"
        segs, _, built, sc, tc = oracle_scene(oracle_api, name)
        tiles_x, tiles_y = (sc.width + 15) // 16, (sc.height + 15) // 16
        per_tile = tm.tile_entries(tc, tiles_x, tiles_y)
        counts.append(max(len(v) for v in per_tile.values()))
        for layers in per_tile.values():
            c = tm.heavy_class(len(layers))
            if c is not None:
                classes.add(c)
            pos = {int(l): i for i, l in enumerate(layers)}
            for i, l in enumerate(layers):
                role, k = extremes.crowd_clip_role(int(l), n)
                if role in ("clip", "clip_carry"):
                    last = max((pos[m] for m in range(int(l) + 1, int(l) + k + 1) if m in pos), default=i)
                    crossing += (i // 32) != (last // 32)
        clips = [l for l in range(n) if extremes.crowd_clip_role(l, n)[0] == "clip_carry"]
        carry_clips += int(np.isin(tc.gap_keys[:, 2], clips).sum())
    assert classes == {0, 1, 2, 3}, (classes, counts)
    assert crossing > 0, "no clip range crosses a 32-entry group"
    assert carry_clips > 0, "no clip layer reaches a tile only as a carry"


def test_nan_blends_produce_nan_channels_encoded_as_zero(oracle_api):
    """Luminosity of a grey outside [0, 1] over grey divides by zero in clip_color!: the channel
    is NaN in both blend forms, and the reference's encoder turns a NaN from CPU arithmetic into
    byte 0 (its bits end in 0x00), in the solid-fold tile column 0 and in the per-pixel triangle."""
    from oracle import oracle
    assert np.isnan(oracle.blend_lane(oracle_api.hooks, BlendMode.Luminosity, [0.5] * 3, [1.5] * 3)).all()
    assert np.isnan(oracle.blend_lane(oracle_api.hooks, BlendMode.Luminosity, [0.5] * 3, [-0.5] * 3)).all()
    assert np.isnan(oracle.blend_scalar(oracle_api.hooks, BlendMode.Luminosity, [0.5, 0.5, 0.5, 1.0],
                                        [1.5, 1.5, 1.5, 1.0])[:3]).all()
    _, buf, _, sc, _ = oracle_scene(oracle_api, "nan_blends")
    img = buf.reshape(sc.height, sc.width, 4)
    assert (img[:, :16] == [0, 0, 0, 255]).all()   # solid-fold column
    assert (img[10, 45] == [0, 0, 0, 255]).all()   # per-pixel triangle


def test_long_diagonal_is_one_line_of_twelve_thousand_segments(oracle_api):
    comp, _, sc = extremes.build(oracle_api, "long_diagonal")
    r = oracle_api.Renderer(0)
    r.render(comp, np.zeros(sc.width * sc.height * 4, np.uint8), sc.width, sc.height, RGBA, CLEAR)
    lines = r.lines()
    assert len(lines["orders"]) == 256
    assert lines["lengths"].max() > 12000


def test_grid_and_far_geometry_reaches_beyond_the_frame(oracle_api):
    segs, buf, _, sc, tc = oracle_scene(oracle_api, "grid_and_far")
    d = tm.decode(segs)
    assert np.any(d["tx"] >= (sc.width + 15) // 16) and np.any(d["ty"] >= (sc.height + 15) // 16)
    assert np.any(d["tx"] == -1) and np.any(d["ty"] == -1)


# --- the model, on hand-made segment lists --------------------------------------------------
def seg(tx, ty, layer, lx, ly, cover, dam=0):
    return ((ty + 1) << 53) | ((tx + 1) << 41) | (layer << 20) | (lx << 16) | (ly << 12) | ((dam & 0x3F) << 6) | (cover & 0x3F)


def counts(segs, rules, width=64, height=16, crop=None):
    s = np.array(sorted(segs, key=lambda v: v >> 20), np.uint64)
    return tm.table_counts(s, width, height, rules, crop)


@pytest.mark.parametrize("copies,gaps", [(7, 3), (8, 3), (9, 3), (15, 3), (16, 0), (17, 3), (32, 0), (33, 3)])
def test_model_i8_wrap_of_a_row_cover(copies, gaps):
    """`copies` segments of cover +16 in row 5 of tile 0: the carry is 16 * copies wrapped to
    i8; a multiple of 256 is empty (no carry-only entries in tiles 1-3), 128 is not."""
    tc = counts([seg(0, 0, 3, 2, 5, 16)] * copies, {3: FillRule.NonZero})
    assert (tc.cells, tc.gaps, tc.entries) == (1, gaps, 1 + gaps)
    assert sorted(tc.gaps_per_tile) == [(0, t) for t in range(1, 1 + gaps)]


@pytest.mark.parametrize("cover,rule,gaps", [(16, 1, 3), (32, 1, 0), (-32, 1, 0), (48, 1, 3), (64, 1, 0),
                                              (32, 0, 3), (-16, 1, 3), (-128, 1, 0), (-128, 0, 3)])
def test_model_even_odd_masks_with_31(cover, rule, gaps):
    segs = [seg(0, 0, 1, 0, 9, 16 if cover > 0 else -16)] * (abs(cover) // 16)
    assert counts(segs, {1: rule}).gaps == gaps


def test_model_cover_predicates_match_the_reference():
    assert tm.cover_is_empty([0] * 16, 0) and not tm.cover_is_empty([0] * 15 + [1], 0)
    assert tm.cover_is_empty([32, -64, 96, 0] * 4, 1) and not tm.cover_is_empty([16] + [0] * 15, 1)
    assert tm.cover_is_full([16] * 8 + [-16] * 8, 0) and not tm.cover_is_full([16] * 15 + [-128], 0)
    assert not tm.cover_is_full([128] * 16, 0)  # -128: i8 abs wraps
    assert tm.cover_is_full([48] * 8 + [-16] * 8, 1) and not tm.cover_is_full([32] * 16, 1)


def test_model_carry_ends_where_the_cover_sums_to_zero():
    # tile 0: +16 in row 0; tile 2: -16 in row 0 -> carry-only entry in tile 1 only
    tc = counts([seg(0, 0, 0, 3, 0, 16), seg(2, 0, 0, 3, 0, -16)], {0: 0})
    assert (tc.cells, tc.gaps) == (2, 1) and tc.gaps_per_tile == {(0, 1): 1}


def test_model_covers_left_of_the_crop():
    """Crop from tile 2: a layer whose cells all lie left of it is queued for tile 2 even with an
    empty cover, once; with a non-empty cover it spans tiles 2-3; a cell at tile 2 takes the
    carry itself; cells right of the crop or in rows outside it are counted but carry nothing."""
    crop = Rect((32, 64), (0, 16))
    empty_left = [seg(0, 0, 0, 1, 4, 16), seg(0, 0, 0, 1, 4, -16), seg(1, 0, 0, 5, 4, 3)] + [seg(1, 0, 0, 5, 4, -3)]
    tc = counts(empty_left, {0: 0}, crop=crop)
    assert (tc.cells, tc.gaps, tc.gaps_per_tile) == (2, 1, {(0, 2): 1})
    full_left = [seg(-1, 0, 1, 15, 0, 16)]
    tc = counts(full_left, {1: 0}, crop=crop)
    assert (tc.gaps, tc.gaps_per_tile) == (2, {(0, 2): 1, (0, 3): 1})
    taken = [seg(0, 0, 2, 0, 0, 16), seg(2, 0, 2, 0, 0, 4)]
    tc = counts(taken, {2: 0}, crop=crop)
    assert (tc.cells, tc.gaps, tc.gaps_per_tile) == (2, 1, {(0, 3): 1})
    outside = [seg(3, 0, 4, 0, 0, 16), seg(0, 1, 5, 0, 0, 16)]  # right of the crop / row 1 of a one-row crop
    tc = counts(outside, {}, width=64, height=32, crop=Rect((0, 48), (0, 16)))
    assert (tc.cells, tc.gaps) == (2, 0)
    # the same cells without the crop
    tc = counts(outside, {}, width=64, height=32)
    assert (tc.cells, tc.gaps) == (2, 3)


def test_model_runs_on_a_random_mixed_scene(oracle_api):
    comp = oracle_api.Composition()
    synth.random_mixed(oracle_api, comp, 300, 513, 259, 22)
    r = oracle_api.Renderer(0)
    r.render(comp, np.zeros(513 * 259 * 4, np.uint8), 513, 259, RGBA, CLEAR)
    segs = r.segments()
    tc = tm.table_counts(segs, 513, 259, {})
    assert tc.cells == np.unique(segs >> np.uint64(20)).size > 1000
    assert tc.gaps == sum(tc.gaps_per_tile.values()) > 500
    assert all(0 <= ty < 17 and 0 <= tx < 33 for ty, tx in tc.gaps_per_tile)
