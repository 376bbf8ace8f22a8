"""A NumPy model of the counts of the painter tables (kernels_tables.cu), computed from the
sorted pixel segments alone, without the oracle's painter.

`Renderer.counters()` reports
  cells    every run of sorted segments with equal (tile_y, tile_x, layer), i.e. the distinct
           `segment >> 20` values: the cells pass counts all of them, also those outside the
           crop or the frame (they get the sentinel key and no carries);
  entries  cells + carry-only entries: the tiles a layer spans without segments of its own in
           them, where the running cover it carries in is not empty.

The carry walk is the reference's (cpu/painter/mod.rs:486-568, layer_workbench/mod.rs:196-342)
in plain integers: per (tile_y, layer) group, cells in tile_x order, covers summed per pixel
row and wrapped to i8; after every cell the tiles up to the next cell (or the crop's right
edge) get a carry-only entry unless the running cover is empty under the layer's fill rule
(`Cover::is_empty`, mod.rs:187-198); a layer whose segments all lie left of the crop is still
queued for the crop's first tile (covers_left_of_row, mod.rs:501-522). Only cells of painted
tile rows that are not right of the crop take part.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import numpy as np

SORT_SHIFT = 20


def wrap_i8(v):
    return ((np.asarray(v, np.int64) + 128) % 256) - 128


def cover_is_empty(cover, fill_rule: int) -> bool:
    """Cover::is_empty for one cell's 16 i8 row covers."""
    c = wrap_i8(cover)
    if fill_rule == 0:
        return bool(np.all(c == 0))
    return bool(np.all((np.abs(c) & 31) == 0))


def cover_is_full(cover, fill_rule: int) -> bool:
    """Cover::is_full (mod.rs:200-214); i8 abs wraps (-128 stays -128)."""
    c = wrap_i8(cover)
    a = wrap_i8(np.abs(c))
    if fill_rule == 0:
        return bool(np.all(a == 16))
    return bool(np.all((a & 31) == 16))


@dataclass
class TableCounts:
    cells: int
    gaps: int
    entries: int
    gaps_per_tile: Dict[Tuple[int, int], int]     # (tile_y, tile_x) -> carry-only entries
    cell_sizes: np.ndarray                        # segments per cell, in sorted order
    cell_starts: np.ndarray                       # first segment of every cell
    row_covers: np.ndarray                        # (cells, 16) unwrapped per-row cover sums
    cell_keys: np.ndarray                         # (tile_y, tile_x, layer) of every cell, (cells, 3)
    gap_keys: np.ndarray                          # (tile_y, tile_x, layer) of every carry-only entry


def decode(segs: np.ndarray):
    s = np.asarray(segs, np.uint64)
    return {
        "ty": ((s >> np.uint64(53)) & np.uint64(0x7FF)).astype(np.int64) - 1,
        "tx": ((s >> np.uint64(41)) & np.uint64(0xFFF)).astype(np.int64) - 1,
        "layer": ((s >> np.uint64(20)) & np.uint64(0x1FFFFF)).astype(np.int64),
        "ly": ((s >> np.uint64(12)) & np.uint64(0xF)).astype(np.int64),
        "cover": ((s & np.uint64(0x3F)).astype(np.int64) ^ 0x20) - 0x20,
    }


def tile_crop(width: int, height: int, crop=None):
    """(tx_lo, tx_hi, ty_lo, ty_hi, tiles_x, tiles_y) of a frame and an optional pixel crop
    (binding.Rect), as the renderer derives them."""
    tiles_x, tiles_y = (width + 15) // 16, (height + 15) // 16
    if crop is None:
        return 0, tiles_x, 0, tiles_y, tiles_x, tiles_y
    tx_lo = min(crop.horizontal[0] // 16, tiles_x)
    tx_hi = max(min((crop.horizontal[1] + 15) // 16, tiles_x), tx_lo)
    ty_lo = min(crop.vertical[0] // 16, tiles_y)
    ty_hi = max(min((crop.vertical[1] + 15) // 16, tiles_y), ty_lo)
    return tx_lo, tx_hi, ty_lo, ty_hi, tiles_x, tiles_y


def table_counts(segs: np.ndarray, width: int, height: int, fill_rules: Dict[int, int], crop=None) -> TableCounts:
    """Counts of the painter tables for sorted segments (sorted on bits [20, 64)).
    fill_rules: layer -> 0 (NonZero) / 1 (EvenOdd); layers without an entry count as NonZero."""
    segs = np.asarray(segs, np.uint64)
    tx_lo, tx_hi, ty_lo, ty_hi, _, _ = tile_crop(width, height, crop)
    keys = segs >> np.uint64(SORT_SHIFT)
    if keys.size:
        assert np.all(keys[1:] >= keys[:-1]), "segments are not sorted"
    head = np.ones(keys.size, bool)
    head[1:] = keys[1:] != keys[:-1]
    starts = np.flatnonzero(head)
    n_cells = starts.size
    sizes = np.diff(np.append(starts, keys.size))
    d = decode(segs)
    cell_of = np.cumsum(head) - 1
    row_covers = np.zeros((n_cells, 16), np.int64)
    np.add.at(row_covers, (cell_of, d["ly"]), d["cover"])
    cty, ctx, clay = d["ty"][starts], d["tx"][starts], d["layer"][starts]
    cell_keys = np.stack([cty, ctx, clay], 1) if n_cells else np.zeros((0, 3), np.int64)

    relevant = (cty >= ty_lo) & (cty < ty_hi) & (ctx < tx_hi)
    idx = np.flatnonzero(relevant)
    order = idx[np.lexsort((ctx[idx], clay[idx], cty[idx]))]  # (tile_y, layer, tile_x)
    gaps_per_tile: Dict[Tuple[int, int], int] = {}
    gap_keys = []
    n_gaps = 0
    j = 0
    while j < order.size:
        c0 = order[j]
        ty, layer = int(cty[c0]), int(clay[c0])
        rule = int(fill_rules.get(layer, 0)) & 1
        k = j
        while k < order.size and cty[order[k]] == ty and clay[order[k]] == layer:
            k += 1
        run = np.zeros(16, np.int64)
        for q in range(j, k):
            c = order[q]
            run = wrap_i8(run + row_covers[c])
            t = int(ctx[c])
            next_t = int(ctx[order[q + 1]]) if q + 1 < k else tx_hi
            lo, hi = max(t + 1, tx_lo), min(next_t, tx_hi)
            tiles = []
            if not cover_is_empty(run, rule):
                tiles = list(range(lo, hi))
            elif t < tx_lo < next_t and tx_lo < tx_hi:
                tiles = [tx_lo]
            for tx in tiles:
                gaps_per_tile[(ty, tx)] = gaps_per_tile.get((ty, tx), 0) + 1
                gap_keys.append((ty, tx, layer))
            n_gaps += len(tiles)
        j = k
    return TableCounts(n_cells, n_gaps, n_cells + n_gaps, gaps_per_tile, sizes, starts, row_covers, cell_keys,
                       np.array(gap_keys, np.int64).reshape(-1, 3))


def tile_entries(tc: TableCounts, tiles_x: int, tiles_y: int) -> Dict[Tuple[int, int], np.ndarray]:
    """Layers of the entries of every painted tile inside the frame, in painting order."""
    keys = np.concatenate([tc.cell_keys, tc.gap_keys])
    inside = (keys[:, 0] >= 0) & (keys[:, 0] < tiles_y) & (keys[:, 1] >= 0) & (keys[:, 1] < tiles_x)
    keys = keys[inside]
    keys = keys[np.lexsort((keys[:, 2], keys[:, 1], keys[:, 0]))]
    out: Dict[Tuple[int, int], np.ndarray] = {}
    if keys.size:
        tile = keys[:, 0] * tiles_x + keys[:, 1]
        cut = np.flatnonzero(np.diff(tile)) + 1
        for part in np.split(keys, cut):
            out[(int(part[0, 0]), int(part[0, 1]))] = part[:, 2].copy()
    return out


def pixel_areas(segs: np.ndarray) -> np.ndarray:
    """Sum of the doubled areas per (tile, layer, pixel) of sorted segments (unwrapped)."""
    s = np.asarray(segs, np.uint64)
    cover = ((s & np.uint64(0x3F)).astype(np.int64) ^ 0x20) - 0x20
    dam = ((s >> np.uint64(6)) & np.uint64(0x3F)).astype(np.int64)
    _, inv = np.unique(s >> np.uint64(12), return_inverse=True)
    return np.bincount(inv.ravel(), weights=(dam * cover).astype(np.float64)).astype(np.int64)


def heavy_class(entries: int, classes: int = 4) -> Optional[int]:
    """Class of a tile's entry count in the painter's heavy-tile lists (paint_common.cuh:
    2^(c+4) <= entries < 2^(c+5), the last class open-ended); None below kHeavyMin = 16."""
    if entries < 16:
        return None
    return min(entries.bit_length() - 5, classes - 1)
