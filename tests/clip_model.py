"""A NumPy model of the painter's tile walk with clips, built from an oracle's sorted pixel segments and
the props every layer was given: each tile's entries and their per-pixel coverages, the optimizer
passes that mark them (skip_trivial_clips, skip_fully_covered_layers) and the clip state of the walk,
giving layer coverage masks, ID frames and layer statistics.

The passes and the clip state are restated from the reference painter (cpu/painter/mod.rs:300-335
and 449-464, layer_workbench/passes/skip_trivial_clips.rs and skip_fully_covered_layers.rs), not
from the oracle's C++, so that a contract the oracle and the kernels share is checked against a
reading of its own. Coverages are integers until the end: a pixel's doubled area is its cell areas
plus 32 x the covers left of it in its row (the carried cover included), in int64; coverage is that
over 512 (clamped for NonZero, folded for EvenOdd), so every mask value is k / 512 or a product of
two such values, exact in float32.

The mask of a layer o is its coverage x clip mask in the painter's walk of the composition cut off
above o: the walk starts at the tile's first entry and restarts its clip state at every entry
skip_fully_covered_layers could choose as the painter's first layer. IDs follow the painter's own
walk, from the top-most such entry."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from forma_b200.binding import ID_NONE, BlendMode, FillRule, unpack_segments

import oracle_stats

U32 = 0xFFFFFFFF


@dataclass
class Layer:
    """What the walk needs of a layer's props."""
    even_odd: bool
    clip: int | None     # Func::Clip(n): n; None for Func::Draw
    clipped: bool        # Func::Draw with is_clipped
    opaque: bool         # Func::Draw, a solid Over fill of alpha 1

    @staticmethod
    def of(props) -> "Layer":
        d = props.func.draw
        solid = d is not None and d.fill.solid is not None
        return Layer(props.fill_rule == FillRule.EvenOdd, props.func.clip, d is not None and d.is_clipped,
                     solid and d.blend_mode == BlendMode.Over and d.fill.solid.a == 1.0)


@dataclass
class Entry:
    """One (tile, layer) pair: the layer has segments in the tile or carries a non-empty cover into it."""
    order: int
    layer: Layer
    cov: np.ndarray      # [16 rows, 16 columns] float64
    full: bool           # no segments, and the carried cover is full in every row
    mask: bool = True    # painted (skip_trivial_clips keeps it)
    skip_clipping: bool = False

    @property
    def is_clip(self):
        return self.layer.clip is not None

    @property
    def applies_clip(self):
        return self.layer.clipped and not self.skip_clipping

    @property
    def may_start(self):
        """skip_fully_covered_layers may start the painter here."""
        return self.mask and not self.is_clip and not self.applies_clip and self.full and self.layer.opaque


def coverage(da, even_odd):
    if even_odd:
        return (512 - np.abs((da & 1023) - 512)) / 512.0
    return np.minimum(np.abs(da) / 512.0, 1.0)


def cover_is_empty(c, even_odd):
    return not np.any(c % 32 if even_odd else c)


def cover_is_full(c, even_odd):
    a = np.abs(c)
    return bool(np.all(a % 32 == 16 if even_odd else a == 16))


def skip_trivial_clips(entries):
    clip = None  # [is_full, last_layer_id, entry, is_used]
    for e in entries:
        if not e.mask:
            continue
        if e.is_clip:
            clip = [e.full, (e.order + e.layer.clip) & U32, e, False]
            if e.full:
                e.mask = False
        if e.layer.clipped:
            if clip is not None and e.order <= clip[1]:
                if clip[0]:
                    e.skip_clipping = True
                else:
                    clip[3] = True
            else:
                e.mask = False
        if clip is not None and e.order > clip[1]:
            if not clip[3]:
                clip[2].mask = False
            clip = None
    if clip is not None and not clip[3]:
        clip[2].mask = False


class ClipState:
    """The painter's clip state (cpu/painter/mod.rs:300-335, clip_at 449-464)."""

    def __init__(self):
        self.active, self.last, self.mask = False, 0, None

    def before(self, order):
        if self.active and self.last < order:
            self.active = False

    def clip_at(self, e):
        if not self.active:
            self.active, self.last = True, (e.order + e.layer.clip) & U32
        self.mask = e.cov

    def value(self, e):
        """The painted coverage of Draw entry e, or None where the painter skips it."""
        if e.applies_clip:
            return e.cov * self.mask if self.active else None
        return e.cov


class Model:
    def __init__(self, segs, layers, width, height):
        """segs: an oracle's sorted segments; layers: {order: Props} of the layers that have props."""
        self.w, self.h = width, height
        self.tx_n, self.ty_n = -(-width // 16), -(-height // 16)
        self.props = {o: Layer.of(p) for o, p in layers.items()}
        self.tiles = {}
        s = unpack_segments(np.asarray(segs, np.uint64))
        W = 16 * self.tx_n
        x = s["tile_x"] * 16 + s["local_x"]
        for ty in range(self.ty_n):
            row = (s["tile_y"] == ty) & (x < W)
            per = {t: [] for t in range(self.tx_n)}
            for order in np.unique(s["layer_id"][row]):
                lay = self.props[int(order)]
                m = row & (s["layer_id"] == order)
                xs, ys = x[m], s["local_y"][m]
                area = np.zeros((16, W), np.int64)
                inside = xs >= 0
                np.add.at(area, (ys[inside], xs[inside]), s["double_area"][m][inside])
                cov_col = np.zeros((16, W + 1), np.int64)
                np.add.at(cov_col, (ys, np.clip(xs + 1, 0, W)), s["cover"][m])
                run = np.cumsum(cov_col, axis=1)  # run[:, X]: covers left of column X
                cov = coverage(area + 32 * run[:, :W], lay.even_odd)
                segs_in = np.zeros(self.tx_n, bool)
                segs_in[np.unique(xs[inside] // 16)] = True
                for tx in range(self.tx_n):
                    carry = run[:, 16 * tx]
                    if segs_in[tx] or not cover_is_empty(carry, lay.even_odd):
                        full = not segs_in[tx] and cover_is_full(carry, lay.even_odd)
                        per[tx].append(Entry(int(order), lay, cov[:, 16 * tx:16 * tx + 16], full))
            for tx, entries in per.items():
                if entries:
                    skip_trivial_clips(entries)
                    self.tiles[tx, ty] = entries

    def _put(self, out, tx, ty, plane):
        h, w = min(16, self.h - 16 * ty), min(16, self.w - 16 * tx)
        out[16 * ty:16 * ty + h, 16 * tx:16 * tx + w] = plane[:h, :w]

    def first_painted(self, entries):
        """skip_fully_covered_layers: the index of the top-most entry the painter starts from."""
        for k in range(len(entries) - 1, -1, -1):
            if entries[k].may_start:
                return k
        return 0

    def masks(self, first, n):
        """F32 planes [n, h, w] of orders [first, first + n)."""
        out = np.zeros((n, self.h, self.w), np.float32)
        for (tx, ty), entries in self.tiles.items():
            st = ClipState()
            for e in entries:
                if e.may_start:
                    st.active = False
                plane = None
                if not e.mask:
                    if e.is_clip:
                        plane = e.cov  # not painted: its own coverage, no clip state
                else:
                    st.before(e.order)
                    if e.is_clip:
                        st.clip_at(e)
                        plane = e.cov
                    else:
                        plane = st.value(e)
                if plane is not None and first <= e.order < first + n:
                    self._put(out[e.order - first], tx, ty, plane)
        return out

    def ids(self, min_coverage):
        """The ID frame [h, w]: the top-most painted Draw layer whose coverage x clip > min_coverage."""
        out = np.full((self.h, self.w), ID_NONE, np.uint32)
        for (tx, ty), entries in self.tiles.items():
            tile = np.full((16, 16), ID_NONE, np.uint32)
            st = ClipState()
            for e in entries[self.first_painted(entries):]:
                if not e.mask:
                    continue
                st.before(e.order)
                if e.is_clip:
                    st.clip_at(e)
                    continue
                v = st.value(e)
                if v is not None:
                    tile[v > min_coverage] = e.order
            self._put(out, tx, ty, tile)
        return out

    def stats(self, first, n, min_coverage, rect=None):
        rect = rect or (0, self.w, 0, self.h)
        return oracle_stats.reduce(self.masks(first, n), self.ids(min_coverage), first, min_coverage, rect)

    def counts(self):
        """{(tx, ty): number of entries} of the tiles with entries."""
        return {t: len(e) for t, e in self.tiles.items()}
