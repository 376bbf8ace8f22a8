"""A NumPy model of the layer cache's decisions, tile by tile, restated from the reference painter
(layer_workbench/passes/tile_unchanged.rs, the visible-unchanged rule of
skip_fully_covered_layers.rs:38-89, CachedTile::convert_optimizer_op and update_* in
cpu/painter/mod.rs:600-714, and BufferLayerCache in cpu/renderer.rs:94-110, 217-223), not from the
oracle's C++ or the kernels.

A tile's entries come from tests/clip_model.py (built from the oracle's sorted segments, with the
`full`, opaque and skip_trivial_clips marks), plus the reference's queue of layers left of the first
painted tile of a row: every layer with a segment left of that tile is queued there, even when its
covers sum to zero, and so counts in the tile's cached layer count.

Per tile the model gives NONE (nothing written), SOLID (the solid tile's bytes) or PAINT, and the new
record (layer count and solid bytes, each optional). The bytes a frame writes are those of an uncached
frame of the same composition: a SOLID tile's bytes are its pixel (0, 0) there.

`errors` plants a model error, so that the tests can show each one is caught:
- "removed": layers_were_removed is always false;
- "unmapped": solid bytes are compared and stored before the channel mapping;
- "clear": the clear colour's check is dropped (taken as unchanged)."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

import clip_model

NONE, SOLID, PAINT = "none", "solid", "paint"


@dataclass
class Record:
    """CachedTile: layer_count and solid_color, each None until set."""
    count: int | None = None
    solid: bytes | None = None


@dataclass
class CacheState:
    """BufferLayerCache: size, clear colour and tile records."""
    size: tuple | None = None
    clear: tuple | None = None
    tiles: dict = field(default_factory=dict)

    def clear_all(self):  # BufferLayerCache::clear
        self.clear = None
        self.tiles = {}


def tile_rect(w, h, crop):
    tx, ty = -(-w // 16), -(-h // 16)
    if crop is None:
        return 0, tx, 0, ty
    (x0, x1), (y0, y1) = crop
    return min(x0 // 16, tx), min(-(-x1 // 16), tx), min(y0 // 16, ty), min(-(-y1 // 16), ty)


def entries(segs, props, w, h, crop):
    """{(tx, ty): [clip_model.Entry]} of the tiles in the crop's tile rectangle, as the painter's
    workbench holds them (mod.rs:500-522: the first tile of a row queues every layer left of it)."""
    m = clip_model.Model(segs, props, w, h)
    tx_lo, tx_hi, ty_lo, ty_hi = tile_rect(w, h, crop)
    s = clip_model.unpack_segments(np.asarray(segs, np.uint64))
    x = s["tile_x"].astype(np.int64) * 16 + s["local_x"]
    out = {}
    for ty in range(ty_lo, ty_hi):
        left = set(int(o) for o in np.unique(s["layer_id"][(s["tile_y"] == ty) & (x < 16 * tx_lo)]))
        for tx in range(tx_lo, tx_hi):
            es = m.tiles.get((tx, ty), [])
            if tx == tx_lo and left - {e.order for e in es}:
                have = {e.order for e in es}
                es = [clip_model.Entry(e.order, e.layer, e.cov, e.full) for e in es]  # marks redone below
                es += [clip_model.Entry(o, m.props[o], np.zeros((16, 16)), False) for o in left - have]
                es.sort(key=lambda e: e.order)
                clip_model.skip_trivial_clips(es)
            out[tx, ty] = es
    return out


def decide(es, props, rec, unchanged, clear_unchanged, errors=()):
    """One tile: tile_unchanged, then skip_fully_covered_layers' visible-unchanged rule and its fold.
    Returns NONE, SOLID (a foldable solid tile, before the byte comparison) or PAINT; updates rec.count."""
    layers = len(es)
    previous, rec.count = rec.count, layers  # update_layer_count(Some(layers))
    removed, is_unchanged = True, False  # PassesSharedState::reset
    if previous is not None:
        removed = layers < previous
        is_unchanged = previous == layers and all(unchanged.get(e.order, False) for e in es)
    if "removed" in errors:
        removed = False
    if (clear_unchanged or "clear" in errors) and is_unchanged:
        return NONE
    visible_unchanged, interesting, start = not removed, None, 0
    for k in range(len(es) - 1, -1, -1):
        e = es[k]
        if not e.mask:
            continue
        if not unchanged.get(e.order, False):
            visible_unchanged = False
        if e.applies_clip or not e.full:
            interesting = interesting or "incomplete"
        elif e.layer.opaque:
            interesting = interesting or "opaque"
            start = k
            break
    if interesting == "incomplete":
        return PAINT
    if interesting == "opaque":
        if visible_unchanged:
            return NONE
        start += 1
    for e in es[start:]:
        if not e.mask:
            continue
        d = props[e.order].func.draw
        if d is None or d.fill.solid is None:
            return PAINT
    return SOLID


def same_color(a, b):
    """Color's PartialEq: per channel f32 ==, so -0 == +0 and NaN is never equal."""
    return a is not None and b is not None and all(np.float32(x) == np.float32(y) for x, y in zip(a, b))


@dataclass
class FrameInput:
    """What the model needs of one cached frame."""
    cache: object           # the cache's key: frames with the same key share records
    w: int
    h: int
    crop: tuple | None      # ((x0, x1), (y0, y1)) in pixels
    clear: tuple            # (r, g, b, a)
    segs: np.ndarray        # the oracle's sorted segments of the frame
    props: dict             # {order: Props} of the layers in the composition
    unchanged: dict         # {order: bool}: the layer's bit for the cache's id
    plain: np.ndarray       # [h, w, 4] uint8: an uncached frame of the same composition and colours
    unmapped: np.ndarray    # [h, w, 4] uint8: the same frame with channels RGBA (for the planted "unmapped")
    reset: bool = False     # cache.clear() was called since the cache's last frame


class CacheModel:
    def __init__(self, errors=()):
        self.errors = tuple(errors)
        self.caches = {}

    def frame(self, f: FrameInput, before: np.ndarray):
        """The expected frame ([h, w, 4], from `before`) and {(tx, ty): op} of the frame's tiles."""
        c = self.caches.setdefault(f.cache, CacheState())
        if f.reset:
            c.clear_all()
        if c.size != (f.w, f.h):  # renderer.rs:103-110
            c.size = (f.w, f.h)
            c.clear_all()
        clear_unchanged = same_color(c.clear, f.clear)
        out, ops = before.copy(), {}
        for (tx, ty), es in entries(f.segs, f.props, f.w, f.h, f.crop).items():
            rec = c.tiles.setdefault((tx, ty), Record())
            op = decide(es, f.props, rec, f.unchanged, clear_unchanged, self.errors)
            sl = np.s_[16 * ty:16 * ty + 16, 16 * tx:16 * tx + 16]
            if op == SOLID:  # convert_optimizer_op
                b = bytes((f.unmapped if "unmapped" in self.errors else f.plain)[16 * ty, 16 * tx])
                op = NONE if rec.solid == b else SOLID
                rec.solid = b
            elif op == PAINT:
                rec.solid = None
            if op != NONE:
                out[sl] = f.plain[sl]
            ops[tx, ty] = op
        c.clear = f.clear  # renderer.rs:217-219
        return out, ops


def count(ops, op):
    return sum(1 for v in ops.values() if v == op)
