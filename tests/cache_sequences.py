"""Named edit sequences under layer caches. Each sequence is a function of `Session`, which runs it on
one library (`api`): the same calls on the oracle and on the CUDA library give frames that must be
equal byte for byte. Before every cached frame a seeded half of the frame's tiles is overwritten with
a marker, so a comparison of two frames also compares the set of tiles each frame wrote.

A session keeps a shadow of what the reference's layer cache decides from (composition/layer.rs):
each layer's props, transform, enabled flag, last order and `is_unchanged` bits, and each renderer's
cache ids. With `record=True` (the oracle) every cached frame also gives a cache_model.FrameInput,
so that tests/cache_model.py can predict it.

Each sequence states the condition it exists for as `want` counts on its frames: the number of tiles
the model decides are NONE, SOLID (written solid) and PAINT (painted) in that frame, checked by
tests/test_cache_model.py. Uncached calls between cached frames (`Session.between`) run through a
hook: the GPU tests pass one that makes ID, mask, statistics, float, over, view and batch calls of the
renderer; they take no cache and leave every cache as it was, so on the oracle they are not made."""
from __future__ import annotations

import numpy as np

import cache_model
import synth
from forma_b200.binding import (BGRA, RGBA, BlendMode, Color, Fill, FillRule, Func, GradientBuilder, GradientType, Point,
                                Props, Rect, Style, Texture)

MARKER = np.array([0xA5, 0x5A, 0x3C, 0xC3], np.uint8)
FILL = 0x6B
CLEAR = Color(0.9, 0.85, 0.8, 1.0)
NAN = float("nan")


def draw(fill, blend=BlendMode.Over, clipped=False, rule=FillRule.NonZero):
    return Props(fill_rule=rule, func=Func.Draw(Style(is_clipped=clipped, fill=fill, blend_mode=blend)))


def solid(r, g, b, a=1.0, **kw):
    return draw(Fill.Solid(Color(r, g, b, a)), **kw)


def clip(n):
    return Props(func=Func.Clip(n))


def gradient(x0, y0, x1, y1):
    gb = GradientBuilder(Point(x0, y0), Point(x1, y1)).type(GradientType.Radial)
    for c in (Color(0.9, 0.1, 0.2, 1.0), Color(0.1, 0.8, 0.3, 0.7), Color(0.2, 0.3, 0.9, 1.0)):
        gb.color(c)
    return draw(Fill.Gradient(gb.build()))


TEXELS = np.linspace(0.0, 1.0, 4 * 4 * 4, dtype=np.float32).reshape(4, 4, 4)


def texture(scale=1.0):
    return draw(Fill.Texture(Texture((0.25, 0.0, 0.0, 0.25, 0.0, 0.0), TEXELS * np.float32(scale))))


def same(a, b):
    """Props' PartialEq: floats by ==, so -0 == +0 and NaN is never equal. An Image is equal only to
    itself (styling.rs: its data pointer); the same texels set again on a layer are the same image."""
    if isinstance(a, float) or isinstance(b, float):
        return isinstance(a, (int, float)) and isinstance(b, (int, float)) and np.float32(a) == np.float32(b)
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        f16 = lambda v: np.asarray(v, np.float32).astype(np.float16).view(np.uint16)
        return isinstance(a, np.ndarray) and isinstance(b, np.ndarray) and a.shape == b.shape and np.array_equal(f16(a), f16(b))
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if hasattr(a, "__dataclass_fields__"):
        return type(a) is type(b) and all(same(getattr(a, k), getattr(b, k)) for k in a.__dataclass_fields__)
    return a == b


class Shadow:
    """A layer as the reference's cache sees it."""

    def __init__(self, handle):
        self.h, self.props, self.transform, self.enabled, self.order, self.bits = handle, Props(), None, True, None, set()


class Cache:
    def __init__(self, session, ri, handle, cid, key):
        self.s, self.ri, self.h, self.id, self.key = session, ri, handle, cid, key
        self.buf, self.shape, self.reset = None, None, False

    def clear(self):
        self.h.clear()
        self.reset = True


class Session:
    def __init__(self, api, record=False, render=None, between=None, pad=0, seed=0):
        """render(renderer, comp, buf, w, h, stride, channels, clear, crop, cache_handle): a cached frame
        into the flat uint8 buffer `buf` (default: a host frame). between(kind, session): an uncached call."""
        self.api, self.record, self.pad, self.seed = api, record, pad, seed
        self.comp = api.Composition()
        self.renderers, self.ids_used = [], []
        self.layers = {}        # order -> Shadow
        self.detached = []      # shadows out of the composition, still owned by it
        self.frames = []        # per cached frame: (before, after), [h, w, 4] uint8 each
        self.inputs = []        # per cached frame (record): cache_model.FrameInput
        self.wants = []         # (frame index, {op: count or (lo, hi)})
        self.render_fn = render or host_render
        self.between_fn = between
        self.n_keys = 0
        self.renderer(0)

    # -- renderers and caches -------------------------------------------------
    def renderer(self, k):
        while len(self.renderers) <= k:
            self.renderers.append(self.api.Renderer(0))
            self.ids_used.append(set())
        return self.renderers[k]

    def cache(self, ri=0):
        """A new cache on renderer ri, or None where the renderer has no free id (both sides must agree)."""
        h = self.renderer(ri).create_buffer_layer_cache()
        free = [i for i in range(32) if i not in self.ids_used[ri]]
        assert (h is None) == (not free), "cache ids: the library and the shadow disagree"
        if h is None:
            return None
        self.ids_used[ri].add(free[0])
        self.n_keys += 1
        return Cache(self, ri, h, free[0], self.n_keys)

    def free(self, c):
        self.ids_used[c.ri].discard(c.id)
        c.h = None  # LayerCache.__del__ frees it now

    # -- layers ----------------------------------------------------------------
    def add(self, order, paths, props, transform=None):
        sh = Shadow(self.comp.create_layer())
        for p in paths:
            sh.h.insert(p)
        self.set_props_of(sh, props)
        if transform is not None:
            self.set_transform_of(sh, transform)
        self.insert(order, sh)
        return sh

    def insert(self, order, sh):
        old = self.comp.insert(order, sh.h)
        if sh.order != order:  # Layer::set_order
            sh.bits.clear()
        sh.order = order
        if sh in self.detached:
            self.detached.remove(sh)
        if order in self.layers:
            assert old is not None
            self.detached.append(self.layers[order])
        self.layers[order] = sh

    def remove(self, order):
        sh = self.layers.pop(order)
        assert self.comp.remove(order) is not None  # the handle stays valid while detached
        self.detached.append(sh)
        return sh

    def drop(self, order):
        sh = self.remove(order)
        self.detached.remove(sh)
        sh.h.drop()

    def set_props(self, order, props):
        self.set_props_of(self.layers[order], props)

    def set_props_of(self, sh, props):
        if not same(sh.props, props):
            sh.bits.clear()
            sh.props = props
        sh.h.set_props(props)

    def set_transform(self, order, t):
        self.set_transform_of(self.layers[order], t)

    def set_transform_of(self, sh, t):
        t = tuple(float(np.float32(v)) for v in t)
        new = None if same(t, (1.0, 0.0, 0.0, 1.0, 0.0, 0.0)) else t
        if not same(sh.transform, new) and not (sh.transform is None and new is None):
            sh.bits.clear()
            sh.transform = new
        sh.h.set_transform(t)

    def enable(self, order, on=True):
        self.layers[order].enabled = on
        self.layers[order].h.set_is_enabled(on)

    def clear_geometry(self, order, paths=()):
        sh = self.layers[order]
        sh.h.clear()
        sh.bits.clear()
        for p in paths:
            sh.h.insert(p)

    def mixed(self, n, w, h, seed, base=0):
        """synth.random_mixed's layers at orders base, base + 1, ..., through the shadow."""
        s = self

        class L:
            def __init__(self, order):
                self.order, self.paths = order, []

            def insert(self, path):
                self.paths.append(path)
                return self

            def set_props(self, props):
                s.add(self.order, self.paths, props)
                return self

        class C:
            def get_mut_or_insert_default(self, i):
                return L(base + i)
        synth.random_mixed(self.api, C(), n, w, h, seed)

    # -- frames ------------------------------------------------------------------
    def between(self, kind, **kw):
        if self.between_fn is not None:
            self.between_fn(kind, self, **kw)

    def frame(self, c, w, h, clear=CLEAR, channels=RGBA, crop=None, want=None):
        stride = 4 * w + self.pad
        if c.shape != (w, h):
            c.buf, c.shape = np.full(h * stride, FILL, np.uint8), (w, h)
        img = c.buf.reshape(h, stride)[:, :4 * w].reshape(h, w, 4)
        k = len(self.frames)
        rng = np.random.default_rng([self.seed, k])
        tiles = rng.random((-(-h // 16), -(-w // 16))) < 0.5
        mark = np.repeat(np.repeat(tiles, 16, 0), 16, 1)[:h, :w]
        img[mark] = MARKER
        before = img.copy()
        crop_px = None if crop is None else (tuple(crop[0]), tuple(crop[1]))
        rect = None if crop is None else Rect(crop_px[0], crop_px[1])
        unchanged = {o: c.id in sh.bits for o, sh in self.layers.items()}
        ctuple = (clear.r, clear.g, clear.b, clear.a)
        if self.record:
            plain_r = self.api.Renderer(0)
            plain = np.zeros(h * w * 4, np.uint8)
            plain_r.render(self.comp, plain, w, h, channels, clear, rect)
            segs = plain_r.segments()
            unmapped = plain
            if tuple(channels) != tuple(RGBA):
                unmapped = np.zeros(h * w * 4, np.uint8)
                self.api.Renderer(0).render(self.comp, unmapped, w, h, RGBA, clear, rect)
            self.inputs.append(cache_model.FrameInput(
                c.key, w, h, crop_px, ctuple, segs, {o: sh.props for o, sh in self.layers.items()}, unchanged,
                plain.reshape(h, w, 4), unmapped.reshape(h, w, 4), c.reset))
        c.reset = False
        self.render_fn(self.renderer(c.ri), self.comp, c.buf, w, h, stride, channels, clear, rect, c.h)
        self.frames.append((before, img.copy()))
        for sh in self.layers.values():  # renderer.rs:217-223
            if sh.enabled:
                sh.bits.add(c.id)
            else:
                sh.bits.discard(c.id)
        if want:
            self.wants.append((k, want))
        return img


def host_render(r, comp, buf, w, h, stride, channels, clear, crop, cache):
    r.render(comp, buf, w, h, channels, clear, crop, cache, stride=stride)


# ---------------------------------------------------------------------------
# Scenes
# ---------------------------------------------------------------------------

def rect(api, x0, y0, x1, y1):
    return (api.PathBuilder().move_to(Point(x0, y0)).line_to(Point(x0, y1)).line_to(Point(x1, y1)).line_to(Point(x1, y0))
            .line_to(Point(x0, y0)).build())


W, H = 100, 72   # 7 x 5 tiles, the last column and row partial
RW, RH = 400, 296  # the redo scenes: their cells and carry-only entries outgrow the bounds of a small frame


def base(s, w=W, h=H):
    """Orders: 0 a full backdrop; 1 two small squares under 2, in the tiles (2, 0) and (3, 1); 2 a full
    opaque block over the tiles (2..3, 0..1); 3 a translucent band across the frame (carry-only
    entries inside it); 4 a gradient; 5 a clip of 6 and 7; 8 a texture; 9 a translucent layer full
    in tile (2, 0); 10 a gradient full in tile (3, 1). (Vertical edges lie inside pixels: one on a
    tile's border leaves segments in the tile, and the layer is then not full there.)"""
    a = s.api
    s.add(0, [rect(a, -4.0, -4.0, w + 4.0, h + 4.0)], solid(0.2, 0.3, 0.4))
    s.add(1, [rect(a, 36.0, 4.0, 44.0, 12.0), rect(a, 52.0, 20.0, 60.0, 28.0)], solid(0.9, 0.1, 0.1))
    s.add(2, [rect(a, 31.5, -1.0, 64.5, 32.5)], solid(0.1, 0.6, 0.2))
    s.add(3, [rect(a, -2.0, 40.0, w + 2.0, 56.0)], solid(0.8, 0.7, 0.1, 0.5))
    s.add(4, [synth.circle_path(a, 18.0, 20.0, 12.0)], gradient(8.0, 8.0, 32.0, 30.0))
    s.add(5, [synth.circle_path(a, 80.0, 24.0, 14.0)], clip(2))
    s.add(6, [rect(a, 64.0, 8.0, 99.0, 30.0)], solid(0.3, 0.3, 0.9, clipped=True))
    s.add(7, [rect(a, 70.0, 16.0, 90.0, 40.0)], solid(0.9, 0.3, 0.9, 0.75, clipped=True))
    s.add(8, [rect(a, 5.0, 58.0, 30.0, 70.0)], texture())
    s.add(9, [rect(a, 31.5, -1.0, 48.5, 16.0)], solid(0.0, 0.0, 1.0, 0.25))
    s.add(10, [rect(a, 47.5, 16.0, 64.5, 32.5)], gradient(48.0, 16.0, 64.0, 32.0))


# ---------------------------------------------------------------------------
# Sequences
# ---------------------------------------------------------------------------

def equal_edits(s):
    """Edits that must not damage: equal props (solid, gradient, texture, a colour of -0 against +0),
    the current transform, identity on a layer without one, enable on an enabled layer, and a layer
    removed and re-inserted at its order: the frame after them writes nothing."""
    c = s.cache()
    base(s)
    s.set_transform(1, (1.0, 0.0, 0.0, 1.0, 2.0, 1.0))
    s.set_props(9, solid(0.0, 0.0, 1.0, 0.25))
    s.frame(c, W, H, want={"paint": (1, None)})
    s.frame(c, W, H, want={"paint": 0, "solid": 0})
    s.set_props(2, solid(0.1, 0.6, 0.2))
    s.set_props(4, gradient(8.0, 8.0, 32.0, 30.0))
    s.set_props(8, texture())
    s.set_props(9, solid(-0.0, -0.0, 1.0, 0.25))
    s.set_transform(1, (1.0, 0.0, 0.0, 1.0, 2.0, 1.0))
    s.set_transform(3, (1.0, 0.0, 0.0, 1.0, 0.0, 0.0))
    s.enable(6)
    s.insert(7, s.remove(7))
    s.frame(c, W, H, want={"paint": 0, "solid": 0})


def damaging_edits(s):
    """Edits that must damage: one props field, a texture's texels, a NaN colour channel (never equal:
    the tiles are painted again at every frame after it is set again), disable then enable, clear and insert, a dropped layer, an insert at a new order, a
    detached layer inserted."""
    a = s.api
    c = s.cache()
    base(s)
    s.frame(c, W, H)
    s.set_props(3, solid(0.8, 0.7, 0.1, 0.5, blend=BlendMode.Multiply))  # one field
    s.frame(c, W, H, want={"written": (7, None)})
    s.set_props(8, texture(0.5))
    s.frame(c, W, H, want={"paint": (2, 4), "solid": 0})
    s.set_props(4, draw(Fill.Solid(Color(NAN, 0.5, 0.5, 0.5))))
    s.frame(c, W, H, want={"paint": (1, None)})
    s.set_props(4, draw(Fill.Solid(Color(NAN, 0.5, 0.5, 0.5))))
    s.frame(c, W, H, want={"paint": (1, None)})  # NaN != NaN: the same tiles again
    s.frame(c, W, H, want={"written": 0})  # no set_props: the frame set the bits
    s.enable(6, False)
    s.frame(c, W, H, want={"written": (1, None)})
    s.enable(6, True)
    s.frame(c, W, H, want={"paint": (1, None)})
    s.clear_geometry(1, [rect(a, 38.0, 2.0, 46.0, 10.0), rect(a, 54.0, 18.0, 62.0, 26.0)])
    s.frame(c, W, H, want={"paint": 0, "solid": 0})  # under the block: nothing
    s.clear_geometry(8, [rect(a, 6.0, 58.0, 31.0, 70.0)])
    s.frame(c, W, H, want={"paint": (1, None)})
    s.drop(9)
    s.frame(c, W, H, want={"written": (1, None)})
    s.insert(12, s.remove(7))
    s.frame(c, W, H, want={"paint": (1, None)})
    d = s.remove(12)
    s.frame(c, W, H)
    s.insert(11, d)
    s.add(13, [rect(a, 0.0, 0.0, 10.0, 10.0)], solid(1.0, 1.0, 1.0, 0.5))
    s.frame(c, W, H, want={"paint": (1, None)})


def decision_edges(s):
    """Tiles at the cache's decision edges: an equal layer count with another set of layers; a change
    below the full opaque block (no write) and above it (a write); a removal under it (written again:
    layers were removed); a solid tile whose folded colour comes back to the cached bytes."""
    a = s.api
    c = s.cache()
    base(s)
    s.frame(c, W, H)
    s.remove(4)  # the gradient's tiles lose a layer ...
    s.add(11, [synth.circle_path(a, 18.0, 20.0, 12.0)], solid(0.4, 0.4, 0.4, 0.6))  # ... and gain one
    s.frame(c, W, H, want={"paint": (1, None)})
    s.set_props(1, solid(0.1, 0.9, 0.9))  # below the block: not even the gradient's tiles
    s.frame(c, W, H, want={"written": 0})
    s.set_props(9, solid(0.0, 0.0, 1.0, 0.3))  # above it
    s.frame(c, W, H, want={"solid": (1, 1)})
    s.remove(1)  # under it, but a removal: the gradient's tile (3, 1) is painted again
    s.frame(c, W, H, want={"paint": (1, 1), "solid": 0})
    s.set_props(9, solid(0.0, 0.0, 1.0, 0.3000001))  # the same bytes in tile (2, 0)
    s.frame(c, W, H, want={"solid": 0})
    s.set_props(2, solid(0.1, 0.6, 0.2000001))  # the opaque layer itself: its solid tile keeps its bytes
    s.frame(c, W, H, want={"solid": 0})


def frame_state(s):
    """Frame state under one cache: the clear colour changed, -0 against +0 (unchanged), NaN (never
    equal); the channel order changed (solid tiles compare after the mapping, painted unchanged tiles
    keep their old order); a size change; a crop that changes between frames of one size;
    cache.clear()."""
    c = s.cache()
    base(s)
    s.frame(c, W, H, clear=Color(0.0, 0.0, 0.0, 0.5))
    s.frame(c, W, H, clear=Color(-0.0, -0.0, 0.0, 0.5), want={"paint": 0, "solid": 0})
    s.frame(c, W, H, clear=Color(0.0, 0.0, 0.0, 1.0), want={"paint": (1, None)})
    s.frame(c, W, H, clear=Color(NAN, 0.0, 0.0, 1.0), want={"paint": (1, None)})
    s.frame(c, W, H, clear=Color(NAN, 0.0, 0.0, 1.0), want={"paint": (1, None)})
    s.frame(c, W, H, clear=CLEAR)
    s.frame(c, W, H, channels=BGRA, want={"written": 0})  # nothing changed: the old order stays
    s.set_props(2, solid(0.1, 0.6, 0.25))
    s.set_props(2, solid(0.1, 0.6, 0.2))  # the same colour, but changed: its solid tiles fold again
    s.frame(c, W, H, channels=BGRA, want={"solid": (1, None)})
    s.frame(c, W, H, channels=BGRA, want={"paint": 0, "solid": 0})
    s.frame(c, W, H, crop=((20, 70), (10, 50)), want={"paint": 0, "solid": 0})
    s.set_props(3, solid(0.8, 0.7, 0.1, 0.4))
    s.frame(c, W, H, crop=((40, 100), (33, 72)), want={"written": (1, None)})
    s.frame(c, W, H, crop=((0, 40), (30, 72)), want={"written": (1, None)})
    s.frame(c, W, H, want={"solid": 0})
    s.frame(c, W + 17, H - 5, want={"none": 0})
    s.frame(c, W + 17, H - 5, want={"paint": 0, "solid": 0})
    c.clear()
    s.frame(c, W + 17, H - 5, want={"none": 0})


def cache_ids(s):
    """Cache ids: 32 caches on one renderer and the 33rd refused; a freed id taken again while the
    layers still carry its bit; two caches alternating on one composition; two renderers, each with
    cache id 0, on one composition (their ids name the same bit of every layer)."""
    base(s, 48, 40)
    caches = [s.cache() for _ in range(32)]
    assert all(c is not None for c in caches) and s.cache() is None
    for c in caches[::7]:
        s.frame(c, 48, 40)
    s.frame(caches[7], 48, 40, want={"paint": 0, "solid": 0})
    s.free(caches[7])
    c7 = s.cache()
    assert c7.id == 7
    s.frame(c7, 48, 40, want={"none": 0})  # a new cache: everything is written, whatever the bits say
    s.frame(c7, 48, 40, want={"paint": 0, "solid": 0})
    for c in caches[:7] + caches[8:]:
        s.free(c)
    a, b = c7, s.cache()
    s.set_props(9, solid(0.5, 0.5, 0.5, 0.5))
    s.frame(a, 48, 40, want={"written": (1, None)})
    s.frame(b, 48, 40, want={"none": 0})
    s.frame(a, 48, 40, want={"paint": 0, "solid": 0})
    s.set_props(9, solid(0.5, 0.5, 0.6, 0.5))
    s.frame(b, 48, 40, want={"written": (1, None)})
    s.frame(a, 48, 40, want={"written": (1, None)})  # b's frame set b's bit, not a's
    r1 = s.cache(1)
    assert r1.id == 0 and s.renderers[1] is not s.renderers[0]
    s.free(a)
    s.free(b)
    r0 = s.cache(0)
    assert r0.id == 0
    s.frame(r0, 48, 40)
    s.frame(r1, 48, 40, want={"none": 0})
    s.set_props(2, solid(0.7, 0.6, 0.2))
    s.frame(r1, 48, 40, want={"written": (1, None)})
    s.frame(r0, 48, 40, want={"paint": 0, "solid": 0})


def between_frames(s):
    """Between cached frames: a compaction (most of the geometry cleared) and an evict, then uncached
    frames of the same renderer (RGBA, IDs, masks, statistics, float, over, views, batch, and a much
    smaller composition), each of which must leave the cache as it was."""
    a = s.api
    c = s.cache()
    base(s)
    s.mixed(60, W, H, 31, base=20)
    s.frame(c, W, H)
    for o in range(20, 70):
        s.clear_geometry(o)
    s.frame(c, W, H, want={"paint": (1, None)})
    s.add(70, [rect(a, 10.0, 10.0, 30.0, 20.0)], solid(0.2, 0.9, 0.2, 0.5))
    s.frame(c, W, H)
    s.between("evict")  # the device's copy of the composition is dropped
    s.frame(c, W, H, want={"paint": 0, "solid": 0})
    for kind in ("rgba", "ids", "masks", "stats", "linear", "over", "views", "batch", "small"):
        s.between(kind)
        s.frame(c, W, H, want={"paint": 0, "solid": 0})
        s.set_props(70, solid(0.2, 0.9, 0.2, 0.5 if kind in ("ids", "stats", "over", "batch") else 0.6))
        s.between(kind)
        s.frame(c, W, H, want={"paint": (1, None)})


def redo_growth(s):
    """The scene grows past the renderer's sync-free bounds between two cached frames: 400 layers
    appear under a full opaque layer, whose tiles must not be written."""
    a = s.api
    w, h = RW, RH
    c = s.cache()
    s.add(500, [rect(a, -2.0, -2.0, w + 2.0, h + 2.0)], solid(0.3, 0.5, 0.7))
    s.add(501, [rect(a, 20.5, 20.5, 60.5, 40.5)], solid(0.9, 0.9, 0.1, 0.5))
    s.frame(c, w, h)
    s.frame(c, w, h, want={"written": 0})
    s.mixed(400, w, h, 77)
    s.frame(c, w, h, want={"none": (400, None), "solid": 0})
    s.set_props(501, solid(0.9, 0.9, 0.1, 0.6))
    s.frame(c, w, h, want={"paint": (1, None)})


def redo_after_small(s):
    """A cached frame right after a small uncached call of the same renderer (an ID frame of a tiny
    composition): its bounds are those of the small call."""
    w, h = RW, RH
    c = s.cache()
    s.mixed(400, w, h, 78)
    s.add(500, [rect(s.api, 100.5, -2.0, w + 2.0, h + 2.0)], solid(0.3, 0.5, 0.7))
    s.frame(c, w, h)
    s.frame(c, w, h, want={"written": 0})
    s.between("small_ids")
    s.frame(c, w, h, want={"written": 0})
    s.set_props(5, solid(0.1, 0.2, 0.3, 0.5))
    s.between("small_ids")
    s.frame(c, w, h)


def random_edits(seed, frames, n_layers):
    def run(s):
        """A seeded sequence of random_mixed frames with edits drawn from every list above."""
        rng = np.random.default_rng(seed)
        w, h = int(rng.integers(80, 200)), int(rng.integers(60, 150))
        c = s.cache()
        s.mixed(n_layers, w, h, seed)
        s.add(n_layers + 1, [rect(s.api, 0.3 * w, -1.0, 0.6 * w, h + 1.0)], solid(0.2, 0.2, 0.2))
        clear = CLEAR
        for k in range(frames):
            orders = sorted(s.layers)
            o = int(orders[rng.integers(len(orders))])
            e = int(rng.integers(12))
            if e == 0:
                s.set_props(o, s.layers[o].props)
            elif e == 1:
                s.set_props(o, solid(*rng.random(3).tolist(), float(rng.choice([1.0, 0.5]))))
            elif e == 2:
                s.set_transform(o, (1.0, 0.0, 0.0, 1.0, float(rng.integers(-8, 8)), float(rng.integers(-8, 8))))
            elif e == 3:
                s.enable(o, not s.layers[o].enabled)
            elif e == 4:
                s.insert(o, s.remove(o))
            elif e == 5 and len(orders) > 4:
                s.drop(o)
            elif e == 6:
                free = max(orders) + 1 + int(rng.integers(3))
                s.insert(free, s.remove(o))
            elif e == 7:
                clear = Color(*rng.random(3).tolist(), 1.0) if rng.random() < 0.5 else clear
            elif e == 8:
                s.set_transform(o, s.layers[o].transform or (1.0, 0.0, 0.0, 1.0, 0.0, 0.0))
            crop = None
            if e == 9:
                x0, y0 = int(rng.integers(0, w // 2)), int(rng.integers(0, h // 2))
                crop = ((x0, w), (y0, h))
            s.frame(c, w, h, clear=clear, crop=crop)
    run.__name__ = f"random_{seed}"
    return run


SEQUENCES = {f.__name__: f for f in (equal_edits, damaging_edits, decision_edges, frame_state, cache_ids, between_frames,
                                     redo_growth, redo_after_small, random_edits(11, 12, 60), random_edits(12, 16, 150),
                                     random_edits(13, 20, 400))}
# The sequences that set up a sync-free redo for a cached device frame (see tests/test_gpu_cache_limits.py).
REDO = ("redo_growth", "redo_after_small")


def run(name, api, **kw):
    s = Session(api, seed=sum(map(ord, name)), **kw)
    SEQUENCES[name](s)
    return s
