"""Named, deterministic scenes for the clip walk of the ID, mask and statistics paths (tests/clip_model.py):
clips nested around a full opaque layer, clip edge cases, clip ranges near 2^32, heavy tiles, windows,
frame edges and thresholds. Each scene builds for either API and carries a check that its model reaches
the edge it is named for (a tile's entries, which set its heavy class, and their flags); tests run the check
before using it.

`record(api, build)` builds any scene and returns the props every layer was given, which the
binding cannot read back."""
from __future__ import annotations

import contextlib
from dataclasses import dataclass, field
from typing import Callable, Optional

import numpy as np

from forma_b200.binding import (BlendMode, Color, Fill, FillRule, Func, GradientBuilder, Layer, Point, Props, Rect,
                                Style)

RED, GREEN, BLUE = Color(1.0, 0.0, 0.0, 1.0), Color(0.0, 1.0, 0.0, 1.0), Color(0.0, 0.0, 1.0, 1.0)
CLEAR = Color(1.0, 1.0, 1.0, 0.0)
LAYER_LIMIT = (1 << 21) - 1
THRESHOLDS = (0.0, 0.25, float(np.nextafter(np.float32(0.25), np.float32(0))), 511.0 / 512.0,
              float(np.nextafter(np.float32(1.0), np.float32(0))))


@contextlib.contextmanager
def _recording(props):
    orig = Layer.set_props

    def set_props(layer, p):
        props[layer._h] = p
        return orig(layer, p)
    Layer.set_props = set_props
    try:
        yield
    finally:
        Layer.set_props = orig


def record(api, build, max_order=1 << 21):
    """(comp, {order: Props}) of the layers `build` attached (Props() where it set none)."""
    by_handle = {}
    comp = api.Composition()
    with _recording(by_handle):
        build(api, comp)
    layers, n, o = {}, len(comp), 0
    while len(layers) < n and o < max_order:
        layer = comp.get(o)
        if layer is not None:
            layers[o] = by_handle.get(layer._h, Props())
        o += 1
    return comp, layers


def draw(color=GREEN, clipped=False, blend=BlendMode.Over, rule=FillRule.NonZero):
    return Props(fill_rule=rule, func=Func.Draw(Style(is_clipped=clipped, fill=Fill.Solid(color), blend_mode=blend)))


def clip(n, rule=FillRule.NonZero):
    return Props(fill_rule=rule, func=Func.Clip(n))


def gradient_draw():
    gb = GradientBuilder(Point(0.0, 0.0), Point(16.0, 0.0))
    gb.color(RED)
    gb.color(BLUE)
    return Props(func=Func.Draw(Style(fill=Fill.Gradient(gb.build()))))


@dataclass
class Scene:
    width: int
    height: int
    layers: list                # (order, (x0, y0, x1, y1) or a list of rects, Props, enabled)
    check: Callable             # (model) -> None: asserts the edge the scene is named for
    windows: list = field(default_factory=list)  # extra (first_order, n_orders)
    crop: Optional[Rect] = None

    def build(self, api, comp):
        for order, rects, props, enabled in self.layers:
            pb = api.PathBuilder()
            for (x0, y0, x1, y1) in ([rects] if isinstance(rects[0], (int, float)) else rects):
                pb.move_to(Point(x0, y0)).line_to(Point(x0, y1)).line_to(Point(x1, y1)).line_to(Point(x1, y0))
            layer = comp.get_mut_or_insert_default(order).insert(pb.build())
            if props is not None:
                layer.set_props(props)
            if not enabled:
                layer.set_is_enabled(False)

    def n_orders(self):
        return max(o for o, *_ in self.layers) + 1


def L(order, r, props, enabled=True):
    return (order, r, props, enabled)


# --- checks ---------------------------------------------------------------------------------------------


def entries_at(model, tile):
    return [e.order for e in model.tiles.get(tile, [])]


def expect_entries(tile, orders):
    def check(model):
        assert entries_at(model, tile) == orders, (tile, entries_at(model, tile), orders)
    return check


def expect(tile, orders, **flags):
    """Entry orders of `tile`, and per flag name a list of the orders it holds for (mask, full, may_start, skip_clipping)."""
    def check(model):
        expect_entries(tile, orders)(model)
        es = model.tiles[tile]
        for name, want in flags.items():
            got = [e.order for e in es if getattr(e, name)]
            assert got == want, (tile, name, got, want)
    return check


def all_of(*checks):
    def check(model):
        for c in checks:
            c(model)
    return check


# --- clip nesting around a full opaque layer ---------------------------------------------------------------

FULL = (-4, -4, 40, 20)
OUTER = L(0, (0, -4, 8.5, 20), clip(10))
INNER = L(5, (0, -4, 12.5, 20), clip(20))
TOP = L(15, (2, -4, 14, 20), draw(GREEN, clipped=True))

SCENES = {
    # The painter starts at layer 3, so clip 5 opens a fresh range and layer 15 is painted.
    "nest_restart": Scene(16, 16, [OUTER, L(3, FULL, draw(RED)), INNER, TOP],
                          expect((0, 0), [0, 3, 5, 15], mask=[0, 3, 5, 15], may_start=[3])),
    "nest_no_opaque": Scene(16, 16, [OUTER, INNER, TOP], expect((0, 0), [0, 5, 15], may_start=[])),
    "nest_clipped_between": Scene(16, 16, [OUTER, L(3, FULL, draw(RED)), L(4, (1, -4, 6, 20), draw(BLUE, clipped=True)), INNER, TOP],
                                  expect((0, 0), [0, 3, 4, 5, 15], mask=[0, 3, 4, 5, 15], may_start=[3])),
    "nest_inner_shorter": Scene(16, 16, [L(0, (0, -4, 8.5, 20), clip(30)), L(3, FULL, draw(RED)), L(5, (0, -4, 12.5, 20), clip(2)),
                                         L(6, (2, -4, 14, 20), draw(GREEN, clipped=True)),
                                         L(7, (3, -4, 11, 20), draw(BLUE, clipped=True)),
                                         L(9, (1, -4, 15, 20), draw(GREEN, clipped=True))],
                                expect((0, 0), [0, 3, 5, 6, 7, 9], mask=[0, 3, 5, 6, 7], may_start=[3])),
    "nest_inner_longer": Scene(16, 16, [L(0, (0, -4, 8.5, 20), clip(6)), L(2, (0, -4, 6, 20), draw(BLUE, clipped=True)),
                                        L(3, FULL, draw(RED)), L(5, (0, -4, 12.5, 20), clip(40)),
                                        L(9, (2, -4, 14, 20), draw(GREEN, clipped=True)),
                                        L(44, (3, -4, 11, 20), draw(BLUE, clipped=True))],
                               expect((0, 0), [0, 2, 3, 5, 9, 44], mask=[0, 2, 3, 5, 9, 44], may_start=[3])),
    # Full layers that are not a first layer the painter may choose: no restart.
    "nest_partial": Scene(16, 16, [OUTER, L(3, (-4, -4, 40, 12.5), draw(RED)), INNER, TOP], expect((0, 0), [0, 3, 5, 15], may_start=[])),
    "nest_gradient": Scene(16, 16, [OUTER, L(3, FULL, gradient_draw()), INNER, TOP], expect((0, 0), [0, 3, 5, 15], may_start=[])),
    "nest_multiply": Scene(16, 16, [OUTER, L(3, FULL, draw(RED, blend=BlendMode.Multiply)), INNER, TOP],
                           expect((0, 0), [0, 3, 5, 15], may_start=[])),
    "nest_translucent": Scene(16, 16, [OUTER, L(3, FULL, draw(Color(1.0, 0.0, 0.0, 0.5))), INNER, TOP],
                              expect((0, 0), [0, 3, 5, 15], may_start=[])),
    # A full opaque layer that is clipped itself (not a first layer), and one whose full clip lifts its clipping (a first layer).
    "nest_clipped_opaque": Scene(16, 16, [L(0, (0, -4, 8.5, 20), clip(10)), L(3, FULL, draw(RED, clipped=True)), INNER, TOP],
                                 expect((0, 0), [0, 3, 5, 15], may_start=[])),
    "nest_full_clip_opaque": Scene(48, 16, [L(0, (-4, -4, 60, 20), clip(3)), L(3, FULL, draw(RED, clipped=True)), INNER,
                                            L(6, (2, -4, 14, 20), draw(GREEN, clipped=True))],
                                   expect((1, 0), [0, 3], mask=[3], full=[0, 3], may_start=[3], skip_clipping=[3])),
    # --- clip edge cases ---
    "clip_zero": Scene(32, 32, [L(0, (0, 0, 30, 30), draw(RED)), L(1, (4, 4, 20.5, 20.5), clip(0)),
                                L(2, (2, 2, 28, 28), draw(GREEN, clipped=True)), L(3, (6, 6, 10, 10), clip(0)), L(4, (1, 1, 9, 9), draw(BLUE))],
                       expect((0, 0), [0, 1, 2, 3, 4], mask=[0, 4])),
    # Clip 0 covers tile (1, 0) as a carried cover: a full clip lifts the clipping of layers 1 and 2.
    "clip_full": Scene(48, 16, [L(0, (-4, -4, 60, 20), clip(2)), L(1, (18, 2, 29.5, 13), draw(GREEN, clipped=True)),
                                L(2, (16, 0, 32, 16), draw(BLUE, clipped=True)), L(3, (20, 4, 26, 10), draw(RED, clipped=True))],
                       expect((1, 0), [0, 1, 2, 3], mask=[1, 2], full=[0], skip_clipping=[1, 2])),
    # Unused clips are not painted; their planes are their own coverage.
    "clip_unused": Scene(32, 32, [L(0, (3, 3, 20.5, 27), clip(1)), L(2, (8, 8, 24, 24), draw(RED)), L(3, (6, 1, 30, 18), clip(5)),
                                  L(11, (2, 2, 31, 31), draw(GREEN, clipped=True))],
                         expect((0, 0), [0, 2, 3, 11], mask=[2])),
    # A clip replaced by the next one before its range ends stays painted, used or not (skip_trivial_clips only
    # drops the clip it tracks).
    "clip_replaced": Scene(32, 32, [L(0, (3, 3, 20.5, 27), clip(1)), L(1, (8, 8, 24, 24), draw(RED)), L(2, (6, 1, 30, 18), clip(5)),
                                    L(9, (2, 2, 31, 31), draw(GREEN, clipped=True))],
                           expect((0, 0), [0, 1, 2, 9], mask=[0, 1])),
    "clip_disabled": Scene(32, 32, [L(0, (3, 3, 28.5, 27), clip(10)), L(1, (1, 1, 14, 30), clip(10), False),
                                    L(2, (2, 2, 31, 31), draw(GREEN, clipped=True)), L(3, (6, 1, 30, 18), clip(1), False),
                                    L(4, (2, 5, 20, 31), draw(BLUE, clipped=True))],
                           expect((0, 0), [0, 2, 4], mask=[0, 2, 4])),
    "clip_none_below": Scene(32, 32, [L(0, (2, 2, 31, 31), draw(GREEN, clipped=True)), L(1, (1, 1, 18, 18), draw(RED)),
                                      L(2, (4, 4, 28, 28), draw(BLUE, clipped=True))],
                             expect((0, 0), [0, 1, 2], mask=[1])),
    # An EvenOdd clip of winding 2: coverage 0 wherever it has segments, an empty carry elsewhere. Where it is an entry
    # it still opens the clip state, so layer 2 is painted with a zero mask there.
    "clip_even_odd_zero": Scene(64, 32, [L(0, (0, 0, 64, 32), draw(RED)),
                                         L(1, [(8, 4, 40, 28), (8, 4, 40, 28)], clip(4, FillRule.EvenOdd)),
                                         L(2, (2, 2, 62, 30), draw(GREEN, clipped=True)), L(3, (4, 8, 60, 24), clip(4)),
                                         L(4, (2, 6, 62, 26), draw(BLUE, clipped=True))],
                                all_of(expect((0, 0), [0, 1, 2, 3, 4], mask=[0, 1, 2, 3, 4]), expect_entries((1, 0), [0, 2, 3, 4]),
                                       lambda m: [(e.cov == 0).all() for e in m.tiles[0, 0] if e.order == 1] == [True])),
    # --- clip ranges near 2^32 (the order plus the range wraps, or just does not) ---
    "range_u32_max": Scene(32, 16, [L(0, (0, 0, 32, 16), draw(RED)), L(1, (2, 2, 20.5, 14), clip(0xFFFFFFFF)),
                                    L(2, (1, 1, 30, 15), draw(GREEN, clipped=True))],
                           expect((0, 0), [0, 1, 2], mask=[0])),
    "range_u32_max_minus_1": Scene(32, 16, [L(0, (0, 0, 32, 16), draw(RED)), L(1, (2, 2, 20.5, 14), clip(0xFFFFFFFE)),
                                            L(2, (1, 1, 30, 15), draw(GREEN, clipped=True))],
                                   expect((0, 0), [0, 1, 2], mask=[0, 1, 2])),
    "range_u32_minus_2p20": Scene(32, 16, [L(0, (0, 0, 32, 16), draw(RED)), L(1, (2, 2, 20.5, 14), clip(0xFFFFFFFF - (1 << 20))),
                                           L(2, (1, 1, 30, 15), draw(GREEN, clipped=True)),
                                           L((1 << 20) + 1, (3, 3, 26.5, 13), clip(0xFFFFFFFF - (1 << 20))),
                                           L((1 << 20) + 2, (1, 4, 30, 12), draw(BLUE, clipped=True))],
                                  expect((0, 0), [0, 1, 2, (1 << 20) + 1, (1 << 20) + 2], mask=[0, 1, 2]),
                                  windows=[((1 << 20) + 1, 2)]),
}


# --- heavy tiles ---------------------------------------------------------------------------------------------


def heavy(n, clips):
    """n entries in tile (0, 0) of a 32 x 32 frame: small rects, every 8th a clip of the next 6 (clips) or none."""
    layers = []
    for i in range(n):
        x0, y0 = (i * 5) % 11 + 0.25 * (i % 4), (i * 7) % 11 + 0.5 * (i % 2)
        r = (x0, y0, x0 + 3.5 + i % 3, y0 + 4.25)
        if clips and i % 8 == 0:
            props = clip(6)
        elif clips and i % 8 in (1, 2, 3, 5, 7):
            props = draw(Color(0.1 * (i % 10), 0.5, 1.0, 1.0), clipped=True)
        else:
            props = draw(Color(0.1 * (i % 10), 0.3, 0.6, 0.5 + 0.5 * (i % 2)))
        layers.append(L(i, r, props))
    check = expect_entries((0, 0), list(range(n)))
    windows = [(f, k) for f in (31, 32, 33) if f < n for k in (1, 3)] + [(n - 1, 2)]
    return Scene(32, 32, layers, check, windows)


for _n in (15, 16, 31, 32, 33, 64, 65, 257):
    SCENES[f"heavy_{_n}"] = heavy(_n, False)
    SCENES[f"heavy_{_n}_clips"] = heavy(_n, True)

# --- windows ---------------------------------------------------------------------------------------------------

SCENES["windows"] = Scene(48, 32, [L(0, (0, 0, 48, 32), draw(RED)), L(1, (3, 2, 40.5, 30), clip(5)),
                                   L(2, (1, 1, 46, 31), draw(GREEN, clipped=True)), L(4, (5, 5, 30, 30), draw(BLUE, clipped=True)),
                                   L(5, (2, 2, 20, 20), draw(BLUE)), L(6, (1, 1, 44, 20), draw(GREEN, clipped=True)),
                                   L(9, (4, 4, 44, 28), clip(3)), L(11, (1, 1, 46, 31), draw(RED, clipped=True)),
                                   L(LAYER_LIMIT, (7, 3, 27.5, 19), draw(GREEN))],
                          expect((0, 0), [0, 1, 2, 4, 5, 6, 9, 11, LAYER_LIMIT], mask=[0, 1, 2, 4, 5, 6, 9, 11, LAYER_LIMIT]),
                          # K = 1 on a clip, a clipped layer, an absent order; starting and ending inside clip ranges
                          windows=[(1, 1), (2, 1), (3, 1), (9, 1), (11, 1), (2, 3), (4, 2), (0, 3), (10, 2), (6, 5),
                                   (LAYER_LIMIT, 1), (LAYER_LIMIT - 1, 2)])

# --- frame edges: full layers over partial edge tiles ---------------------------------------------------------

for _w, _h in ((1, 17), (7, 15), (8, 1), (9, 17), (15, 15), (17, 1), (17, 17)):
    SCENES[f"edge_{_w}x{_h}"] = Scene(_w, _h, [L(0, (-8, -8, 40, 40), draw(RED)), L(1, (-8, -8, 40, 40), draw(Color(0.0, 0.5, 1.0, 0.5))),
                                               L(2, (0.5, -8, 40, 12.5), clip(1)), L(3, (-8, 0.5, 40, 40), draw(GREEN, clipped=True)),
                                               L(4, (-8, -8, 3.5, 40), draw(BLUE))],
                                      # (at width 1 the rasterizer leaves layer 4 no segments: it is carried in full)
                                      expect((0, 0), [0, 1, 2, 3, 4], full=[0, 1, 4] if _w < 4 else [0, 1],
                                             may_start=[0, 4] if _w < 4 else [0]))

# --- thresholds: coverage 0.5 x clip 0.5 = 0.25 exactly ---------------------------------------------------------

SCENES["quarter"] = Scene(32, 32, [L(0, (0, 0, 32, 32), draw(RED)), L(1, (0, 0, 10.5, 32), clip(2)),
                                   L(2, (10, 0, 30, 32), draw(GREEN, clipped=True)), L(3, (0, 0, 20.5, 32), draw(BLUE)),
                                   L(4, (20, 0, 32, 32), draw(GREEN))],
                          all_of(expect((0, 0), [0, 1, 2, 3], mask=[0, 1, 2, 3]), expect_entries((1, 0), [0, 2, 3, 4])))


def props_of(sc):
    """{order: Props} of the scene's enabled layers (the model's input)."""
    return {o: p if p is not None else Props() for o, _, p, enabled in sc.layers if enabled}
