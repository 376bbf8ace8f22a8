"""Scenes at the limits of the painter and its tables: dense cells, deep winding, crowded
tiles and rasterizer extremes. Every builder takes `(api, comp)` like `scenes.py` and
`synth.py`, so the CUDA library and the oracle build identical compositions, and returns the
fill rule of every layer it styled (what `tables_model.py` needs besides the segments).

Moderate scenes never reach these paths: no cell of the other parity scenes has 2016
segments (the painter's packed-cell fold, a cell longer than one 2048-segment CTA tile of
the cells pass), no pixel sums an area beyond i16, no layer winds to a multiple of 8 or 16,
and clips appear only in 64x64 scenes with a handful of layers.

Pitfall when building dense geometry: consecutive lines whose direction changes by less than
`MAX_ANGLE_ERROR` are merged into one spline (path.rs:213-262), and the angle difference is
folded modulo pi, so a near-reversing zig-zag counts as "unchanged". A 2400-stroke zig-zag
inside one tile flattens to 3 points, while a 2000-stroke one gives 28 025 segments in one
cell. The builders below make dense geometry from strokes whose direction really changes
(the pixel star turns by about 137 degrees at every point) or from separate contours, and
`test_extremes_scenes.py` checks that every scene still reaches its target condition.

All coordinates are float32 (the builders hand float32 arrays or float32-exact values to the
path builder), and |coordinate| < 2^26 px: beyond that the float-to-int conversions of the
C++ oracle are undefined behaviour.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, Dict, Optional

import numpy as np

from synth import SplitMix64, f32
from forma_b200.binding import (BlendMode, Color, Fill, FillRule, Func, GradientBuilder, GradientType, Point, Props,
                                Rect, Style, Texture)

GOLDEN_ANGLE = 2.39996  # radians, about 137.5 degrees


def polyline(api, xy, contour_len: Optional[int] = None):
    """One path from float32 points (n, 2): a single closed contour, or contours of
    `contour_len` points each."""
    xy = np.asarray(xy, np.float32).reshape(-1, 2)
    n = xy.shape[0]
    cmds = np.ones(n, np.uint8)
    cmds[0 if contour_len is None else slice(0, n, contour_len)] = 0
    return api.PathBuilder().extend(cmds, xy.ravel()).build()


def star_points(px: int, py: int, n: int) -> np.ndarray:
    """A "pixel star": n chords inside pixel (px, py), each turning by about 137 degrees.
    Closed, it gives exactly n pixel segments, all in one pixel."""
    ang = np.arange(n) * GOLDEN_ANGLE
    return np.stack([px + 0.5 + 0.45 * np.cos(ang), py + 0.5 + 0.45 * np.sin(ang)], 1).astype(np.float32)


def rect_points(x0, y0, x1, y1, reverse=False) -> np.ndarray:
    p = [(x0, y0), (x0, y1), (x1, y1), (x1, y0)]
    return np.array(p[::-1] if reverse else p, np.float32)


def solid(c: Color, rule=FillRule.NonZero, blend=BlendMode.Over, clipped=False) -> Props:
    return Props(fill_rule=rule, func=Func.Draw(Style(fill=Fill.Solid(c), blend_mode=blend, is_clipped=clipped)))


@dataclass
class Extreme:
    build: Callable
    width: int
    height: int
    crop: Optional[Rect] = None
    raster: bool = False  # also compare the unsorted segments of rasterize_only
    tags: tuple = ()


@dataclass
class Built:
    rules: Dict[int, int]
    animate: Optional[Callable] = None  # animate(frame): changes the composition between cached frames
    notes: dict = field(default_factory=dict)


# ---------------------------------------------------------------------------
# Dense cells
# ---------------------------------------------------------------------------
STAR_SIZES = (63, 64, 65, 2015, 2016, 2017, 2047, 2048, 2049, 4032, 4033, 6000)


def dense_stars(api, comp):
    """Every STAR_SIZES star in its own tile and layer, under both fill rules (NonZero in tile
    row 0, EvenOdd in tile row 2), over a translucent layer whose cover reaches the stars'
    tiles as a carry."""
    rules = {}
    under = comp.get_mut_or_insert_default(0)
    under.insert(polyline(api, rect_points(3.25, 2.5, 250.75, 61.5))).set_props(solid(Color(0.1, 0.6, 0.3, 0.5)))
    rules[0] = FillRule.NonZero
    for r, rule in enumerate((FillRule.NonZero, FillRule.EvenOdd)):
        for i, n in enumerate(STAR_SIZES):
            order = 1 + r * len(STAR_SIZES) + i
            px, py = 16 * i + (5 * i + 3) % 16, 32 * r + (7 * i + 2) % 16
            comp.get_mut_or_insert_default(order).insert(polyline(api, star_points(px, py, n))).set_props(
                solid(Color(0.9, f32(0.05 * i), 0.2, 0.85), rule))
            rules[order] = rule
    return Built(rules)


# Cells of one tile row in sorted order: starts at 0, 2048, 3048, 10048, 12288, 14336, 18432.
# The first ends on 2048, the second starts on it; the third spans CTA tiles 1-4 of the cells
# pass, two of which hold no cell head; the fourth ends on 12288; the fifth is exactly CTA tile
# 6; the sixth is exactly CTA tiles 7-8 (tile 8 without a head); the seventh starts on 18432.
BOUNDARY_CELLS = (2048, 1000, 7000, 2240, 2048, 4096, 65)


def cell_boundaries(api, comp):
    rules = {}
    for i, n in enumerate(BOUNDARY_CELLS):
        rule = FillRule.EvenOdd if i % 2 else FillRule.NonZero
        comp.get_mut_or_insert_default(i).insert(polyline(api, star_points(16 * i + 2 + i, 3 + 2 * i, n))).set_props(
            solid(Color(0.2, 0.3, f32(0.1 * i), 0.9), rule))
        rules[i] = rule
    return Built(rules)


SAW_CYCLES = 2500


def sawtooth(api, comp):
    """One entry with tens of thousands of segments over a whole tile: SAW_CYCLES strokes down
    pixel column 3 of tile (2, 1), each followed by a diagonal back up to another column and a
    horizontal step. The pixels of column 3 sum a cover of 16 * SAW_CYCLES, beyond i16: the
    painter's packed cells must fold it back to i8 before it carries into their area half."""
    x0, y0 = 32.0, 16.0
    pts = []
    for c in range(SAW_CYCLES):
        v = (3 + 1 + (c * 5) % 15) % 16  # never column 3
        pts += [(x0 + 3.5, y0), (x0 + 3.5, y0 + 16.0), (x0 + v + 0.25, y0)]
    backdrop = comp.get_mut_or_insert_default(0)
    backdrop.insert(polyline(api, rect_points(0.0, 0.0, 96.0, 48.0))).set_props(solid(Color(0.0, 0.1, 0.3, 1.0)))
    comp.get_mut_or_insert_default(1).insert(polyline(api, pts)).set_props(solid(Color(1.0, 0.8, 0.1, 0.7)))
    comp.get_mut_or_insert_default(2).insert(polyline(api, pts)).set_props(
        solid(Color(0.3, 0.8, 0.9, 0.6), FillRule.EvenOdd))
    return Built({0: FillRule.NonZero, 1: FillRule.NonZero, 2: FillRule.EvenOdd})


# ---------------------------------------------------------------------------
# Deep winding
# ---------------------------------------------------------------------------
WINDINGS = (7, 8, 9, 15, 16, 17, 127, 128, 129, 255, 256, 257, 300)
WIND_W, WIND_H = 320, 32 * len(WINDINGS)


def deep_winding(how: str, rule: int):
    """K coincident copies of a rectangle with fractional edges, one layer per K of WINDINGS
    (tile rows 2j, 2j + 1), over an opaque backdrop. how: "insert" (K inserts of one path into
    the layer), "contours" (one path of K contours) or "mixed" (contours, every fourth one
    reversed). Even layers are translucent (a dropped carry shows), odd ones opaque."""
    def build(api, comp):
        rules = {0: FillRule.NonZero}
        comp.get_mut_or_insert_default(0).insert(polyline(api, rect_points(0.0, 0.0, WIND_W, WIND_H))).set_props(
            solid(Color(0.05, 0.1, 0.2, 1.0)))
        for j, k in enumerate(WINDINGS):
            y0 = 32.0 * j
            layer = comp.get_mut_or_insert_default(1 + j)
            if how == "insert":
                path = polyline(api, rect_points(19.25, y0 + 5.5, 300.75, y0 + 27.25))
                for _ in range(k):
                    layer.insert(path)
            else:
                pts = np.concatenate([rect_points(19.25, y0 + 5.5, 300.75, y0 + 27.25, reverse=how == "mixed" and i % 4 == 3)
                                      for i in range(k)])
                layer.insert(polyline(api, pts, contour_len=4))
            alpha = 0.6 if j % 2 == 0 else 1.0
            layer.set_props(solid(Color(0.9, f32(0.07 * j), 0.3, alpha), rule))
            rules[1 + j] = rule
        return Built(rules)
    return build


# ---------------------------------------------------------------------------
# Crowded tiles
# ---------------------------------------------------------------------------
CROWDS = (15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 1000, 5000)
CROWD_W, CROWD_H = 128, 64  # the crowd covers tiles x 2..5, y 1..2


def _texture(rng: SplitMix64) -> np.ndarray:
    h, w = 3 + rng.randint(5), 2 + rng.randint(6)
    img = np.array([[[rng.uniform(), rng.uniform(), rng.uniform(), rng.uniform(0.3, 1.0)] for _ in range(w)]
                    for _ in range(h)], np.float32)
    return img


def _gradient(rng: SplitMix64, i: int, cx: float, cy: float):
    n = 2 + i % 15  # 2..16 stops
    gb = GradientBuilder(Point(f32(cx - 20.0), f32(cy - 7.0)), Point(f32(cx + 25.0), f32(cy + 11.0)))
    if rng.randint(2):
        gb.type(GradientType.Radial)
    if i % 3 == 0:  # explicit stops: uneven and repeated
        stops = sorted(rng.uniform() for _ in range(n))
        if n > 2:
            stops[1] = stops[0]
            stops[-1] = 1.0
        for s in stops:
            gb.color_with_stop(Color(rng.uniform(), rng.uniform(), rng.uniform(), rng.uniform(0.3, 1.0)), s)
    else:
        for _ in range(n):
            gb.color(Color(rng.uniform(), rng.uniform(), rng.uniform(), rng.uniform(0.3, 1.0)))
    return gb.build()


def crowd_clip_role(i: int, n: int):
    """("clip", clip_layers) / ("clipped", None) / (None, None) of layer i of a crowd of n."""
    m = i % 64
    if m == 29:
        return "clip", 6          # 30..35: straddles a 32-entry group when the tile holds every layer
    if m == 13:
        return "clip_carry", 3    # a clip that reaches the middle tiles only as a carry
    if m == 40:
        return "clip", 1          # back-to-back clips: 40 (41), 42 (43, 44)
    if m == 42:
        return "clip", 2
    if 30 <= m <= 35 or 14 <= m <= 16 or m in (41, 43, 44) or m == 50:  # 50: clipped, outside any clip
        return "clipped", None
    return None, None


def crowded(n: int):
    """n layers over the tiles x 2..5, y 1..2 of a 128 x 64 frame: carry-only covers (rectangles
    whose edges lie outside the crowd), partial shapes, opaque solid Over layers at several depths
    (some covering only part of the crowd), gradients of 2-16 stops, rotated / scaled textures
    sampled beyond their edges, all 16 blend modes, and clips (see crowd_clip_role). `animate`
    moves a layer deep in the stack."""
    def build(api, comp):
        rng = SplitMix64(1000 + n)
        rules = {}
        opaque_at = {n // 4, n // 2, (3 * n) // 4}
        for i in range(n):
            role, clip_n = crowd_clip_role(i, n)
            kind = rng.randint(4)
            cx, cy = rng.uniform(32.0, 96.0), rng.uniform(16.0, 48.0)
            if role == "clip_carry" or kind == 0 or i in opaque_at:
                x0 = 5.25 + rng.randint(4) if i not in opaque_at else 32.0 + 16.0 * (i % 2)
                pts = rect_points(x0, 16.0 + rng.randint(3), 122.75 - rng.randint(4), 48.0 - rng.randint(3))
            elif kind == 1:  # triangle inside the crowd
                pts = np.array([(cx, cy), (f32(cx + rng.uniform(-30, 30)), f32(cy + rng.uniform(-20, 20))),
                                (f32(cx + rng.uniform(-30, 30)), f32(cy + rng.uniform(-20, 20)))], np.float32)
            elif kind == 2:  # a small quad polygon that may straddle tile edges
                e = rng.uniform(2.0, 12.0)
                pts = np.array([(cx - e, cy), (cx, cy - e), (cx + e, cy), (cx, cy + e)], np.float32)
            else:  # two contours, one of them reversed
                pts = np.concatenate([rect_points(f32(cx - 9.5), f32(cy - 5.25), f32(cx + 7.75), f32(cy + 6.5)),
                                      rect_points(f32(cx - 3.5), f32(cy - 2.25), f32(cx + 3.75), f32(cy + 2.5), reverse=True)])
            path = polyline(api, pts, contour_len=4 if kind == 3 and role != "clip_carry" and i not in opaque_at else None)
            rule = FillRule.EvenOdd if rng.randint(4) == 0 else FillRule.NonZero
            if role in ("clip", "clip_carry"):
                props = Props(fill_rule=rule, func=Func.Clip(clip_n))
            elif i in opaque_at:
                props = solid(Color(rng.uniform(), rng.uniform(), rng.uniform(), 1.0), rule)
            else:
                mode = i % 16
                fk = rng.randint(3)
                if fk == 0:
                    fill = Fill.Solid(Color(rng.uniform(), rng.uniform(), rng.uniform(), rng.uniform(0.2, 1.0)))
                elif fk == 1:
                    fill = Fill.Gradient(_gradient(rng, i, cx, cy))
                else:
                    a = rng.uniform(0.0, 6.283)
                    s = rng.uniform(0.05, 0.6)
                    ux, uy = f32(s * np.cos(a)), f32(s * np.sin(a))
                    fill = Fill.Texture(Texture((ux, uy, f32(-uy * 1.5), f32(ux * 1.5), rng.uniform(-6.0, 6.0),
                                                 rng.uniform(-6.0, 6.0)), _texture(rng)))
                props = Props(fill_rule=rule, func=Func.Draw(Style(fill=fill, blend_mode=mode,
                                                                   is_clipped=role == "clipped")))
            comp.get_mut_or_insert_default(i).insert(path).set_props(props)
            rules[i] = rule
        deep = n // 3

        def animate(frame: int):
            comp.get(deep).set_transform([1.0, 0.0, 0.0, 1.0, f32(0.25 * frame), f32(-0.5 * frame)])
        return Built(rules, animate, {"deep_layer": deep})
    return build


def nan_blends(api, comp):
    """Non-separable blend modes whose clip_color! divides by zero, so that a channel becomes NaN
    (the reference encodes such a channel as byte 0), and over a destination channel of 0.
    Tile column 0 is covered by whole layers only (the solid-tile fold, scalar blend); the other
    columns are painted per pixel. Luminosity of a colour outside [0, 1] over a grey backdrop:
    set_lum! leaves r = g = b = l with l > 1 (x - l = 0) or l < 0 (l - n = 0)."""
    rules = {}
    layers = [
        (rect_points(0.0, 0.0, 64.0, 32.0), solid(Color(0.5, 0.5, 0.5, 1.0))),
        (rect_points(16.0, 0.0, 32.0, 32.0), solid(Color(1.0, 0.0, 1.0, 1.0))),           # dst green = 0
        (rect_points(0.0, 0.0, 16.0, 32.0), solid(Color(1.5, 1.5, 1.5, 1.0), blend=BlendMode.Luminosity)),
        (np.array([(34.25, 2.5), (61.5, 9.75), (40.0, 29.5)], np.float32),
         solid(Color(-0.5, -0.5, -0.5, 0.9), blend=BlendMode.Luminosity)),
        (np.array([(17.5, 3.0), (30.25, 15.5), (18.0, 28.75)], np.float32),
         Props(func=Func.Draw(Style(fill=Fill.Texture(Texture((0.3, 0.1, -0.2, 0.45, 2.0, -3.0),
                                                              _texture(SplitMix64(5)))),
                                    blend_mode=BlendMode.Color)))),
        (np.array([(20.0, 20.0), (60.0, 16.0), (50.0, 31.0)], np.float32),
         Props(func=Func.Draw(Style(fill=Fill.Gradient(_gradient(SplitMix64(6), 7, 40.0, 20.0)),
                                    blend_mode=BlendMode.Hue)))),
        (np.array([(2.0, 30.0), (63.0, 1.0), (63.0, 30.0)], np.float32),
         solid(Color(0.0, 0.2, 0.9, 0.7), blend=BlendMode.Saturation)),
    ]
    for i, (pts, props) in enumerate(layers):
        comp.get_mut_or_insert_default(i).insert(polyline(api, pts)).set_props(props)
        rules[i] = props.fill_rule
    return Built(rules)


# ---------------------------------------------------------------------------
# Rasterizer extremes
# ---------------------------------------------------------------------------
def long_diagonal(api, comp):
    """One path of 256 lines (one CTA of the emit pass): the full 7680 x 4320 diagonal, then a
    zig-zag back along it (alternating sides: every line turns)."""
    k = np.arange(1, 255)
    t = 1.0 - k / 255.0
    side = np.where(k % 2 == 0, 1.0, -1.0) * (12.0 + (k % 7))
    back = np.stack([7680.0 * t + side * 0.49, 4320.0 * t - side * 0.87], 1)
    pts = np.concatenate([[(0.0, 0.0), (7680.0, 4320.0)], back]).astype(np.float32)
    comp.get_mut_or_insert_default(0).insert(polyline(api, pts)).set_props(solid(Color(0.2, 0.2, 0.8, 0.9)))
    return Built({0: FillRule.NonZero})


def grid_and_far(api, comp):
    """Lines exactly on pixel and tile grid lines, sub-1/16-px lines, and geometry far right of,
    below, left of and above the frame (up to 2^20 px: tile fields wrap as in PixelSegment::new)."""
    rules = {}
    shapes = [
        rect_points(16.0, 16.0, 64.0, 48.0),                     # tile grid
        rect_points(37.0, 5.0, 59.0, 91.0),                      # pixel grid
        rect_points(100.0, 100.0, 100.03125, 140.0),             # 1/32 px wide
        rect_points(120.0, 70.0, 180.0, 70.04),                  # sub-1/16 px tall
        np.array([(130.0, 130.0), (130.05, 130.02), (130.01, 130.06)], np.float32),  # sub-1/16 px triangle
        np.array([(200.0, 20.0), (1048576.0, 40.0), (1048576.0, 1048576.0), (220.0, 250.0)], np.float32),
        np.array([(-1048576.0, -1048576.0), (60.0, 200.0), (90.0, 1048576.0)], np.float32),
        np.array([(250.0, 250.0), (700000.0, 255.5), (250.5, 900000.0)], np.float32),
        rect_points(-3.0, 96.0, 260.0, 112.0),                   # across the whole frame on tile rows
        np.array([(0.0, 0.0), (256.0, 256.0), (0.0, 256.0)], np.float32),  # 45 degrees through tile corners
    ]
    for i, pts in enumerate(shapes):
        rule = FillRule.EvenOdd if i % 3 == 2 else FillRule.NonZero
        comp.get_mut_or_insert_default(i).insert(polyline(api, pts)).set_props(
            solid(Color(f32(0.09 * i), 0.5, 0.7, 0.75), rule))
        rules[i] = rule
    return Built(rules)


# ---------------------------------------------------------------------------
# Registry
# ---------------------------------------------------------------------------
SCENES: Dict[str, Extreme] = {
    "dense_stars": Extreme(dense_stars, 256, 64, tags=("dense",)),
    "cell_boundaries": Extreme(cell_boundaries, 128, 16, tags=("boundaries",)),
    "sawtooth": Extreme(sawtooth, 96, 48, tags=("sawtooth",)),
    "nan_blends": Extreme(nan_blends, 64, 32, tags=("nan",)),
    "long_diagonal": Extreme(long_diagonal, 7680, 4320, raster=True),
    "grid_and_far": Extreme(grid_and_far, 256, 256, raster=True),
}
for _how in ("insert", "contours", "mixed"):
    for _rn, _rule in (("nz", FillRule.NonZero), ("eo", FillRule.EvenOdd)):
        SCENES[f"winding_{_how}_{_rn}"] = Extreme(deep_winding(_how, _rule), WIND_W, WIND_H, tags=("winding",))
# A crop whose left edge lies inside the rectangles (tile 4, then mid-tile 75 px): the covers
# left of the painted columns reach them through the covers-left-of-row rule.
SCENES["winding_insert_nz_crop"] = Extreme(deep_winding("insert", FillRule.NonZero), WIND_W, WIND_H,
                                           Rect((64, WIND_W), (0, WIND_H)), tags=("winding", "crop"))
SCENES["winding_mixed_eo_crop"] = Extreme(deep_winding("mixed", FillRule.EvenOdd), WIND_W, WIND_H,
                                          Rect((75, 290), (0, WIND_H)), tags=("winding", "crop"))
for _n in CROWDS:
    SCENES[f"crowd_{_n}"] = Extreme(crowded(_n), CROWD_W, CROWD_H, tags=("crowd",))


def build(api, name: str):
    """(composition, Built, Extreme) of scene `name` for `api`."""
    sc = SCENES[name]
    comp = api.Composition()
    return comp, sc.build(api, comp), sc
