"""Scenes for the painter's per-pixel styling: fills, blend modes, clips and fill rules at their
limits on every paint path, with hostile colours, degenerate gradients, textures sampled off
their edges and values that straddle the sRGB and f16 encoders. Every scene is a pure function
of its name; its builder takes `(api, comp)` so that the CUDA library and the oracle build the
same composition, and records the props of every layer it styled so that `PathModel` can
tell, from the oracle's segments, which of the painter's paths each (tile, layer) takes:

  fold     every visible layer of the tile is full and solid (blend_solid, one colour)
  fast     solid fill, BlendMode::Over (the inline pair arithmetic)
  pair     separable mode (< 12), solid or 2-4-stop gradient (blend_pair_separable, GradRec)
  generic  textures, gradients of 5+ stops, the four non-separable modes (blend_pixel_generic)

plus `masked` (clipped outside any clip, or a clip nothing uses), `culled` (under the top-most
full opaque layer), `zero` (no coverage in the tile, or clipped with no clip active) and `clip`.
The declared conditions of each scene (`Built.expect` and `Built.check`) are proved by
tests/test_style_scenes.py without a GPU; tests/test_gpu_styles.py compares the device with
the oracle at tolerance 0.

Cells sit on even tile columns and rows, so that a cell's clip can reach past its tile into
empty tiles. All coordinates are multiples of 1/4 and every colour is float32-exact."""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional

import numpy as np

from synth import SplitMix64, f32
from forma_b200.binding import (BlendMode, Color, Fill, FillRule, Func, GradientBuilder, GradientType, Point, Props,
                                Style, Texture, unpack_segments)

INF, NAN = float("inf"), float("nan")
SUB_MIN, SUB_MAX = float(np.float32(2.0 ** -149)), float(np.nextafter(np.float32(2.0 ** -126), np.float32(0)))
ONE_DOWN, ONE_UP = float(np.nextafter(np.float32(1), np.float32(0))), float(np.nextafter(np.float32(1), np.float32(2)))
ALPHAS = (0.0, 1.0, ONE_DOWN, ONE_UP, 2.0, -0.5)
# Values the separable modes branch on (dodge, burn, hard and soft light: 0, 0.25, 0.5, 1), exact.
EXACT = (0.0, 0.25, 0.5, 1.0, 0.75, 1.5, 2.0, 0.125, 3.0)
# Backdrop texels: exact for the texel conversion (f16_from), including -0 and negative values,
# which it maps to +0 and |v|.
BACKDROP = (0.0, -0.0, 0.25, 0.5, 1.0, 0.75, 1.5, 2.0, 0.125, -0.5, 3.0)
BACKDROP_ALPHA = (1.0, 1.0, 1.0, 0.5, 1.0, 0.25, 1.0, 0.0)

PATHS = ("fold", "fast", "pair", "generic")


@dataclass
class Built:
    layers: Dict[int, Props] = field(default_factory=dict)
    # (layer, (tile_x, tile_y) or None, path, needs an inactive f32x8 group, needs a pair with
    # one active and one inactive column): each must hold in the path model.
    expect: List[tuple] = field(default_factory=list)
    # check(model) -> list of failed conditions, for conditions over the whole scene.
    check: Optional[Callable] = None
    notes: dict = field(default_factory=dict)


@dataclass
class StyleScene:
    build: Callable
    width: int
    height: int
    clear: Color = Color(1.0, 1.0, 1.0, 1.0)
    family: str = ""
    tags: tuple = ()


def rect(x0, y0, x1, y1):
    return [(x0, y0), (x0, y1), (x1, y1), (x1, y0)]


def path(api, contours):
    pb = api.PathBuilder()
    for c in contours:
        pb.move_to(Point(f32(c[0][0]), f32(c[0][1])))
        for x, y in c[1:]:
            pb.line_to(Point(f32(x), f32(y)))
    return pb.build()


def add(api, comp, b: Built, order: int, contours, props: Props):
    comp.get_mut_or_insert_default(order).insert(path(api, contours)).set_props(props)
    b.layers[order] = props


def draw(fill: Fill, mode=BlendMode.Over, rule=FillRule.NonZero, clipped=False) -> Props:
    return Props(fill_rule=rule, func=Func.Draw(Style(fill=fill, blend_mode=mode, is_clipped=clipped)))


def gradient(start, end, colors, stops=None, radial=False):
    gb = GradientBuilder(Point(f32(start[0]), f32(start[1])), Point(f32(end[0]), f32(end[1])))
    if radial:
        gb.type(GradientType.Radial)
    for k, c in enumerate(colors):
        s = None if stops is None else stops[k]
        if s is None:
            gb.color(c)
        else:
            gb.color_with_stop(c, s)
    return Fill.Gradient(gb.build())


def backdrop(api, comp, b: Built, w: int, h: int, order: int = 0):
    """A whole-frame texture layer whose texel (x, y) is pixel (x, y): exact values per pixel."""
    y, x = np.mgrid[0:h, 0:w]
    img = np.zeros((h, w, 4), np.float32)
    for c in range(3):
        img[..., c] = np.array(BACKDROP, np.float32)[(3 * x + 5 * y + 7 * c) % len(BACKDROP)]
    img[..., 3] = np.array(BACKDROP_ALPHA, np.float32)[(x + 2 * y) % len(BACKDROP_ALPHA)]
    add(api, comp, b, order, [rect(-1.0, 0.0, w + 1.0, h)], draw(Fill.Texture(Texture((1.0, 0.0, 0.0, 1.0, 0.0, 0.0), img))))


def exact_color(rng: SplitMix64, alphas=(1.0, 0.5, 0.75)) -> Color:
    return Color(EXACT[rng.randint(len(EXACT))], EXACT[rng.randint(len(EXACT))], EXACT[rng.randint(len(EXACT))],
                 alphas[rng.randint(len(alphas))])


# ---------------------------------------------------------------------------
# The path matrix
# ---------------------------------------------------------------------------
# (name, stops, radial, texture); stops 0: solid
FILLS = {"solid": (0, False, False), "lin2": (2, False, False), "lin3": (3, False, False), "lin4": (4, False, False),
         "lin5": (5, False, False), "lin16": (16, False, False), "rad2": (2, True, False), "rad4": (4, True, False),
         "rad5": (5, True, False), "tex": (0, False, True)}
CLIPS = ("none", "partial", "full", "outside")
CELL_TEXTURE = np.array([[[EXACT[(3 * i + j + c) % len(EXACT)] for c in range(3)] + [(1.0, 0.5, 0.75)[(i + j) % 3]]
                          for j in range(5)] for i in range(3)], np.float32)  # 3 x 5


def cell_shape(x0, y0):
    """Two overlapping rectangles in rows 2-6 and columns 3-9 of the tile at (x0, y0): column 2
    and rows 8-15 stay empty (pair (2, 3) has one active column, the lower f32x8 groups none);
    the overlap winds twice (filled under NonZero, a hole under EvenOdd)."""
    return [rect(x0 + 3.0, y0 + 2.0, x0 + 6.5, y0 + 5.5), rect(x0 + 5.0, y0 + 4.0, x0 + 9.5, y0 + 6.75)]


def cell_fill(kind: str, x0, y0, colors: List[Color]) -> Fill:
    n, radial, tex = FILLS[kind]
    if tex:
        return Fill.Texture(Texture((0.5, 0.0, 0.0, 0.75, -0.5 * x0 - 1.0, -0.75 * y0 - 0.5), CELL_TEXTURE))
    if n == 0:
        return Fill.Solid(colors[0])
    if radial:
        return gradient((x0 + 3.0, y0 + 2.0), (x0 + 9.0, y0 + 6.0), colors[:n], radial=True)
    return gradient((x0 + 2.0, y0 + 0.0), (x0 + 10.0, y0 + 7.0), colors[:n])


def expected_path(kind: str, mode: int) -> str:
    n, _, tex = FILLS[kind]
    if n == 0 and not tex and mode == BlendMode.Over:
        return "fast"
    if mode < 12 and not tex and n <= 4:
        return "pair"
    return "generic"


def matrix(kinds, modes, clips, rules, palette: Callable):
    """Cells for every (kind, mode, clip, rule), 16 per tile row of cells (every other tile)."""
    cells = [(k, m, c, r) for k in kinds for c in clips for r in rules for m in modes]

    def build(api, comp):
        b = Built()
        cols = 16
        rows = (len(cells) + cols - 1) // cols
        backdrop(api, comp, b, 32 * cols, 32 * rows)
        rng = SplitMix64(len(cells) * 131 + len(kinds))
        order = 1
        for i, (kind, mode, clip, rule) in enumerate(cells):
            x0, y0 = 32.0 * (i % cols), 32.0 * (i // cols)
            colors = palette(rng)
            if clip == "partial":
                add(api, comp, b, order, [rect(x0 + 5.25, y0 + 0.5, x0 + 14.0, y0 + 7.5)], Props(func=Func.Clip(1)))
                order += 1
            elif clip == "full":  # reaches the cell's tile as a full carry only
                add(api, comp, b, order, [rect(x0 - 8.0, y0 - 8.0, x0 + 24.0, y0 + 24.0)], Props(func=Func.Clip(1)))
                order += 1
            add(api, comp, b, order, cell_shape(x0, y0), draw(cell_fill(kind, x0, y0, colors), mode, rule, clip != "none"))
            want = "masked" if clip == "outside" else expected_path(kind, mode)
            b.expect.append((order, (2 * (i % cols), 2 * (i // cols)), want, want != "masked", want != "masked"))
            b.notes.setdefault("cells", []).append((order, kind, mode, clip, rule, colors))
            order += 1
        return b
    rows = (len(cells) + 15) // 16
    return build, 512, 32 * rows


def exact_palette(rng):
    return [exact_color(rng) for _ in range(16)]


# ---------------------------------------------------------------------------
# Hostile colours
# ---------------------------------------------------------------------------
HOSTILE = {
    "beyond": (-2.5, -0.25, 1.25, 7.0, 65504.0, -1e6),
    "zeros": (0.0, -0.0),
    "subnormal": (SUB_MIN, -SUB_MIN, SUB_MAX, -SUB_MAX),
    "inf": (INF, -INF),
    "nan": (NAN,),
}
HOSTILE_CLEAR = {
    "beyond": Color(-0.5, 1.5, 0.25, 1.0),
    "zeros": Color(-0.0, 0.0, -0.0, 1.0),
    "subnormal": Color(SUB_MIN, -SUB_MAX, 0.5, 0.5),
    "inf": Color(0.5, INF, 0.25, 1.0),
    "nan": Color(0.5, 0.5, NAN, 1.0),
    "alpha": Color(0.25, 0.5, 0.75, ONE_UP),
}
HOSTILE_KINDS = ("solid", "lin2", "lin4", "lin5", "rad4")


def hostile_palette(cls: str, channel: Optional[int]):
    """Stop / solid colours: one value of the class in one channel (`channel`, or a random one,
    alpha included), exact values elsewhere; alphas from ALPHAS."""
    def pal(rng):
        out = []
        for _ in range(16):
            v = [EXACT[rng.randint(len(EXACT))] for _ in range(3)] + [ALPHAS[rng.randint(len(ALPHAS))]]
            if cls != "alpha":
                ch = channel if channel is not None else rng.randint(4)
                v[ch] = HOSTILE[cls][rng.randint(len(HOSTILE[cls]))]
            out.append(Color(*v))
        return out
    return pal


def fold_scene(palette: Callable, seed: int):
    """Sixteen tile rows, one per blend mode: in tile column 0 two full bands (that mode, then
    another) over the clear colour, in columns 2-3 the same bands above an opaque layer. The
    bands start left of those tiles, which hold them as full carries and fold to one colour."""
    def build(api, comp):
        b = Built()
        rng = SplitMix64(seed)
        order = 0
        for m in range(16):
            y0 = 16.0 * m
            cs = palette(rng)
            add(api, comp, b, order, [rect(-1.0, y0, 32.0, y0 + 16.0)], draw(Fill.Solid(cs[0]), m))
            add(api, comp, b, order + 1, [rect(-1.0, y0, 32.0, y0 + 16.0)], draw(Fill.Solid(cs[1]), (m + 5) % 16))
            # from tile 1 on: an opaque layer, then the same two bands again (tile 1 holds their
            # left edges and is painted per pixel; tiles 2-3 hold them as full carries)
            add(api, comp, b, order + 2, [rect(31.5, y0, 65.0, y0 + 16.0)], draw(Fill.Solid(Color(0.25, 0.5, 0.75, 1.0))))
            add(api, comp, b, order + 3, [rect(31.5, y0, 65.0, y0 + 16.0)], draw(Fill.Solid(cs[0]), m))
            add(api, comp, b, order + 4, [rect(31.5, y0, 65.0, y0 + 16.0)], draw(Fill.Solid(cs[1]), (m + 5) % 16))
            b.expect.append((order + 1, (0, m), "fold", False, False))
            for tx in (2, 3):
                b.expect.append((order + 4, (tx, m), "fold", False, False))
            order += 5
        return b
    return build, 64, 256


def defect(color: Color, clear_neg_zero=False):
    """The triangle (0, 0)-(4, 0)-(0, 6), solid Over, in a 16 x 16 frame: columns 0-3 of rows 0-7
    have coverage, every other f32x8 group of the tile has none and must keep the clear colour."""
    def build(api, comp):
        b = Built()
        add(api, comp, b, 0, [[(0.0, 0.0), (4.0, 0.0), (0.0, 6.0)]], draw(Fill.Solid(color)))
        b.expect.append((0, (0, 0), "fast", True, False))
        return b
    return build, 16, 16


# ---------------------------------------------------------------------------
# Gradient edges
# ---------------------------------------------------------------------------
def _cells_scene(cells, seed: int, h: int = 256):
    """cells: (name, fill(x0, y0, rng) -> Fill, mode, expected path, shape); one per tile pair."""
    def build(api, comp):
        b = Built()
        backdrop(api, comp, b, 512, h)
        rng = SplitMix64(seed)
        for i, (name, fill, mode, want, shape) in enumerate(cells):
            x0, y0 = 32.0 * (i % 16), 32.0 * (i // 16)
            add(api, comp, b, 1 + i, shape(x0, y0), draw(fill(x0, y0, rng), mode))
            b.expect.append((1 + i, (2 * (i % 16), 2 * (i // 16)), want, False, False))
            b.notes.setdefault("cells", []).append((1 + i, name))
        return b
    return build, 512, h


def tall(x0, y0):
    """Most of the tile, over both f32x8 groups of every column (one pixel column partly)."""
    return [rect(x0 + 0.5, y0 + 0.25, x0 + 16.0, y0 + 15.75)]


def _grad_cells():
    P = [Color(0.0, 1.0, 0.25, 1.0), Color(1.0, 0.5, 0.0, 0.5), Color(0.25, 0.0, 1.0, 1.0), Color(0.5, 0.75, 0.5, 0.75),
         Color(1.0, 0.25, 0.75, 1.0), Color(0.0, 0.0, 0.5, 0.25)]

    def g(start, end, n, stops=None, radial=False, origin=True):
        def f(x0, y0, rng):
            s = (x0 + start[0], y0 + start[1]) if origin else start
            e = (x0 + end[0], y0 + end[1]) if origin else end
            return gradient(s, e, [P[(k + int(x0) // 32) % len(P)] for k in range(n)], stops, radial)
        return f
    cases = [
        ("same_point_linear", g((5.0, 5.0), (5.0, 5.0), 3)),
        ("same_point_radial", g((5.0, 5.0), (5.0, 5.0), 3, radial=True)),
        ("dx0", g((3.0, 0.0), (3.0, 16.0), 4)),
        ("dy0", g((0.0, 3.0), (16.0, 3.0), 4)),
        ("far_start", g((-1e6, -3.0), (8.0, 12.0), 3, origin=False)),
        ("far_start_radial", g((1e6, 0.0), (1e6 + 8.0, 0.0), 2, radial=True, origin=False)),
        ("repeated", g((0.0, 0.0), (16.0, 8.0), 4, (0.0, 0.5, 0.5, 1.0))),
        ("repeated_ends", g((0.0, 0.0), (16.0, 8.0), 4, (0.0, 0.0, 1.0, 1.0))),
        ("decreasing", g((0.0, 0.0), (16.0, 8.0), 3, (1.0, 0.5, 0.0))),
        ("unsorted", g((0.0, 0.0), (16.0, 8.0), 4, (0.25, 0.75, 0.5, 1.0))),
        ("unsorted5", g((0.0, 0.0), (16.0, 8.0), 5, (0.25, 0.75, 0.5, 1.0, 0.125))),
        ("mixed_implicit", g((0.0, 0.0), (16.0, 8.0), 4, (None, 0.125, None, None))),
        ("inset", g((0.0, 0.0), (12.0, 12.0), 2, (0.25, 0.75))),
        ("inset4", g((0.0, 0.0), (12.0, 12.0), 4, (0.25, 0.375, 0.5, 0.75), radial=True)),
        ("on_stops4", g((0.0, 0.0), (16.0, 0.0), 4, (0.0, 3.0 / 16.0, 7.0 / 16.0, 1.0))),
        ("on_stops5", g((0.0, 0.0), (16.0, 0.0), 5, (0.0, 3.0 / 16.0, 7.0 / 16.0, 10.0 / 16.0, 1.0))),
        ("on_stops_radial", g((0.0, 0.0), (16.0, 0.0), 4, (0.0, 4.0 / 16.0, 8.0 / 16.0, 1.0), radial=True)),
        ("exactly4", g((2.0, 1.0), (14.0, 13.0), 4)),
        ("exactly5", g((2.0, 1.0), (14.0, 13.0), 5)),
        ("rows", g((0.0, 0.0), (1.0, 16.0), 3)),
    ]
    cells = []
    for name, f in cases:
        n = len(f(0.0, 0.0, None).gradient.stops)
        for mode in (BlendMode.Over, BlendMode.HardLight, BlendMode.SoftLight, BlendMode.Hue):
            want = "pair" if mode < 12 and n <= 4 else "generic"
            cells.append((f"{name}_{BlendMode.NAMES[mode]}", f, mode, want, tall))
    return cells


# ---------------------------------------------------------------------------
# Gradient stack: the one-entry-ahead GradRec load
# ---------------------------------------------------------------------------
STACK = 72
STACK_MASKED = (33, 34, 65, 66)  # tile A: positions 31, 32, 63, 64; B: 32, 33, 64, 65; C: 33, 34, 65, 66
STACK_ZERO = (20, 30, 40, 62, 71)


def gradient_stack(api, comp):
    """Tiles A (0, 0), B (2, 0) and C (4, 0) over a backdrop hold STACK gradient layers of 2-4 stops
    each with its own stops and colours and a separable mode; layer 1 reaches B and C, layer 2
    only C, which shifts the stack's positions by one and two entries. Layers STACK_MASKED are
    clipped outside any clip (masked out), layers STACK_ZERO wind twice under EvenOdd (segments,
    zero coverage)."""
    b = Built()
    backdrop(api, comp, b, 96, 16)
    add(api, comp, b, 1, [rect(32.0 + 1.0, 0.0, 96.0, 16.0)], draw(Fill.Solid(Color(0.5, 0.25, 1.0, 0.5)), BlendMode.Screen))
    add(api, comp, b, 2, [rect(64.0 + 2.0, 0.0, 96.0, 16.0)], draw(Fill.Solid(Color(1.0, 0.5, 0.0, 0.75)), BlendMode.Multiply))
    rng = SplitMix64(77)
    for i in range(STACK):
        order = 3 + i
        n = 2 + i % 3
        stops = sorted({0.0, 1.0} | {float(np.float32(rng.uniform(0.05, 0.95))) for _ in range(n - 2)})
        while len(stops) < n:
            stops.append(1.0)
        a, c = float(rng.randint(8)), float(rng.randint(8))
        contours = []
        for t in range(3):
            x0 = 32.0 * t
            if order in STACK_ZERO:
                r = rect(x0 + 1.0 + a, 1.0 + c, x0 + 9.0 + a, 9.0 + c)
                contours += [r, r]
            else:
                contours.append(rect(x0 + 0.25 * (1 + i % 7) + a, 0.5 + 0.25 * (i % 5), x0 + 7.5 + a, 8.25 + c))
        colors = [exact_color(rng, (1.0, 0.5, 0.75, 0.25)) for _ in range(n)]
        fill = gradient((1.0 + i % 5, 0.0), (15.0, 3.0 + i % 11), colors, stops, radial=i % 4 == 3)
        rule = FillRule.EvenOdd if order in STACK_ZERO else FillRule.NonZero
        add(api, comp, b, order, contours, draw(fill, i % 12, rule, clipped=order in STACK_MASKED))

    def check(model):
        fails, masked_at_boundary, pair_across = [], [], []
        for tile in ((0, 0), (2, 0), (4, 0)):
            ents = model.entries(tile)
            grads = [e for e in ents if e.small_gradient]
            if len(grads) < 65:
                fails.append(f"tile {tile}: {len(grads)} gradient entries")
            if not any(e.path == "zero" and e.small_gradient for e in ents):
                fails.append(f"tile {tile}: no zero-coverage gradient entry")
            path = {e.pos: e.path for e in ents}
            masked_at_boundary += [tile for p in (31, 32) if path.get(p) == "masked"]
            pair_across += [(tile, p) for p in (31, 63) if path.get(p) == path.get(p + 1) == "pair"]
        if not masked_at_boundary:
            fails.append("no tile has a masked entry at position 31 or 32")
        if {p for _, p in pair_across} != {31, 63}:
            fails.append(f"pair-path entries on both sides of a group boundary only at {pair_across}")
        return fails
    b.check = check
    return b


# ---------------------------------------------------------------------------
# Texture edges
# ---------------------------------------------------------------------------
H16 = {"zero": 0.0, "negzero": -0.0, "sub_min": 2.0 ** -24, "sub_max": 2.0 ** -14 - 2.0 ** -24, "max": 65504.0,
       "above": 1e5, "inf": INF, "nan": NAN, "neg": -0.75, "neg_big": -300.0, "one": 1.0, "half": 0.5}


def texel_image(w, h, seed):
    vals = list(H16.values())
    rng = SplitMix64(seed)
    img = np.zeros((h, w, 4), np.float32)
    for y in range(h):
        for x in range(w):
            img[y, x, :3] = [vals[rng.randint(len(vals))] for _ in range(3)]
            img[y, x, 3] = 1.0
    return img


def _tex_cells():
    big = float(2 ** 33)
    xfs = {
        "identity": lambda x0, y0: (1.0, 0.0, 0.0, 1.0, -x0, -y0),
        "past_edges": lambda x0, y0: (0.75, 0.25, -0.25, 0.75, -x0 * 0.75 - 3.0, -y0 * 0.75 + 2.0),
        "negative": lambda x0, y0: (1.0, 0.0, 0.0, 1.0, -1e4, -1e4),
        "above_2_32": lambda x0, y0: (1.0, 0.0, 0.0, 1.0, big, big),
        "huge_scale": lambda x0, y0: (3e38, 0.0, 0.0, -3e38, -x0 * 3e38, 0.0),
        "inf": lambda x0, y0: (INF, 0.0, 0.0, 1.0, 0.0, -y0),
        "neg_inf": lambda x0, y0: (1.0, 0.0, 0.0, -INF, -x0, 0.0),
        "nan": lambda x0, y0: (NAN, 0.0, 0.0, 1.0, 0.0, -y0),
        "nan_y": lambda x0, y0: (1.0, 0.0, NAN, 0.0, -x0, 0.0),
        "zero": lambda x0, y0: (0.0, 0.0, 0.0, 0.0, 2.0, 1.0),
        "fraction": lambda x0, y0: (0.37, 0.0, 0.0, 0.29, -x0 * 0.37 + 0.5, -y0 * 0.29 - 0.5),
    }
    sizes = {"1x1": (1, 1), "1xN": (1, 7), "Nx1": (9, 1), "5x4": (5, 4), "16x16": (16, 16)}
    cells = []
    k = 0
    for sname, (tw, th) in sizes.items():
        img = texel_image(tw, th, 31 + k)
        for xname, xf in xfs.items():
            def fill(x0, y0, rng, xf=xf, img=img):
                with np.errstate(over="ignore", invalid="ignore"):
                    return Fill.Texture(Texture(tuple(float(np.float32(v)) for v in xf(x0, y0)), img))
            mode = (BlendMode.Over, BlendMode.Multiply, BlendMode.Luminosity)[k % 3]
            cells.append((f"{sname}_{xname}", fill, mode, "generic", tall))
            k += 1
    return cells


# ---------------------------------------------------------------------------
# Encoder sweep
# ---------------------------------------------------------------------------
SWEEPS = [  # (r0, r1), (g0, g1), (b0, b1) across 256 columns
    ((-0.01, 0.01), (0.0, 0.0062616), (0.0031308, 0.0031309)),
    ((0.99, 1.01), (0.995, 1.0001), (0.0, 1.0)),
    ((0.2, 0.21), (0.5, 0.502), (0.7, 0.7012)),
    ((65480.0, 65540.0), (1.0, 1.0 + 2.0 ** -9), (2.0 ** -15, 2.0 ** -13)),
]
# Solid colours painted once as a folded tile and once per pixel: the sRGB knee, byte
# boundaries and their neighbours, f16 halfway values and values above 65504.
ENC_COLORS = [
    Color(0.0031308, float(np.nextafter(np.float32(0.0031308), np.float32(1))), 0.04045, 1.0),
    Color(0.5 / 255.0, 1.5 / 255.0, 254.5 / 255.0, 1.0),
    Color(1.0 + 2.0 ** -11, 1.0 + 3.0 * 2.0 ** -11, 2048.0 + 1.0, 1.0),
    Color(65504.0, 65519.0, 65520.0, 1.0),
    Color(1e6, -65520.0, 2.0 ** -25, 1.0),
    Color(-0.0, 2.0 ** -24 * 1.5, 0.999, 1.0),
    Color(0.2140, 0.2141, 0.7354, 1.0),
    Color(NAN, 0.5, -INF, 1.0),
]


def encoder_sweep(api, comp):
    """Rows 0-63: four horizontal 2-stop gradients (16 rows each) across 256 columns with the
    ranges of SWEEPS, painted per pixel over an opaque solid layer. Rows 64-191: per colour of
    ENC_COLORS a tile row whose tiles 0-7 fold to the colour (a full band) and whose tiles 8-15
    paint it per pixel (the same band, then a tiny zero-alpha layer in every tile above it)."""
    b = Built()
    add(api, comp, b, 0, [rect(-1.0, 0.0, 257.0, 64.0)], draw(Fill.Solid(Color(0.0, 0.0, 0.0, 1.0))))
    for i, (r, g, bb) in enumerate(SWEEPS):
        y0 = 16.0 * i
        cs = [Color(r[0], g[0], bb[0], 1.0), Color(r[1], g[1], bb[1], 1.0)]
        add(api, comp, b, 1 + i, [rect(-1.0, y0, 257.0, y0 + 16.0)], draw(gradient((0.0, y0), (255.0, y0), cs)))
        for tx in range(16):
            b.expect.append((1 + i, (tx, i), "pair", False, False))
    order = 10
    for j, c in enumerate(ENC_COLORS):
        y0 = 64.0 + 16.0 * j
        add(api, comp, b, order, [rect(-1.0, y0, 257.0, y0 + 16.0)], draw(Fill.Solid(c)))
        specks = [rect(128.0 + 16.0 * t + 7.25, y0 + 9.0, 128.0 + 16.0 * t + 7.75, y0 + 9.5) for t in range(8)]
        add(api, comp, b, order + 1, specks, draw(Fill.Solid(Color(0.25, 0.5, 0.75, 0.0))))
        for tx in range(8):
            b.expect.append((order, (tx, 4 + j), "fold", False, False))
            b.expect.append((order + 1, (8 + tx, 4 + j), "fast", True, True))
        order += 2
    b.notes["solid_rows"] = [(4 + j, c) for j, c in enumerate(ENC_COLORS)]
    return b


# ---------------------------------------------------------------------------
# Registry
# ---------------------------------------------------------------------------
SCENES: Dict[str, StyleScene] = {}


def _reg(name, spec, clear=Color(1.0, 1.0, 1.0, 1.0), family="", tags=()):
    build, w, h = spec
    SCENES[name] = StyleScene(build, w, h, clear, family, tags)


for _k in FILLS:  # 16 modes x 4 clips x 2 rules per fill
    _reg(f"matrix_{_k}", matrix((_k,), range(16), CLIPS, (FillRule.NonZero, FillRule.EvenOdd), exact_palette),
         Color(0.25, 0.5, 0.75, 0.5), "matrix")
_reg("fold_exact", fold_scene(exact_palette, 5), Color(0.5, 0.25, 1.0, 0.5), "fold")
for _cls in list(HOSTILE) + ["alpha"]:
    _channels = (0, 3) if _cls in ("nan", "inf") else (None,)
    for _ch in _channels:
        _nm = _cls if _ch is None else f"{_cls}_{'rgba'[_ch]}"
        _reg(f"hostile_{_nm}", matrix(HOSTILE_KINDS, range(16), ("none", "partial"), (FillRule.NonZero,),
                                      hostile_palette(_cls, _ch)), HOSTILE_CLEAR[_cls], "hostile", (_cls,))
        _reg(f"fold_{_nm}", fold_scene(hostile_palette(_cls, _ch), 11 + len(SCENES)), HOSTILE_CLEAR[_cls], "fold", (_cls,))
for _nm, _c in (("nan_r", Color(NAN, 0.2, 0.2, 1.0)), ("inf_r", Color(INF, 0.2, 0.2, 1.0)), ("inf_a", Color(0.5, 0.2, 0.2, INF))):
    _reg(f"defect_{_nm}", defect(_c), Color(1.0, 1.0, 1.0, 1.0), "defect")
_reg("defect_neg_zero_clear", defect(Color(0.5, 0.2, 0.2, 1.0)), Color(-0.0, 0.5, 0.5, 1.0), "defect")
_reg("gradient_edges", _cells_scene(_grad_cells(), 3, 32 * ((len(_grad_cells()) + 15) // 16)), Color(0.5, 0.5, 0.5, 1.0),
     "gradient")
_reg("gradient_stack", (gradient_stack, 96, 16), Color(0.25, 0.25, 0.25, 1.0), "stack")
_reg("texture_edges", _cells_scene(_tex_cells(), 9, 32 * ((len(_tex_cells()) + 15) // 16)), Color(0.0, 0.0, 0.0, 1.0),
     "texture")
_reg("encoder_sweep", (encoder_sweep, 256, 192), Color(0.0, 0.0, 0.0, 1.0), "encoder")


def build(api, name: str):
    """(composition, Built, StyleScene) of scene `name` for `api`."""
    sc = SCENES[name]
    comp = api.Composition()
    return comp, sc.build(api, comp), sc


# ---------------------------------------------------------------------------
# The path model
# ---------------------------------------------------------------------------
@dataclass
class Entry:
    layer: int
    pos: int             # position in the tile's entry list
    path: str
    small_gradient: bool
    cov: np.ndarray      # (16, 16) coverage in the tile
    active: np.ndarray   # (2, 16) f32x8 group (half, column) has non-zero coverage


def _wrap_i8(v):
    return ((np.asarray(v, np.int64) + 128) % 256) - 128


class PathModel:
    """The painter's decisions per (tile, layer), from the oracle's sorted segments and the
    scene's props: which entries a tile holds (cells or carries), the clip and cull passes,
    the fold, and then per entry the path and the f32x8 activity of blend_at."""

    def __init__(self, segs: np.ndarray, width: int, height: int, layers: Dict[int, Props]):
        self.w, self.h, self.layers = width, height, layers
        s = unpack_segments(segs)
        x = s["tile_x"].astype(np.int64) * 16 + s["local_x"]
        y = s["tile_y"].astype(np.int64) * 16 + s["local_y"]
        self.tx_n, self.ty_n = (width + 15) // 16, (height + 15) // 16
        W, H = 16 * self.tx_n, 16 * self.ty_n
        self.cov, self.has_segs = {}, {}
        for layer in np.unique(s["layer_id"]):
            layer = int(layer)
            m = (s["layer_id"] == layer) & (y >= 0) & (y < H)
            xs, ys, da, cv = x[m], y[m], s["double_area"][m].astype(np.int64), s["cover"][m].astype(np.int64)
            area = np.zeros((H, W), np.int64)
            ins = (xs >= 0) & (xs < W)
            np.add.at(area, (ys[ins], xs[ins]), da[ins])
            cov_col = np.zeros((H, W + 1), np.int64)
            np.add.at(cov_col, (ys, np.clip(xs + 1, 0, W)), cv)
            run = np.cumsum(cov_col, axis=1)
            d = area + 32 * _wrap_i8(run[:, :W])
            rule = layers[layer].fill_rule if layer in layers else FillRule.NonZero
            if rule == FillRule.NonZero:
                c = np.minimum(np.abs(d) / 512.0, 1.0)
            else:
                c = (512 - np.abs((d & 1023) - 512)) / 512.0
            self.cov[layer] = c.astype(np.float32)
            hs = np.zeros((self.ty_n, self.tx_n), bool)
            tin = ins & (ys >= 0)
            hs[ys[tin] // 16, xs[tin] // 16] = True
            self.has_segs[layer] = (hs, run)
        self._tiles = {}

    def _carry(self, layer, tx, ty):
        _, run = self.has_segs[layer]
        return _wrap_i8(run[16 * ty:16 * ty + 16, 16 * tx])

    def entries(self, tile) -> List[Entry]:
        if tile in self._tiles:
            return self._tiles[tile]
        tx, ty = tile
        raw = []
        for layer in sorted(self.cov):
            hs, _ = self.has_segs[layer]
            carry = self._carry(layer, tx, ty)
            rule = self.layers[layer].fill_rule
            segs = bool(hs[ty, tx])
            empty = np.all(carry == 0) if rule == FillRule.NonZero else np.all((np.abs(carry) & 31) == 0)
            if not segs and empty:
                continue
            a = _wrap_i8(np.abs(carry))
            full = not segs and (np.all(a == 16) if rule == FillRule.NonZero else np.all((a & 31) == 16))
            raw.append([layer, segs, full])
        flags = []
        for layer, segs, full in raw:
            p = self.layers[layer]
            st = p.func.draw
            f = {"full": full, "clip": p.func.clip is not None, "clipped": st is not None and st.is_clipped,
                 "masked": False, "skip_clip": False}
            f["opaque"] = (st is not None and st.fill.solid is not None and st.blend_mode == 0 and st.fill.solid.a == 1.0)
            flags.append(f)
        # skip_trivial_clips (paint_kernel_body.cuh Pass B)
        has_clip, clip_full, clip_used, clip_last, clip_i = False, False, False, 0, 0
        for i, (layer, _, _) in enumerate(raw):
            f = flags[i]
            if not (f["clip"] or f["clipped"]):
                if has_clip and layer > clip_last:
                    has_clip = False
                    if not clip_used:
                        flags[clip_i]["masked"] = True
                continue
            if f["clip"]:
                clip_full, clip_last, clip_i, clip_used, has_clip = f["full"], layer + self.layers[layer].func.clip, i, False, True
                if clip_full:
                    f["masked"] = True
            if f["clipped"]:
                if has_clip and layer <= clip_last:
                    if clip_full:
                        f["skip_clip"] = True
                    else:
                        clip_used = True
                else:
                    f["masked"] = True
            if has_clip and layer > clip_last:
                has_clip = False
                if not clip_used:
                    flags[clip_i]["masked"] = True
        if has_clip and not clip_used:
            flags[clip_i]["masked"] = True
        # skip_fully_covered_layers: the top-most full, unclipped, opaque layer
        first, incomplete = 0, False
        for i in range(len(raw) - 1, -1, -1):
            f = flags[i]
            if f["masked"]:
                continue
            clipped = f["clipped"] and not f["skip_clip"]
            if clipped or not f["full"]:
                incomplete = True
            elif f["opaque"]:
                first = i
                break
        folded = False
        if not incomplete:
            folded = all(flags[i]["masked"] or (self.layers[raw[i][0]].func.draw is not None
                                                and self.layers[raw[i][0]].func.draw.fill.solid is not None)
                         for i in range(first, len(raw)))
        out = []
        clip_active, clip_last = False, 0
        for i, (layer, _, _) in enumerate(raw):
            p, f = self.layers[layer], flags[i]
            st = p.func.draw
            cov = self.cov[layer][16 * ty:16 * ty + 16, 16 * tx:16 * tx + 16]
            active = np.stack([(cov[:8] != 0).any(axis=0), (cov[8:] != 0).any(axis=0)])
            small = st is not None and st.fill.gradient is not None and 2 <= len(st.fill.gradient.stops) <= 4
            if f["masked"]:
                path = "masked"
            elif i < first:
                path = "culled"
            elif folded:
                path = "fold"
            else:
                if clip_active and clip_last < layer:
                    clip_active = False
                if p.func.clip is not None:
                    if not clip_active:
                        clip_active, clip_last = True, layer + p.func.clip
                    path = "clip"
                elif not active.any() or (f["clipped"] and not f["skip_clip"] and not clip_active):
                    path = "zero"
                elif st.fill.solid is not None and st.blend_mode == 0:
                    path = "fast"
                elif st.blend_mode < 12 and (st.fill.solid is not None or small):
                    path = "pair"
                else:
                    path = "generic"
            out.append(Entry(layer, i, path, small, cov, active))
        self._tiles[tile] = out
        return out

    def entry(self, tile, layer) -> Optional[Entry]:
        for e in self.entries(tile):
            if e.layer == layer:
                return e
        return None

    def all_entries(self):
        for ty in range(self.ty_n):
            for tx in range(self.tx_n):
                for e in self.entries((tx, ty)):
                    yield (tx, ty), e

    def path_at(self, x: int, y: int) -> str:
        """The paths of the visible entries of the tile holding pixel (x, y), for reports."""
        ents = self.entries((x // 16, y // 16))
        return ", ".join(f"{e.layer}:{e.path}" for e in ents[-6:]) or "clear"


def mixed_pair(active: np.ndarray) -> bool:
    """Some pixel pair (2q, 2q + 1) of an active f32x8 group row has one active column and one inactive one."""
    return bool((active[:, 0::2] != active[:, 1::2]).any())


def check_expectations(model: PathModel, built: Built) -> List[str]:
    fails = []
    for layer, tile, want, need_inactive, need_mixed in built.expect:
        tiles = [tile] if tile is not None else [t for t, e in model.all_entries() if e.layer == layer]
        for t in tiles:
            e = model.entry(t, layer)
            if e is None:
                fails.append(f"layer {layer} has no entry in tile {t}")
                continue
            if e.path != want:
                fails.append(f"layer {layer} in tile {t}: path {e.path}, built for {want}")
            if need_inactive and (e.active.all() or not e.active.any()):
                fails.append(f"layer {layer} in tile {t}: no mix of active and inactive f32x8 groups")
            if need_mixed and not mixed_pair(e.active):
                fails.append(f"layer {layer} in tile {t}: no pixel pair with one active and one inactive column")
    if built.check is not None:
        fails += built.check(model)
    return fails


def value_classes(c: Color) -> set:
    """The hostile classes (HOSTILE keys, "alpha") that colour `c` carries."""
    out = set()
    for k, v in enumerate((c.r, c.g, c.b, c.a)):
        if v == 0.0 and math.copysign(1.0, v) > 0:
            continue  # +0 is an ordinary value; -0 is the hostile one
        for cls, vals in HOSTILE.items():
            if any((math.isnan(v) and math.isnan(u)) or (v == u and math.copysign(1, v) == math.copysign(1, u))
                   for u in vals):
                out.add(cls)
    if c.a in ALPHAS and c.a not in (1.0,):
        out.add("alpha")
    return out


def layer_colors(props: Props) -> List[Color]:
    st = props.func.draw
    if st is None:
        return []
    if st.fill.solid is not None:
        return [st.fill.solid]
    if st.fill.gradient is not None:
        return [c for c, _ in st.fill.gradient.stops]
    return []
