"""Scenes of instance calls (Renderer.render_instances_device): a library composition, a frame size
and the instance tables it is rendered with, plus `twin`, which builds frame b's composition T_b.

The library is a list of prototype specs (Proto): the layer at `order` with its live paths, their
path transform, its props, transform and enabled state, and optionally paths it held before a
Layer::clear (their inserts are dead and must not be drawn). Frame b of an instance call is the
ordinary frame of T_b: for every slot m with a prototype p, the layer at order m holds p's live
paths, p's props (with colours, a Draw fill becomes Solid(colors[b, m])), the transform
transforms[b, m] (or p's own without that table), and is enabled.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np

from forma_b200.binding import (BlendMode, Color, Fill, FillRule, Func, GradientBuilder, GradientType, Point, Props, Style,
                                Texture)

f32 = np.float32
NONE = 0xFFFFFFFF
IDENTITY = [1.0, 0.0, 0.0, 1.0, 0.0, 0.0]
LAYER_LIMIT = 1 << 21


@dataclass
class Proto:
    order: int
    paths: List[List[tuple]] = field(default_factory=list)  # live inserts, in insertion order
    path_xf: Optional[Sequence[float]] = None                # 9 values (Path.transform), every path
    props: Optional[Props] = None                            # None: a solid colour of its own
    xf: Optional[Sequence[float]] = None                     # [ux, vx, uy, vy, tx, ty]
    enabled: bool = False                                    # a library is usually kept disabled
    cleared: List[List[tuple]] = field(default_factory=list)  # inserted, then dropped by Layer::clear


@dataclass
class InstanceScene:
    name: str
    protos: List[Proto]
    width: int
    height: int
    prototypes: np.ndarray                  # [n, M] uint32, NONE = empty slot
    transforms: Optional[np.ndarray] = None  # [n, M, 6] float32
    colors: Optional[np.ndarray] = None      # [n, M, 4] float32
    differ: Sequence[tuple] = ()             # pairs of frames (a, b) whose frames must differ
    heavy: bool = False                      # large: the tests take it only where they say so

    @property
    def n(self) -> int:
        return self.prototypes.shape[0]

    @property
    def m(self) -> int:
        return self.prototypes.shape[1]


def solid(k: int, alpha: float = 1.0) -> Color:
    return Color(((k * 37) % 11) / 10.0, ((k * 53) % 7) / 6.0, ((k * 17) % 5) / 4.0, alpha)


def _props(p: Proto, k: int) -> Props:
    return p.props if p.props is not None else Props(func=Func.Draw(Style(fill=Fill.Solid(solid(k, 0.75)))))


def _path(api, pts, path_xf):
    pb = api.PathBuilder().move_to(Point(*pts[0]))
    for q in pts[1:]:
        pb.line_to(Point(*q))
    path = pb.build()
    return path if path_xf is None else path.transform(path_xf)


def build_library(api, sc: InstanceScene):
    """The scene's library composition on `api` (the binding or the oracle)."""
    comp = api.Composition()
    for k, p in enumerate(sc.protos):
        layer = comp.get_mut_or_insert_default(p.order)
        if p.cleared:
            for pts in p.cleared:
                layer.insert(_path(api, pts, p.path_xf))
            layer.clear()
        for pts in p.paths:
            layer.insert(_path(api, pts, p.path_xf))
        layer.set_props(_props(p, k))
        if p.xf is not None:
            layer.set_transform(p.xf)
        if not p.enabled:
            layer.disable()
    return comp


def _solid_props(props: Props, c) -> Props:
    """props with a Draw layer's fill replaced by Solid(c); a Clip layer's props as they are."""
    if props.func.draw is None:
        return props
    s = props.func.draw
    return Props(fill_rule=props.fill_rule,
                 func=Func.Draw(Style(is_clipped=s.is_clipped, fill=Fill.Solid(Color(*[float(v) for v in c])), blend_mode=s.blend_mode)))


def twin(api, sc: InstanceScene, b: int):
    """T_b on `api`: the composition whose ordinary frame is frame b of the instance call."""
    comp = api.Composition()
    by_order = {p.order: (k, p) for k, p in enumerate(sc.protos)}
    for m in range(sc.m):
        o = int(sc.prototypes[b, m])
        if o == NONE:
            continue
        k, p = by_order[o]
        layer = comp.get_mut_or_insert_default(m)
        for pts in p.paths:
            layer.insert(_path(api, pts, p.path_xf))
        props = _props(p, k)
        if sc.colors is not None:
            props = _solid_props(props, sc.colors[b, m])
        layer.set_props(props)
        if sc.transforms is not None:
            layer.set_transform([float(v) for v in sc.transforms[b, m]])
        elif p.xf is not None:
            layer.set_transform(p.xf)
    return comp


def instances(binding_mod, sc: InstanceScene):
    return binding_mod.Instances(sc.prototypes, sc.transforms, sc.colors)


# ---------------------------------------------------------------------------
# Shapes
# ---------------------------------------------------------------------------
def star(cx, cy, r0, r1, n, phase=0.0):
    return [(cx + (r1 if i % 2 else r0) * math.cos(phase + math.pi * i / n), cy + (r1 if i % 2 else r0) * math.sin(phase + math.pi * i / n))
            for i in range(2 * n)]


def rect(x0, y0, x1, y1):
    return [(x0, y0), (x1, y0), (x1, y1), (x0, y1)]


def poly(cx, cy, r, n, phase=0.0):
    return [(cx + r * math.cos(phase + 2 * math.pi * i / n), cy + r * math.sin(phase + 2 * math.pi * i / n)) for i in range(n)]


def move(tx, ty):
    return [1.0, 0.0, 0.0, 1.0, float(tx), float(ty)]


def _about(angle, cx, cy, scale=1.0, tx=0.0, ty=0.0):
    c, s = f32(scale * math.cos(angle)), f32(scale * math.sin(angle))
    return [float(c), float(-s), float(s), float(c), float(f32(cx + tx) - (c * f32(cx) - s * f32(cy))),
            float(f32(cy + ty) - (s * f32(cx) + c * f32(cy)))]


def _table(rows, width=6):
    return np.asarray(rows, f32).reshape(len(rows), -1, width)


# ---------------------------------------------------------------------------
# Scenes
# ---------------------------------------------------------------------------
def _repeats() -> InstanceScene:
    """Six library shapes around the origin, repeated within and across frames, with empty slots;
    frames 0 and 1 draw the same two overlapping shapes in reversed orders."""
    protos = [Proto(0, [rect(-12, -9, 12, 9)]), Proto(1, [star(0, 0, 6, 15, 5)]), Proto(2, [poly(0, 0, 11, 6)]),
              Proto(3, [rect(-5, -14, 5, 14)]), Proto(4, [star(0, 0, 4, 10, 7, 0.3)]), Proto(7, [poly(0, 0, 8, 3, 0.5)], enabled=True)]
    P = np.array([[2, 3, 0, 1, NONE, 4],
                  [3, 2, 0, 1, NONE, 4],
                  [1, 1, 1, NONE, 7, 7],
                  [NONE, NONE, NONE, NONE, NONE, NONE]], np.uint32)
    T = np.zeros((4, 6, 6), f32)
    spots = [(30, 30), (34, 33), (12, 50), (52, 12), (0, 0), (50, 50)]
    for b in range(4):
        for m in range(6):
            x, y = spots[1 - m if b == 1 and m < 2 else m]  # frame 1: the pair of frame 0 in place, stacked the other way
            T[b, m] = _about(0.4 * m, 0, 0, 1.0, 8 + 9 * m, 10 + 8 * m) if b == 2 else move(x, y)
    return InstanceScene("repeats", protos, 64, 64, P, T, None, differ=[(0, 1), (0, 2), (2, 3)])


def _inserts() -> InstanceScene:
    """A prototype of two inserts with a path transform, one cleared and drawn again (its first
    geometry is dead), one without geometry, and prototypes with transforms of their own that the
    frames keep (no transforms table)."""
    rot = [0.8, -0.6, 0.0, 0.6, 0.8, 0.0, 0.0, 0.0, 1.0]
    protos = [Proto(5, [rect(4, 4, 20, 16), star(30, 20, 4, 9, 5)], path_xf=rot, xf=move(6, 3)),
              Proto(6, [poly(40, 40, 12, 5)], cleared=[rect(0, 0, 60, 60), star(30, 30, 10, 28, 6)]),
              Proto(9),
              Proto(11, [star(20, 44, 5, 14, 4)], xf=[0.9, 0.2, -0.2, 0.9, 4.0, -6.0], enabled=True)]
    P = np.array([[5, 6, 9, 11], [11, 9, 6, 5], [6, 6, NONE, 5]], np.uint32)
    return InstanceScene("inserts", protos, 64, 48, P, None, None, differ=[(0, 2)])


def _gradient():
    g = GradientBuilder(Point(0, 0), Point(40, 30)).color(Color(1, 0, 0, 1)).color(Color(0, 0, 1, 0.5)).color(Color(0, 1, 0, 1))
    return g.build()


def _radial():
    return GradientBuilder(Point(20, 20), Point(36, 20)).type(GradientType.Radial).color(Color(1, 1, 0, 1)).color(Color(0, 0.5, 1, 1)).build()


def _texture():
    img = np.zeros((4, 4, 4), f32)
    for i in range(4):
        for j in range(4):
            img[i, j] = [(i + 1) / 4.0, (j + 1) / 4.0, ((i + j) % 3) / 2.0, 1.0]
    return Texture((4.0, 0.0, 0.0, 4.0, 2.0, 3.0), img)


def _styles() -> InstanceScene:
    """Gradient and texture prototypes without colours: their fills are served as they are, in
    each frame's own coordinates."""
    protos = [Proto(0, [rect(0, 0, 40, 30)], props=Props(func=Func.Draw(Style(fill=Fill.Gradient(_gradient()))))),
              Proto(1, [star(20, 20, 8, 18, 6)], props=Props(func=Func.Draw(Style(fill=Fill.Gradient(_radial()))))),
              Proto(2, [rect(4, 4, 36, 28)], props=Props(func=Func.Draw(Style(fill=Fill.Texture(_texture())))))]
    P = np.array([[0, 2, 1], [2, 1, 0]], np.uint32)
    T = _table([[move(2, 2), move(20, 10), move(8, 20)], [move(24, 0), move(0, 24), move(10, 12)]])
    return InstanceScene("styles", protos, 64, 64, P, T, None, differ=[(0, 1)])


def _colors_blend() -> InstanceScene:
    """Colours: a non-separable blend prototype, an even-odd one, a gradient made solid and a
    translucent one, each instance recoloured per frame."""
    protos = [Proto(0, [rect(0, 0, 48, 40)], props=Props(func=Func.Draw(Style(fill=Fill.Solid(solid(3)))))),
              Proto(1, [star(24, 20, 8, 20, 5)], props=Props(func=Func.Draw(Style(fill=Fill.Solid(solid(4)), blend_mode=BlendMode.Hue)))),
              Proto(2, [rect(4, 4, 30, 30), rect(10, 10, 24, 24)], props=Props(fill_rule=FillRule.EvenOdd,
                                                                             func=Func.Draw(Style(fill=Fill.Gradient(_gradient()))))),
              Proto(3, [poly(30, 24, 14, 7)], props=Props(func=Func.Draw(Style(fill=Fill.Solid(solid(5, 0.5)), blend_mode=BlendMode.Multiply))))]
    P = np.array([[0, 1, 2, 3], [0, 3, 1, 2], [2, 1, 1, 0]], np.uint32)
    C = np.zeros((3, 4, 4), f32)
    for b in range(3):
        for m in range(4):
            C[b, m] = [((b + 2 * m) % 5) / 4.0, ((3 * b + m) % 4) / 3.0, ((b * m) % 3) / 2.0, (1.0, 0.5, 0.75, 1.0)[(b + m) % 4]]
    T = _table([[move(0, 0), move(8, 6), move(30, 20), move(12, 10)]] * 3)
    return InstanceScene("colors_blend", protos, 64, 56, P, T, C, differ=[(0, 1), (1, 2)])


def _clip_leak() -> InstanceScene:
    """A Clip prototype whose range (8 layers) runs past the frame's M = 3 slots, clipped Draw
    prototypes above it, and frames of 20 rows (not whole tiles): nothing of one frame's clip may
    reach the next frame's instances."""
    protos = [Proto(0, [rect(8, 4, 40, 16)], props=Props(func=Func.Clip(8))),
              Proto(1, [rect(0, 0, 48, 20)], props=Props(func=Func.Draw(Style(is_clipped=True, fill=Fill.Solid(solid(1)))))),
              Proto(2, [star(24, 10, 4, 10, 5)], props=Props(func=Func.Draw(Style(fill=Fill.Solid(solid(2))))))]
    P = np.array([[0, 1, 1], [1, 2, 1], [2, 0, 1], [1, 1, 2]], np.uint32)
    T = _table([[move(0, 0), move(0, 0), move(4, 2)], [move(0, 2), move(0, 0), move(8, 2)], [move(0, 0), move(0, 0), move(0, 0)],
                [move(0, 1), move(6, 0), move(0, 0)]])
    return InstanceScene("clip_leak", protos, 48, 20, P, T, None, differ=[(0, 1), (2, 3)])


def _nonfinite() -> InstanceScene:
    """NaN and infinite translations, which render as render_device renders them."""
    nan, inf = float("nan"), float("inf")
    protos = [Proto(0, [rect(0, 0, 20, 20)]), Proto(1, [star(30, 30, 6, 14, 5)])]
    P = np.array([[0, 1, 0], [1, 0, 1]], np.uint32)
    T = _table([[[1.0, 0.0, 0.0, 1.0, nan, 3.0], move(4, 4), [1.0, 0.0, 0.0, 1.0, inf, -inf]],
                [[1.0, 0.0, 0.0, 1.0, -inf, 0.0], [1.0, 0.0, 0.0, 1.0, 2.0, nan], move(20, 20)]])
    return InstanceScene("nonfinite", protos, 48, 48, P, T, None, differ=[(0, 1)])


def _library(n=511, m=8, shapes=64, size=64, seed=11) -> InstanceScene:
    """511 frames of 64 x 64 (max_views(64)), 8 slots each, from a library of 64 shapes: the
    synthetic-data workload, with per-instance transforms and colours and a few empty slots."""
    rng = np.random.default_rng(seed)
    protos = []
    for k in range(shapes):
        kind = k % 3
        r = 6 + (k * 7) % 9
        pts = star(0, 0, r * 0.45, r, 4 + k % 5, 0.1 * k) if kind == 0 else poly(0, 0, r, 3 + k % 6, 0.2 * k) if kind == 1 else rect(-r, -r * 0.6, r, r * 0.6)
        protos.append(Proto(k, [pts]))
    P = rng.integers(0, shapes, (n, m)).astype(np.uint32)
    P[rng.random((n, m)) < 0.05] = NONE
    T = np.zeros((n, m, 6), f32)
    for b in range(n):
        for j in range(m):
            a, s = rng.uniform(0, 2 * math.pi), rng.uniform(0.5, 1.0)
            T[b, j] = _about(a, 0, 0, s, rng.uniform(4, size - 4), rng.uniform(4, size - 4))
    C = np.concatenate([rng.random((n, m, 3)), np.where(rng.random((n, m, 1)) < 0.7, 1.0, 0.6)], axis=2).astype(f32)
    return InstanceScene("library_511x64", protos, size, size, P, T, C, differ=[(0, 1), (1, 510)], heavy=True)


def glyph_protos(count=90):
    """`count` glyph-sized shapes (8 to 14 px) of one or two contours, a font of sorts."""
    protos = []
    for k in range(count):
        r = 4 + (k % 4)
        outer = star(0, 0, r * 0.5, r, 3 + k % 6, 0.17 * k) if k % 2 else poly(0, 0, r, 4 + k % 5, 0.11 * k)
        paths = [outer] if k % 3 else [outer, rect(-r * 0.25, -r * 0.25, r * 0.25, r * 0.25)]
        protos.append(Proto(k, paths, props=Props(fill_rule=FillRule.EvenOdd, func=Func.Draw(Style(fill=Fill.Solid(solid(k)))))))
    return protos


def glyph_tables(count=20000, n_protos=90, w=1920, h=1080, seed=5):
    """[1, count] prototypes and translations of a page of text: rows of glyphs 12 px apart."""
    rng = np.random.default_rng(seed)
    P = rng.integers(0, n_protos, (1, count)).astype(np.uint32)
    T = np.zeros((1, count, 6), f32)
    per_row = (w - 16) // 12
    for i in range(count):
        T[0, i] = move(8 + 12 * (i % per_row) + rng.uniform(-0.5, 0.5), 8 + 13 * ((i // per_row) % ((h - 16) // 13)))
    return P, T


def _glyphs() -> InstanceScene:
    """One 1920 x 1080 frame of 20 000 glyph-sized instances of 90 prototypes."""
    P, T = glyph_tables()
    return InstanceScene("glyphs_1080p", glyph_protos(), 1920, 1080, P, T, None, heavy=True)


def _scenes() -> Dict[str, InstanceScene]:
    out = [_repeats(), _inserts(), _styles(), _colors_blend(), _clip_leak(), _nonfinite(), _library(), _glyphs()]
    return {s.name: s for s in out}


SCENES = _scenes()
LIGHT = [k for k, s in SCENES.items() if not s.heavy]
