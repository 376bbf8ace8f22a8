"""Scenes at the limits of stage 1: the host-built flatten program (host_path.cpp), the device's
quad expansion and point evaluation (quad_expand_kernel, flatten_eval_kernel), path transforms
at the GeomPresTransform boundary, and the band filter of Renderer::flush_geometry.

Builders take `api` (and `comp` for the renderable scenes) like `extremes.py`, so the CUDA
library and the oracle build identical paths. Every coordinate is float32 (handed over as
float32-exact values) with |coordinate| < 2^26 px.

- PATHS: name -> PathScene(build(api) -> [Path], ...). Compared point by point (flatten stage),
  plain and through every transform of TRANSFORMS when `transforms` is set. `device=False`
  scenes are checked on the CPU only (their point count exceeds the pre-flight cap); `finite`
  is False for paths whose points may be NaN / infinite (weights <= 0, projective w -> 0): they
  are never rendered.
- RENDER: name -> RenderScene(build(api, comp), width, height): whole frames.
- BANDS: name -> RenderScene whose inserts sit 0 ... 1 px from the edges of BAND (rows
  [BAND_LO, BAND_HI)), rendered in band sequences.

Notes on the targets:
- Long splines: a spline's running curvature is an f32 sum; a collinear quad adds exactly 2.0.
  From 2^23 on a quad can add exactly 1, and past 2^25 nothing at all, so the reference's quad
  walk (one index per path, one step per point) can fall behind the kernel's bisection. The
  `lagging_walk_*` scenes get there: a chain of collinear quads followed by a quad whose
  curvature is 1 + 2^-22 or so (the running total lands on an integer, so the last evaluated point
  does not reach the spline's last quad), and a 2^25 spiral with a stalled collinear tail.
- `collinear_then_curve_*`: pi equals a collinear quad's running curvature exactly while the
  step is below 1, so evaluating the quad that reaches pi and the next one give different points.
- The encoding switch: the point encoding is used when 36 B per spline exceed 9 B per point;
  `crossover_47` has 12 splines and 47 points (point records), `crossover_48` 12 and 48
  (exactly equal: spline records).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Dict, List, Tuple

import numpy as np

from forma_b200.binding import Color, Fill, FillRule, Func, Point, Props, Rect, Style

f32 = np.float32
MAX_ERROR = 1.0 / 16.0
MAX_ANGLE_ERROR = 0.001
K_EPS = float(np.finfo(np.float32).eps)  # 2^-23

W, H = 256, 256
BAND_LO, BAND_HI = 64, 128                 # tile rows 4..7
BAND = Rect((0, W), (BAND_LO, BAND_HI))
INNER_BAND = Rect((0, W), (80, 112))       # tile rows 5..6: inside BAND
OUTER_BAND = Rect((0, W), (160, 224))      # tile rows 10..13: outside BAND


def P(x, y) -> Point:
    return Point(float(f32(x)), float(f32(y)))


def nextup(v: float) -> float:
    return float(np.nextafter(f32(v), f32(np.inf)))


@dataclass
class PathScene:
    build: Callable
    device: bool = True        # compared on the device (the point count fits the pre-flight budget)
    finite: bool = True        # every point finite: may be rendered and transformed
    transforms: bool = False   # also compared through every transform of TRANSFORMS
    tags: Tuple[str, ...] = ()


@dataclass
class RenderScene:
    build: Callable            # build(api, comp) -> notes dict
    width: int = W
    height: int = H
    tags: Tuple[str, ...] = ()


def solid(c: Color, rule=FillRule.NonZero) -> Props:
    return Props(fill_rule=rule, func=Func.Draw(Style(fill=Fill.Solid(c))))


# ---------------------------------------------------------------------------
# Shapes
# ---------------------------------------------------------------------------
def quad_circle(api, cx, cy, r, n=8, pb=None, turns=1):
    """A circle of n quads per turn (control points on the tangents)."""
    pb = pb or api.PathBuilder()
    th = np.linspace(0.0, 2 * np.pi * turns, n * turns + 1)
    h = 1.0 / np.cos(np.pi / n)
    pb.move_to(P(cx + r, cy))
    for i in range(1, len(th)):
        m = 0.5 * (th[i - 1] + th[i])
        end = (cx + r, cy) if i == len(th) - 1 and turns == 1 else (cx + r * np.cos(th[i]), cy + r * np.sin(th[i]))
        pb.quad_to(P(cx + r * h * np.cos(m), cy + r * h * np.sin(m)), P(*end))
    return pb


def shape_set(api, s: float, ox: float, oy: float) -> List:
    """The scale-sweep shapes at scale s around (ox, oy): a quad circle, a cubic S, a rational
    quad arc and a polygon."""
    out = [quad_circle(api, ox, oy, 100 * s).build()]
    pb = api.PathBuilder()
    pb.move_to(P(ox - 100 * s, oy))
    pb.cubic_to(P(ox - 30 * s, oy - 120 * s), P(ox + 30 * s, oy + 120 * s), P(ox + 100 * s, oy))
    out.append(pb.build())
    pb = api.PathBuilder()
    pb.move_to(P(ox - 100 * s, oy))
    pb.rat_quad_to(P(ox, oy - 100 * s), P(ox + 100 * s, oy), float(f32(np.sqrt(0.5))))
    out.append(pb.build())
    ang = np.arange(7) * 2.39996
    pb = api.PathBuilder()
    pb.move_to(P(ox + 100 * s, oy))
    for a in ang[1:]:
        pb.line_to(P(ox + 100 * s * np.cos(a), oy + 100 * s * np.sin(a)))
    out.append(pb.build())
    return out


SCALES = tuple(2.0 ** e for e in (-10, -6, -3, 0, 3, 6, 10, 14, 17))
OFFSETS = (0.0, 2.0 ** 12, 2.0 ** 22)


def scale_sweep(api):
    out = []
    for s in SCALES:
        for o in OFFSETS:
            out += shape_set(api, s, o + 128.0, o + 128.0)
    return out


def scale_sweep_huge(api):
    """2^20 ... 2^24 px shapes (2^24 stays below 2^26 with the 100x radius only as 2^18 * 100)."""
    return [p for s in (2.0 ** 18,) for p in shape_set(api, s, 128.0, 128.0)]


# ---------------------------------------------------------------------------
# Degenerate primitives
# ---------------------------------------------------------------------------
def degenerate(api):
    out = []

    def path(*ops, start=(10.0, 10.0)):
        pb = api.PathBuilder()
        pb.move_to(P(*start))
        for op in ops:
            getattr(pb, op[0])(*[P(*p) if isinstance(p, tuple) else p for p in op[1:]])
        return pb.build()
    out.append(path(("cubic_to", (100.0, 100.0), (10.0, 100.0), (100.0, 10.0))))            # cusp-like crossing
    out.append(path(("cubic_to", (60.0, 60.0), (60.0, 60.0), (110.0, 10.0))))               # coincident inner points
    out.append(path(("cubic_to", (10.0, 10.0), (110.0, 110.0), (110.0, 110.0))))            # coincident end points
    out.append(path(("cubic_to", (160.0, 110.0), (-40.0, 110.0), (110.0, 10.0))))           # loop
    out.append(path(("cubic_to", (110.0, 10.0), (10.0, 10.0), (110.0, 10.0))))              # collinear cubic, reversing
    out.append(path(("quad_to", (10.0, 10.0), (90.0, 50.0))))                               # p1 == p0
    out.append(path(("quad_to", (90.0, 50.0), (90.0, 50.0))))                               # p1 == p2
    out.append(path(("quad_to", (10.0, 10.0), (10.0, 10.0))))                               # all three equal
    out.append(path(("quad_to", (90.0, 90.0), (10.0, 10.0))))                               # closed quad
    out.append(path(("quad_to", (120.0, 10.0), (60.0, 10.0))))                             # collinear reversal
    out.append(path(("quad_to", (60.0, 10.0), (110.0, 10.0))))                             # collinear, midpoint
    out.append(path(("rat_quad_to", (90.0, 90.0), (10.0, 10.0), 3.0)))                     # closed rational quad
    # lines shorter than MAX_ERROR and shorter than kEps
    for step in (0.05, 0.0625, 0.07, 1e-7, 1e-8):
        pb = api.PathBuilder()
        pb.move_to(P(50.0, 50.0))
        x = f32(50.0)
        for i in range(12):
            x = f32(x + f32(step))
            pb.line_to(P(float(x), 50.0 + (i % 2) * step))
        pb.line_to(P(60.0, 70.0))
        out.append(pb.build())
    # direction changes of MAX_ANGLE_ERROR +- a little, near 0 and near the fold at pi
    for base in (0.0, np.pi):
        for d in (-4e-7, -1e-7, 0.0, 1e-7, 4e-7):
            turn = base + MAX_ANGLE_ERROR + d
            pb = api.PathBuilder()
            pb.move_to(P(20.0, 20.0))
            x, y, a = 20.0, 20.0, 0.3
            for _ in range(6):
                x, y = x + 40.0 * np.cos(a), y + 40.0 * np.sin(a)
                pb.line_to(P(x, y))
                a += turn
            out.append(pb.build())
    # move_to only, repeated move_to, the empty path
    pb = api.PathBuilder()
    pb.move_to(P(5.0, 5.0))
    out.append(pb.build())
    pb = api.PathBuilder()
    pb.move_to(P(5.0, 5.0)).move_to(P(7.0, 9.0)).line_to(P(30.0, 40.0)).move_to(P(1.0, 2.0)).move_to(P(3.0, 4.0))
    out.append(pb.build())
    out.append(api.PathBuilder().build())
    return out


# ---------------------------------------------------------------------------
# Long splines
# ---------------------------------------------------------------------------
SPIRAL_QUADS = 100_000


def spiral(api, n=SPIRAL_QUADS, cx=128.0, cy=128.0):
    """A smooth spiral of n quads (one spline): r = 200 + c theta over 500 turns, each quad's
    control point where the tangents at its ends meet (turns of about 2 degrees, so that the
    float32 rounding of the points stays far below MAX_ANGLE_ERROR)."""
    th = np.linspace(0.0, 2 * np.pi * 500, n + 1)
    c = 1800.0 / th[-1]
    r = 200.0 + c * th
    pts = np.stack([r * np.cos(th), r * np.sin(th)], 1)
    tan = np.stack([c * np.cos(th) - r * np.sin(th), c * np.sin(th) + r * np.cos(th)], 1)
    a, b, ta, tb = pts[:-1], pts[1:], tan[:-1], tan[1:]
    d = b - a
    den = ta[:, 0] * tb[:, 1] - ta[:, 1] * tb[:, 0]
    s = (d[:, 0] * tb[:, 1] - d[:, 1] * tb[:, 0]) / den
    ctrl = a + s[:, None] * ta
    off = np.array([cx, cy])
    xy = np.concatenate([pts[:1], np.stack([ctrl, b], 1).reshape(-1, 2)]) + off
    cmds = np.concatenate([[0], np.full(n, 2)]).astype(np.uint8)
    return api.PathBuilder().extend(cmds, xy.astype(np.float32).ravel()).build()


def collinear_chain(api, n, x0=-40.0, y0=100.0, step=2.0, tail=None, pb=None, close=True):
    """n collinear quads along +x (control point at the middle: the fall-back curvature 2.0),
    optionally followed by `tail(pb, x, y)`."""
    pb = pb or api.PathBuilder()
    xs = (x0 + step * np.arange(n + 1)).astype(np.float32)
    mids = (0.5 * (xs[1:].astype(np.float64) + xs[:-1])).astype(np.float32)
    xy = np.empty((2 * n + 1, 2), np.float32)
    xy[0] = (xs[0], y0)
    xy[1::2, 0], xy[2::2, 0] = mids, xs[1:]
    xy[1:, 1] = y0
    pb.extend(np.concatenate([[0], np.full(n, 2)]).astype(np.uint8), xy.ravel())
    if tail:
        tail(pb, float(xs[-1]), y0)
    return pb


# A tangent-continuous quad (192, 100) -> (196, 100) -> (200, LAG_Y) at the end of a chain along
# y = 100: its curvature is 1 + 4e-5 (just above the collinear fall-back), so after 4096 collinear
# quads (running curvature 8192, half an ulp 2^-11) the total lands on 8193 exactly.
LAG_Y = 100.2501220703125
CURVE_H = 0.5  # curvature about 1.41: after a chain of n quads the step is (2n + 1.41) / (2n + 2) < 1


def lagging_walk_small(api):
    """4096 collinear quads + the LAG_Y quad, then a second contour (a circle): the reference's
    walk ends the first spline on its next-to-last quad and evaluates the circle's points on
    the first contour's last quad."""
    def tail(pb, x, y):
        pb.quad_to(P(x + 4.0, y), P(x + 8.0, LAG_Y))
    pb = collinear_chain(api, 4096, x0=-8000.0, y0=100.0, step=2.0, tail=tail)
    quad_circle(api, 128.0, 160.0, 40.0, pb=pb)
    return pb.build()


def collinear_then_curve(api, n):
    def tail(pb, x, y):
        pb.quad_to(P(x + 16.0, y), P(x + 32.0, y + CURVE_H))
    return collinear_chain(api, n, x0=20.0, y0=60.0, step=f32(150.0 / max(n, 1)), tail=tail).build()


def spiral_2p25(api, stalled: bool):
    """A circle of radius 2^23 wound 1400 times (running curvature past 2^25, 36 M points),
    then, when `stalled`, six collinear quads along the end tangent that add nothing to it, and a
    second contour. Without the tail the walk keeps up (spline records); with it, it falls behind
    (point records with the walk's choices)."""
    R, turns, n = 2.0 ** 23, 1400, 8
    th = np.linspace(0.0, 2 * np.pi * turns, n * turns + 1)
    h = 1.0 / np.cos(np.pi / n)
    pts = np.stack([R * np.cos(th), R * np.sin(th)], 1)
    m = 0.5 * (th[1:] + th[:-1])
    ctrl = np.stack([R * h * np.cos(m), R * h * np.sin(m)], 1)
    xy = np.concatenate([pts[:1], np.stack([ctrl, pts[1:]], 1).reshape(-1, 2)]).astype(np.float32)
    pb = api.PathBuilder().extend(np.concatenate([[0], np.full(len(th) - 1, 2)]).astype(np.uint8), xy.ravel())
    if stalled:
        x, y = float(xy[-1, 0]), float(xy[-1, 1])
        for k in range(6):
            pb.quad_to(P(x, y + 8 * k + 4), P(x, y + 8 * k + 8))
    pb.move_to(P(0.0, 0.0))
    pb.quad_to(P(50.0, 0.0), P(50.0, 50.0))
    pb.line_to(P(0.0, 50.0))
    return pb.build()


# ---------------------------------------------------------------------------
# Rational
# ---------------------------------------------------------------------------
WEIGHTS = (1e-3, 1e-2, 0.1, 0.5, 1.0, 2.0, 10.0, 100.0, 1e3)
BAD_WEIGHTS = (0.0, -1e-3, -0.5, -1.0)


def rational(api, weights=WEIGHTS):
    out = []
    for w in weights:
        w = float(f32(w))
        pb = api.PathBuilder()
        pb.move_to(P(30.0, 200.0))
        pb.rat_quad_to(P(128.0, 20.0), P(226.0, 200.0), w)
        out.append(pb.build())
        for w2 in (1.0, w):
            pb = api.PathBuilder()
            pb.move_to(P(30.0, 200.0))
            pb.rat_cubic_to(P(60.0, 20.0), P(200.0, 20.0), P(226.0, 200.0), w, float(f32(w2)))  # mult = max(w1, w2, 1)
            out.append(pb.build())
    return out


# ---------------------------------------------------------------------------
# Encodings
# ---------------------------------------------------------------------------
CROSSOVER_R = {47: 224.002197265625, 48: 237.36119079589844}  # 12 splines; 47 / 48 points


def crossover(api, r, ox=0.0, oy=0.0):
    """10 zig-zag lines, then a quad of radius r: 12 splines (the lines, the quad, the closing
    line); the quad's subdivisions move the point count across 4 points per spline."""
    pb = api.PathBuilder()
    pb.move_to(P(ox, oy))
    for i in range(10):
        pb.line_to(P(ox + 4.0 * (i + 1), oy + (3.0 if i % 2 == 0 else 0.0)))
    x0 = ox + 40.0
    pb.quad_to(P(x0 + r, oy), P(x0 + r, oy + r))
    return pb.build()


def encodings(api):
    return [crossover(api, CROSSOVER_R[47]), crossover(api, CROSSOVER_R[48])]


# ---------------------------------------------------------------------------
# Transforms (3x3, row-major: x' = m0 x + m1 y + m2, y' = m3 x + m4 y + m5, w = m6 x + m7 y + m8)
# ---------------------------------------------------------------------------
def _rot(a, s=1.0, tx=0.0, ty=0.0):
    c, n = float(f32(s * np.cos(a))), float(f32(s * np.sin(a)))
    return [c, -n, tx, n, c, ty, 0.0, 0.0, 1.0]


SX_EDGE = float(f32(1.0 + 2.0 ** -21))   # ux^2 == 1 + MAX_ERROR / 65536 exactly in f32
SY_EDGE = float(f32(1.0 + 2.0 ** -20))   # vy^2 == 1 + MAX_ERROR / 32768 exactly in f32
XF_LIMIT = float(f32(1.0 + MAX_ERROR / 65536.0))
TRANSFORMS: Dict[str, List[float]] = {
    "identity": [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0],
    "translate": [1.0, 0.0, 37.25, 0.0, 1.0, -12.5, 0.0, 0.0, 1.0],
    "sx_at_limit": [SX_EDGE, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0],
    "sx_above_limit": [nextup(SX_EDGE), 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0],
    "sx_limit_value": [XF_LIMIT, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0],
    "sx_limit_value_up": [nextup(XF_LIMIT), 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0],
    "sy_at_limit": [1.0, 0.0, 0.0, 0.0, SY_EDGE, 0.0, 0.0, 0.0, 1.0],
    "sy_above_limit": [1.0, 0.0, 0.0, 0.0, nextup(SY_EDGE), 0.0, 0.0, 0.0, 1.0],
    "m8_two": [2.0, 0.0, 10.0, 0.0, 2.0, 20.0, 0.0, 0.0, 2.0],
    "m8_eps": [1.0, 0.0, 3.0, 0.0, 1.0, 4.0, 0.0, 0.0, 1.0 + K_EPS],
    "m8_2eps": [1.0, 0.0, 3.0, 0.0, 1.0, 4.0, 0.0, 0.0, 1.0 + 2 * K_EPS],
    "m8_half": [0.5, 0.0, 1.0, 0.0, 0.5, 1.0, 0.0, 0.0, 0.5],
    "m6_at_eps": [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, K_EPS, 0.0, 1.0],
    "m6_above_eps": [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, nextup(K_EPS), 0.0, 1.0],
    "m7_at_eps": [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, -K_EPS, 1.0],
    "m7_above_eps": [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, -nextup(K_EPS), 1.0],
    "reflect_x": [-1.0, 0.0, 256.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0],
    "reflect_y": [1.0, 0.0, 0.0, 0.0, -1.0, 256.0, 0.0, 0.0, 1.0],
    "swap_xy": [0.0, 1.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0],
    "scale_up_2": [2.0, 0.0, 0.0, 0.0, 2.0, 0.0, 0.0, 0.0, 1.0],
    "scale_down_half": [0.5, 0.0, 64.0, 0.0, 0.5, 64.0, 0.0, 0.0, 1.0],
    "projective": [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 1e-3, 5e-4, 1.0],
    "projective_strong": [0.9, 0.2, 5.0, -0.1, 1.1, 3.0, 2e-3, -1e-3, 1.2],
}
for _k in range(24):
    TRANSFORMS[f"rotate_{_k * 15}"] = _rot(_k * np.pi / 12, 1.0, 128.0, 128.0)
TRANSFORMS["rotate_37_shrink"] = _rot(0.65, 0.75, 10.0, 20.0)
CHAINS = (("rotate_30", "translate"), ("scale_up_2", "rotate_45"), ("projective", "rotate_90"),
          ("rotate_45", "projective"), ("sx_above_limit", "sx_at_limit"))
# projective transforms whose w reaches 0 or below over the path: non-finite points, flatten stage only
DEGENERATE_TRANSFORMS = {
    "w_to_zero": [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, float(f32(-1.0 / 226.0)), 0.0, 1.0],
    "w_negative": [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, -0.01, 0.0, 1.0],
}


def transform_sample(api):
    """Paths pushed through TRANSFORMS: a circle, a cubic, a rational arc, a polygon, lines only."""
    out = shape_set(api, 0.8, 128.0, 128.0)
    out.append(crossover(api, 30.0, 20.0, 20.0))
    return out


def degenerate_weights(api):
    return rational(api, BAD_WEIGHTS)


PATHS: Dict[str, PathScene] = {
    "scale_sweep": PathScene(scale_sweep),
    "scale_sweep_huge": PathScene(scale_sweep_huge),
    "degenerate": PathScene(degenerate, transforms=True),
    "spiral_1e5": PathScene(lambda api: [spiral(api)]),
    "collinear_chain": PathScene(lambda api: [collinear_chain(api, 20_000, x0=-20000.0, y0=100.0).build()]),
    "collinear_then_curve": PathScene(lambda api: [collinear_then_curve(api, n) for n in (1, 4, 64, 1000)]),
    "lagging_walk_small": PathScene(lambda api: [lagging_walk_small(api)], tags=("lags",)),
    "spiral_2p25_keeps_up": PathScene(lambda api: [spiral_2p25(api, False)], device=False, tags=("2p25",)),
    "spiral_2p25_stalled": PathScene(lambda api: [spiral_2p25(api, True)], device=False, tags=("2p25", "lags")),
    "rational": PathScene(rational, transforms=True),
    "rational_bad_weights": PathScene(degenerate_weights, finite=False),
    "encodings": PathScene(encodings, transforms=True),
    "transform_sample": PathScene(transform_sample, transforms=True),
}


# ---------------------------------------------------------------------------
# Renderable scenes
# ---------------------------------------------------------------------------
def _styled(layer, color, rule):
    layer.set_props(solid(color, rule))
    return layer


def render_scale_sweep(api, comp):
    """The sweep's shapes that fit the segment budget: the small ones in the frame, the large
    ones far to its right (their lines are culled, their points still evaluated)."""
    for i, (s, o) in enumerate(((2.0 ** -6, 0.0), (2.0 ** -3, 0.0), (0.5, 0.0), (1.0, 0.0), (2.0 ** 10, 2.0 ** 22),
                                (2.0 ** 14, 2.0 ** 22))):
        lay = _styled(comp.get_mut_or_insert_default(i), Color(0.2, f32(0.1 * i), 0.7, 0.6), FillRule.EvenOdd)
        for p in shape_set(api, s, 128.0 + o, 128.0):
            lay.insert(p)
    return {}


def render_long(api, comp):
    _styled(comp.get_mut_or_insert_default(0), Color(0.9, 0.3, 0.1, 0.7), FillRule.EvenOdd).insert(spiral(api))
    _styled(comp.get_mut_or_insert_default(1), Color(0.1, 0.5, 0.2, 0.8), FillRule.NonZero).insert(lagging_walk_small(api))
    lay = _styled(comp.get_mut_or_insert_default(2), Color(0.3, 0.3, 0.9, 0.5), FillRule.NonZero)
    for n in (1, 4, 64, 1000):
        lay.insert(collinear_then_curve(api, n))
    return {}


def render_rational_mix(api, comp):
    """Rational and polynomial inserts in one batch (48-byte QuadUp records for all)."""
    lay = _styled(comp.get_mut_or_insert_default(0), Color(0.6, 0.2, 0.5, 0.6), FillRule.NonZero)
    for i, p in enumerate(rational(api)):
        lay.insert(p)
        lay.insert(quad_circle(api, 20.0 + 24.0 * (i % 10), 30.0 + 20.0 * (i // 10), 9.0).build())
    return {}


def render_encodings(api, comp):
    """Point- and spline-encoded inserts alternating job by job in one batch (zig-zag polylines
    and circles), then the two paths on either side of the crossover."""
    lay = _styled(comp.get_mut_or_insert_default(0), Color(0.1, 0.1, 0.1, 0.8), FillRule.EvenOdd)
    for i in range(24):
        x, y = 12.0 + 10.0 * i, 20.0 + 9.0 * i
        if i % 2 == 0:
            pb = api.PathBuilder()
            pb.move_to(P(x, y))
            for k in range(1, 30):
                pb.line_to(P(x + 0.7 * k, y + (5.0 if k % 2 else 0.0)))
            lay.insert(pb.build())
        else:
            lay.insert(quad_circle(api, x, y, 9.0).build())
    lay.insert(crossover(api, CROSSOVER_R[47]))
    lay.insert(crossover(api, CROSSOVER_R[48]))
    return {}


def render_transforms(api, comp):
    i = 0
    for name, m in TRANSFORMS.items():
        if name.startswith("projective"):
            continue
        lay = _styled(comp.get_mut_or_insert_default(i), Color(f32(0.02 * i), 0.4, 0.6, 0.35), FillRule.NonZero)
        for p in transform_sample(api):
            lay.insert(p.transform(m))
        i += 1
    return {}


RENDER: Dict[str, RenderScene] = {
    "scale_sweep": RenderScene(render_scale_sweep),
    "long_splines": RenderScene(render_long),
    "rational_mix": RenderScene(render_rational_mix),
    "encodings_alternating": RenderScene(render_encodings),
    "transforms": RenderScene(render_transforms),
}


# ---------------------------------------------------------------------------
# Band-filter scenes: inserts whose bounds sit 0 ... 1 px from an edge of BAND
# ---------------------------------------------------------------------------
EDGE_GAPS = (0.0, 0.01, 0.03, 0.25, 0.5, 0.51, 0.75, 1.0)


def _edges():
    """(edge, body, y_ext): an insert whose extreme row is y_ext = edge +- gap, with its body
    above (body = -1: y_ext is its largest y) or below it (body = +1: its smallest y)."""
    for edge in (BAND_LO, BAND_HI):
        for body in (-1, 1):
            for sign in (-1, 1):
                for gap in EDGE_GAPS:
                    if sign > 0 or gap > 0:
                        yield edge, body, float(f32(edge + sign * gap))


def _x(i):
    return 2.0 + 4.0 * (i % 62)


def band_rotated(api, comp):
    """A thin rectangle rotated by 30 degrees through a geometry-preserving path transform;
    its lowest (or highest) transformed corner is the extreme row."""
    lay = _styled(comp.get_mut_or_insert_default(0), Color(0.8, 0.2, 0.2, 0.7), FillRule.NonZero)
    base = api.PathBuilder()
    base.move_to(P(0.0, 0.0)).line_to(P(0.0, 4.0)).line_to(P(12.0, 4.0)).line_to(P(12.0, 0.0))
    base = base.build()
    a = np.pi / 6
    c, s = float(f32(np.cos(a))), float(f32(np.sin(a)))
    ymax = s * 12.0 + c * 4.0  # y' = s x + c y + ty: smallest at corner (0, 0), largest at (12, 4)
    for i, (edge, body, y_ext) in enumerate(_edges()):
        ty = y_ext - ymax if body < 0 else y_ext
        lay.insert(base.transform([c, -s, _x(i), s, c, float(f32(ty)), 0.0, 0.0, 1.0]))
    return {}


def band_rational_outside(api, comp):
    """Rational quads whose end points lie 30 px beyond their extreme row and whose control
    point lies beyond the curve: the curve's apex (not an end point) is the extreme row."""
    lay = _styled(comp.get_mut_or_insert_default(0), Color(0.2, 0.6, 0.2, 0.7), FillRule.NonZero)
    for i, (edge, body, y_ext) in enumerate(_edges()):
        w = (0.5, 1.0, 2.0)[i % 3]
        y0 = y_ext + body * 30.0
        y1 = ((1.0 + w) * y_ext - y0) / w  # apex of the symmetric quad: (y0 + w y1) / (1 + w)
        x = _x(i)
        pb = api.PathBuilder()
        pb.move_to(P(x, y0))
        pb.rat_quad_to(P(x + 2.0, y1), P(x + 4.0, y0), w)
        lay.insert(pb.build())
    return {}


def band_unbounded(api, comp):
    """Inserts with bounded == false: a quad whose middle weight lies in (-1, 0), finite on its
    whole length but outside the hull rule, with an end point at the extreme row."""
    lay = _styled(comp.get_mut_or_insert_default(0), Color(0.2, 0.2, 0.8, 0.7), FillRule.NonZero)
    for i, (edge, body, y_ext) in enumerate(_edges()):
        x = _x(i)
        pb = api.PathBuilder()
        pb.move_to(P(x, y_ext))
        pb.rat_quad_to(P(x + 2.0, y_ext + body * 10.0), P(x + 4.0, y_ext + body * 20.0), (-0.25, -0.5, -0.9)[i % 3])
        pb.line_to(P(x + 4.0, y_ext + body * 2.0))
        lay.insert(pb.build())
    return {}


def band_rounding(api, comp):
    """Polygons whose extreme row is a shallow zig-zag of 0.01 px: a line that lies within 1/32 px
    of an edge has its pixel segment rounded onto the edge's row (rasterizer.rs:111-156), so an
    insert whose points all stay above BAND_LO can still paint the band's first row. The filter's
    half-pixel margin keeps such inserts."""
    lay = _styled(comp.get_mut_or_insert_default(0), Color(0.7, 0.5, 0.1, 0.7), FillRule.NonZero)
    for i, (edge, body, y_ext) in enumerate(_edges()):
        x, inner = _x(i), y_ext + body * 0.01
        pb = api.PathBuilder()
        pb.move_to(P(x, y_ext + body * 10.0))
        pb.line_to(P(x + 1.0, inner)).line_to(P(x + 2.0, y_ext)).line_to(P(x + 3.0, inner))
        pb.line_to(P(x + 4.0, y_ext + body * 10.0))
        lay.insert(pb.build())
    return {}


BANDS: Dict[str, RenderScene] = {
    "rounding": RenderScene(band_rounding),
    "rotated": RenderScene(band_rotated, tags=("xf",)),
    "rational_outside": RenderScene(band_rational_outside),
    "unbounded": RenderScene(band_unbounded),
}
