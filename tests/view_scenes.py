"""Scenes of views (Renderer.render_views): a composition, a frame size and the views it is
rendered through, plus the host-side model the tests hold the device to.

A view V = [ux, vx, uy, vy, tx, ty] turns a layer with transform T into one with C = V ∘ T
(`compose`, exact `fmaf` from line_model) and a layer without one into one with C = V. The
oracle renders view b of a scene as an ordinary frame with C set on every layer (`set_view`).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np

import extremes
import line_model as lm
import line_scenes as ls
import scenes

f32 = np.float32
IDENTITY = [1.0, 0.0, 0.0, 1.0, 0.0, 0.0]
SEGMENT_BUDGET = 50_000_000  # pixel segments per call of an in-limit scene


def compose(v: Sequence[float], t: Optional[Sequence[float]]) -> List[float]:
    """C = V ∘ T in forma_layer_set_transform order, as line setup composes it."""
    if t is None:
        return [float(f32(x)) for x in v]
    vux, vvx, vuy, vvy, vtx, vty = (f32(x) for x in v)
    tux, tvx, tuy, tvy, ttx, tty = (f32(x) for x in t)
    with np.errstate(all="ignore"):
        c = [lm.fmaf(vux, tux, vvx * tuy), lm.fmaf(vux, tvx, vvx * tvy),
             lm.fmaf(vuy, tux, vvy * tuy), lm.fmaf(vuy, tvx, vvy * tvy),
             lm.fmaf(vux, ttx, lm.fmaf(vvx, tty, vtx)), lm.fmaf(vuy, ttx, lm.fmaf(vvy, tty, vty))]
    return [float(x) for x in c]


def about(k: int, cx: float, cy: float, ulps: int = 0) -> List[float]:
    """A rotation by k * 90 degrees (one ulp off with `ulps`) about (cx, cy)."""
    c, s = ls._rot(k, ulps)
    return ls._about(c, s, cx, cy)


def e2e_views(size: int) -> List[List[float]]:
    """Rotations by k * 90 degrees and one ulp off, reflections, a shear, zoom-outs, fractional
    and +-2^20 px translations, about the frame's centre."""
    m = size / 2.0
    return [about(1, m, m), about(2, m, m), about(3, m, m), about(1, m, m, ulps=1),
            [-1.0, 0.0, 0.0, 1.0, float(size), 0.0],          # mirror x
            [1.0, 0.25, 0.0, 0.9375, -3.5, 1.25],             # shear + fractional translation
            [0.5, 0.0, 0.0, 0.5, m / 2 + 0.375, m / 2 - 0.625],  # zoom-out
            [1.0, 0.0, 0.0, -1.0, 2.0 ** 20, 2.0 ** 20 + size],  # mirror y, 2^20 px below (culled: empty frame)
            [1.0, 0.0, 0.0, 1.0, -(2.0 ** 20), 0.25]]  # -2^20 px: lines left of the frame, rasterized there


@dataclass
class ViewScene:
    name: str
    build: Optional[Callable]  # (api, comp) -> {order: layer transform or None}; None: `specs`
    width: int
    height: int
    views: List[List[float]]
    specs: Optional[List[ls.LayerSpec]] = None  # line_scenes layers (with layer and path transforms)
    straddles: bool = False  # some view has lines above and below it, next to a neighbour with content
    over: bool = False       # the views together reach the 2^30 segment limit


def _orders(api, comp, xf=None):
    """{order: transform} of every layer of `comp` (probing orders until all are found)."""
    out, n, o = {}, len(comp), 0
    while len(out) < n:
        if comp.get(o) is not None:
            out[o] = None if xf is None else xf.get(o)
        o += 1
    return out


def _e2e(name):
    def build(api, comp):
        scenes.E2E[name](api, comp)
        return _orders(api, comp)
    return build


def _extreme(name):
    def build(api, comp):
        extremes.SCENES[name].build(api, comp)
        return _orders(api, comp)
    return build


def _paris(api, comp):
    import os

    from forma_b200 import svg
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    paths = svg.PathList.load(os.path.join(root, "tests", "data", "paris30k_paths.npz"))
    svg.compose(api, comp, paths, scale=1080.0 / 1060.0)
    return _orders(api, comp)


def _straddle_layers():
    """Rectangles and a star that cross the top and bottom edge of a 64 x 40 view, with layer and
    path transforms mixed in one composition."""
    return [
        ls.LayerSpec(0, None, [ls.rect(4, -12, 30, 10), ls.rect(34, 30, 60, 55)]),
        ls.LayerSpec(1, [0.8, -0.6, 0.6, 0.8, 10.0, -5.0], [ls.star(32, 20, 6, 30, 7)]),
        ls.LayerSpec(2, [1.0, 0.0, 0.0, 1.0, 0.5, 0.25], [ls.rect(-8, 35, 70, 45)],
                     path_xf=[0.5, 0.0, 8.0, 0.0, 0.5, 0.0, 0.0, 0.0, 1.0]),
        ls.LayerSpec(3, [0.6, 0.0, 0.0, 0.6, 3.0, 2.0], [ls.rect(10, -20, 50, 60)], even_odd=True),
    ]


def _long_layers(n_lines: int):
    """`n_lines` long horizontal-ish lines of about 2^24 px each on one layer (line_scenes' long
    lines): ~2^24 segments per line per view."""
    span = float(2 ** 24)
    paths = [[(-span / 2, 1.0 + k), (span / 2, 2.0 + k), (span / 2, 3.0 + k), (-span / 2, 2.0 + k)] for k in range(n_lines)]
    return [ls.LayerSpec(0, None, paths)]


FAR = 2.0 ** 20
ROTATIONS = ((0.8, 0.6), (0.6, -0.8), (-0.28, 0.96), (0.96, 0.28))


def far_compose_views(sign: float = 1.0) -> List[List[float]]:
    """Rotations whose translation cancels the layer's +-2^20 px one (_far_layers): C.tx and C.ty
    are sums at 2^20 px, where one rounding is 1/8 px, so the nesting of the two fmaf calls shows."""
    out = []
    for k, (c, s) in enumerate(ROTATIONS):
        c, s = float(f32(c)), float(f32(s))
        tx, ty = sign * FAR + 0.3, sign * FAR - 0.7
        out.append([c, -s, s, c, -(c * tx - s * ty) + 24.0 + k, -(s * tx + c * ty) + 20.0 - k])
    return out


FAR_POINTS_XF = [float(f32(0.8)), float(f32(-0.6)), float(f32(0.6)), float(f32(0.8)), 0.0, 0.0]


def far_points_views() -> List[List[float]]:
    """Rotations that bring the layer's points (about 2^20 px from the origin, rotated by
    FAR_POINTS_XF) back into the frame: 1 ulp of C's linear part moves them by about 1/10 px, so
    the order of the two products in C.ux ... C.vy shows."""
    t = FAR_POINTS_XF
    X, Y = t[0] * FAR + t[1] * FAR, t[2] * FAR + t[3] * FAR
    out = []
    for k, (c, s) in enumerate(ROTATIONS):
        c, s = float(f32(c)), float(f32(s))
        out.append([c, -s, s, c, -(c * X - s * Y) + 24.0 + k, -(s * X + c * Y) + 20.0 - k])
    return out


def nesting_matters(v: Sequence[float], t: Sequence[float]) -> bool:
    """Whether C.tx or C.ty changes when the two fmaf calls are nested the other way."""
    vux, vvx, vuy, vvy, vtx, vty = (f32(x) for x in v)
    ttx, tty = f32(t[4]), f32(t[5])
    c = compose(v, t)
    return (float(lm.fmaf(vvx, tty, lm.fmaf(vux, ttx, vtx))) != c[4]) or (float(lm.fmaf(vvy, tty, lm.fmaf(vuy, ttx, vty))) != c[5])


def linear_order_matters(v: Sequence[float], t: Sequence[float]) -> bool:
    """Whether some of C.ux ... C.vy changes when the two products of its fmaf are swapped."""
    vux, vvx, vuy, vvy = (f32(x) for x in v[:4])
    tux, tvx, tuy, tvy = (f32(x) for x in t[:4])
    with np.errstate(all="ignore"):
        swapped = [lm.fmaf(vvx, tuy, vux * tux), lm.fmaf(vvx, tvy, vux * tvx),
                   lm.fmaf(vvy, tuy, vuy * tux), lm.fmaf(vvy, tvy, vuy * tvx)]
    return [float(x) for x in swapped] != compose(v, t)[:4]


def _far_layers(sign: float = 1.0):
    """A star and a rectangle moved +-2^20 px away by their layer transform (brought back by the views)."""
    t = [1.0, 0.0, 0.0, 1.0, sign * FAR + 0.3, sign * FAR - 0.7]
    return [ls.LayerSpec(0, t, [ls.star(0, 0, 4, 14, 9)]), ls.LayerSpec(1, t, [ls.rect(-10, -3, 12, 5)], even_odd=True)]


def _far_point_layers():
    """A star and a rectangle whose points lie about 2^20 px from the origin, under a rotation."""
    return [ls.LayerSpec(0, FAR_POINTS_XF, [ls.star(FAR, FAR, 4, 14, 9)]),
            ls.LayerSpec(1, FAR_POINTS_XF, [ls.rect(FAR - 10, FAR - 3, FAR + 12, FAR + 5)], even_odd=True)]


def _inf_layers():
    """A rectangle and a contour whose points have x = -inf. Without a transform its line is
    skipped (both ends at the same y); under an identity applied as a transform, 0 * -inf makes y
    NaN and the line is kept: the rule that a composed identity is no transform shows in the count."""
    inf = float("inf")
    return [ls.LayerSpec(0, None, [ls.rect(4, 4, 40, 30)]), ls.LayerSpec(1, None, [[(-inf, 10.0), (-inf, 20.0), (-inf, 33.0)]])]


def _scenes() -> List[ViewScene]:
    out = []
    for name in sorted(scenes.E2E):
        out.append(ViewScene(f"e2e_{name}", _e2e(name), 64, 64, e2e_views(64)))
    shift = [[1.0, 0.0, 0.0, 1.0, 0.0, dy] for dy in (-20.0, -7.5, 0.0, 9.25, 20.0)]
    out.append(ViewScene("straddle", None, 64, 40, shift + [about(1, 32, 20)], _straddle_layers(), straddles=True))
    out.append(ViewScene("straddle_h100", None, 64, 100, shift + e2e_views(64)[:4], _straddle_layers()))
    for name in ("dense_stars", "nan_blends", "crowd_64", "winding_mixed_eo"):
        if name in extremes.SCENES:
            sc = extremes.SCENES[name]
            m = sc.width / 2.0, sc.height / 2.0
            out.append(ViewScene(f"extreme_{name}", _extreme(name), sc.width, sc.height,
                                 [IDENTITY, about(2, *m), [0.75, 0.0, 0.0, 0.75, 10.0, 3.0], [-1.0, 0.0, 0.0, 1.0, float(sc.width), 0.0]]))
    out.append(ViewScene("far_compose", None, 48, 40, far_compose_views(), _far_layers()))
    # One view whose every line lies 2^20 px left of the frame: its tile columns wrap (int16) into
    # columns 1 ... 5, which the sort must still order.
    out.append(ViewScene("far_left", _e2e("radial_gradient"), 64, 64, [[1.0, 0.0, 0.0, 1.0, -(2.0 ** 20), 0.25]]))
    out.append(ViewScene("far_compose_neg", None, 48, 40, far_compose_views(-1.0), _far_layers(-1.0)))
    out.append(ViewScene("far_points", None, 48, 40, far_points_views(), _far_point_layers()))
    out.append(ViewScene("inf_points", None, 48, 40, [IDENTITY, [1.0, 0.0, 0.0, 1.0, 0.5, 0.25]], _inf_layers()))
    # Odd sizes: heights 1, 100 and 1080, widths that are not multiples of 16.
    out.append(ViewScene("odd_h1", _e2e("clipping"), 61, 1, [[1.0, 0.0, 0.0, 1.0, 0.0, -float(y)] for y in range(0, 64, 4)]))
    out.append(ViewScene("odd_h100", _e2e("radial_gradient"), 77, 100, e2e_views(64)[:5]))
    out.append(ViewScene("odd_h1080", _e2e("texture"), 33, 1080, [[1.0, 0.0, 0.0, 1.0, 0.0, 0.0], about(2, 16.5, 540.0)]))
    # Paris: 16 translated 960 x 540 tiles of the 1920 x 1080 drawing, and 4 rotated or zoomed-out views.
    tiles = [[1.0, 0.0, 0.0, 1.0, -960.0 * (k % 2) - 480.0 * (k // 8), -540.0 * ((k // 2) % 2) - 270.0 * ((k // 4) % 2)]
             for k in range(16)]
    out.append(ViewScene("paris_tiles", _paris, 960, 540, tiles))
    out.append(ViewScene("paris_views", _paris, 1920, 1080,
                         [about(1, 960, 540), about(3, 960, 540, ulps=1), [0.5, 0.0, 0.0, 0.5, 480.0, 270.0],
                          [0.7, -0.7, 0.7, 0.7, 500.0, -400.0]]))
    # At the limit: n * rows == 2046 (max_views), with content in the first and the last view.
    out.append(ViewScene("limit_h16", _e2e("covers"), 64, 16,
                         [[1.0, 0.0, 0.0, 1.0, 0.0, -16.0 * (k % 4)] for k in range(2046)]))
    out.append(ViewScene("limit_h1000", _e2e("linear_gradient"), 64, 1000,  # 32 views of 63 rows: 2016 rows
                         [IDENTITY if k % 2 else about(2, 32, 32) for k in range(32)]))
    # Two views each below 2^30 segments, at or above it together.
    out.append(ViewScene("segment_limit", None, 64, 64,
                         [IDENTITY, [1.0, 0.0, 0.0, 1.0, 0.0, 10.0]], _long_layers(20), over=True))
    return out


SCENES: Dict[str, ViewScene] = {s.name: s for s in _scenes()}
IN_LIMIT = [n for n, s in SCENES.items() if not s.over]
OVER_LIMIT = [n for n, s in SCENES.items() if s.over]
LIMIT_SCENES = ["limit_h16", "limit_h1000"]  # n = max_views(height)


def build(api, sc: ViewScene):
    """(composition, {order: layer transform or None}) of scene `sc` on `api`."""
    if sc.specs is not None:
        comp, _, _ = ls.build(api, sc.specs)
        return comp, {s.order: (list(s.xf) if s.xf is not None else None) for s in sc.specs}
    comp = api.Composition()
    return comp, sc.build(api, comp)


def set_view(comp, xf: Dict[int, Optional[Sequence[float]]], v: Sequence[float]) -> None:
    """Every layer of `comp` gets C = v ∘ T: the ordinary frame equal to view `v`."""
    for order, t in xf.items():
        comp.get(order).set_transform(compose(v, t))


def rows(height: int) -> int:
    return (height + 15) // 16


def view_model(oracle_api, sc: ViewScene, v: Sequence[float]) -> dict:
    """line_model replayed on the composed transforms of view `v` (frame coordinates) of a scene
    built from line_scenes layers."""
    layers = [lm.LayerXf(s.order, compose(v, s.xf), s.enabled) for s in sc.specs]
    _, _, inserts = ls.build(oracle_api, sc.specs)
    x, y, ids = lm.point_buffer([(k, *p.segments()) for k, p in inserts])
    rec = lm.replay(x, y, ids, layers, sc.width, sc.height, (0.0, float(sc.height)))
    rec["counts"] = lm.counts(rec["length"], len(x))
    return rec


def outside_rows(rec: dict, height: int) -> tuple:
    """(lines of the view that reach above row 0, lines that reach below `height`)."""
    y0, dy, keep = rec["y0"] / 16.0, rec["dy"] / 16.0, rec["keep"]
    lo, hi = np.minimum(y0, y0 + dy), np.maximum(y0, y0 + dy)
    return int(np.sum(keep & (lo < 0))), int(np.sum(keep & (hi > height)))
