"""Scenes at the limits of line setup and rasterization (tests/line_model.py replays them).

Every scene is a list of layers, each with an order, an optional layer transform and polylines
(optionally under a path transform), built the same way on any API. `Scene.reached(model)` says
whether the scene reaches the condition it is there for; tests/test_line_scenes.py checks that
on the CPU before tests/test_gpu_lines.py lets the device see it.

- In-limit scenes (`over` False) are rendered on both sides and compared at tolerance 0.
- Over-limit scenes (`over` True) have a true pixel-segment total of 2^30 or more: the renderer
  refuses them with FORMA_ERR_CAPACITY and the oracle refuses those above 2^32 - 1.
- `ORIGINS` are single-segment lines for `rasterize_only` at widths up to 2^31, whose segment
  words tests/test_line_scenes.py derives by hand.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, List, Optional, Sequence

import numpy as np

import line_model as lm
from forma_b200.binding import Color, Fill, FillRule, Func, Point, Props, Style

W, H = 512, 384
f32 = np.float32


@dataclass
class LayerSpec:
    order: int
    xf: Optional[Sequence[float]] = None          # [ux, vx, uy, vy, tx, ty]
    paths: List[List[tuple]] = field(default_factory=list)
    path_xf: Optional[Sequence[float]] = None     # 9 values, Path.transform
    enabled: bool = True
    even_odd: bool = False


@dataclass
class Scene:
    name: str
    target: str
    layers: List[LayerSpec]
    reached: Callable[[dict], bool]
    width: int = W
    height: int = H
    over: bool = False
    crops: Sequence[tuple] = ()


def _color(k):
    return Color(((k * 37) % 11) / 10.0, ((k * 53) % 7) / 6.0, ((k * 17) % 5) / 4.0, 0.75)


def build_path(api, pts):
    pb = api.PathBuilder().move_to(Point(*pts[0]))
    for p in pts[1:]:
        pb.line_to(Point(*p))
    return pb.build()


def build(api, layers: Sequence[LayerSpec]):
    """(composition, [LayerXf], inserts for line_model.point_buffer) of `layers` on `api`."""
    comp = api.Composition()
    model_layers, inserts = [], []
    for k, spec in enumerate(layers):
        layer = comp.get_mut_or_insert_default(spec.order)
        for pts in spec.paths:
            path = build_path(api, pts)
            if spec.path_xf is not None:
                path = path.transform(spec.path_xf)
            layer.insert(path)
            inserts.append((k, path))
        layer.set_props(Props(fill_rule=FillRule.EvenOdd if spec.even_odd else FillRule.NonZero,
                              func=Func.Draw(Style(fill=Fill.Solid(_color(k))))))
        if spec.xf is not None:
            layer.set_transform(spec.xf)
        if not spec.enabled:
            layer.disable()
        model_layers.append(lm.LayerXf(spec.order, spec.xf, spec.enabled))
    return comp, model_layers, inserts


def model(oracle_api, scene: Scene, band=(-3.0e38, 3.0e38)) -> dict:
    """Replays line setup of the scene from the oracle's flattened points."""
    _, layers, inserts = build(oracle_api, scene.layers)
    x, y, ids = lm.point_buffer([(k, *p.segments()) for k, p in inserts])
    rec = lm.replay(x, y, ids, layers, scene.width, scene.height, band)
    rec["counts"] = lm.counts(rec["length"], len(x))
    rec["n_points"] = len(x)
    return rec


def star(cx, cy, r0, r1, n, phase=0.0):
    out = []
    for i in range(2 * n):
        r = r1 if i % 2 else r0
        a = phase + math.pi * i / n
        out.append((cx + r * math.cos(a), cy + r * math.sin(a)))
    return out


def rect(x0, y0, x1, y1):
    return [(x0, y0), (x1, y0), (x1, y1), (x0, y1)]


def _rot(k, ulps=0):
    c = [1.0, 0.0, -1.0, 0.0][k % 4]
    s = [0.0, 1.0, 0.0, -1.0][k % 4]
    if ulps:
        c = float(np.nextafter(f32(c), f32(0))) if c else float(np.nextafter(f32(0), f32(1)) * ulps)
        s = float(np.nextafter(f32(s), f32(0))) if s else float(np.nextafter(f32(0), f32(1)) * ulps)
    return c, s


def _about(c, s, cx, cy):
    """[ux, vx, uy, vy, tx, ty] of a rotation (c, s) about (cx, cy), in float32."""
    c, s, cx, cy = f32(c), f32(s), f32(cx), f32(cy)
    tx = cx - (c * cx - s * cy)
    ty = cy - (s * cx + c * cy)
    return [float(c), float(-s), float(s), float(c), float(tx), float(ty)]


def _fma_nesting_operands():
    """A rotation and points where fmaf(ux, x, fmaf(vx, y, tx)) differs from
    fmaf(vx, y, fmaf(ux, x, tx)), for x and y both, found by a seeded search."""
    rng = np.random.default_rng(11)
    a = 0.5235988
    xf = [math.cos(a), -math.sin(a), math.sin(a), math.cos(a), 170.3, 20.7]
    ux, vx, uy, vy, tx, ty = (f32(v) for v in xf)
    pts = []
    while len(pts) < 24:
        p = rng.uniform(40, 300, size=2).astype(np.float32)
        ax = lm.fmaf(ux, p[0], lm.fmaf(vx, p[1], tx))
        bx = lm.fmaf(vx, p[1], lm.fmaf(ux, p[0], tx))
        ay = lm.fmaf(uy, p[0], lm.fmaf(vy, p[1], ty))
        by = lm.fmaf(vy, p[1], lm.fmaf(uy, p[0], ty))
        if ax != bx or ay != by:
            pts.append((float(p[0]), float(p[1])))
    return xf, pts


def _nesting_matters(xf):
    """True when, on some kept line, the start point the model replays differs from what the two
    fmaf calls of the layer affine nested the other way give."""
    ux, vx, uy, vy, tx, ty = (f32(v) for v in xf)

    def reached(rec):
        x, y = rec["source_points"]
        k = rec["keep"]
        ax = lm.fmaf(vx, y[k], lm.fmaf(ux, x[k], tx))
        ay = lm.fmaf(vy, y[k], lm.fmaf(uy, x[k], ty))
        p0x, p0y = rec["end_points"][0][k], rec["end_points"][1][k]
        return int(k.sum()) >= 16 and bool(np.any(ax != p0x)) and bool(np.any(ay != p0y))
    return reached


def _tri(x):
    """A right triangle with legs of x px: 2 x + 1 pixel segments when x is at least the frame's
    width (only the diagonal survives the skip rules), 3 x - 1 inside the frame."""
    return [(0.5, 0.5), (x, 0.5), (x, x)]


# Zig-zag above the frame: 300 points whose lines are all skipped (y <= 0), so that the paths on
# either side of it fall in different CTAs of the count pass.
FILLER = [(1.0 + 0.01 * i, -1.0 - (i % 2)) for i in range(300)]


def _scan_saturates(rec):
    """Several CTAs with segments, each CTA's sum below 2^32, their running sum past it."""
    b = [int(v) for v in rec["counts"].block_sums]
    return sum(v > 0 for v in b) >= 2 and max(b) < 2 ** 32 and sum(b) > 2 ** 32 and (sum(b) & lm.U32_MAX) < lm.SEGMENT_LIMIT


SUB = float(np.nextafter(f32(0), f32(1)) * 2 ** 9)  # 2^-140: a subnormal scale


def _scenes() -> List[Scene]:
    out = []
    blob = [star(100, 100, 30, 70, 7), rect(20.25, 30.5, 90.75, 60.03125)]
    # Rotations by k * 90 degrees about the frame's centre and one ulp off each.
    layers = []
    for k in range(4):
        for ulps in (0, 1):
            c, s = _rot(k, ulps)
            layers.append(LayerSpec(len(layers), _about(c, s, W / 2, H / 2), blob))
    out.append(Scene("rotations", "rotations by k * 90 degrees and one ulp off them", layers,
                     lambda rec: int(rec["keep"].sum()) > 100, crops=((0, W, 100, 260),)))
    # Reflections and shears (column norms within the GeomPresTransform limit).
    out.append(Scene("reflect_shear", "reflections and shears", [
        LayerSpec(0, [-1, 0, 0, 1, W, 0], blob),
        LayerSpec(1, [1, 0, 0, -1, 0, H], blob),
        LayerSpec(2, [1, 0.6, 0, 0.8, 150, 50], blob),
        LayerSpec(3, [0.8, 0, 0.6, 1, 200, 30], blob, even_odd=True),
    ], lambda rec: int(rec["keep"].sum()) > 60))
    # Shrinks to subnormal scales: dx / dy subnormal, 1 / dy infinite, both find_param branches.
    out.append(Scene("subnormal", "subnormal dx and dy, infinite 1/dx and 1/dy", [
        LayerSpec(0, [SUB, 0, 0, SUB, 0, 0], blob),
        LayerSpec(1, [1, 0, 0, SUB, 0, 0], blob),
        LayerSpec(2, [SUB, 0, 0, 1, 0, 0], blob),
        LayerSpec(3, [SUB * 0.5, 0, 0, SUB * 0.25, 0, 2 ** -126], blob),
    ], lambda rec: bool(np.any(np.isinf(rec["b"])) and np.any(np.isinf(rec["a"]))
                        and np.any(np.isfinite(rec["b"]) & (rec["b"] > 0) & np.isinf(rec["a"])))))
    # Translations far out, and back in through float32 rounding.
    far = [[(x + 2 ** 22, y + 2 ** 22) for x, y in p] for p in blob]
    out.append(Scene("translations", "translations of +-2^22, +-2^27, +-2^31 px and -inf", [
        LayerSpec(0, [1, 0, 0, 1, -2 ** 22, -2 ** 22], far),
        LayerSpec(1, [1, 0, 0, 1, 2 ** 22, 0], blob),
        LayerSpec(2, [1, 0, 0, 1, -2 ** 27, 0], blob),
        LayerSpec(3, [1, 0, 0, 1, 2 ** 27, 2 ** 27], blob),
        LayerSpec(4, [1, 0, 0, 1, -2 ** 31, 10], blob),
        LayerSpec(5, [1, 0, 0, 1, 2 ** 31, 0], blob),
        LayerSpec(6, [1, 0, 0, 1, -math.inf, 0], blob),
        LayerSpec(7, [1, 0, 0, 1, 0, -2 ** 27], blob),
    ], lambda rec: bool(np.any(rec["keep"] & np.isinf(rec["x0"]))) and bool(np.any(rec["keep"] & (rec["x0"] <= -2.0 ** 31)))))
    # NaN in the linear part and in the translation (geom_pres_ok accepts NaN).
    out.append(Scene("nan", "NaN in the linear part or the translation", [
        LayerSpec(0, [math.nan, 0, 0, 1, 0, 0], blob),
        LayerSpec(1, [1, 0, 0, 1, math.nan, 0], blob),
        LayerSpec(2, [1, math.nan, 0, 1, 0, 0], blob),
        LayerSpec(3, [1, 0, 0, 1, 50, 0], blob),
    ], lambda rec: bool(np.any(rec["keep"] & np.isnan(rec["x0"])))))
    # Operands where the nesting of the two fmaf calls changes the result.
    xf, pts = _fma_nesting_operands()
    out.append(Scene("fma_nesting", "operands where the nesting order of the two fmaf calls matters",
                     [LayerSpec(0, xf, [pts[i:i + 3] for i in range(0, len(pts), 3)])],
                     _nesting_matters(xf)))
    # End points exactly on the skip boundaries, and on rounding ties (half sub-pixels).
    h = 1.0 / 32.0
    edges = [
        [(5, 0), (7, -3), (9, 0)], [(20, 0), (22, 3), (24, 0)],
        [(40, H), (42, H + 3), (44, H)], [(60, H), (62, H - 3), (64, H)],
        [(W, 50), (W + 3, 60), (W, 70)], [(W - 1, 80), (W + 3, 90), (W - 1, 100)],
        [(100 + h, 100 + h), (101 + 3 * h, 120 + h), (103, 100.5 + h)],
        [(150, 150), (151, 151), (152, 150), (151, 149)],
        [(200 + 0.5 + h, 140 - h), (202.5 - h, 170 + 5 * h), (205.5, 140)],
    ]
    out.append(Scene("edges", "end points on y = 0, y = height, x = width, integers and half sub-pixels", [
        LayerSpec(0, None, edges), LayerSpec(1, [1, 0, 0, 1, 0.5, 0.25], edges),
    ], lambda rec: bool(np.any(rec["end_points"][1] == 0) and np.any(rec["end_points"][2] == W)),
        crops=((0, W, 16, 96), (0, W, 80, 144), (0, W, 368, 384))))
    # Band edges under a crop: layer transforms turn the band filter off, only the per-line cull applies.
    bands = []
    for e in (16.0, 96.0):
        for dy in (-1.0 / 16.0, -1.0 / 32.0, 0.0, 1.0 / 32.0):
            y = e + dy
            bands.append([(10 + 30 * len(bands) % 480, y), (25 + 30 * len(bands) % 480, y - 5), (40 + 30 * len(bands) % 480, y)])
            bands.append([(12 + 30 * len(bands) % 480, y), (27 + 30 * len(bands) % 480, y + 5), (42 + 30 * len(bands) % 480, y)])
    out.append(Scene("band_edges", "end points on and 1/16, 1/32 px off the band edges of a crop", [
        LayerSpec(0, [1, 0, 0, 1, 0, 0.0], bands), LayerSpec(1, None, bands),
    ], lambda rec: bool(np.any(rec["end_points"][1] == f32(16.0 - 1.0 / 16.0))), crops=((0, W, 16, 96), (0, W, 17, 95))))
    # Tile wrap: segments at y and x around 2^20 px wrap through `as i16` into tile row / column 0.
    # (Long thin spikes are merged away by the flattening: the shapes are right triangles.)
    out.append(Scene("tile_wrap", "lines into y, x ~ 2^20 px whose tiles wrap through i16", [
        LayerSpec(0, None, [[(10, 10), (20, 10), (20, 2 ** 20)]]),
        LayerSpec(1, None, [[(10, 20), (2 ** 20, 20), (2 ** 20, 40)]]),
    ], lambda rec: int(rec["counts"].total) > 2 ** 20))
    # The same to the other side: one end in the frame, the other 2^20 px above or left of it. The
    # skip rules keep such a line (only a line with both ends outside is dropped), and its tiles
    # wrap through i16 into every value of the tile_y / tile_x field: the sort's plan must keep
    # all of that field's bits although the frame itself needs two or three.
    out.append(Scene("far_up", "a line from inside the frame to y ~ -2^20 px: tile rows wrap into all 11 bits", [
        LayerSpec(0, None, [[(10, 20), (2 ** 20, 20), (10, -2 ** 20)]]),
        LayerSpec(1, None, blob),
    ], lambda rec: bool(np.any(rec["keep"] & (np.minimum(rec["y0"], rec["y0"] + rec["dy"]) < -32770 * 256.0)
                               & (np.maximum(rec["y0"], rec["y0"] + rec["dy"]) > 0)))))
    out.append(Scene("far_left_line", "a line from inside the frame to x ~ -2^20 px: tile columns wrap into all 12 bits", [
        LayerSpec(0, None, [[(20, 10), (20, 2 ** 20), (-2 ** 20, 10)]]),
        LayerSpec(1, None, blob),
    ], lambda rec: bool(np.any(rec["keep"] & (np.minimum(rec["x0"], rec["x0"] + rec["dx"]) < -32770 * 256.0)
                               & (np.maximum(rec["x0"], rec["x0"] + rec["dx"]) > 0)))))
    # Long lines: one line of ~6e6 segments has every segment of its CTA, the other 255 lines
    # (zig-zags above the frame or right of it) have none, at CTA positions 0 and 255 too.
    zig = [(1 + 0.01 * i, -1.0 - (i % 2)) for i in range(100)] + [(3.0e6, 3.0e6)]
    zig += [(3.0e6 + 1 + 0.5 * i, -1.0 - (i % 2)) for i in range(160)]
    out.append(Scene("long_lines", "one line of ~6e6 segments, alone in its CTA", [
        LayerSpec(0, None, [zig]),
    ], lambda rec: (int(rec["length"].max()) > 2 ** 22 and int(rec["length"][0]) == 0 and int(rec["length"][255]) == 0
                    and int(rec["counts"].block_sums[0]) == int(rec["length"].max()))))
    # Layer and path transforms together: a GeomPresTransform path transform and a projective one.
    c, s = math.cos(0.3), math.sin(0.3)
    out.append(Scene("layer_and_path", "a layer affine over a GeomPres and a projective path transform", [
        LayerSpec(0, _about(c, s, 200, 150), blob, path_xf=[c, -s, 40, s, c, 10, 0, 0, 1]),
        LayerSpec(1, [0.9, 0.1, -0.1, 0.9, 30, 40], blob, path_xf=[1, 0.2, 0, 0.1, 1, 0, 0.0005, 0.0002, 1]),
    ], lambda rec: int((rec["keep"] & (rec["orders"] == 0)).sum()) > 0 and int((rec["keep"] & (rec["orders"] == 1)).sum()) > 0))
    # Over the limit (`reached` also requires the renderer's status to be FORMA_ERR_CAPACITY).
    out.append(Scene("exactly_2p30", "a true total of exactly 2^30", [
        # only the diagonal of the large triangle survives the skip rules (2 X + 1 segments); the
        # small one lies in the frame (3 x - 1): 2 (2^29 - 96) + 1 + 3 * 64 - 1 = 2^30
        LayerSpec(0, None, [[(0.5, 0.5), (2.0 ** 29 - 96, 0.5), (2.0 ** 29 - 96, 2.0 ** 29 - 96)], _tri(64.0)]),
    ], lambda rec: rec["counts"].total == 2 ** 30, over=True))
    out.append(Scene("past_2p30", "a true total of 2^30 + 1, below 2^32", [
        LayerSpec(0, None, [_tri(2.0 ** 29)]),
    ], lambda rec: rec["counts"].total == 2 ** 30 + 1, over=True))
    out.append(Scene("wrap_2p32", "a true total of 2^32 + 7, which wraps to 7", [
        LayerSpec(0, None, [_tri(2.0 ** 30)] * 2 + [_tri(2.0)]),
    ], lambda rec: rec["counts"].total == 2 ** 32 + 7 and int(rec["counts"].prefix_u32[-1]) == 7, over=True))
    out.append(Scene("scan_wrap", "2^32 + 7 spread over CTAs: each CTA sum fits u32, the device-wide scan does not", [
        LayerSpec(0, None, [_tri(2.0 ** 30), FILLER, _tri(2.0 ** 30), FILLER, _tri(2.0)]),
    ], _scan_saturates, over=True))
    out.append(Scene("block_wrap", "nine triangles of 2^29 + 1 segments in one CTA", [
        LayerSpec(0, None, [_tri(2.0 ** 28)] * 9),
    ], lambda rec: int(rec["counts"].block_sums[0]) > 2 ** 32
        and (int(rec["counts"].block_sums[0]) & lm.U32_MAX) < lm.SEGMENT_LIMIT, over=True))
    out.append(Scene("span_3e38", "one line from (-3e38, 5) to (3e38, 20)", [
        LayerSpec(0, None, [[(-3.0e38, 5), (3.0e38, 20), (3.0e38, 30)]]),
    ], lambda rec: bool(rec["saturated"].any()) and int(rec["counts"].prefix_u32[-1]) < lm.SEGMENT_LIMIT, over=True))
    return out


def _over_reached(rec):
    c = rec["counts"]
    return c.status == lm.FORMA_ERR_CAPACITY


SCENES = {s.name: s for s in _scenes()}
for _s in SCENES.values():
    if _s.over:
        _s.reached = (lambda f: lambda rec: _over_reached(rec) and f(rec))(_s.reached)
IN_LIMIT = [n for n, s in SCENES.items() if not s.over]
OVER_LIMIT = [n for n, s in SCENES.items() if s.over]

# Single-segment vertical lines for rasterize_only at width 2^31: (x px, y0, y1). Their sub-pixel
# x (16 x) is 2^31 and more from 2^27 px on; the last one goes through a NaN layer transform.
ORIGIN_WIDTH = 2 ** 31
ORIGINS = [(2.0 ** 26, 5.25, 5.75), (2.0 ** 27 - 64, 6.25, 6.75), (2.0 ** 27, 7.25, 7.75), (2.0 ** 28, 8.25, 8.75),
           (2.0 ** 30, 9.25, 9.75), (math.nan, 10.25, 10.75)]


def origin_layers():
    """Each origin as a right triangle whose first line is the vertical one, (x, y0) -> (x, y1):
    one pixel segment with t0 = 0 and t1 = 1."""
    out = []
    for k, (x, y0, y1) in enumerate(ORIGINS):
        if math.isnan(x):
            out.append(LayerSpec(k, [math.nan, 0, 0, 1, 0, 0], [[(0.0, y0), (0.0, y1), (64.0, y1)]]))
        else:
            step = 2.0 ** max(6, math.frexp(x)[1] - 20)
            out.append(LayerSpec(k, None, [[(x, y0), (x, y1), (x + step, y1)]]))
    return out
