"""Scenes of poses (Renderer.render_poses): a composition, a frame size and the pose tables it is
rendered with, plus `set_pose`, which puts a composition (binding or oracle) into pose b.

A pose gives each layer at an order of the window [first_order, first_order + K) its own
transform and visibility for one frame. Frame b of a poses call is the ordinary frame of the
composition after `set_pose(comp, scene, orders, b)`: set_transform(transforms[b, k]) when the
scene has transforms, set_is_enabled(visible[b, k]) when it has visibility, for every layer
attached at an order of the window.
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np

import line_scenes as ls
import scenes
import synth
import view_scenes as vs

f32 = np.float32
IDENTITY = [1.0, 0.0, 0.0, 1.0, 0.0, 0.0]
LAYER_LIMIT = 1 << 21
E2E_K = 66  # the window of the e2e scenes: every layer of each, and orders without one


@dataclass
class PoseScene:
    name: str
    build: Callable            # api -> (composition, sorted list of attached orders)
    width: int
    height: int
    first_order: int
    transforms: Optional[np.ndarray]  # [n, K, 6] float32, or None
    visible: Optional[np.ndarray]     # [n, K] uint8, or None
    differ: Sequence[tuple] = ()      # pairs of frames (a, b) whose poses must differ
    heavy: bool = False               # large: the GPU tests take it only where they say so

    @property
    def n(self) -> int:
        return (self.transforms if self.transforms is not None else self.visible).shape[0]

    @property
    def n_orders(self) -> int:
        return (self.transforms if self.transforms is not None else self.visible).shape[1]


def window_orders(sc: PoseScene, orders: Sequence[int]) -> List[int]:
    """The attached orders inside the scene's window."""
    return [o for o in orders if sc.first_order <= o < sc.first_order + sc.n_orders]


def set_pose(comp, sc: PoseScene, orders: Sequence[int], b: int) -> None:
    """Puts `comp` (built by sc.build, with attached `orders`) into pose b of the scene."""
    for o in window_orders(sc, orders):
        k = o - sc.first_order
        layer = comp.get(o)
        if sc.transforms is not None:
            layer.set_transform([float(x) for x in sc.transforms[b, k]])
        if sc.visible is not None:
            layer.set_is_enabled(bool(sc.visible[b, k]))


def poses(api_binding, sc: PoseScene):
    """The binding's Poses value of the scene."""
    return api_binding.Poses(sc.first_order, sc.transforms, sc.visible)


def _orders(comp) -> List[int]:
    out, n, o = [], len(comp), 0
    while len(out) < n:
        if comp.get(o) is not None:
            out.append(o)
        o += 1
    return out


def _e2e(name):
    def build(api):
        comp = api.Composition()
        scenes.E2E[name](api, comp)
        return comp, _orders(comp)
    return build


def _specs(specs: List[ls.LayerSpec]):
    def build(api):
        comp, _, _ = ls.build(api, specs)
        return comp, sorted(s.order for s in specs)
    return build


def _about(angle: float, cx: float, cy: float, scale: float = 1.0) -> List[float]:
    c, s = f32(scale * math.cos(angle)), f32(scale * math.sin(angle))
    cx, cy = f32(cx), f32(cy)
    return [float(c), float(-s), float(s), float(c), float(cx - (c * cx - s * cy)), float(cy - (s * cx + c * cy))]


def _ulp_identity() -> List[float]:
    one_down = float(np.nextafter(f32(1.0), f32(0.0)))
    tiny = float(np.nextafter(f32(0.0), f32(1.0)))
    return [one_down, tiny, 0.0, one_down, 0.0, tiny]


def e2e_pose_table(n_orders: int, size: int) -> np.ndarray:
    """Six poses of K layers: per layer a different rotation, shear, zoom-out, translation or an
    ulp-near identity (and the identity itself), about the frame's centre."""
    m = size / 2.0
    kinds = [
        lambda b, k: _about(0.3 * (b + 1) + 0.7 * k, m, m),
        lambda b, k: [1.0, 0.25 * ((b + k) % 3 - 1), 0.0, 0.9375, -3.5 + b, 1.25 - k],
        lambda b, k: _about(0.0, m, m, 0.5 + 0.125 * ((b + k) % 3)),
        lambda b, k: [1.0, 0.0, 0.0, 1.0, 2.5 * (b - k), -1.75 * b],
        lambda b, k: _ulp_identity(),
        lambda b, k: IDENTITY,
    ]
    t = np.empty((6, n_orders, 6), f32)
    for b in range(6):
        for k in range(n_orders):
            t[b, k] = kinds[(b + k) % len(kinds)](b, k)
    return t


def _straddle_specs(disabled: bool = False):
    specs = vs._straddle_layers()
    if disabled:
        specs[1].enabled = False
    return specs


def _window_edge_specs():
    """Layers inside a window [3, 9) (orders 3, 5, 8; orders 4, 6, 7 empty), and outside it layers
    with their own transform, one disabled."""
    return [
        ls.LayerSpec(0, [0.8, -0.6, 0.6, 0.8, 10.0, -5.0], [ls.rect(2, 2, 30, 20)]),
        ls.LayerSpec(1, None, [ls.star(40, 20, 5, 15, 6)], enabled=False),
        ls.LayerSpec(3, None, [ls.rect(10, 10, 40, 30)]),
        ls.LayerSpec(5, [1.0, 0.0, 0.0, 1.0, 3.0, 2.0], [ls.star(30, 20, 4, 12, 5)]),
        ls.LayerSpec(8, None, [ls.rect(20, 5, 60, 35)], even_odd=True),
        ls.LayerSpec(12, [0.5, 0.0, 0.0, 0.5, 8.0, 4.0], [ls.rect(0, 0, 64, 40)]),
    ]


def _top_order_specs():
    """Layers at the last orders of the layer field, and one far below them."""
    top = LAYER_LIMIT - 1
    return [ls.LayerSpec(0, None, [ls.rect(0, 0, 64, 40)]),
            ls.LayerSpec(top - 5, None, [ls.star(20, 20, 4, 16, 7)]),
            ls.LayerSpec(top, [1.0, 0.0, 0.0, 1.0, 5.0, 0.0], [ls.rect(30, 8, 60, 36)])]


def _spaceship_build(api):
    comp = api.Composition()
    synth.spaceship_scene(api, comp, 400, 1920, 1080, 43)
    return comp, list(range(402))


def spaceship_table(n_frames: int = 200):
    """The transforms of synth.spaceship_scene's animate(f), f < n_frames, for orders 1 ... 401
    (the backdrop at order 0 stays): the same motion function, the same float32 roundings."""
    w, h = 1920, 1080
    rng = synth.SplitMix64(43)
    movers = []
    for i in range(401):
        ship = i == 400
        if not ship:
            rng.uniform(8.0, 60.0)
        k = 3 if ship else 6 + rng.randint(5)
        for _ in range(k):
            if not ship:
                rng.uniform(0.7, 1.3)
        rng.uniform(0.3, 0.8)
        movers.append((rng.uniform(0.0, w), rng.uniform(0.0, h), rng.uniform(-120.0, 120.0), rng.uniform(-120.0, 120.0)))
    t = np.empty((n_frames, 401, 6), f32)
    dt = 1.0 / 60.0
    for f in range(n_frames):
        for j, (x0, y0, vx, vy) in enumerate(movers):
            t[f, j] = [1.0, 0.0, 0.0, 1.0, synth.f32((x0 + vx * dt * f) % w), synth.f32((y0 + vy * dt * f) % h)]
    return t


def _paris_build(api):
    from forma_b200 import svg
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    paths = svg.PathList.load(os.path.join(root, "tests", "data", "paris30k_paths.npz"))
    comp = api.Composition()
    svg.compose(api, comp, paths, scale=1080.0 / 1060.0)
    return comp, _orders(comp)


PARIS_LAYERS = 50620


def paris_table(n_frames: int = 16, n_orders: int = PARIS_LAYERS) -> np.ndarray:
    """Every layer its own translation per frame: a 960 x 540 tile of the drawing, jittered per layer."""
    rng = np.random.default_rng(5)
    t = np.zeros((n_frames, n_orders, 6), f32)
    t[:, :, 0] = t[:, :, 3] = 1.0
    for b in range(n_frames):
        ox, oy = -480.0 * (b % 3), -270.0 * ((b // 3) % 3)
        t[b, :, 4] = (ox + rng.uniform(-6.0, 6.0, n_orders)).astype(f32)
        t[b, :, 5] = (oy + rng.uniform(-6.0, 6.0, n_orders)).astype(f32)
    return t


LIBRARY_SHAPES = 64


def _library_build(api):
    """64 shapes: stars, rectangles and circles of 6 to 20 px about the origin, some translucent."""
    from forma_b200.binding import Color, Fill, Func, Props, Style
    comp = api.Composition()
    for k in range(LIBRARY_SHAPES):
        r = 6.0 + (k * 7) % 15
        if k % 3 == 0:
            path = ls.build_path(api, ls.star(0.0, 0.0, r * 0.45, r, 5 + k % 4))
        elif k % 3 == 1:
            path = ls.build_path(api, ls.rect(-r, -r * 0.6, r, r * 0.6))
        else:
            path = synth.circle_path(api, 0.0, 0.0, r)
        col = Color(((k * 37) % 11) / 10.0, ((k * 53) % 7) / 6.0, ((k * 17) % 5) / 4.0, 1.0 if k % 4 else 0.6)
        comp.get_mut_or_insert_default(k).insert(path).set_props(Props(func=Func.Draw(Style(fill=Fill.Solid(col)))))
    return comp, list(range(LIBRARY_SHAPES))


def library_tables(n_frames: int = 511, size: int = 64):
    """Frame b: a random subset of the library, each shape at a random offset (and a few rotated)."""
    rng = np.random.default_rng(11)
    vis = (rng.random((n_frames, LIBRARY_SHAPES)) < 0.2).astype(np.uint8)
    t = np.zeros((n_frames, LIBRARY_SHAPES, 6), f32)
    ang = np.where(rng.random((n_frames, LIBRARY_SHAPES)) < 0.25, rng.uniform(0, 2 * np.pi, (n_frames, LIBRARY_SHAPES)), 0.0)
    t[:, :, 0] = np.cos(ang).astype(f32)
    t[:, :, 1] = -np.sin(ang).astype(f32)
    t[:, :, 2] = np.sin(ang).astype(f32)
    t[:, :, 3] = np.cos(ang).astype(f32)
    t[:, :, 4] = rng.uniform(-8.0, size + 8.0, (n_frames, LIBRARY_SHAPES)).astype(f32)
    t[:, :, 5] = rng.uniform(-8.0, size + 8.0, (n_frames, LIBRARY_SHAPES)).astype(f32)
    return t, vis


def _vis(rows: Sequence[Sequence[int]]) -> np.ndarray:
    return np.asarray(rows, np.uint8)


def _xf(rows) -> np.ndarray:
    return np.asarray(rows, f32)


def _scenes() -> List[PoseScene]:
    out = []
    for name in sorted(scenes.E2E):  # (the texture scene has 64 layers, the others up to 7)
        out.append(PoseScene(f"e2e_{name}", _e2e(name), 64, 64, 0, e2e_pose_table(E2E_K, 64), None, differ=[(0, 1)]))
    # Clips: moved off their clipped layers, hidden (the clipped layer has no active clip and is not
    # drawn), clipped layers hidden. Orders 0 ... 6 of e2e clipping (1 is Clip(4)).
    off = IDENTITY[:4] + [40.0, 40.0]
    out.append(PoseScene("clip_moved", _e2e("clipping"), 64, 64, 1, _xf([[IDENTITY], [off], [[1.0, 0.0, 0.0, 1.0, -20.0, 3.0]]]), None,
                         differ=[(0, 1), (1, 2)]))
    out.append(PoseScene("clip_hidden", _e2e("clipping"), 64, 64, 0,
                         None, _vis([[1, 1, 1, 1, 1, 1, 1], [1, 0, 1, 1, 1, 1, 1], [1, 1, 0, 1, 1, 0, 0], [0, 0, 1, 1, 0, 1, 1]]),
                         differ=[(0, 1), (0, 2), (1, 3)]))
    out.append(PoseScene("clip2_both", _e2e("clipping2"), 64, 64, 1,
                         _xf([[IDENTITY, IDENTITY], [_about(0.5, 32, 32), IDENTITY], [IDENTITY, [1, 0, 0, 1, 9.0, -4.0]]]),
                         _vis([[1, 1], [1, 1], [0, 1]]), differ=[(0, 1), (1, 2)]))
    # Gradients and textures moved (they stay in frame coordinates).
    for name in ("linear_gradient", "radial_gradient", "texture"):
        t = np.stack([np.tile(_xf(p), (E2E_K, 1)) for p in ([1, 0, 0, 1, 10.0, -6.0], _about(1.1, 32, 32), _about(0.0, 32, 32, 0.6))])
        out.append(PoseScene(f"moved_{name}", _e2e(name), 64, 64, 0, t, None, differ=[(0, 1)]))
    # inf_points under an identity pose (no transform: the -inf line stays skipped) and a real one.
    out.append(PoseScene("inf_points", _specs(vs._inf_layers()), 48, 40, 0,
                         _xf([[IDENTITY, IDENTITY], [IDENTITY, [1.0, 0.0, 0.0, 1.0, 0.5, 0.25]], [[1.0, 0.0, 0.0, 1.0, 0.5, 0.0], IDENTITY]]),
                         None, differ=[(0, 1)]))
    # NaN and infinite translations (forma_layer_set_transform accepts them).
    nan, inf = float("nan"), float("inf")
    out.append(PoseScene("nonfinite", _specs(_straddle_specs()), 64, 40, 0,
                         _xf([[[1, 0, 0, 1, nan, 0.0], IDENTITY, [1, 0, 0, 1, 0.0, inf], IDENTITY],
                              [IDENTITY, [0.8, -0.6, 0.6, 0.8, -inf, 2.0], IDENTITY, [0.6, 0, 0, 0.6, nan, nan]],
                              [IDENTITY] * 4]), None, differ=[(0, 1), (1, 2)]))
    # A disabled layer shown and an enabled layer hidden; visibility only and transforms only, on
    # both layer-record paths (straddle has layer transforms: 36-byte records; e2e none: 4 bytes).
    out.append(PoseScene("show_hide", _specs(_straddle_specs(disabled=True)), 64, 40, 0, None,
                         _vis([[1, 1, 1, 1], [0, 1, 0, 1], [1, 0, 1, 0], [0, 0, 0, 0]]), differ=[(0, 1), (1, 2), (2, 3)]))
    out.append(PoseScene("show_hide_bits", _e2e("covers"), 64, 64, 0, None,
                         _vis([[1, 0, 1, 0], [0, 1, 0, 1], [1, 1, 1, 1]]), differ=[(0, 1), (1, 2)]))
    out.append(PoseScene("transform_only", _specs(_straddle_specs(disabled=True)), 64, 40, 0,
                         np.stack([np.tile(_xf(_about(0.4 * b, 32, 20)), (4, 1)) for b in range(5)]), None, differ=[(0, 1)]))
    # Window edges: K = 1; a window with empty orders and untouched layers around it; a window past
    # the last order; a window at the top of the layer field (first_order + K = 2^21).
    out.append(PoseScene("k1", _specs(_window_edge_specs()), 64, 40, 5, _xf([[[1, 0, 0, 1, 5.0 * b, -2.0 * b]] for b in range(4)]),
                         _vis([[1], [0], [1], [1]]), differ=[(0, 1), (0, 2)]))
    wt = np.stack([np.stack([_about(0.2 * b + 0.1 * k, 32, 20) for k in range(6)]) for b in range(3)]).astype(f32)
    out.append(PoseScene("window_gaps", _specs(_window_edge_specs()), 64, 40, 3, wt,
                         _vis([[1, 1, 1, 1, 1, 1], [0, 0, 1, 1, 1, 0], [1, 0, 0, 0, 0, 1]]), differ=[(0, 1), (1, 2)]))
    out.append(PoseScene("window_past_end", _specs(_window_edge_specs()), 64, 40, 13,
                         np.tile(_xf(_about(0.5, 32, 20)), (2, 3, 1)), _vis([[0, 0, 0], [1, 1, 1]])))
    top_t = np.tile(_xf(IDENTITY), (3, 8, 1))
    top_t[1, 2] = [0.6, -0.8, 0.8, 0.6, 30.0, -10.0]
    top_t[2, 7] = [1.0, 0.0, 0.0, 1.0, -12.0, 4.0]
    out.append(PoseScene("window_top", _specs(_top_order_specs()), 64, 40, LAYER_LIMIT - 8, top_t,
                         _vis([[1] * 8, [1] * 8, [1, 1, 0, 1, 1, 1, 1, 1]]), differ=[(0, 1), (0, 2)]))
    # Workloads: the spaceship animation, paris with every layer its own translation, a shape library.
    out.append(PoseScene("spaceship1080p", _spaceship_build, 1920, 1080, 1, spaceship_table(), None, differ=[(0, 199)], heavy=True))
    out.append(PoseScene("paris_poses", _paris_build, 960, 540, 0, paris_table(), None, differ=[(0, 1)], heavy=True))
    lt, lv = library_tables()
    out.append(PoseScene("library_511x64", _library_build, 64, 64, 0, lt, lv, differ=[(0, 1), (1, 510)], heavy=True))
    return out


SCENES: Dict[str, PoseScene] = {s.name: s for s in _scenes()}
LIGHT = [n for n, s in SCENES.items() if not s.heavy]
HEAVY = [n for n, s in SCENES.items() if s.heavy]
