"""Scenes of pose fills (Renderer.render_poses* with Poses(colors=...)): a composition, a frame
size and the pose tables it is rendered with, plus `set_pose_fill`, which puts a composition
(binding or oracle) into the state of frame b.

Frame b of a call with colours is the ordinary frame of the composition after `set_pose` (the
transforms and visibility, see tests/pose_scenes.py) and, for every layer attached at an order of
the window whose func is Draw(style), set_props with the layer's own props except that the fill is
Fill.Solid(colors[b, k]). The binding keeps no Props on a Layer, so every scene records the props
each layer was given while it was built (`record_props`).
"""
from __future__ import annotations

import dataclasses
import weakref
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np

import line_scenes as ls
import pose_scenes as ps
import scenes
from forma_b200 import binding
from forma_b200.binding import BlendMode, Color, Fill, Func, Props, Style

f32 = np.float32
NAN, INF = float("nan"), float("inf")
ONE_DOWN = float(np.nextafter(f32(1.0), f32(0.0)))


@dataclass
class FillScene:
    name: str
    build: Callable            # api -> (composition, sorted list of attached orders); props recorded
    width: int
    height: int
    first_order: int
    colors: Optional[np.ndarray]      # [n, K, 4] float32, or None
    transforms: Optional[np.ndarray] = None  # [n, K, 6] float32, or None
    visible: Optional[np.ndarray] = None     # [n, K] uint8, or None
    heavy: bool = False

    def _table(self):
        return next(t for t in (self.colors, self.transforms, self.visible) if t is not None)

    @property
    def n(self) -> int:
        return self._table().shape[0]

    @property
    def n_orders(self) -> int:
        return self._table().shape[1]


# The props each layer of a composition was given while its scene was built, by order.
_PROPS: "weakref.WeakKeyDictionary" = weakref.WeakKeyDictionary()


def record_props(build):
    """Wraps a scene builder (api -> (comp, orders)): Layer.set_props is recorded while it runs, and
    the last props of every attached layer (Props() for a layer never given any) are kept for
    `props_of`."""
    def wrapped(api):
        seen = {}
        original = binding.Layer.set_props

        def set_props(layer, props):
            seen[layer._h] = props
            return original(layer, props)
        binding.Layer.set_props = set_props
        try:
            comp, orders = build(api)
        finally:
            binding.Layer.set_props = original
        _PROPS[comp] = {o: seen.get(comp.get(o)._h, Props()) for o in orders}
        return comp, orders
    return wrapped


def props_of(comp) -> Dict[int, Props]:
    return _PROPS[comp]


def filled(props: Props, color) -> Optional[Props]:
    """props with the fill replaced by Fill.Solid(color), or None for a Clip layer."""
    if props.func.draw is None:
        return None
    style = dataclasses.replace(props.func.draw, fill=Fill.Solid(Color(*[float(c) for c in color])))
    return Props(fill_rule=props.fill_rule, func=Func.Draw(style))


def set_pose_fill(comp, sc: FillScene, orders: Sequence[int], b: int) -> None:
    """Puts `comp` (built by sc.build, with attached `orders`) into the state of frame b."""
    if sc.transforms is not None or sc.visible is not None:
        ps.set_pose(comp, sc, orders, b)
    if sc.colors is None:
        return
    props = props_of(comp)
    for o in ps.window_orders(sc, orders):
        p = filled(props[o], sc.colors[b, o - sc.first_order])
        if p is not None:
            comp.get(o).set_props(p)


def poses(sc: FillScene):
    """The binding's Poses value of the scene."""
    return binding.Poses(sc.first_order, sc.transforms, sc.visible, sc.colors)


def random_colors(n: int, k: int, seed: int, alpha=(0.25, 1.0)) -> np.ndarray:
    """[n, K, 4] colours in [0, 1], alpha uniform in `alpha`, a quarter of the alphas exactly 1."""
    rng = np.random.default_rng(seed)
    c = rng.random((n, k, 4)).astype(f32)
    c[..., 3] = rng.uniform(alpha[0], alpha[1], (n, k)).astype(f32)
    c[..., 3][rng.random((n, k)) < 0.25] = 1.0
    return c


def _e2e(name):
    return record_props(ps._e2e(name))


def _specs(specs):
    return record_props(ps._specs(specs))


FULL = ls.rect(-8.0, -8.0, 80.0, 56.0)  # covers a 64 x 40 frame: full in every tile


def _flips_build(api):
    """Full layers below, inside and above a clip range, with small layers between: order 0 an
    opaque full backdrop, 1 a star, 2 a full layer, 3 Clip(3) of a circle, 4 a full clipped layer,
    5 a full unclipped layer inside the open clip range, 6 a clipped star, 7 a full layer above the
    clip range, 8 a star on top."""
    def solid(a, clipped=False, mode=BlendMode.Over):
        return Props(func=Func.Draw(Style(is_clipped=clipped, fill=Fill.Solid(Color(0.2, 0.4, 0.6, a)), blend_mode=mode)))
    layers = [
        (0, FULL, solid(1.0)),
        (1, ls.star(20, 20, 5, 15, 6), solid(0.8)),
        (2, FULL, solid(0.5)),
        (3, ls.star(32, 20, 8, 19, 7), Props(func=Func.Clip(3))),
        (4, FULL, solid(1.0, clipped=True)),
        (5, FULL, solid(0.5)),
        (6, ls.star(40, 22, 4, 14, 5), solid(0.9, clipped=True)),
        (7, FULL, solid(0.5)),
        (8, ls.rect(44, 4, 60, 30), solid(0.7, mode=BlendMode.Multiply)),
    ]
    comp = api.Composition()
    for order, pts, props in layers:
        comp.get_mut_or_insert_default(order).insert(ls.build_path(api, pts)).set_props(props)
    return comp, [o for o, _, _ in layers]


def _alpha_rows(alphas: Sequence[Sequence[float]]) -> np.ndarray:
    """Frames of the flips scene: per frame and order an alpha, the colour channels vary by order."""
    n, k = len(alphas), len(alphas[0])
    c = np.zeros((n, k, 4), f32)
    for j in range(k):
        c[:, j, :3] = [(0.1 + 0.09 * j) % 1.0, (0.7 - 0.07 * j) % 1.0, (0.3 + 0.13 * j) % 1.0]
    c[..., 3] = np.asarray(alphas, f32)
    return c


def _scenes() -> List[FillScene]:
    out = []
    # Every e2e scene recoloured (solid, gradient and texture layers become solid; the 16 blend
    # modes keep their mode), window of E2E_K orders, the last frame with every alpha 1.
    for name in sorted(scenes.E2E):
        c = random_colors(3, ps.E2E_K, 100 + len(out))
        c[2, :, 3] = 1.0
        out.append(FillScene(f"e2e_{name}", _e2e(name), 64, 64, 0, c))
    # The blend layer alone recoloured, over the scene's own gradient: the mode reads the pose slot.
    for mode, mname in enumerate(BlendMode.NAMES):
        c = _alpha_rows([[1.0], [0.6], [ONE_DOWN]])
        c[1, 0, :3] = [0.9, 0.1, 0.5]
        out.append(FillScene(f"blend_top_{mname}", _e2e(f"blend_modes__{mname}"), 64, 64, 1, c))
    # Clip layers inside the window: their colours are garbage and must not be read.
    c = random_colors(3, 7, 7)
    c[:, 1] = [NAN, INF, -INF, NAN]
    out.append(FillScene("clip_ignored", _e2e("clipping"), 64, 64, 0, c))
    c = random_colors(2, 2, 8)
    c[:, 0] = [1e30, -1e30, NAN, 7.0]
    out.append(FillScene("clip2_ignored", _e2e("clipping2"), 64, 64, 1, c))
    # Alpha flips of full layers: 1 -> 0.5 and 0.5 -> 1 below, inside and above the clip range.
    out.append(FillScene("alpha_flips", record_props(_flips_build), 64, 40, 0, _alpha_rows([
        [1.0, 0.8, 0.5, 1.0, 1.0, 0.5, 0.9, 0.5, 0.7],
        [0.5, 0.8, 1.0, 1.0, 0.5, 1.0, 0.9, 1.0, 0.7],
        [1.0, 0.8, 1.0, 1.0, 1.0, 1.0, 0.9, 0.5, 0.7],
        [0.5, 0.8, 0.5, 1.0, 0.5, 0.5, 0.9, 1.0, 1.0],
    ])))
    # Alpha exactly 1, one ulp below, 0, above 1 and negative.
    out.append(FillScene("alpha_edges", record_props(_flips_build), 64, 40, 0, _alpha_rows([
        [1.0, ONE_DOWN, 1.0, 1.0, ONE_DOWN, 1.0, 0.0, ONE_DOWN, 1.0],
        [ONE_DOWN, 0.0, ONE_DOWN, 1.0, 1.0, ONE_DOWN, 1.5, 1.0, -0.25],
        [0.0, 1.5, 0.0, 1.0, 0.0, 0.0, -0.25, 2.0, 0.0],
        [-0.25, -1.0, 1.5, 1.0, 1.5, -0.5, 1.0, 0.0, ONE_DOWN],
    ])))
    # NaN and infinite components.
    c = _alpha_rows([[1.0] * 9, [0.5] * 9, [1.0] * 9])
    c[0, 2] = [NAN, 0.5, 0.5, 1.0]
    c[0, 5] = [0.5, INF, -INF, 0.5]
    c[1, 0] = [0.2, 0.2, 0.2, NAN]
    c[1, 7] = [INF, INF, INF, INF]
    c[2, 4] = [-INF, NAN, 1.0, 1.0]
    c[2, 8] = [NAN, NAN, NAN, NAN]
    out.append(FillScene("nonfinite_colors", record_props(_flips_build), 64, 40, 0, c))
    # Colours with transforms and visibility, and with each of them alone.
    for base in ("window_gaps", "clip2_both", "show_hide", "clip_moved"):
        p = ps.SCENES[base]
        out.append(FillScene(f"{base}_filled", record_props(p.build), p.width, p.height, p.first_order,
                             random_colors(p.n, p.n_orders, 30 + len(out)), p.transforms, p.visible))
    out.append(FillScene("colors_visible_only", _specs(ps._straddle_specs(disabled=True)), 64, 40, 0,
                         random_colors(4, 4, 40), None, ps.SCENES["show_hide"].visible))
    # Window edges: K = 1, empty orders in the window, a window past the last order, and the top of
    # the layer field (first_order + K = 2^21).
    edge = ps._window_edge_specs
    out.append(FillScene("fill_k1", _specs(edge()), 64, 40, 5, random_colors(4, 1, 50)))
    out.append(FillScene("fill_window_gaps", _specs(edge()), 64, 40, 3, random_colors(3, 6, 51)))
    out.append(FillScene("fill_window_past_end", _specs(edge()), 64, 40, 13, random_colors(2, 3, 52)))
    top = ps.SCENES["window_top"]
    out.append(FillScene("fill_window_top", _specs(ps._top_order_specs()), 64, 40, ps.LAYER_LIMIT - 8, random_colors(3, 8, 53),
                         top.transforms, top.visible))
    # Workloads: the spaceship animation with per-frame colours, the shape library with random
    # colours, paris with every layer recoloured.
    ship = ps.SCENES["spaceship1080p"]
    out.append(FillScene("spaceship_filled", record_props(ps._spaceship_build), 1920, 1080, 1, random_colors(200, 401, 60),
                         ship.transforms, heavy=True))
    lib = ps.SCENES["library_511x64"]
    out.append(FillScene("library_filled", record_props(ps._library_build), 64, 64, 0, random_colors(511, ps.LIBRARY_SHAPES, 61),
                         lib.transforms, lib.visible, heavy=True))
    out.append(FillScene("paris_filled", record_props(ps._paris_build), 960, 540, 0, random_colors(16, ps.PARIS_LAYERS, 62),
                         ps.paris_table(), heavy=True))
    return out


SCENES: Dict[str, FillScene] = {s.name: s for s in _scenes()}
LIGHT = [n for n, s in SCENES.items() if not s.heavy]
HEAVY = [n for n, s in SCENES.items() if s.heavy]
