"""Scenes of batches (Renderer.render_batch): a list of distinct compositions, a frame size, and
the frames, each naming the composition it shows (repeats allowed).

Every frame of a batch must equal the oracle's ordinary frame of its composition. The host-side
rule the tests hold the device to is the slice rule of the layer field (`order_bases`): the
distinct compositions, in order of first appearance, get consecutive slices of n_orders each
(largest attached order + 1, or 0).
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import Callable, Dict, List, Sequence

import numpy as np

import line_scenes as ls
import scenes
import synth
import view_scenes as vs
from forma_b200.binding import Color, Fill, Func, Props, Style

ORDER_FIELD = 1 << 21        # the layer field of the sort key holds orders [0, 2^21)
SEGMENT_BUDGET = 50_000_000  # pixel segments per call of an in-limit scene


@dataclass
class BatchScene:
    name: str
    builders: List[Callable]  # (api) -> composition, one per distinct composition
    width: int
    height: int
    frames: List[int]         # per frame: index into `builders`
    over: str = ""            # "orders" / "segments": the call is refused for that limit


def _e2e(name):
    def build(api):
        comp = api.Composition()
        scenes.E2E[name](api, comp)
        return comp
    return build


def _specs(specs):
    def build(api):
        return ls.build(api, specs)[0]
    return build


def _random(seed, n_layers=24, size=64):
    def build(api):
        comp = api.Composition()
        synth.random_mixed(api, comp, n_layers, size, size, seed)
        return comp
    return build


def _empty(api):
    return api.Composition()


def _all_disabled(api):
    comp = api.Composition()
    scenes.E2E["covers"](api, comp)
    o = 0
    for _ in range(len(comp)):
        while comp.get(o) is None:
            o += 1
        comp.get(o).set_is_enabled(False)
        o += 1
    return comp


def _sparse(api):
    """Two layers, the second at order 10^6: a slice of 10^6 + 1 orders, nearly all empty."""
    comp = api.Composition()
    comp.get_mut_or_insert_default(3).insert(scenes.square(api)).set_props(scenes.solid(Color(0.2, 0.4, 0.9, 1.0)))
    comp.get_mut_or_insert_default(1_000_000).insert(scenes.circle(api)).set_props(scenes.solid(Color(0.9, 0.3, 0.1, 0.8)))
    return comp


def _long_clip(api):
    """A Clip(1000) at order 1 whose range runs far past the composition's last order (3)."""
    comp = api.Composition()
    comp.get_mut_or_insert_default(0).insert(scenes.square(api)).set_props(scenes.solid(Color(0.0, 0.0, 0.0, 0.7)))
    comp.get_mut_or_insert_default(1).insert(scenes.inner_circle(api)).set_props(Props(func=Func.Clip(1000)))
    comp.get_mut_or_insert_default(3).insert(scenes.triangle(api)).set_props(
        Props(func=Func.Draw(Style(fill=Fill.Solid(Color(0.5, 0.5, 1.0, 0.7)), is_clipped=True))))
    return comp


def _low_orders(api):
    """Clipped and unclipped draws at orders 0 ... 5: inside the Clip(1000) range of _long_clip if
    slices leaked across frames."""
    comp = api.Composition()
    comp.get_mut_or_insert_default(0).insert(scenes.square(api)).set_props(scenes.solid(Color(0.1, 0.8, 0.2, 0.9)))
    for o in range(1, 6):
        comp.get_mut_or_insert_default(o).insert(scenes.custom_circle(api, 12.0 + 8 * o, 30.0, 10.0)).set_props(
            Props(func=Func.Draw(Style(fill=Fill.Solid(Color(0.9, 0.2, 0.1 * o, 0.6)), is_clipped=o % 2 == 1))))
    return comp


def _out_of_order(api):
    """Layers inserted against their order (5, then 2, then 4): the segments are not emitted in
    layer order, so the sort needs the layer digits."""
    comp = api.Composition()
    comp.get_mut_or_insert_default(5).insert(scenes.circle(api)).set_props(scenes.solid(Color(0.9, 0.1, 0.1, 0.6)))
    comp.get_mut_or_insert_default(2).insert(scenes.square(api)).set_props(scenes.solid(Color(0.1, 0.1, 0.9, 0.8)))
    comp.get_mut_or_insert_default(4).insert(scenes.triangle(api)).set_props(scenes.solid(Color(0.1, 0.9, 0.1, 0.5)))
    return comp


def _top_order(order):
    """One square at `order`: a slice of order + 1 orders."""
    def build(api):
        comp = api.Composition()
        comp.get_mut_or_insert_default(order).insert(scenes.square(api)).set_props(scenes.solid(Color(0.3, 0.6, 0.9, 1.0)))
        return comp
    return build


PARIS_SCALE = 1080.0 / 1060.0
PARIS_TILE = (960, 540)


def paris_tile_offsets() -> List[tuple]:
    """(x, y) of the 16 960 x 540 tiles of the 1920 x 1080 drawing, those of view_scenes' paris_tiles."""
    return [(960.0 * (k % 2) + 480.0 * (k // 8), 540.0 * ((k // 2) % 2) + 270.0 * ((k // 4) % 2)) for k in range(16)]


_PARIS = {}


def _paris_paths():
    from forma_b200 import svg
    if "paths" not in _PARIS:
        root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
        _PARIS["paths"] = svg.PathList.load(os.path.join(root, "tests", "data", "paris30k_paths.npz"))
    return _PARIS["paths"]


def paris_tile_paths(k: int):
    """The paths of the drawing whose control points' box meets tile k, moved into the tile (in the
    file's units, before the scale)."""
    from forma_b200 import svg
    p = _paris_paths()
    ox, oy = paris_tile_offsets()[k]
    tw, th = PARIS_TILE
    lo = np.minimum.reduceat(p.pts, p.pt_off[:-1], axis=0) * PARIS_SCALE
    hi = np.maximum.reduceat(p.pts, p.pt_off[:-1], axis=0) * PARIS_SCALE
    keep = np.nonzero((hi[:, 0] >= ox) & (lo[:, 0] <= ox + tw) & (hi[:, 1] >= oy) & (lo[:, 1] <= oy + th))[0]
    n_rat = np.add.reduceat((p.cmd == svg.RATQUAD).astype(np.int64), p.cmd_off[:-1])
    n_rat[np.diff(p.cmd_off) == 0] = 0
    w_off = np.concatenate([[0], np.cumsum(n_rat)])
    shift = np.array([ox, oy], np.float32) / np.float32(PARIS_SCALE)
    cmd, pts, weights, cmd_off, pt_off = [], [], [], [0], [0]
    for i in keep:
        cmd.append(p.cmd[p.cmd_off[i]:p.cmd_off[i + 1]])
        pts.append(p.pts[p.pt_off[i]:p.pt_off[i + 1]] - shift)
        weights.append(p.weights[w_off[i]:w_off[i + 1]])
        cmd_off.append(cmd_off[-1] + len(cmd[-1]))
        pt_off.append(pt_off[-1] + len(pts[-1]))
    return svg.PathList(np.concatenate(cmd).astype(np.uint8), np.concatenate(pts).astype(np.float32),
                        np.array(cmd_off, np.int64), np.array(pt_off, np.int64), p.color[keep], p.fill_rule[keep],
                        np.concatenate(weights).astype(np.float32), p.blend[keep], p.grad[keep], p.gradients)


def _paris_tile(k):
    def build(api):
        from forma_b200 import svg
        comp = api.Composition()
        svg.compose(api, comp, paris_tile_paths(k), scale=PARIS_SCALE)
        return comp
    return build


def _scenes() -> List[BatchScene]:
    out = []
    # Every e2e scene (gradients, textures, clips, all blend modes, both fill rules) and compositions
    # with layer transforms (view_scenes' straddle and far layers), each once.
    e2e = [_e2e(n) for n in sorted(scenes.E2E)]
    xf = [_specs(vs._straddle_layers()), _specs(vs._far_layers())]
    mixed = e2e[:9] + xf[:1] + e2e[9:] + xf[1:]
    out.append(BatchScene("e2e_all", mixed, 64, 64, list(range(len(mixed)))))
    # Repeated and interleaved: A, B, A, C, A.
    abc = [_e2e("texture"), _e2e("linear_gradient"), _specs(vs._straddle_layers())]
    out.append(BatchScene("repeats", abc, 64, 64, [0, 1, 0, 2, 0]))
    out.append(BatchScene("repeats_h40", abc, 64, 40, [0, 1, 0, 2, 0, 1]))
    # Compositions whose segments are emitted in layer order and one whose are not.
    out.append(BatchScene("mixed_order", [_e2e("covers"), _out_of_order, _e2e("clipping")], 64, 64, [0, 1, 2, 1, 0]))
    # Empty, all disabled, sparse, between ordinary compositions.
    out.append(BatchScene("degenerate", [_e2e("covers"), _empty, _all_disabled, _sparse, _e2e("radial_gradient")], 64, 64,
                          [0, 1, 2, 3, 4, 1]))
    # A clip past its composition's last order next to low orders of the next composition.
    out.append(BatchScene("clip_leak", [_long_clip, _low_orders, _e2e("clipping")], 64, 64, [0, 1, 2, 1, 0]))
    # Heights that are not multiples of 16, widths that are not either.
    out.append(BatchScene("odd_h37", [_e2e("clipping2"), _e2e("radial_gradient"), _random(5)], 61, 37, [0, 1, 2, 2, 0]))
    out.append(BatchScene("odd_h1", [_e2e("clipping"), _e2e("covers")], 61, 1, [0, 1] * 8))
    # n = max_views(height): 2046 frames of 16 rows, content in the first and the last.
    out.append(BatchScene("limit_h16", [_e2e("covers"), _random(11, 8, 16), _e2e("pixel")], 64, 16,
                          [k % 3 for k in range(2046)]))
    out.append(BatchScene("limit_h1000", [_e2e("linear_gradient"), _e2e("texture")], 64, 1000, [k % 2 for k in range(32)]))
    # Paris split into its 16 tiles, one composition each.
    out.append(BatchScene("paris_tiles", [_paris_tile(k) for k in range(16)], *PARIS_TILE, list(range(16))))
    # 511 distinct random compositions of 64 x 64.
    out.append(BatchScene("random_511", [_random(1000 + k) for k in range(511)], 64, 64, list(range(511))))
    # The order field: 2^21 orders exactly, and one more.
    half = ORDER_FIELD // 2
    out.append(BatchScene("orders_at_limit", [_top_order(half - 1), _top_order(half - 1)], 64, 64, [0, 1, 0]))
    out.append(BatchScene("orders_over", [_top_order(half - 1), _top_order(half)], 64, 64, [0, 1], over="orders"))
    # Two frames each below 2^30 pixel segments, above it together.
    out.append(BatchScene("segment_limit", [_specs(vs._long_layers(20))], 64, 64, [0, 0], over="segments"))
    return out


SCENES: Dict[str, BatchScene] = {s.name: s for s in _scenes()}
IN_LIMIT = [n for n, s in SCENES.items() if not s.over]
LIMIT_SCENES = ["limit_h16", "limit_h1000"]  # n = max_views(height)


def rows(height: int) -> int:
    return (height + 15) // 16


def max_frames(height: int) -> int:
    """forma_renderer_max_views(height), which bounds batches too."""
    return 0 if height == 0 or height > 32768 else 2046 // rows(height)


def build(api, sc: BatchScene):
    """(the distinct compositions, the composition of every frame) of scene `sc` on `api`."""
    distinct = [b(api) for b in sc.builders]
    return distinct, [distinct[k] for k in sc.frames]


def n_orders(comp) -> int:
    """Largest attached order + 1, or 0 (probing orders until all layers are found)."""
    n, o, found, top = len(comp), 0, 0, -1
    while found < n:
        if comp.get(o) is not None:
            found += 1
            top = o
        o += 1
    return top + 1


def order_bases(frames: Sequence, counts: Dict[int, int]) -> List[int]:
    """The order base of every frame: the distinct compositions (by id()) in order of first
    appearance get consecutive slices of counts[id(comp)] orders."""
    base, seen, out = 0, {}, []
    for comp in frames:
        if id(comp) not in seen:
            seen[id(comp)] = base
            base += counts[id(comp)]
        out.append(seen[id(comp)])
    return out


def order_sum(frames: Sequence, counts: Dict[int, int]) -> int:
    return sum(counts[k] for k in {id(c): None for c in frames})
