"""Pose scenes at the limits the poses calls document (include/forma_b200.h: render_poses;
DESIGN.md "Poses", Limits): full stacks, odd heights, far and long lines, the transforms of
tests/line_scenes.py delivered as poses, crowded tiles with pose fills, window shapes and the
segment limit.

Every scene is a pure function of its name and names the condition it is there for. Frame b of a
call is the ordinary frame of the composition put into pose b (pose_fill_scenes.set_pose_fill:
transforms, visibility and colours). Scenes built from line_scenes layers (`specs`) are replayed
by tests/line_model.py frame by frame: frame b's lines are the single frame's lines of the layers
`frame_layers(sc, b)` gives, so tests/test_pose_limit_scenes.py proves each condition and budget
on the CPU before tests/test_gpu_pose_limits.py lets a device see the scene.
"""
from __future__ import annotations

import functools
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np

import extremes
import line_model as lm
import line_scenes as ls
import pose_fill_scenes as pfs
import pose_scenes as ps
import view_scenes as vs

f32 = np.float32
IDENTITY = ps.IDENTITY
U32 = 0xFFFFFFFF
NAN = float("nan")
SEGMENT_BUDGET = vs.SEGMENT_BUDGET  # pixel segments of an in-limit call, all frames together
POINT_BUDGET = 20_000_000           # point pairs line setup visits in one call: n times the points
TABLE_BUDGET = 1 << 30              # bytes of pose records (32 n K) and pose style table (112 (S + n K))
FAR_LEFT = -(2.0 ** 19)             # px: frames whose lines all lie left of it are the stacked calls' exception


def max_views(height: int) -> int:
    """forma_renderer_max_views: 2046 stacked tile rows."""
    return 0 if height == 0 or height > 32768 else 2046 // ((height + 15) // 16)


@dataclass
class LimitScene:
    name: str
    condition: str                    # what the scene is there for
    build: Callable                   # api -> (composition, sorted attached orders); props recorded
    width: int
    height: int
    first_order: int
    tables: Callable                  # () -> (transforms [n, K, 6] | None, visible [n, K] | None, colors [n, K, 4] | None)
    specs: Optional[List[ls.LayerSpec]] = None  # line_scenes layers: replayed by line_model
    kind: str = "in"                  # "in"; "over": the frames together reach 2^30 segments; "saturate": 2^32 - 1
    far: Sequence[int] = ()           # frames whose every line lies more than 2^19 px left of the frame
    big: bool = False                 # tables of 100 MB and more

    @functools.cached_property
    def _t(self):
        return self.tables()

    @property
    def transforms(self):
        return self._t[0]

    @property
    def visible(self):
        return self._t[1]

    @property
    def colors(self):
        return self._t[2]

    @property
    def n(self) -> int:
        return next(t for t in self._t if t is not None).shape[0]

    @property
    def n_orders(self) -> int:
        return next(t for t in self._t if t is not None).shape[1]

    @property
    def rows(self) -> int:
        return (self.height + 15) // 16


def record_index(order: int, first_order: int, n_orders: int, b: int, wrap: bool = True) -> Optional[int]:
    """The pose record line setup reads for the layer at `order` in frame b, or None (the layer's
    own state): b K + (order - first_order) when that difference, taken as an unsigned 32-bit value,
    is below K. One compare tests both ends of the window. (`wrap=False` is the error of a signed
    compare, which gives the orders below the window the records of the frame before.)"""
    k = (order - first_order) & U32 if wrap else order - first_order
    return b * n_orders + k if k < n_orders else None


def frame_layers(sc: LimitScene, b: int, lookup=record_index) -> List[lm.LayerXf]:
    """line_model layers of frame b: every layer's transform and enabled state after the pose edits
    (a pose transform equal to the identity is no transform, as forma_layer_set_transform has it)."""
    T = None if sc.transforms is None else sc.transforms.reshape(-1, 6)
    V = None if sc.visible is None else sc.visible.reshape(-1)
    out = []
    for s in sc.specs:
        xf, enabled = (None if s.xf is None else list(s.xf)), s.enabled
        r = lookup(s.order, sc.first_order, sc.n_orders, b)
        if r is not None:
            if T is not None:
                t = [float(v) for v in T[r]]
                xf = None if t == IDENTITY else t
            if V is not None:
                enabled = bool(V[r])
        out.append(lm.LayerXf(s.order, xf, enabled))
    return out


def record_props(build):
    return pfs.record_props(build)


def _specs(specs):
    return record_props(ps._specs(specs))


def _shift(dx: float, dy: float) -> List[float]:
    return [1.0, 0.0, 0.0, 1.0, float(dx), float(dy)]


def neighbour_shifts(height: int) -> List[float]:
    """Translations in y that move a layer by exactly one frame or one frame's tile rows, and 1/16 px
    either side of the latter: a remap or bound off by one row puts segments into a neighbour's rows."""
    r16 = 16.0 * ((height + 15) // 16)
    return [0.0, float(height), -float(height), r16, -r16, r16 + 0.0625, r16 - 0.0625, -(r16 + 0.0625), -(r16 - 0.0625)]


def edge_layers(w: float, h: float) -> List[ls.LayerSpec]:
    """Layers over the top and the bottom edge of a w x h frame: two 4-byte-path layers, one with its
    own transform (the 36-byte layer records), and a disabled layer that the poses show."""
    return [
        ls.LayerSpec(0, None, [ls.rect(2, -6, w * 0.4, 6), ls.rect(w * 0.5, h - 5, w - 3, h + 7)]),
        ls.LayerSpec(1, [0.8, -0.6, 0.6, 0.8, 3.0, -2.0], [ls.star(w / 2, h / 2, 3, max(h, 12.0) * 0.75, 7)]),
        ls.LayerSpec(2, None, [ls.rect(-4, h / 2 - 3.25, w + 4, h / 2 + 2.5)], even_odd=True),
        ls.LayerSpec(3, None, [ls.rect(w * 0.25, -17, w * 0.75, h + 17)], enabled=False),  # (over a whole tile row either side)
    ]


def stack_tables(n: int, height: int, k_orders: int = 4):
    """Frame b, layer k: a neighbour shift (cycling with b + 2 k) and 0.5 k px right; visibility
    varies from frame to frame, the first and the last frame show every layer."""
    d = neighbour_shifts(height)

    def make():
        t = np.empty((n, k_orders, 6), f32)
        v = np.empty((n, k_orders), np.uint8)
        for b in range(n):
            for k in range(k_orders):
                t[b, k] = _shift(0.5 * k, d[(b + 2 * k) % len(d)])
                v[b, k] = (b * 5 + k * 3) % 7 != 0
        v[0] = v[-1] = 1
        return t, v, None
    return make


def _fixed(t=None, v=None, c=None):
    return lambda: (None if t is None else np.asarray(t, f32), None if v is None else np.asarray(v, np.uint8),
                    None if c is None else np.asarray(c, f32))


def _stack(name, w, h, n, condition):
    specs = edge_layers(w, h)
    return LimitScene(name, condition, _specs(specs), w, h, 0, stack_tables(n, h), specs)


def _line_xf_scenes() -> List[LimitScene]:
    """Every in-limit layer transform of tests/line_scenes.py as a pose on the scene's layers without
    their transforms, between identity frames: once on a composition whose layers have no transform
    of their own (4-byte layer records), once where each has one (36-byte records)."""
    out = []
    own_xf = [1.0, 0.0, 0.0, 1.0, 0.5, 0.25]
    for name in ls.IN_LIMIT:
        src = ls.SCENES[name]
        if not any(s.xf is not None for s in src.layers):
            continue
        orders = [s.order for s in src.layers]
        K = max(orders) + 1
        posed = np.tile(np.asarray(IDENTITY, f32), (K, 1))
        for s in src.layers:
            if s.xf is not None:
                posed[s.order] = s.xf
        t = np.stack([np.tile(np.asarray(IDENTITY, f32), (K, 1)), posed, np.tile(np.asarray(IDENTITY, f32), (K, 1)), posed])
        for own in (False, True):
            specs = [ls.LayerSpec(s.order, own_xf if own else None, s.paths, s.path_xf, s.enabled, s.even_odd) for s in src.layers]
            out.append(LimitScene(f"lines_{name}{'_own' if own else ''}", f"line_scenes {name}: {src.target}, as poses",
                                  _specs(specs), src.width, src.height, 0, _fixed(t), specs))
    return out


def _extreme_build(name):
    def build(api):
        comp = api.Composition()
        extremes.SCENES[name].build(api, comp)
        return comp, ps._orders(comp)
    return record_props(build)


def crowd_tables(n_orders: int, seed: int):
    """Three frames of every order of a crowded scene: the first with opaque colours; the second with
    every third layer moved by (1.5, -2) px, every seventh hidden and alphas cycling through 0, 1, NaN
    and 0.5; the third with every fifth layer hidden, every fourth turned by 90 degrees about (64, 32)
    and random colours."""
    def make():
        rng = np.random.default_rng(seed)
        K = n_orders
        t = np.tile(np.asarray(IDENTITY, f32), (3, K, 1))
        v = np.ones((3, K), np.uint8)
        c = rng.random((3, K, 4)).astype(f32)
        c[0, :, 3] = 1.0
        k = np.arange(K)
        t[1, k % 3 == 0] = _shift(1.5, -2.0)
        v[1, k % 7 == 3] = 0
        c[1, :, 3] = np.asarray([0.0, 1.0, NAN, 0.5], f32)[k % 4]
        v[2, k % 5 == 1] = 0
        t[2, k % 4 == 2] = vs.about(1, 64.0, 32.0)
        return t, v, c
    return make


# Orders the extreme scenes attach (test_pose_limit_scenes checks that the window covers them).
CROWDED = {"dense_stars": 64, "nan_blends": 8, "winding_mixed_eo": 64, "crowd_129": 129, "crowd_1000": 1000, "crowd_5000": 5000}


def _far_up_specs():
    """A triangle 2^21 px below the frame, which a pose of -2^21 px brings to one end in the frame and
    the other 2^20 px above it (more than 32767 tile rows: its rows wrap), and a star in the frame."""
    y = 2.0 ** 21
    return [ls.LayerSpec(0, None, [[(10.0, 20.0 + y), (2.0 ** 20, 20.0 + y), (10.0, y - 2.0 ** 20)]]),
            ls.LayerSpec(1, None, [ls.star(32, 20, 6, 16, 7)])]


def _long_specs():
    return vs._long_layers(20)


def _long_tables(n: int):
    """Translations only (poses cannot scale up): frame b moves the long lines down by 3 b px."""
    return _fixed([[_shift(0.0, 3.0 * b)] for b in range(n)])


def _sparse_window_tables(n: int, n_orders: int, layers: Sequence[int], colors: bool = False):
    """Identity everywhere but at the attached orders of the window; visibility all ones but for one
    layer per frame; optional colours. Frame b moves the layer at orders[j] by (2 b - j, b + 1.5 j)."""
    def make():
        t = np.tile(np.asarray(IDENTITY, f32), (n, n_orders, 1))
        v = np.ones((n, n_orders), np.uint8)
        for b in range(n):
            for j, o in enumerate(layers):
                if o < n_orders:
                    t[b, o] = _shift(2.0 * (b % 7) - j, (b % 5) + 1.5 * j)
            v[b, layers[b % len(layers)] % n_orders] = 0 if b % 3 == 1 else 1
        c = pfs.random_colors(n, n_orders, 91) if colors else None
        return t, v, c
    return make


def _sparse_specs(orders: Sequence[int], w: float, h: float) -> List[ls.LayerSpec]:
    return [ls.LayerSpec(o, None, [ls.star(w * (0.2 + 0.15 * j), h * 0.5, 4, min(w, h) * 0.3, 5 + j)]) for j, o in enumerate(orders)]


def _scenes() -> List[LimitScene]:
    out = []
    # Full stacks: n = max_views(height), content in the first and the last frame.
    out.append(_stack("limit_h16", 64, 16, 2046, "n = 2046 frames of one tile row"))
    out.append(_stack("limit_h1", 61, 1, 2046, "n = 2046 frames one pixel high"))
    out.append(_stack("limit_h17", 64, 17, 1023, "n = 1023 frames of two tile rows, the second one pixel high"))
    out.append(_stack("limit_h1000", 64, 1000, 32, "n = 32 frames of 63 tile rows"))
    # Odd heights: the device frames are repacked.
    out.append(_stack("odd_h37", 64, 37, 9, "height 37: layers moved across the bottom edge, repacked frames"))
    out.append(_stack("odd_h100", 77, 100, 9, "77 x 100: layers moved across the bottom edge, repacked frames"))
    out.append(_stack("odd_h1080", 33, 1080, 9, "33 x 1080: layers moved across the bottom edge, repacked frames"))
    # Far lines.
    specs = edge_layers(64, 40)
    far = np.stack([np.tile(np.asarray(_shift(0.5 * (b % 2), 0.25 * b), f32), (4, 1)) for b in range(5)])
    far[1, :, 4] = far[3, :, 4] = -(2.0 ** 20)
    out.append(LimitScene("far_left", "frames 1 and 3 move every layer 2^20 px left: all their lines lie left of -2^19 px",
                          _specs(specs), 64, 40, 0, _fixed(far, [[1, 1, 1, 1], [1, 1, 1, 1], [1, 0, 1, 1], [1, 1, 1, 0], [1, 1, 1, 1]]),
                          specs, far=(1, 3)))
    specs = _far_up_specs()
    out.append(LimitScene("far_up", "a pose takes a line from inside the frame to 2^20 px above it: its rows wrap",
                          _specs(specs), 64, 40, 0,
                          _fixed([[IDENTITY, IDENTITY], [_shift(0, -2.0 ** 21), IDENTITY], [_shift(0.5, -2.0 ** 21 + 0.5), _shift(3, 1)],
                                  [IDENTITY, _shift(-2, 0)]]), specs))
    specs = [ls.LayerSpec(k, None, [ls.star(40 + 60 * k, 40, 10, 30, 6)]) for k in range(4)]
    out.append(LimitScene("far_translations", "pose translations of +-2^31 px and -inf, between ordinary frames",
                          _specs(specs), 256, 80, 0,
                          _fixed([[IDENTITY] * 4, [_shift(-2.0 ** 31, 0), _shift(2.0 ** 31, 0), _shift(0, -2.0 ** 31), _shift(float("-inf"), 0)],
                                  [_shift(3, 2)] * 4, [_shift(float("-inf"), 0), IDENTITY, _shift(-2.0 ** 31, 7.5), _shift(0, 2.0 ** 31)]]),
                          specs, far=(1,)))  # frame 1: what survives lies at x = -2^31 and -inf
    out += _line_xf_scenes()
    # Crowded tiles with pose fills (every blend mode, clips, dense cells, deep winding).
    for j, (name, k) in enumerate(CROWDED.items()):
        sc = extremes.SCENES[name]
        out.append(LimitScene(f"crowded_{name}", f"extremes {name} with layers moved, hidden and recoloured per frame",
                              _extreme_build(name), sc.width, sc.height, 0, crowd_tables(k, 200 + j)))
    # Window shapes.
    specs = edge_layers(64, 40)
    specs[3].enabled = True
    out.append(LimitScene("window_from_1", "a window [1, 4) above a layer at order 0: the unsigned compare wraps for it",
                          _specs(specs), 64, 40, 1,
                          _fixed([[_shift(5.0 * b + k, 3.0 * b - 2 * k) for k in range(3)] for b in range(4)], np.ones((4, 3))), specs))
    orders = [0, 1000, ps.LAYER_LIMIT - 1]
    specs = _sparse_specs(orders, 64, 40)
    out.append(LimitScene("window_2p21", "first_order 0, K = 2^21, n = 2 on three layers: 128 MB of pose records",
                          _specs(specs), 64, 40, 0, _sparse_window_tables(2, ps.LAYER_LIMIT, orders), specs, big=True))
    orders = [0, 3, 65535, 65536, 70000]
    specs = _sparse_specs(orders, 64, 1000)
    out.append(LimitScene("window_k2p16", "K = 2^16, 33 frames of 63 rows: chunks of 32 and 1 frame",
                          _specs(specs), 64, 1000, 0, _sparse_window_tables(33, 1 << 16, orders, colors=True), specs, big=True))
    out.append(LimitScene("window_odd_k", "K = 2^16 + 1, 35 frames of 63 rows: chunks start at odd visibility bytes",
                          _specs(specs), 64, 1000, 0, _sparse_window_tables(35, (1 << 16) + 1, orders, colors=True), specs, big=True))
    specs = [ls.LayerSpec(o, None, [ls.star(30 + 7 * k, 40 + 5 * k, 10, 40, 5)]) for k, o in enumerate((9, 2, 300, 5, 0, 77))]
    out.append(LimitScene("out_of_order", "inserts out of layer order (layers_in_order false): the sort orders layer digits",
                          _specs(specs), 256, 128, 0, _sparse_window_tables(4, 301, (9, 2, 300, 5, 0, 77)), specs))
    # The segment limit: every frame below 2^30 segments, the call at 2^30 and more, and at 2^32 - 1.
    specs = _long_specs()
    out.append(LimitScene("segment_limit", "two frames below 2^30 segments each, at least 2^30 together",
                          _specs(specs), 64, 64, 0, _long_tables(2), specs, kind="over"))
    out.append(LimitScene("segment_saturate", "eight frames below 2^30 segments each: the count saturates at 2^32 - 1",
                          _specs(specs), 64, 64, 0, _long_tables(8), specs, kind="saturate"))
    return out


SCENES: Dict[str, LimitScene] = {s.name: s for s in _scenes()}
IN_LIMIT = [n for n, s in SCENES.items() if s.kind == "in"]
OVER_LIMIT = [n for n, s in SCENES.items() if s.kind != "in"]
STACKS = ["limit_h16", "limit_h1", "limit_h17", "limit_h1000"]          # n = max_views(height)
ODD = ["odd_h37", "odd_h100", "odd_h1080"]
WINDOWS = ["window_from_1", "window_2p21", "window_k2p16", "window_odd_k", "out_of_order"]


def points(oracle_api, sc: LimitScene):
    """(x, y, layer index per point) of the composition's flattened points (specs scenes)."""
    _, _, inserts = ls.build(oracle_api, sc.specs)
    return lm.point_buffer([(k, *p.segments()) for k, p in inserts])


def frame_model(sc: LimitScene, pts, b: int, lookup=record_index) -> dict:
    """line_model's line records of frame b (frame coordinates, band [0, height)) and their counts."""
    x, y, ids = pts
    rec = lm.replay(x, y, ids, frame_layers(sc, b, lookup), sc.width, sc.height, (0.0, float(sc.height)))
    rec["counts"] = lm.counts(rec["length"], len(x))
    return rec


def touched_rows(rec: dict) -> tuple:
    """(first, last) tile row of every kept line, in frame coordinates (floor of sub-pixel y / 256)."""
    keep = rec["keep"]
    y0, dy = rec["y0"][keep].astype(np.float64), rec["dy"][keep].astype(np.float64)
    with np.errstate(invalid="ignore"):
        lo, hi = np.floor(np.minimum(y0, y0 + dy) / 256.0), np.floor(np.maximum(y0, y0 + dy) / 256.0)
    return lo, hi


def stacked_row(b: int, t: int, rows: int, remap: bool = True) -> int:
    """The biased tile_y a frame-b segment of frame tile row t gets in the stack: b rows + t + 1 for the
    frame's rows, 0 for every other (`remap=False`: the error of moving every row)."""
    ty = t + 1
    return ty + b * rows if (not remap or (ty - 1) & U32 < rows) else 0


def frame_bound(b: int, rows: int) -> int:
    """The tile_y bound the count pass reports for a frame-b line."""
    return (b + 1) * rows
