"""ctypes binding over the C ABI of include/forma_b200.h.

This is the reference-side stub a maintainer would write (INTEGRATION.md shows
the Rust `extern "C"` equivalent). The classes mirror the names and argument
meaning of the reference's public API (forma/src/lib.rs:128-154): `Point`,
`PathBuilder`, `Path`, `Order`, `Color`, `GradientBuilder`, `Props`/`Style`/
`Fill`, `Composition`, `Layer`, `Renderer`, channel constants `RGBA`, `BGRA`…

`Api(lib, prefix)` is generic over the symbol prefix so that the test-only CPU
oracle (oracle/oracle.py, prefix ``fo_``) can be driven by the same
scene-building code as the product library (prefix ``forma_``); nothing in
this module knows about the oracle.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np

# ---------------------------------------------------------------------------
# Plain data (forma/src/styling.rs, forma/src/math/point.rs)
# ---------------------------------------------------------------------------


@dataclass(frozen=True)
class Point:
    x: float
    y: float


@dataclass(frozen=True)
class Color:
    """Linear RGBA, forma/src/styling.rs:28-33 (default: opaque black, :52-61)."""

    r: float = 0.0
    g: float = 0.0
    b: float = 0.0
    a: float = 1.0


class FillRule:
    NonZero = 0
    EvenOdd = 1


class GradientType:
    Linear = 0
    Radial = 1


class BlendMode:
    Over, Multiply, Screen, Overlay, Darken, Lighten, ColorDodge, ColorBurn = range(8)
    HardLight, SoftLight, Difference, Exclusion, Hue, Saturation, Color, Luminosity = range(8, 16)
    NAMES = [
        "Over", "Multiply", "Screen", "Overlay", "Darken", "Lighten", "ColorDodge", "ColorBurn",
        "HardLight", "SoftLight", "Difference", "Exclusion", "Hue", "Saturation", "Color", "Luminosity",
    ]


class Channel:
    Red, Green, Blue, Alpha, Zero, One = range(6)


# forma/src/cpu/channel.rs:57-62
RGBA = (Channel.Red, Channel.Green, Channel.Blue, Channel.Alpha)
BGRA = (Channel.Blue, Channel.Green, Channel.Red, Channel.Alpha)
RGB0 = (Channel.Red, Channel.Green, Channel.Blue, Channel.Zero)
BGR0 = (Channel.Blue, Channel.Green, Channel.Red, Channel.Zero)
RGB1 = (Channel.Red, Channel.Green, Channel.Blue, Channel.One)
BGR1 = (Channel.Blue, Channel.Green, Channel.Red, Channel.One)

LAYER_LIMIT = (1 << 21) - 1
ID_NONE = 0xFFFFFFFF  # FORMA_ID_NONE: no layer hits the pixel (see Renderer.render_ids)


class OrderError(ValueError):
    pass


class GeomPresTransformError(ValueError):
    pass


class FormaError(RuntimeError):
    pass


@dataclass
class Gradient:
    type: int
    start: Point
    end: Point
    stops: List[Tuple[Color, float]]


class GradientBuilder:
    """forma/src/styling.rs:84-139. Stops are resolved by the library."""

    def __init__(self, start: Point, end: Point):
        self._type = GradientType.Linear
        self._start, self._end = start, end
        self._stops: List[Tuple[Color, float]] = []

    def type(self, t: int) -> "GradientBuilder":
        self._type = t
        return self

    def color(self, color: Color) -> "GradientBuilder":
        self._stops.append((color, -1.0))
        return self

    def color_with_stop(self, color: Color, stop: float) -> "GradientBuilder":
        if not (0.0 <= stop <= 1.0):
            raise ValueError("gradient stops must be between 0.0 and 1.0")
        self._stops.append((color, stop))
        return self

    def build(self) -> Optional[Gradient]:
        if len(self._stops) < 2:
            return None
        return Gradient(self._type, self._start, self._end, list(self._stops))


@dataclass
class Texture:
    """Texture{transform, image} with the image given as linear RGBA floats
    (Image::from_linear_rgba, styling.rs:320-327). transform = (ux, uy, vx, vy, tx, ty)."""

    transform: Tuple[float, float, float, float, float, float]
    linear_rgba: np.ndarray  # (h, w, 4) float32


@dataclass
class Fill:
    solid: Optional[Color] = None
    gradient: Optional[Gradient] = None
    texture: Optional[Texture] = None

    @staticmethod
    def Solid(c: Color) -> "Fill":
        return Fill(solid=c)

    @staticmethod
    def Gradient(g: Gradient) -> "Fill":
        return Fill(gradient=g)

    @staticmethod
    def Texture(t: Texture) -> "Fill":
        return Fill(texture=t)


@dataclass
class Style:
    is_clipped: bool = False
    fill: Fill = field(default_factory=lambda: Fill.Solid(Color()))
    blend_mode: int = BlendMode.Over


@dataclass
class Func:
    draw: Optional[Style] = None
    clip: Optional[int] = None

    @staticmethod
    def Draw(style: Style) -> "Func":
        return Func(draw=style)

    @staticmethod
    def Clip(n: int) -> "Func":
        return Func(clip=n)


@dataclass
class Props:
    fill_rule: int = FillRule.NonZero
    func: Func = field(default_factory=lambda: Func.Draw(Style()))


# ---------------------------------------------------------------------------
# C structs
# ---------------------------------------------------------------------------


class _CColor(C.Structure):
    _fields_ = [("r", C.c_float), ("g", C.c_float), ("b", C.c_float), ("a", C.c_float)]


class _CStop(C.Structure):
    _fields_ = [("color", _CColor), ("stop", C.c_float)]


class _CProps(C.Structure):
    _fields_ = [
        ("fill_rule", C.c_uint32), ("func", C.c_uint32), ("clip_layers", C.c_uint32),
        ("is_clipped", C.c_uint32), ("blend_mode", C.c_uint32), ("fill_type", C.c_uint32),
        ("color", _CColor), ("gradient_type", C.c_uint32),
        ("start", C.c_float * 2), ("end", C.c_float * 2),
        ("n_stops", C.c_uint32), ("stops", C.POINTER(_CStop)),
        ("tex_transform", C.c_float * 6), ("tex_width", C.c_uint32), ("tex_height", C.c_uint32),
        ("tex_linear_rgba", C.POINTER(C.c_float)),
    ]


class _CRect(C.Structure):
    _fields_ = [("hor_start", C.c_uint64), ("hor_end", C.c_uint64), ("vert_start", C.c_uint64), ("vert_end", C.c_uint64)]


class _CMasks(C.Structure):  # forma_masks
    _fields_ = [("ptr", C.c_void_p), ("first_order", C.c_uint32), ("n_orders", C.c_uint32), ("format", C.c_uint32),
                ("stride", C.c_uint64), ("plane_stride", C.c_uint64)]


class _CStats(C.Structure):  # forma_stats
    _fields_ = [("ptr", C.c_void_p), ("first_order", C.c_uint32), ("n_orders", C.c_uint32), ("min_coverage", C.c_float)]


class _CPoses(C.Structure):  # forma_poses
    _fields_ = [("first_order", C.c_uint32), ("n_orders", C.c_uint32), ("transforms", C.c_void_p), ("visible", C.c_void_p),
                ("colors", C.c_void_p)]


class _CInstances(C.Structure):  # forma_instances
    _fields_ = [("n_instances", C.c_uint32), ("prototypes", C.c_void_p), ("transforms", C.c_void_p), ("colors", C.c_void_p)]


def _is_cuda_array(a) -> bool:
    return a is not None and hasattr(a, "__cuda_array_interface__")


class _CudaTable:
    """A pose table in device memory, from an object with __cuda_array_interface__: its address,
    shape and bytes per frame (a chunk of frames [f, f + c) starts at ptr + f * row_bytes). It
    keeps the object alive and is never copied."""

    def __init__(self, name, a, typestrs, what="Poses"):
        cai = a.__cuda_array_interface__
        shape, typestr = tuple(int(s) for s in cai["shape"]), cai["typestr"]
        if typestr not in typestrs:
            raise ValueError(f"{what}: {name} of CUDA type {typestr!r}, not {' or '.join(map(repr, typestrs))}")
        if cai.get("mask") is not None:
            raise ValueError(f"{what}: {name} is a masked CUDA array")
        itemsize = int(typestr[2:])
        strides = cai.get("strides")
        if strides is not None:  # C-contiguous: each dimension longer than 1 steps over the ones after it
            step = itemsize
            for n, s in reversed(list(zip(shape, strides))):
                if n > 1 and s != step:
                    raise ValueError(f"{what}: {name} is not a C-contiguous CUDA array (strides {tuple(strides)})")
                step *= n
        self.owner, self.ptr, self.shape = a, int(cai["data"][0]), shape
        self.ndim = len(shape)
        self.row_bytes = itemsize * int(np.prod(shape[1:], dtype=np.int64)) if shape else 0


class Poses:
    """The per-frame layer states of a poses call (see include/forma_b200.h: forma_poses): in frame
    b, the layer at order first_order + k takes transforms[b, k] ([n, K, 6] float32, set_transform
    order [ux, vx, uy, vy, tx, ty]), is enabled where visible[b, k] ([n, K] bool / uint8) is
    non-zero, and, when it draws, fills with the solid linear RGBA colour colors[b, k] ([n, K, 4]
    float32; its fill rule, clipping and blend mode stay). Any table may be None (that state stays
    the layer's own), not all three; the tables given must agree on n and K.

    Each table may also be a CUDA array on the renderer's device: any object with
    __cuda_array_interface__, such as a torch CUDA tensor, C-contiguous, float32 transforms and
    colours, uint8 or bool visibility. It is read where it is, on the renderer's stream (see
    include/forma_b200.h: forma_poses), never copied or moved to the host; anything else is refused
    with ValueError. Host and CUDA tables can be mixed."""

    def __init__(self, first_order: int, transforms=None, visible=None, colors=None):
        if transforms is None and visible is None and colors is None:
            raise ValueError("Poses: transforms, visible, colors or several of them")
        self.first_order = int(first_order)
        if _is_cuda_array(transforms):
            self.transforms = _CudaTable("transforms", transforms, ("<f4",))
        else:
            self.transforms = None if transforms is None else np.ascontiguousarray(np.asarray(transforms, dtype=np.float32))
        if _is_cuda_array(visible):
            self.visible = _CudaTable("visible", visible, ("|u1", "|b1"))
        else:
            self.visible = None if visible is None else np.ascontiguousarray(np.asarray(visible).astype(np.uint8))
        if _is_cuda_array(colors):
            self.colors = _CudaTable("colors", colors, ("<f4",))
        else:
            if colors is not None and (not isinstance(colors, np.ndarray) or colors.dtype != np.float32):
                raise ValueError("Poses: colors must be a float32 array [n, K, 4]")
            self.colors = None if colors is None else np.ascontiguousarray(colors)
        if self.transforms is not None and (self.transforms.ndim != 3 or self.transforms.shape[2] != 6):
            raise ValueError(f"Poses: transforms of shape {self.transforms.shape}, not [n, K, 6]")
        if self.visible is not None and self.visible.ndim != 2:
            raise ValueError(f"Poses: visible of shape {self.visible.shape}, not [n, K]")
        if self.colors is not None and (self.colors.ndim != 3 or self.colors.shape[2] != 4):
            raise ValueError(f"Poses: colors of shape {self.colors.shape}, not [n, K, 4]")
        shapes = {t.shape[:2] for t in (self.transforms, self.visible, self.colors) if t is not None}
        if len(shapes) != 1:
            raise ValueError(f"Poses: the tables disagree on [n, K]: {sorted(shapes)}")
        self.n, self.n_orders = shapes.pop()

    def __len__(self) -> int:
        return self.n


NO_INSTANCE = 0xFFFFFFFF  # FORMA_NO_INSTANCE: an empty instance slot


class Instances:
    """The instance slots of an instance-scene call (see include/forma_b200.h: forma_instances):
    frame b draws, in slot m, a copy of the layer at order prototypes[b, m] ([n, M] integers; -1 or
    NO_INSTANCE = an empty slot) as the layer m of its own composition, enabled, with the transform
    transforms[b, m] ([n, M, 6] float32, set_transform order [ux, vx, uy, vy, tx, ty]; None: the
    prototype's own) and, when it draws, the solid linear RGBA fill colors[b, m] ([n, M, 4] float32;
    None: the prototype's own props). IDs, masks and statistics of the call are indexed by m.

    Each table may also be a CUDA array on the renderer's device (__cuda_array_interface__, such as
    a torch CUDA tensor, C-contiguous): int32 or uint32 prototypes (int32 -1 is NO_INSTANCE),
    float32 transforms and colours. It is read where it is, never copied by the binding; the
    library reads a CUDA prototypes table back to the host, since it decides the launch sizes.
    Host and CUDA tables can be mixed."""

    def __init__(self, prototypes, transforms=None, colors=None):
        if prototypes is None:
            raise ValueError("Instances: a prototypes table [n, M] is required")
        if _is_cuda_array(prototypes):
            self.prototypes = _CudaTable("prototypes", prototypes, ("<u4", "<i4"), "Instances")
        else:
            p = np.asarray(prototypes)
            if p.dtype.kind not in "iu":
                raise ValueError(f"Instances: prototypes of type {p.dtype}, not integers")
            p = p.astype(np.int64)
            if p.size and (p.min() < -1 or p.max() > NO_INSTANCE):
                raise ValueError("Instances: prototypes must be layer orders, -1 or NO_INSTANCE")
            self.prototypes = np.ascontiguousarray((p & NO_INSTANCE).astype(np.uint32))
        if _is_cuda_array(transforms):
            self.transforms = _CudaTable("transforms", transforms, ("<f4",), "Instances")
        else:
            self.transforms = None if transforms is None else np.ascontiguousarray(np.asarray(transforms, dtype=np.float32))
        if _is_cuda_array(colors):
            self.colors = _CudaTable("colors", colors, ("<f4",), "Instances")
        else:
            if colors is not None and (not isinstance(colors, np.ndarray) or colors.dtype != np.float32):
                raise ValueError("Instances: colors must be a float32 array [n, M, 4]")
            self.colors = None if colors is None else np.ascontiguousarray(colors)
        if self.prototypes.ndim != 2:
            raise ValueError(f"Instances: prototypes of shape {self.prototypes.shape}, not [n, M]")
        if self.transforms is not None and (self.transforms.ndim != 3 or self.transforms.shape[2] != 6):
            raise ValueError(f"Instances: transforms of shape {self.transforms.shape}, not [n, M, 6]")
        if self.colors is not None and (self.colors.ndim != 3 or self.colors.shape[2] != 4):
            raise ValueError(f"Instances: colors of shape {self.colors.shape}, not [n, M, 4]")
        shapes = {t.shape[:2] for t in (self.prototypes, self.transforms, self.colors) if t is not None}
        if len(shapes) != 1:
            raise ValueError(f"Instances: the tables disagree on [n, M]: {sorted(shapes)}")
        self.n, self.n_instances = shapes.pop()
        if self.n_instances == 0:
            raise ValueError("Instances: M = 0 slots per frame")

    def __len__(self) -> int:
        return self.n


# forma_layer_stats, one 48-byte record per frame and order (see include/forma_b200.h).
STATS_DTYPE = np.dtype([("area", np.uint64), ("pixels", np.uint32), ("visible", np.uint32), ("box", np.uint32, (4,)),
                        ("visible_box", np.uint32, (4,))])


def split_stats(t):
    """The fields of device records, a [..., 12] int32 tensor (or array) of forma_layer_stats: a dict
    of `area` (int64), `pixels`, `visible` ([...], int64) and `box`, `visible_box` ([..., 4], int64),
    the unsigned values of the records."""
    w = (t.astype(np.int64) if isinstance(t, np.ndarray) else t.long()) & 0xFFFFFFFF  # the words as unsigned 32-bit values
    return {"area": w[..., 0] | (w[..., 1] << 32), "pixels": w[..., 2], "visible": w[..., 3], "box": w[..., 4:8],
            "visible_box": w[..., 8:12]}


class _CTimings(C.Structure):
    _fields_ = [
        ("line_setup_ms", C.c_double), ("rasterize_ms", C.c_double), ("sort_ms", C.c_double),
        ("paint_ms", C.c_double), ("n_lines", C.c_uint64), ("n_segments", C.c_uint64),
    ]


@dataclass
class Timings:
    line_setup_ms: float
    rasterize_ms: float
    sort_ms: float
    paint_ms: float
    n_lines: int
    n_segments: int


def _timings(t: Optional[_CTimings]) -> Optional[Timings]:
    return Timings(t.line_setup_ms, t.rasterize_ms, t.sort_ms, t.paint_ms, t.n_lines, t.n_segments) if t is not None else None


@dataclass
class Rect:
    """cpu::Rect::new(horizontal, vertical), pixel ranges (cpu/renderer.rs:38-53)."""

    horizontal: Tuple[int, int]
    vertical: Tuple[int, int]


# Every symbol include/forma_b200.h declares (without prefix), with signature.
_f, _u8p, _u32p, _u64p, _fp = C.c_float, C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_float)
_vp = C.c_void_p
SIGNATURES = {
    "last_error": (C.c_char_p, []),
    "path_builder_new": (_vp, []),
    "path_builder_free": (None, [_vp]),
    "path_builder_move_to": (None, [_vp, _f, _f]),
    "path_builder_line_to": (None, [_vp, _f, _f]),
    "path_builder_quad_to": (None, [_vp, _f, _f, _f, _f]),
    "path_builder_cubic_to": (None, [_vp, _f, _f, _f, _f, _f, _f]),
    "path_builder_rat_quad_to": (None, [_vp, _f, _f, _f, _f, _f]),
    "path_builder_rat_cubic_to": (None, [_vp, _f, _f, _f, _f, _f, _f, _f, _f]),
    "path_builder_extend": (None, [_vp, _u8p, C.c_uint64, _fp]),
    "path_builder_build": (_vp, [_vp]),
    "path_transform": (_vp, [_vp, _fp]),
    "path_free": (None, [_vp]),
    "path_segments": (C.c_int, [_vp, C.POINTER(_fp), C.POINTER(_fp), C.POINTER(_u8p), _u64p]),
    "path_program_stats": (None, [_vp, _u64p]),
    "path_program_records": (None, [_vp, C.POINTER(_vp), _u64p, C.POINTER(_vp), C.POINTER(_u8p), _u64p, C.POINTER(_vp),
                                    _u64p, C.POINTER(C.c_int), _fp]),
    "composition_new": (_vp, []),
    "composition_free": (None, [_vp]),
    "composition_create_layer": (_vp, [_vp]),
    "composition_insert": (_vp, [_vp, C.c_uint32, _vp, C.POINTER(C.c_int)]),
    "composition_remove": (_vp, [_vp, C.c_uint32]),
    "composition_get": (_vp, [_vp, C.c_uint32]),
    "composition_get_mut_or_insert_default": (_vp, [_vp, C.c_uint32, C.POINTER(C.c_int)]),
    "composition_len": (C.c_uint64, [_vp]),
    "layer_drop": (None, [_vp, _vp]),
    "layer_geom_id": (C.c_uint64, [_vp]),
    "layer_insert": (C.c_int, [_vp, _vp, _vp]),
    "layer_clear": (C.c_int, [_vp, _vp]),
    "layer_set_is_enabled": (C.c_int, [_vp, _vp, C.c_int]),
    "layer_is_enabled": (C.c_int, [_vp]),
    "layer_set_transform": (C.c_int, [_vp, _vp, _fp]),
    "layer_set_props": (C.c_int, [_vp, _vp, C.POINTER(_CProps)]),
    "renderer_new": (_vp, [C.c_int]),
    "renderer_free": (None, [_vp]),
    "layer_cache_new": (_vp, [_vp]),
    "layer_cache_free": (None, [_vp, _vp]),
    "layer_cache_clear": (None, [_vp]),
    "renderer_render": (C.c_int, [_vp, _vp, _vp, C.c_uint64, C.c_uint64, C.c_uint64, _u32p, _fp, C.POINTER(_CRect), _vp, C.POINTER(_CTimings)]),
    "renderer_render_device": (C.c_int, [_vp, _vp, _vp, C.c_uint64, C.c_uint64, C.c_uint64, _u32p, _fp, C.POINTER(_CRect), _vp, C.POINTER(_CTimings)]),
    "renderer_render_ids": (C.c_int, [_vp, _vp, _vp, C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(_CRect), _f, C.POINTER(_CTimings)]),
    "renderer_render_ids_device": (C.c_int, [_vp, _vp, _vp, C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(_CRect), _f,
                                             C.POINTER(_CTimings)]),
    "renderer_render_device_with_ids": (C.c_int, [_vp, _vp, _vp, C.c_uint64, C.c_uint64, C.c_uint64, _u32p, _fp, C.POINTER(_CRect),
                                                  _vp, C.c_uint64, _f, C.POINTER(_CTimings)]),
    "renderer_max_views": (C.c_uint32, [C.c_uint64]),
    "renderer_render_views": (C.c_int, [_vp, _vp, _fp, C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, _u32p, _fp,
                                        C.POINTER(_CTimings)]),
    "renderer_render_views_device": (C.c_int, [_vp, _vp, _fp, C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, _u32p,
                                               _fp, C.POINTER(_CTimings)]),
    "renderer_render_batch": (C.c_int, [_vp, C.POINTER(_vp), C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, _u32p,
                                        _fp, C.POINTER(_CTimings)]),
    "renderer_render_batch_device": (C.c_int, [_vp, C.POINTER(_vp), C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64,
                                               _u32p, _fp, C.POINTER(_CTimings)]),
    "renderer_render_views_ids": (C.c_int, [_vp, _vp, _fp, C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, _f,
                                            C.POINTER(_CTimings)]),
    "renderer_render_views_ids_device": (C.c_int, [_vp, _vp, _fp, C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64,
                                                   _u32p, _fp, _vp, C.c_uint64, C.c_uint64, _f, C.POINTER(_CTimings)]),
    "renderer_render_batch_ids": (C.c_int, [_vp, C.POINTER(_vp), C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, _f,
                                            C.POINTER(_CTimings)]),
    "renderer_render_batch_ids_device": (C.c_int, [_vp, C.POINTER(_vp), C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64,
                                                   C.c_uint64, _u32p, _fp, _vp, C.c_uint64, C.c_uint64, _f, C.POINTER(_CTimings)]),
    "renderer_render_linear": (C.c_int, [_vp, _vp, _vp, C.c_uint64, C.c_uint64, C.c_uint64, _u32p, _fp, C.POINTER(_CRect), C.c_uint32,
                                         C.POINTER(_CTimings)]),
    "renderer_render_linear_device": (C.c_int, [_vp, _vp, _vp, C.c_uint64, C.c_uint64, C.c_uint64, _u32p, _fp, C.POINTER(_CRect),
                                                C.c_uint32, C.POINTER(_CTimings)]),
    "renderer_render_views_linear": (C.c_int, [_vp, _vp, _fp, C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, _u32p,
                                               _fp, C.c_uint32, C.POINTER(_CTimings)]),
    "renderer_render_views_linear_device": (C.c_int, [_vp, _vp, _fp, C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64,
                                                      _u32p, _fp, C.c_uint32, C.POINTER(_CTimings)]),
    "renderer_render_batch_linear": (C.c_int, [_vp, C.POINTER(_vp), C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64,
                                               _u32p, _fp, C.c_uint32, C.POINTER(_CTimings)]),
    "renderer_render_batch_linear_device": (C.c_int, [_vp, C.POINTER(_vp), C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64,
                                                      C.c_uint64, _u32p, _fp, C.c_uint32, C.POINTER(_CTimings)]),
    "renderer_render_over_device": (C.c_int, [_vp, _vp, _vp, C.c_uint64, C.c_uint64, C.c_uint64, _u32p, C.POINTER(_CRect), C.c_uint32,
                                              C.POINTER(_CTimings)]),
    "renderer_render_views_over_device": (C.c_int, [_vp, _vp, _fp, C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64,
                                                    _u32p, C.c_uint32, C.POINTER(_CTimings)]),
    "renderer_render_batch_over_device": (C.c_int, [_vp, C.POINTER(_vp), C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64,
                                                    C.c_uint64, _u32p, C.c_uint32, C.POINTER(_CTimings)]),
    "renderer_render_masks": (C.c_int, [_vp, _vp, C.POINTER(_CMasks), C.c_uint64, C.c_uint64, C.POINTER(_CRect), C.POINTER(_CTimings)]),
    "renderer_render_masks_device": (C.c_int, [_vp, _vp, C.POINTER(_CMasks), C.c_uint64, C.c_uint64, C.POINTER(_CRect), _vp,
                                               C.c_uint64, _u32p, _fp, C.POINTER(_CTimings)]),
    "renderer_render_views_masks_device": (C.c_int, [_vp, _vp, _fp, C.c_uint32, C.POINTER(_CMasks), C.c_uint64, C.c_uint64, _vp,
                                                     C.c_uint64, C.c_uint64, _u32p, _fp, C.POINTER(_CTimings)]),
    "renderer_render_batch_masks_device": (C.c_int, [_vp, C.POINTER(_vp), C.c_uint32, C.POINTER(_CMasks), C.c_uint64, C.c_uint64,
                                                     _vp, C.c_uint64, C.c_uint64, _u32p, _fp, C.POINTER(_CTimings)]),
    "renderer_render_stats": (C.c_int, [_vp, _vp, C.POINTER(_CStats), C.c_uint64, C.c_uint64, C.POINTER(_CRect), C.POINTER(_CTimings)]),
    "renderer_render_stats_device": (C.c_int, [_vp, _vp, C.POINTER(_CStats), C.c_uint64, C.c_uint64, C.POINTER(_CRect), _vp,
                                               C.c_uint64, _u32p, _fp, C.POINTER(_CTimings)]),
    "renderer_render_views_stats_device": (C.c_int, [_vp, _vp, _fp, C.c_uint32, C.POINTER(_CStats), C.c_uint64, C.c_uint64, _vp,
                                                     C.c_uint64, C.c_uint64, _u32p, _fp, C.POINTER(_CTimings)]),
    "renderer_render_batch_stats_device": (C.c_int, [_vp, C.POINTER(_vp), C.c_uint32, C.POINTER(_CStats), C.c_uint64, C.c_uint64,
                                                     _vp, C.c_uint64, C.c_uint64, _u32p, _fp, C.POINTER(_CTimings)]),
    "renderer_render_poses": (C.c_int, [_vp, _vp, C.POINTER(_CPoses), C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64,
                                        _u32p, _fp, C.POINTER(_CTimings)]),
    "renderer_render_poses_device": (C.c_int, [_vp, _vp, C.POINTER(_CPoses), C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64,
                                               C.c_uint64, _u32p, _fp, C.POINTER(_CTimings)]),
    "renderer_render_poses_ids": (C.c_int, [_vp, _vp, C.POINTER(_CPoses), C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64,
                                            C.c_uint64, _f, C.POINTER(_CTimings)]),
    "renderer_render_poses_ids_device": (C.c_int, [_vp, _vp, C.POINTER(_CPoses), C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64,
                                                   C.c_uint64, _u32p, _fp, _vp, C.c_uint64, C.c_uint64, _f, C.POINTER(_CTimings)]),
    "renderer_render_poses_masks_device": (C.c_int, [_vp, _vp, C.POINTER(_CPoses), C.c_uint32, C.POINTER(_CMasks), C.c_uint64,
                                                     C.c_uint64, _vp, C.c_uint64, C.c_uint64, _u32p, _fp, C.POINTER(_CTimings)]),
    "renderer_render_poses_stats_device": (C.c_int, [_vp, _vp, C.POINTER(_CPoses), C.c_uint32, C.POINTER(_CStats), C.c_uint64,
                                                     C.c_uint64, _vp, C.c_uint64, C.c_uint64, _u32p, _fp, C.POINTER(_CTimings)]),
    "renderer_render_poses_linear": (C.c_int, [_vp, _vp, C.POINTER(_CPoses), C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64,
                                               C.c_uint64, _u32p, _fp, C.c_uint32, C.POINTER(_CTimings)]),
    "renderer_render_poses_linear_device": (C.c_int, [_vp, _vp, C.POINTER(_CPoses), C.c_uint32, _vp, C.c_uint64, C.c_uint64,
                                                      C.c_uint64, C.c_uint64, _u32p, _fp, C.c_uint32, C.POINTER(_CTimings)]),
    "renderer_render_poses_over_device": (C.c_int, [_vp, _vp, C.POINTER(_CPoses), C.c_uint32, _vp, C.c_uint64, C.c_uint64, C.c_uint64,
                                                    C.c_uint64, _u32p, C.c_uint32, C.POINTER(_CTimings)]),
    "renderer_render_instances_device": (C.c_int, [_vp, _vp, C.POINTER(_CInstances), C.c_uint32, _vp, C.c_uint64, C.c_uint64,
                                                   C.c_uint64, C.c_uint64, _u32p, _fp, C.POINTER(_CTimings)]),
    "renderer_render_instances_ids_device": (C.c_int, [_vp, _vp, C.POINTER(_CInstances), C.c_uint32, _vp, C.c_uint64, C.c_uint64,
                                                       C.c_uint64, C.c_uint64, _u32p, _fp, _vp, C.c_uint64, C.c_uint64, _f,
                                                       C.POINTER(_CTimings)]),
    "renderer_render_instances_masks_device": (C.c_int, [_vp, _vp, C.POINTER(_CInstances), C.c_uint32, C.POINTER(_CMasks), C.c_uint64,
                                                         C.c_uint64, _vp, C.c_uint64, C.c_uint64, _u32p, _fp, C.POINTER(_CTimings)]),
    "renderer_render_instances_stats_device": (C.c_int, [_vp, _vp, C.POINTER(_CInstances), C.c_uint32, C.POINTER(_CStats), C.c_uint64,
                                                         C.c_uint64, _vp, C.c_uint64, C.c_uint64, _u32p, _fp, C.POINTER(_CTimings)]),
    "renderer_launch_count": (C.c_uint64, [_vp]),
    "renderer_stage_times": (None, [_vp, C.POINTER(C.c_double)]),
    "renderer_counters": (None, [_vp, _u64p]),
    "renderer_host_slices": (C.c_int, [_vp, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "renderer_kernel_times": (None, [_vp, C.POINTER(C.c_double), _u32p]),
    "renderer_set_stream": (None, [_vp, _vp]),
    "shared_frame_create": (C.c_int, [C.c_int, C.c_uint64, C.POINTER(C.c_void_p), C.c_char_p]),
    "shared_frame_open": (C.c_int, [C.c_int, C.c_char_p, C.POINTER(C.c_void_p)]),
    "shared_frame_close": (C.c_int, [C.c_int, _vp]),
    "shared_frame_free": (C.c_int, [C.c_int, _vp]),
    "composition_evict": (None, [_vp]),
    "composition_point_count": (C.c_uint64, [_vp]),
    "renderer_lines": (C.c_uint64, [_vp, C.c_uint64, _u32p, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _u32p]),
    "renderer_segments": (C.c_uint64, [_vp, C.c_uint64, _u64p]),
    "renderer_rasterize_only": (C.c_uint64, [_vp, _vp, C.c_uint64, C.c_uint64, C.c_uint64, _u64p]),
    "renderer_sort_u64": (C.c_int, [_vp, _u64p, C.c_uint64]),
    "debug_sort_plan": (C.c_int, [C.c_int, _u64p, _u8p]),
    "renderer_sort_pairs": (C.c_int, [_vp, C.c_int, C.c_int, _u64p, _u32p, C.c_uint64, C.c_uint64]),
    "renderer_sort_bounds": (None, [_vp, _u64p]),
    "renderer_sort_counts": (C.c_uint64, [_vp, C.c_int, _u32p, _u32p, C.c_uint64]),
    "renderer_sort_mode": (C.c_uint32, [_vp]),
    "debug_selftest": (C.c_int, [C.c_int, _u64p]),
    "renderer_multi_new": (_vp, [C.POINTER(C.c_int), C.c_int]),
    "renderer_multi_free": (None, [_vp]),
    "renderer_multi_device_count": (C.c_int, [_vp]),
    "renderer_multi_render": (C.c_int, [_vp, _vp, _vp, C.c_uint64, C.c_uint64, C.c_uint64, _u32p, _fp, C.POINTER(_CRect), C.POINTER(_CTimings)]),
    "renderer_multi_render_device": (C.c_int, [_vp, _vp, _vp, C.c_uint64, C.c_uint64, C.c_uint64, _u32p, _fp, C.POINTER(_CRect), C.POINTER(_CTimings)]),
    "renderer_multi_bands": (C.c_int, [_vp, _u32p, C.POINTER(C.c_double)]),
    "renderer_row_costs": (C.c_uint64, [_vp, C.c_uint64, _u64p]),
    "set_option": (C.c_int, [C.c_char_p, C.c_int]),
    "get_option": (C.c_int, [C.c_char_p, C.POINTER(C.c_int)]),
}


# The ID-frame entry points. A library may be built without them (it then loads, and the ID
# methods of Renderer fail); `Api.attach` can take them from a companion library.
ID_FRAME_SYMBOLS = ("renderer_render_ids", "renderer_render_ids_device", "renderer_render_device_with_ids")
# The entry points of views (Renderer.render_views): the CUDA library has them, other libraries
# with this binding's symbols may not (the view methods of Renderer then fail).
VIEW_SYMBOLS = ("renderer_max_views", "renderer_render_views", "renderer_render_views_device")
# The same for batches (Renderer.render_batch).
BATCH_SYMBOLS = ("renderer_render_batch", "renderer_render_batch_device")
# The same for the ID frames of views and batches (Renderer.render_views_ids, render_batch_ids).
STACK_ID_SYMBOLS = ("renderer_render_views_ids", "renderer_render_views_ids_device", "renderer_render_batch_ids",
                    "renderer_render_batch_ids_device")


# The same for the inspection entry points of the sort (sort_plan, Renderer.sort_pairs, sort_bounds).
SORT_DEBUG_SYMBOLS = ("debug_sort_plan", "renderer_sort_pairs", "renderer_sort_bounds", "renderer_sort_counts", "renderer_sort_mode")
# The same for linear float frames (Renderer.render_linear, render_views_linear, render_batch_linear).
LINEAR_SYMBOLS = ("renderer_render_linear", "renderer_render_linear_device", "renderer_render_views_linear",
                  "renderer_render_views_linear_device", "renderer_render_batch_linear", "renderer_render_batch_linear_device")

# The same for frames over a background (Renderer.render_over_device, render_views_over_device,
# render_batch_over_device).
OVER_SYMBOLS = ("renderer_render_over_device", "renderer_render_views_over_device", "renderer_render_batch_over_device")

# The same for layer coverage masks (Renderer.render_masks, render_masks_device, render_views_masks_device,
# render_batch_masks_device).
MASK_SYMBOLS = ("renderer_render_masks", "renderer_render_masks_device", "renderer_render_views_masks_device",
                "renderer_render_batch_masks_device")
# The same for layer statistics (Renderer.render_stats, render_stats_device, render_views_stats_device,
# render_batch_stats_device).
STATS_SYMBOLS = ("renderer_render_stats", "renderer_render_stats_device", "renderer_render_views_stats_device",
                 "renderer_render_batch_stats_device")
# The same for poses (Renderer.render_poses, render_poses_device, render_poses_ids{,_device},
# render_poses_masks_device, render_poses_stats_device, render_poses_linear{,_device},
# render_poses_over_device).
POSE_SYMBOLS = ("renderer_render_poses", "renderer_render_poses_device", "renderer_render_poses_ids",
                "renderer_render_poses_ids_device", "renderer_render_poses_masks_device", "renderer_render_poses_stats_device",
                "renderer_render_poses_linear", "renderer_render_poses_linear_device", "renderer_render_poses_over_device")
# The same for instance scenes (Renderer.render_instances_device, render_instances_ids_device,
# render_instances_masks_device, render_instances_stats_device).
INSTANCE_SYMBOLS = ("renderer_render_instances_device", "renderer_render_instances_ids_device",
                    "renderer_render_instances_masks_device", "renderer_render_instances_stats_device")
# Value formats of mask planes: name -> (FORMA_MASK_*, bytes per value, numpy dtype).
MASK_FORMATS = {"f32": (0, 4, np.float32), "u8": (1, 1, np.uint8)}


def mask_format(fmt: str):
    """(FORMA_MASK_* code, bytes per value, numpy dtype) of "f32" or "u8"."""
    if fmt not in MASK_FORMATS:
        raise ValueError(f"mask format {fmt!r}: 'f32' or 'u8'")
    return MASK_FORMATS[fmt]


# Pixel formats of linear frames: name -> (FORMA_PIXEL_*, bytes per pixel, element dtype).
PIXEL_FORMATS = {"f16": (1, 8, np.float16), "f32": (2, 16, np.float32)}
# ... and of frames over a background, which may be sRGB8 as well.
OVER_FORMATS = {"srgb8": (0, 4, np.uint8), **PIXEL_FORMATS}


def pixel_format(fmt: str):
    """(FORMA_PIXEL_* code, bytes per pixel, numpy dtype) of "f16" or "f32"."""
    if fmt not in PIXEL_FORMATS:
        raise ValueError(f"pixel format {fmt!r}: 'f16' or 'f32'")
    return PIXEL_FORMATS[fmt]


def over_format(fmt: str):
    """(FORMA_PIXEL_* code, bytes per pixel, numpy dtype) of "srgb8", "f16" or "f32"."""
    if fmt not in OVER_FORMATS:
        raise ValueError(f"pixel format {fmt!r}: 'srgb8', 'f16' or 'f32'")
    return OVER_FORMATS[fmt]


_OPTIONAL_SYMBOLS = frozenset(ID_FRAME_SYMBOLS + VIEW_SYMBOLS + BATCH_SYMBOLS + STACK_ID_SYMBOLS + SORT_DEBUG_SYMBOLS +
                              LINEAR_SYMBOLS + OVER_SYMBOLS + MASK_SYMBOLS + STATS_SYMBOLS + POSE_SYMBOLS + INSTANCE_SYMBOLS)


class Api:
    """Typed access to one shared library exporting `<prefix><name>` symbols."""

    def __init__(self, lib: C.CDLL, prefix: str, optional: Sequence[str] = ()):
        self.lib, self.prefix = lib, prefix
        for name, (res, args) in SIGNATURES.items():
            try:
                fn = getattr(lib, prefix + name)
            except AttributeError:
                if name in optional or name in _OPTIONAL_SYMBOLS:
                    continue
                raise
            fn.restype, fn.argtypes = res, args
            setattr(self, name + "_fn" if name in ("set_option", "get_option") else name, fn)

    def attach(self, lib: C.CDLL, names: Sequence[str]) -> "Api":
        """Binds `names` (keys of SIGNATURES) from `lib`, a library with the same symbol prefix
        that works on this library's objects."""
        for name in names:
            fn = getattr(lib, self.prefix + name)
            fn.restype, fn.argtypes = SIGNATURES[name]
            setattr(self, name, fn)
        return self

    def check(self, status: int, what: str) -> None:
        if status == 0:
            return
        msg = self.last_error().decode() if hasattr(self, "last_error") else ""
        if status == 2:
            raise OrderError(f"{what}: exceeded layer limit ({LAYER_LIMIT})")
        raise FormaError(f"{what}: status {status} {msg}")

    def set_option(self, name: str, value: int) -> None:
        """Schedule switch of the library (see include/forma_b200.h: forma_set_option)."""
        self.check(self.__dict__["set_option_fn"](name.encode(), int(value)), f"set_option({name})")

    def get_option(self, name: str) -> int:
        v = C.c_int(0)
        self.check(self.__dict__["get_option_fn"](name.encode(), C.byref(v)), f"get_option({name})")
        return int(v.value)

    def sort_plan(self, layout: int, bound: Sequence[int]) -> bytes:
        """The library's sort plan for the field bounds `bound` (least significant field first)
        under layout 0 (segments) or 1 (carry keys): n_passes, total_bits, then 10 bytes per pass
        (shift[3], width[3], lsh[3], bits). No device is touched."""
        b = (C.c_uint64 * 3)(*[int(v) for v in bound])
        out = (C.c_uint8 * 62)()
        self.check(self.debug_sort_plan(layout, b, out), "sort_plan")
        return bytes(out)

    # Constructors bound to this library -----------------------------------
    def PathBuilder(self) -> "PathBuilder":
        return PathBuilder(self)

    def Composition(self) -> "Composition":
        return Composition(self)

    def Renderer(self, device: int = 0) -> "Renderer":
        return Renderer(self, device)

    def MultiRenderer(self, devices: Sequence[int]) -> "MultiRenderer":
        return MultiRenderer(self, devices)

    def SharedFrame(self, device: int, nbytes: int, handle: Optional[bytes] = None) -> "SharedFrame":
        return SharedFrame(self, device, nbytes, handle)


class SharedFrame:
    """A frame in one GPU's HBM that other processes paint into over NVLink
    (forma_shared_frame_*): the owner passes `handle` (64 bytes) to the other
    ranks, which construct theirs with it; `ptr` goes to Renderer.render_device.
    `__cuda_array_interface__` lets torch / cupy view the bytes without a copy."""

    def __init__(self, api: "Api", device: int, nbytes: int, handle: Optional[bytes] = None):
        self._api, self.device, self.nbytes, self.owner = api, device, nbytes, handle is None
        p = C.c_void_p()
        if self.owner:
            buf = C.create_string_buffer(64)
            api.check(api.shared_frame_create(device, nbytes, C.byref(p), buf), "shared_frame_create")
            self.handle = buf.raw
        else:
            self.handle = bytes(handle)
            api.check(api.shared_frame_open(device, self.handle, C.byref(p)), "shared_frame_open")
        self.ptr = int(p.value)

    @property
    def __cuda_array_interface__(self):
        return {"shape": (self.nbytes,), "typestr": "|u1", "data": (self.ptr, False), "version": 2}

    def close(self):
        if self.ptr:
            (self._api.shared_frame_free if self.owner else self._api.shared_frame_close)(self.device, C.c_void_p(self.ptr))
            self.ptr = 0


# Flatten-program records (forma_b200/csrc/device_types.h), as Path.program() returns them.
SPLINE_REC = np.dtype([("p0x", "<f4"), ("p0y", "<f4"), ("p2x", "<f4"), ("p2y", "<f4"), ("step", "<f4"),
                       ("first_quad", "<u4"), ("n_quads", "<u4"), ("first_point", "<u4"), ("info", "<u4")])
POINT_REC = np.dtype([("a", "<f4"), ("b", "<f4")])  # kind 2 / 3: a holds the quad index's bits
QUAD_REC = np.dtype([("px", "<f4", 3), ("py", "<f4", 3), ("pw", "<f4", 3), ("x0", "<f4"), ("dx_recip", "<f4"),
                     ("k0", "<f4"), ("dk", "<f4"), ("curv_recip", "<f4"), ("prev_curv", "<f4"), ("total", "<f4"),
                     ("step", "<f4")])
assert (SPLINE_REC.itemsize, POINT_REC.itemsize, QUAD_REC.itemsize) == (36, 8, 68)


def _np_f32(ptr, n):
    return np.ctypeslib.as_array(ptr, shape=(n,)).copy() if n else np.zeros(0, np.float32)


class Path:
    """forma/src/path.rs:670-766."""

    def __init__(self, api: Api, handle):
        self._api, self._h = api, handle

    def transform(self, m: Sequence[float]) -> "Path":
        arr = (C.c_float * 9)(*[float(v) for v in m])
        return Path(self._api, self._api.path_transform(self._h, arr))

    def program_stats(self) -> dict:
        """Host-side facts of the flatten program (CUDA library only; needs no GPU)."""
        out = (C.c_uint64 * 6)()
        self._api.path_program_stats(self._h, out)
        return dict(zip(("points", "quads", "splines", "point_records", "rational", "contour_ends"), [int(v) for v in out]))

    def program(self) -> dict:
        """The flatten program's records as the host built them (CUDA library only; needs no
        GPU; inspection only): structured arrays "splines" (SPLINE_REC), "points" (POINT_REC),
        "kinds" (uint8 per point record), "quads" (QUAD_REC), plus "bounded" and "bounds"
        (min x, min y, max x, max y) and the program_stats() facts under "stats"."""
        a = self._api
        sp, pp, qp, kp = _vp(), _vp(), _vp(), _u8p()
        ns, nr, nq, bounded = C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_int()
        bounds = (C.c_float * 4)()
        a.path_program_records(self._h, C.byref(sp), C.byref(ns), C.byref(pp), C.byref(kp), C.byref(nr), C.byref(qp),
                               C.byref(nq), C.byref(bounded), bounds)

        def records(ptr, n, dtype):
            if n == 0:
                return np.zeros(0, dtype)
            return np.frombuffer(C.string_at(ptr.value, n * dtype.itemsize), dtype).copy()
        return {
            "splines": records(sp, ns.value, SPLINE_REC),
            "points": records(pp, nr.value, POINT_REC),
            "kinds": np.ctypeslib.as_array(kp, shape=(nr.value,)).copy() if nr.value else np.zeros(0, np.uint8),
            "quads": records(qp, nq.value, QUAD_REC),
            "bounded": bool(bounded.value),
            "bounds": np.array(list(bounds), np.float32),
            "stats": self.program_stats(),
        }

    def segments(self):
        """Flattened points: (x, y, start_new_contour) numpy arrays."""
        x, y, c, n = _fp(), _fp(), _u8p(), C.c_uint64()
        self._api.check(self._api.path_segments(self._h, C.byref(x), C.byref(y), C.byref(c), C.byref(n)), "path_segments")
        k = n.value
        if k == 0:
            return np.zeros(0, np.float32), np.zeros(0, np.float32), np.zeros(0, np.uint8)
        return _np_f32(x, k), _np_f32(y, k), np.ctypeslib.as_array(c, shape=(k,)).copy()

    def __del__(self):
        try:
            self._api.path_free(self._h)
        except Exception:
            pass


class PathBuilder:
    """forma/src/path.rs:776-925."""

    def __init__(self, api: Api):
        self._api = api
        self._h = api.path_builder_new()

    def move_to(self, p: Point) -> "PathBuilder":
        self._api.path_builder_move_to(self._h, p.x, p.y)
        return self

    def line_to(self, p: Point) -> "PathBuilder":
        self._api.path_builder_line_to(self._h, p.x, p.y)
        return self

    def quad_to(self, p1: Point, p2: Point) -> "PathBuilder":
        self._api.path_builder_quad_to(self._h, p1.x, p1.y, p2.x, p2.y)
        return self

    def cubic_to(self, p1: Point, p2: Point, p3: Point) -> "PathBuilder":
        self._api.path_builder_cubic_to(self._h, p1.x, p1.y, p2.x, p2.y, p3.x, p3.y)
        return self

    def rat_quad_to(self, p1: Point, p2: Point, weight: float) -> "PathBuilder":
        self._api.path_builder_rat_quad_to(self._h, p1.x, p1.y, p2.x, p2.y, weight)
        return self

    def rat_cubic_to(self, p1: Point, p2: Point, p3: Point, w1: float, w2: float) -> "PathBuilder":
        self._api.path_builder_rat_cubic_to(self._h, p1.x, p1.y, p2.x, p2.y, p3.x, p3.y, w1, w2)
        return self

    def extend(self, cmds: np.ndarray, xy: np.ndarray) -> "PathBuilder":
        """Bulk move/line/quad/cubic (codes 0..3) with their points (float32, flat)."""
        cmds = np.ascontiguousarray(cmds, np.uint8)
        xy = np.ascontiguousarray(xy, np.float32)
        self._api.path_builder_extend(self._h, cmds.ctypes.data_as(_u8p), cmds.size, xy.ctypes.data_as(_fp))
        return self

    def build(self) -> Path:
        return Path(self._api, self._api.path_builder_build(self._h))

    def __del__(self):
        try:
            self._api.path_builder_free(self._h)
        except Exception:
            pass


def _lower_props(props: Props):
    """Props -> (_CProps, keepalive list)."""
    cp = _CProps()
    keep = []
    cp.fill_rule = props.fill_rule
    if props.func.clip is not None:
        cp.func = 1
        cp.clip_layers = int(props.func.clip)
        return cp, keep
    style = props.func.draw
    cp.func = 0
    cp.is_clipped = 1 if style.is_clipped else 0
    cp.blend_mode = style.blend_mode
    fill = style.fill
    if fill.solid is not None:
        cp.fill_type = 0
        c = fill.solid
        cp.color = _CColor(c.r, c.g, c.b, c.a)
    elif fill.gradient is not None:
        g = fill.gradient
        cp.fill_type = 1
        cp.gradient_type = g.type
        cp.start[0], cp.start[1] = g.start.x, g.start.y
        cp.end[0], cp.end[1] = g.end.x, g.end.y
        stops = (_CStop * len(g.stops))()
        for i, (c, s) in enumerate(g.stops):
            stops[i].color = _CColor(c.r, c.g, c.b, c.a)
            stops[i].stop = s
        keep.append(stops)
        cp.n_stops = len(g.stops)
        cp.stops = C.cast(stops, C.POINTER(_CStop))
    else:
        t = fill.texture
        cp.fill_type = 2
        img = np.ascontiguousarray(t.linear_rgba, dtype=np.float32)
        keep.append(img)
        for i in range(6):
            cp.tex_transform[i] = t.transform[i]
        cp.tex_height, cp.tex_width = img.shape[0], img.shape[1]
        cp.tex_linear_rgba = img.ctypes.data_as(_fp)
    return cp, keep


class Layer:
    """forma/src/composition/layer.rs:61-353. The handle is owned by the
    Composition; `drop()` is Rust's `Drop for Layer`."""

    def __init__(self, comp: "Composition", handle):
        self._c, self._h = comp, handle

    def insert(self, path: Path) -> "Layer":
        a = self._c._api
        a.check(a.layer_insert(self._c._h, self._h, path._h), "Layer::insert")
        return self

    def clear(self) -> "Layer":
        a = self._c._api
        a.check(a.layer_clear(self._c._h, self._h), "Layer::clear")
        return self

    def geom_id(self) -> int:
        return int(self._c._api.layer_geom_id(self._h))

    def set_props(self, props: Props) -> "Layer":
        a = self._c._api
        cp, keep = _lower_props(props)
        a.check(a.layer_set_props(self._c._h, self._h, C.byref(cp)), "Layer::set_props")
        del keep
        return self

    def set_transform(self, t: Sequence[float]) -> "Layer":
        """t = [ux, vx, uy, vy, tx, ty] as GeomPresTransform::try_from([f32; 6])."""
        a = self._c._api
        arr = (C.c_float * 6)(*[float(v) for v in t])
        st = a.layer_set_transform(self._c._h, self._h, arr)
        if st == 1:
            raise GeomPresTransformError("exceeded scaling factor")
        a.check(st, "Layer::set_transform")
        return self

    def is_enabled(self) -> bool:
        return bool(self._c._api.layer_is_enabled(self._h))

    def set_is_enabled(self, enabled: bool) -> "Layer":
        a = self._c._api
        a.check(a.layer_set_is_enabled(self._c._h, self._h, 1 if enabled else 0), "Layer::set_is_enabled")
        return self

    def enable(self) -> "Layer":
        return self.set_is_enabled(True)

    def disable(self) -> "Layer":
        return self.set_is_enabled(False)

    def drop(self) -> None:
        self._c._api.layer_drop(self._c._h, self._h)
        self._h = None


class Composition:
    """forma/src/composition/mod.rs:53-343."""

    def __init__(self, api: Api):
        self._api = api
        self._h = api.composition_new()

    def create_layer(self) -> Layer:
        return Layer(self, self._api.composition_create_layer(self._h))

    def insert(self, order: int, layer: Layer) -> Optional[Layer]:
        st = C.c_int(0)
        old = self._api.composition_insert(self._h, order, layer._h, C.byref(st))
        self._api.check(st.value, "Order::new")
        return Layer(self, old) if old else None

    def remove(self, order: int) -> Optional[Layer]:
        h = self._api.composition_remove(self._h, order)
        return Layer(self, h) if h else None

    def get(self, order: int) -> Optional[Layer]:
        h = self._api.composition_get(self._h, order)
        return Layer(self, h) if h else None

    get_mut = get

    def get_mut_or_insert_default(self, order: int) -> Layer:
        st = C.c_int(0)
        h = self._api.composition_get_mut_or_insert_default(self._h, order, C.byref(st))
        self._api.check(st.value, "Order::new")
        return Layer(self, h)

    def evict(self) -> None:
        """Drop device residency (next render re-uploads from pinned host memory)."""
        self._api.composition_evict(self._h)

    def point_count(self) -> int:
        return int(self._api.composition_point_count(self._h))

    def __len__(self) -> int:
        return int(self._api.composition_len(self._h))

    def is_empty(self) -> bool:
        return len(self) == 0

    def __del__(self):
        try:
            self._api.composition_free(self._h)
        except Exception:
            pass


class LayerCache:
    def __init__(self, renderer: "Renderer", handle):
        self._r, self._h = renderer, handle

    def clear(self):
        self._r._api.layer_cache_clear(self._h)

    def __del__(self):
        try:
            self._r._api.layer_cache_free(self._r._h, self._h)
        except Exception:
            pass


class Renderer:
    """forma/src/cpu/renderer.rs:56-224 — `render` has the same arguments:
    (composition, buffer(width, stride, height), channels, clear_color, crop)."""

    def __init__(self, api: Api, device: int = 0):
        self._api = api
        self._h = api.renderer_new(device)
        if not self._h:
            msg = api.last_error().decode() if hasattr(api, "last_error") else ""
            raise FormaError(f"Renderer::new failed (no CPU fallback exists): {msg}")

    def create_buffer_layer_cache(self) -> Optional[LayerCache]:
        h = self._api.layer_cache_new(self._h)
        return LayerCache(self, h) if h else None

    def _common(self, channels, clear_color, crop):
        ch = (C.c_uint32 * 4)(*channels)
        cc = (C.c_float * 4)(clear_color.r, clear_color.g, clear_color.b, clear_color.a)
        rect = None
        if crop is not None:
            rect = _CRect(crop.horizontal[0], crop.horizontal[1], crop.vertical[0], crop.vertical[1])
        return ch, cc, rect

    def _frame(self, fn, what, composition, ptr, width, height, stride, colors, crop, tail, timings):
        """Calls `fn`, a single-frame entry point: fn(renderer, composition, ptr, width, stride, height,
        [channels, [clear colour,]] crop, *tail, timings), with channels and clear colour when
        `colors` = (channels, clear_color) is given, channels alone when clear_color is None."""
        stride = width * 4 if stride is None else stride
        channels, clear = colors or (RGBA, Color())
        ch, cc, rect = self._common(channels, Color() if clear is None else clear, crop)
        colour_args = () if not colors else (ch,) if clear is None else (ch, cc)
        t = _CTimings() if timings else None
        st = fn(self._h, composition._h, ptr, width, stride, height, *colour_args,
                C.byref(rect) if rect is not None else None, *tail, C.byref(t) if t is not None else None)
        self._api.check(st, what)
        return _timings(t)

    def render(self, composition: Composition, buffer: np.ndarray, width: int, height: int,
               channels=RGBA, clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), crop: Optional[Rect] = None,
               layer_cache: Optional[LayerCache] = None, stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """`buffer`: writable contiguous uint8 host array of >= height*stride bytes.
        timings=False passes a null `forma_timings*`: the call then does not query its stage events
        (stage_times() still can, afterwards)."""
        stride = width * 4 if stride is None else stride
        assert buffer.dtype == np.uint8 and buffer.flags["C_CONTIGUOUS"] and buffer.size >= height * stride
        return self._frame(self._api.renderer_render, "Renderer::render", composition, buffer.ctypes.data_as(C.c_void_p), width,
                           height, stride, (channels, clear_color), crop, (layer_cache._h if layer_cache else None,), timings)

    def render_device(self, composition: Composition, device_ptr: int, width: int, height: int,
                      channels=RGBA, clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), crop: Optional[Rect] = None,
                      layer_cache: Optional[LayerCache] = None, stride: Optional[int] = None,
                      timings: bool = True) -> Optional[Timings]:
        return self._frame(self._api.renderer_render_device, "Renderer::render_device", composition, C.c_void_p(device_ptr), width,
                           height, stride, (channels, clear_color), crop, (layer_cache._h if layer_cache else None,), timings)

    def render_ids(self, composition: Composition, ids: np.ndarray, width: int, height: int, crop: Optional[Rect] = None,
                   stride: Optional[int] = None, min_coverage: float = 0.0, timings: bool = True) -> Optional[Timings]:
        """ID frame into a host array: per pixel the order of the top-most Draw layer whose coverage
        (x clip mask) exceeds `min_coverage`, or ID_NONE. `ids`: writable contiguous uint32 array
        of >= height * stride / 4 elements; `stride` in bytes (default 4 * width). Only the crop's
        tile rectangle is written."""
        stride = width * 4 if stride is None else stride
        assert ids.dtype == np.uint32 and ids.flags["C_CONTIGUOUS"] and ids.size * 4 >= height * stride
        return self._frame(self._api.renderer_render_ids, "Renderer::render_ids", composition, ids.ctypes.data_as(C.c_void_p), width,
                           height, stride, None, crop, (float(min_coverage),), timings)

    def render_ids_device(self, composition: Composition, device_ptr: int, width: int, height: int,
                          crop: Optional[Rect] = None, stride: Optional[int] = None, min_coverage: float = 0.0,
                          timings: bool = True) -> Optional[Timings]:
        """render_ids into device memory (e.g. a torch int32 / uint32 tensor's data_ptr())."""
        return self._frame(self._api.renderer_render_ids_device, "Renderer::render_ids_device", composition, C.c_void_p(device_ptr),
                           width, height, stride, None, crop, (float(min_coverage),), timings)

    def render_device_with_ids(self, composition: Composition, device_ptr: int, ids_device_ptr: int, width: int, height: int,
                               channels=RGBA, clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), crop: Optional[Rect] = None,
                               stride: Optional[int] = None, ids_stride: Optional[int] = None, min_coverage: float = 0.0,
                               timings: bool = True) -> Optional[Timings]:
        """render_device (without a layer cache) and render_ids_device of the same frame from one
        pass through the stages; both pointers are device memory."""
        ids_stride = width * 4 if ids_stride is None else ids_stride
        return self._frame(self._api.renderer_render_device_with_ids, "Renderer::render_device_with_ids", composition,
                           C.c_void_p(device_ptr), width, height, stride, (channels, clear_color), crop,
                           (C.c_void_p(ids_device_ptr), ids_stride, float(min_coverage)), timings)

    def max_views(self, height: int) -> int:
        """The most views of `height` rows one render_views call of the library takes (0: none)."""
        return int(self._api.renderer_max_views(height))

    def _stack(self, fn, what, first_args, n, width, height, rgba, ids, timings, bpp=4, tail=(), chunk=None):
        """Calls `fn`, an entry point of views or batches, on chunks of at most max_views(height)
        frames: first_args(first, count) gives a chunk's leading arguments (views or handles,
        count), then come its targets. rgba = (ptr or None, stride, frame_stride, channels,
        clear_color) and ids = (ptr, stride, frame_stride, min_coverage), either may be None; a
        stride of None takes its default (bpp * width, height * stride; IDs: bpp 4); a clear colour
        of None is not passed (frames over a background). An entry point with both takes the ID
        target's arguments without width and height. `tail` follows the targets. `chunk`: fewer
        frames per call than max_views(height)."""
        chunk = max(min(self.max_views(height), chunk or self.max_views(height)), 1)
        if rgba is not None:
            rgba_ptr, stride, frame_stride = rgba[0], *self._strides(width, height, rgba[1], rgba[2], bpp)
            ch, cc, _ = self._common(rgba[3], Color() if rgba[4] is None else rgba[4], None)
            colour_args = [ch] if rgba[4] is None else [ch, cc]
        if ids is not None:
            ids_ptr, ids_stride, ids_frame_stride = ids[0], *self._strides(width, height, ids[1], ids[2])
        t = None
        for first in range(0, max(n, 1), chunk):
            args = list(first_args(first, min(chunk, n - first)))
            if rgba is not None:
                ptr = C.c_void_p(rgba_ptr + first * frame_stride) if rgba_ptr is not None else None
                args += [ptr, width, stride, height, frame_stride, *colour_args]
            if ids is not None:
                ptr = C.c_void_p(ids_ptr + first * ids_frame_stride)
                layout = [ids_stride, ids_frame_stride] if rgba is not None else [width, ids_stride, height, ids_frame_stride]
                args += [ptr, *layout, float(ids[3])]
            t = _CTimings() if timings else None
            st = fn(self._h, *args, *tail, C.byref(t) if t is not None else None)
            self._api.check(st, what)
        return _timings(t)

    @staticmethod
    def _strides(width, height, stride, frame_stride, bpp=4):
        """Row and frame strides in bytes, by default bpp * width and height * stride."""
        stride = width * bpp if stride is None else stride
        return stride, height * stride if frame_stride is None else frame_stride

    @staticmethod
    def _view_args(composition, views):
        v = np.ascontiguousarray(np.asarray(views, dtype=np.float32).reshape(-1, 6))
        keep = []  # the chunk handed to the library stays alive until the next one

        def args(first, count):
            keep[:] = [np.ascontiguousarray(v[first:first + count])]
            return composition._h, keep[0].ctypes.data_as(_fp), count
        return len(v), args

    @staticmethod
    def _batch_args(comps):
        comps = list(comps)

        def args(first, count):
            part = comps[first:first + count]
            return (_vp * max(len(part), 1))(*[c._h for c in part]), count
        return len(comps), args

    @staticmethod
    def _pose_args(composition, poses: Poses):
        """(n, args) for _stack: a chunk's forma_poses holds its frames' rows of the tables (of a CUDA
        table, the address of its first frame's row)."""
        keep = []  # the chunk's descriptor and tables stay alive until the next one

        def args(first, count):
            t, v, c = (None if a is None else a if isinstance(a, _CudaTable) else np.ascontiguousarray(a[first:first + count])
                       for a in (poses.transforms, poses.visible, poses.colors))
            d = _CPoses(poses.first_order, poses.n_orders,
                        *(None if a is None else a.ptr + first * a.row_bytes if isinstance(a, _CudaTable) else a.ctypes.data
                          for a in (t, v, c)))
            keep[:] = [t, v, c, d]
            return composition._h, C.byref(d), count
        return poses.n, args

    @staticmethod
    def _instance_args(composition, instances: Instances):
        """(n, args, chunk) for _stack: a chunk's forma_instances holds its frames' rows of the tables
        (of a CUDA table, the address of its first frame's row); a chunk holds at most 2^21 // M
        frames, so that its n M orders fit in the layer field."""
        keep = []  # the chunk's descriptor and tables stay alive until the next one

        def args(first, count):
            p, t, c = (None if a is None else a if isinstance(a, _CudaTable) else np.ascontiguousarray(a[first:first + count])
                       for a in (instances.prototypes, instances.transforms, instances.colors))
            d = _CInstances(instances.n_instances,
                            *(None if a is None else a.ptr + first * a.row_bytes if isinstance(a, _CudaTable) else a.ctypes.data
                              for a in (p, t, c)))
            keep[:] = [p, t, c, d]
            return composition._h, C.byref(d), count
        return instances.n, args, max((1 << 21) // instances.n_instances, 1)

    def render_views(self, composition: Composition, views, buffer: np.ndarray, width: int, height: int, channels=RGBA,
                     clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), stride: Optional[int] = None,
                     view_stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """One frame per row of `views`, an (N, 6) array-like of transforms in set_transform order
        [ux, vx, uy, vy, tx, ty], each a frame of the composition with every layer's transform T
        replaced by view ∘ T. Frame b starts at byte b * view_stride (default height * stride) of
        `buffer`, a writable contiguous uint8 host array; `stride` (default 4 * width) is the row
        stride. N may exceed max_views(height): the views are then rendered in chunks. Returns the
        timings of the last chunk."""
        n, args = self._view_args(composition, views)
        stride, view_stride = self._strides(width, height, stride, view_stride)
        assert buffer.dtype == np.uint8 and buffer.flags["C_CONTIGUOUS"]
        assert n == 0 or buffer.size >= (n - 1) * view_stride + (height - 1) * stride + 4 * width
        return self._stack(self._api.renderer_render_views, "Renderer::render_views", args, n, width, height,
                           (buffer.ctypes.data, stride, view_stride, channels, clear_color), None, timings)

    def render_views_device(self, composition: Composition, views, device_ptr: int, width: int, height: int, channels=RGBA,
                            clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), stride: Optional[int] = None,
                            view_stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """render_views into device memory on the renderer's device: with the defaults, the
        data_ptr() of a contiguous [N, height, width, 4] uint8 CUDA tensor."""
        n, args = self._view_args(composition, views)
        return self._stack(self._api.renderer_render_views_device, "Renderer::render_views_device", args, n, width, height,
                           (int(device_ptr), stride, view_stride, channels, clear_color), None, timings)

    def render_batch(self, comps, buffer: np.ndarray, width: int, height: int, channels=RGBA,
                     clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), stride: Optional[int] = None,
                     frame_stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """One frame per composition of the sequence `comps` (repeats allowed), frame c showing
        comps[c] alone, from one pass through the stages. Frame c starts at byte c * frame_stride
        (default height * stride) of `buffer`, a writable contiguous uint8 host array; `stride`
        (default 4 * width) is the row stride. N may exceed max_views(height): the compositions
        are then rendered in chunks. A chunk whose distinct compositions need more than 2^21 layer
        orders raises OrderError. Returns the timings of the last chunk."""
        n, args = self._batch_args(comps)
        stride, frame_stride = self._strides(width, height, stride, frame_stride)
        assert buffer.dtype == np.uint8 and buffer.flags["C_CONTIGUOUS"]
        assert n == 0 or buffer.size >= (n - 1) * frame_stride + (height - 1) * stride + 4 * width
        return self._stack(self._api.renderer_render_batch, "Renderer::render_batch", args, n, width, height,
                           (buffer.ctypes.data, stride, frame_stride, channels, clear_color), None, timings)

    def render_batch_device(self, comps, device_ptr: int, width: int, height: int, channels=RGBA,
                            clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), stride: Optional[int] = None,
                            frame_stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """render_batch into device memory on the renderer's device: with the defaults, the
        data_ptr() of a contiguous [N, height, width, 4] uint8 CUDA tensor."""
        n, args = self._batch_args(comps)
        return self._stack(self._api.renderer_render_batch_device, "Renderer::render_batch_device", args, n, width, height,
                           (int(device_ptr), stride, frame_stride, channels, clear_color), None, timings)

    def render_views_ids(self, composition: Composition, views, ids: np.ndarray, width: int, height: int,
                         ids_stride: Optional[int] = None, ids_view_stride: Optional[int] = None, min_coverage: float = 0.0,
                         timings: bool = True) -> Optional[Timings]:
        """The ID frame (see render_ids) of every view of render_views, in one pass. ID frame b
        starts at byte b * ids_view_stride (default height * ids_stride) of `ids`, a writable
        contiguous uint32 host array; `ids_stride` (default 4 * width) is the row stride in bytes.
        Chunked like render_views."""
        n, args = self._view_args(composition, views)
        s, fs = self._strides(width, height, ids_stride, ids_view_stride)
        assert ids.dtype == np.uint32 and ids.flags["C_CONTIGUOUS"]
        assert n == 0 or ids.size * 4 >= (n - 1) * fs + (height - 1) * s + 4 * width
        return self._stack(self._api.renderer_render_views_ids, "Renderer::render_views_ids", args, n, width, height, None,
                           (ids.ctypes.data, s, fs, min_coverage), timings)

    def render_views_ids_device(self, composition: Composition, views, ids_device_ptr: int, width: int, height: int,
                                rgba_ptr: Optional[int] = None, channels=RGBA, clear_color: Color = Color(1.0, 1.0, 1.0, 1.0),
                                stride: Optional[int] = None, view_stride: Optional[int] = None, ids_stride: Optional[int] = None,
                                ids_view_stride: Optional[int] = None, min_coverage: float = 0.0,
                                timings: bool = True) -> Optional[Timings]:
        """render_views_ids into device memory: with the defaults, the data_ptr() of a contiguous
        [N, height, width] int32 / uint32 CUDA tensor. With `rgba_ptr` (a [N, height, width, 4]
        uint8 tensor's data_ptr() with the default strides) the frames of render_views_device are
        written as well, from the same pass; rgba_ptr=None renders the IDs only."""
        n, args = self._view_args(composition, views)
        return self._stack(self._api.renderer_render_views_ids_device, "Renderer::render_views_ids_device", args, n, width, height,
                           (None if rgba_ptr is None else int(rgba_ptr), stride, view_stride, channels, clear_color),
                           (int(ids_device_ptr), ids_stride, ids_view_stride, min_coverage), timings)

    def render_batch_ids(self, comps, ids: np.ndarray, width: int, height: int, ids_stride: Optional[int] = None,
                         ids_frame_stride: Optional[int] = None, min_coverage: float = 0.0,
                         timings: bool = True) -> Optional[Timings]:
        """The ID frame (see render_ids) of every frame of render_batch, in one pass: frame c holds
        comps[c]'s own layer orders (or ID_NONE). Layout as for render_views_ids; chunked like
        render_batch."""
        n, args = self._batch_args(comps)
        s, fs = self._strides(width, height, ids_stride, ids_frame_stride)
        assert ids.dtype == np.uint32 and ids.flags["C_CONTIGUOUS"]
        assert n == 0 or ids.size * 4 >= (n - 1) * fs + (height - 1) * s + 4 * width
        return self._stack(self._api.renderer_render_batch_ids, "Renderer::render_batch_ids", args, n, width, height, None,
                           (ids.ctypes.data, s, fs, min_coverage), timings)

    def render_batch_ids_device(self, comps, ids_device_ptr: int, width: int, height: int, rgba_ptr: Optional[int] = None,
                                channels=RGBA, clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), stride: Optional[int] = None,
                                frame_stride: Optional[int] = None, ids_stride: Optional[int] = None,
                                ids_frame_stride: Optional[int] = None, min_coverage: float = 0.0,
                                timings: bool = True) -> Optional[Timings]:
        """render_batch_ids into device memory (a contiguous [N, height, width] int32 / uint32 CUDA
        tensor's data_ptr() with the defaults): the labels of a batch of scenes. With `rgba_ptr`
        the frames of render_batch_device are written as well, from the same pass; rgba_ptr=None
        renders the IDs only."""
        n, args = self._batch_args(comps)
        return self._stack(self._api.renderer_render_batch_ids_device, "Renderer::render_batch_ids_device", args, n, width, height,
                           (None if rgba_ptr is None else int(rgba_ptr), stride, frame_stride, channels, clear_color),
                           (int(ids_device_ptr), ids_stride, ids_frame_stride, min_coverage), timings)

    @staticmethod
    def _linear_host(buffer: np.ndarray, dtype, nbytes: int) -> None:
        assert buffer.dtype == dtype and buffer.flags["C_CONTIGUOUS"] and buffer.nbytes >= nbytes, \
            f"a contiguous {np.dtype(dtype).name} array of at least {nbytes} bytes"

    def render_linear(self, composition: Composition, buffer: np.ndarray, width: int, height: int, channels=RGBA,
                      clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), crop: Optional[Rect] = None, format: str = "f32",
                      stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """The frame's linear colour (see include/forma_b200.h: forma_renderer_render_linear): per
        pixel the painter's four values in channel order, before the sRGB encode, as float32
        (format "f32") or float16 ("f16"). `buffer`: a writable contiguous host array of that dtype,
        e.g. [height, width, 4]; `stride` in bytes (default bpp * width, bpp = 16 or 8). Only the
        crop's tile rectangle is written."""
        code, bpp, dtype = pixel_format(format)
        stride = width * bpp if stride is None else stride
        self._linear_host(buffer, dtype, height * stride)
        return self._frame(self._api.renderer_render_linear, "Renderer::render_linear", composition, buffer.ctypes.data_as(C.c_void_p),
                           width, height, stride, (channels, clear_color), crop, (code,), timings)

    def render_linear_device(self, composition: Composition, device_ptr: int, width: int, height: int, channels=RGBA,
                             clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), crop: Optional[Rect] = None, format: str = "f32",
                             stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """render_linear into device memory on the renderer's device: with the defaults, the
        data_ptr() of a contiguous [height, width, 4] float32 / float16 CUDA tensor."""
        code, bpp, _ = pixel_format(format)
        return self._frame(self._api.renderer_render_linear_device, "Renderer::render_linear_device", composition,
                           C.c_void_p(device_ptr), width, height, width * bpp if stride is None else stride, (channels, clear_color),
                           crop, (code,), timings)

    def render_views_linear(self, composition: Composition, views, buffer: np.ndarray, width: int, height: int, channels=RGBA,
                            clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), format: str = "f32", stride: Optional[int] = None,
                            view_stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """render_views as linear float frames (see render_linear): frame b at byte b * view_stride
        (default height * stride) of `buffer`, a writable contiguous host array of the format's
        dtype, e.g. [N, height, width, 4]. Chunked like render_views."""
        code, bpp, dtype = pixel_format(format)
        n, args = self._view_args(composition, views)
        stride, view_stride = self._strides(width, height, stride, view_stride, bpp)
        if n:
            self._linear_host(buffer, dtype, (n - 1) * view_stride + (height - 1) * stride + bpp * width)
        return self._stack(self._api.renderer_render_views_linear, "Renderer::render_views_linear", args, n, width, height,
                           (buffer.ctypes.data, stride, view_stride, channels, clear_color), None, timings, bpp, (code,))

    def render_views_linear_device(self, composition: Composition, views, device_ptr: int, width: int, height: int,
                                   channels=RGBA, clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), format: str = "f32",
                                   stride: Optional[int] = None, view_stride: Optional[int] = None,
                                   timings: bool = True) -> Optional[Timings]:
        """render_views_linear into device memory: with the defaults, the data_ptr() of a
        contiguous [N, height, width, 4] float32 / float16 CUDA tensor."""
        code, bpp, _ = pixel_format(format)
        n, args = self._view_args(composition, views)
        return self._stack(self._api.renderer_render_views_linear_device, "Renderer::render_views_linear_device", args, n, width,
                           height, (int(device_ptr), stride, view_stride, channels, clear_color), None, timings, bpp, (code,))

    def render_batch_linear(self, comps, buffer: np.ndarray, width: int, height: int, channels=RGBA,
                            clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), format: str = "f32", stride: Optional[int] = None,
                            frame_stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """render_batch as linear float frames (see render_linear); layout as for
        render_views_linear, chunked like render_batch."""
        code, bpp, dtype = pixel_format(format)
        n, args = self._batch_args(comps)
        stride, frame_stride = self._strides(width, height, stride, frame_stride, bpp)
        if n:
            self._linear_host(buffer, dtype, (n - 1) * frame_stride + (height - 1) * stride + bpp * width)
        return self._stack(self._api.renderer_render_batch_linear, "Renderer::render_batch_linear", args, n, width, height,
                           (buffer.ctypes.data, stride, frame_stride, channels, clear_color), None, timings, bpp, (code,))

    def render_batch_linear_device(self, comps, device_ptr: int, width: int, height: int, channels=RGBA,
                                   clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), format: str = "f32",
                                   stride: Optional[int] = None, frame_stride: Optional[int] = None,
                                   timings: bool = True) -> Optional[Timings]:
        """render_batch_linear into device memory: with the defaults, the data_ptr() of a
        contiguous [N, height, width, 4] float32 / float16 CUDA tensor."""
        code, bpp, _ = pixel_format(format)
        n, args = self._batch_args(comps)
        return self._stack(self._api.renderer_render_batch_linear_device, "Renderer::render_batch_linear_device", args, n, width,
                           height, (int(device_ptr), stride, frame_stride, channels, clear_color), None, timings, bpp, (code,))

    def render_over_device(self, composition: Composition, device_ptr: int, width: int, height: int, channels=RGBA,
                           crop: Optional[Rect] = None, format: str = "srgb8", stride: Optional[int] = None,
                           timings: bool = True) -> Optional[Timings]:
        """Draws the composition over the pixels already in device memory (see
        include/forma_b200.h: forma_renderer_render_over_device): each pixel's own value, decoded,
        is its clear colour, so the result is render_device's (format "srgb8") or
        render_linear_device's ("f16", "f32") with that clear colour, pixel by pixel. With the
        defaults, the data_ptr() of a contiguous [height, width, 4] uint8 / float16 / float32 CUDA
        tensor. `channels`: a permutation of R, G, B, A (for "srgb8" with A last). Only the crop's
        tile rectangle is read and written."""
        code, bpp, _ = over_format(format)
        return self._frame(self._api.renderer_render_over_device, "Renderer::render_over_device", composition, C.c_void_p(device_ptr),
                           width, height, width * bpp if stride is None else stride, (channels, None), crop, (code,), timings)

    def render_views_over_device(self, composition: Composition, views, device_ptr: int, width: int, height: int, channels=RGBA,
                                 format: str = "srgb8", stride: Optional[int] = None, view_stride: Optional[int] = None,
                                 timings: bool = True) -> Optional[Timings]:
        """render_views over the frames already in device memory (see render_over_device): with the
        defaults, the data_ptr() of a contiguous [N, height, width, 4] uint8 / float16 / float32 CUDA
        tensor. Chunked like render_views."""
        code, bpp, _ = over_format(format)
        n, args = self._view_args(composition, views)
        return self._stack(self._api.renderer_render_views_over_device, "Renderer::render_views_over_device", args, n, width, height,
                           (int(device_ptr), stride, view_stride, channels, None), None, timings, bpp, (code,))

    def render_batch_over_device(self, comps, device_ptr: int, width: int, height: int, channels=RGBA, format: str = "srgb8",
                                 stride: Optional[int] = None, frame_stride: Optional[int] = None,
                                 timings: bool = True) -> Optional[Timings]:
        """render_batch over the frames already in device memory (see render_over_device): frame c
        of comps over frame c of the [N, height, width, 4] tensor. Chunked like render_batch."""
        code, bpp, _ = over_format(format)
        n, args = self._batch_args(comps)
        return self._stack(self._api.renderer_render_batch_over_device, "Renderer::render_batch_over_device", args, n, width, height,
                           (int(device_ptr), stride, frame_stride, channels, None), None, timings, bpp, (code,))

    @staticmethod
    def _mask_layout(width, height, n_orders, format, stride, plane_stride):
        """(FORMA_MASK_* code, bpp, dtype, stride, plane_stride) with the defaults of a contiguous
        [K, height, width] array: stride = bpp * width, plane_stride = height * stride."""
        code, bpp, dtype = mask_format(format)
        stride = width * bpp if stride is None else stride
        return code, bpp, dtype, stride, height * stride if plane_stride is None else plane_stride

    def render_masks(self, composition: Composition, masks: np.ndarray, width: int, height: int, first_order: int,
                     n_orders: Optional[int] = None, crop: Optional[Rect] = None, stride: Optional[int] = None,
                     plane_stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """Layer coverage masks into a host array (see include/forma_b200.h: forma_renderer_render_masks):
        plane k holds the coverage (x clip mask) of layer order first_order + k, amodal, whatever
        the layers above it. `masks`: a writable contiguous float32 ("f32", exact) or uint8 ("u8",
        the alpha byte of sRGB8 frames) array, by default [K, height, width] with K = n_orders
        (default masks.shape[0]); strides in bytes. Only the crop's tile rectangle of each plane
        is written."""
        fmt = {np.dtype(np.float32): "f32", np.dtype(np.uint8): "u8"}.get(masks.dtype)
        assert fmt is not None and masks.flags["C_CONTIGUOUS"], "a contiguous float32 or uint8 array"
        k = masks.shape[0] if n_orders is None else n_orders
        code, bpp, _, stride, plane_stride = self._mask_layout(width, height, k, fmt, stride, plane_stride)
        assert k == 0 or masks.nbytes >= (k - 1) * plane_stride + (height - 1) * stride + bpp * width
        m = _CMasks(masks.ctypes.data, first_order, k, code, stride, plane_stride)
        _, _, rect = self._common(RGBA, Color(), crop)
        t = _CTimings() if timings else None
        st = self._api.renderer_render_masks(self._h, composition._h, C.byref(m), width, height,
                                             C.byref(rect) if rect is not None else None, C.byref(t) if t is not None else None)
        self._api.check(st, "Renderer::render_masks")
        return _timings(t)

    def render_masks_device(self, composition: Composition, masks_ptr: int, width: int, height: int, first_order: int,
                            n_orders: int, format: str = "f32", crop: Optional[Rect] = None, stride: Optional[int] = None,
                            plane_stride: Optional[int] = None, rgba_ptr: Optional[int] = None, channels=RGBA,
                            clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), rgba_stride: Optional[int] = None,
                            timings: bool = True) -> Optional[Timings]:
        """render_masks into device memory: with the defaults, the data_ptr() of a contiguous
        [n_orders, height, width] float32 ("f32") or uint8 ("u8") CUDA tensor. With `rgba_ptr` the
        frame of render_device (no layer cache; default stride 4 * width) is written as well, from
        the same pass."""
        code, _, _, stride, plane_stride = self._mask_layout(width, height, n_orders, format, stride, plane_stride)
        m = _CMasks(int(masks_ptr), first_order, n_orders, code, stride, plane_stride)
        ch, cc, rect = self._common(channels, clear_color, crop)
        t = _CTimings() if timings else None
        st = self._api.renderer_render_masks_device(self._h, composition._h, C.byref(m), width, height,
                                                    C.byref(rect) if rect is not None else None,
                                                    None if rgba_ptr is None else C.c_void_p(int(rgba_ptr)),
                                                    4 * width if rgba_stride is None else rgba_stride, ch, cc,
                                                    C.byref(t) if t is not None else None)
        self._api.check(st, "Renderer::render_masks_device")
        return _timings(t)

    def _stack_masks(self, fn, what, first_args, n, masks_ptr, width, height, first_order, n_orders, format, stride, plane_stride, rgba_ptr,
                     channels, clear_color, rgba_stride, frame_stride, timings, chunk=None):
        """Calls `fn`, the mask entry point of views or batches, on chunks of at most
        max_views(height) frames (see _stack)."""
        code, _, _, stride, plane_stride = self._mask_layout(width, height, n_orders, format, stride, plane_stride)
        rgba_stride, frame_stride = self._strides(width, height, rgba_stride, frame_stride)
        ch, cc, _ = self._common(channels, clear_color, None)
        chunk = max(min(self.max_views(height), chunk or self.max_views(height)), 1)
        t = None
        for first in range(0, max(n, 1), chunk):
            m = _CMasks(int(masks_ptr) + first * n_orders * plane_stride, first_order, n_orders, code, stride, plane_stride)
            rgba = None if rgba_ptr is None else C.c_void_p(int(rgba_ptr) + first * frame_stride)
            t = _CTimings() if timings else None
            st = fn(self._h, *first_args(first, min(chunk, n - first)), C.byref(m), width, height, rgba, rgba_stride, frame_stride, ch, cc,
                    C.byref(t) if t is not None else None)
            self._api.check(st, what)
        return _timings(t)

    def render_views_masks_device(self, composition: Composition, views, masks_ptr: int, width: int, height: int, first_order: int,
                                  n_orders: int, format: str = "f32", stride: Optional[int] = None,
                                  plane_stride: Optional[int] = None, rgba_ptr: Optional[int] = None, channels=RGBA,
                                  clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), rgba_stride: Optional[int] = None,
                                  view_stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """The masks (see render_masks) of every view of render_views_device, in one pass: with the
        defaults, the data_ptr() of a contiguous [N, n_orders, height, width] CUDA tensor; every
        view holds the same orders. With `rgba_ptr` the frames of render_views_device are written
        as well. Chunked like render_views."""
        n, args = self._view_args(composition, views)
        return self._stack_masks(self._api.renderer_render_views_masks_device, "Renderer::render_views_masks_device", args, n, masks_ptr, width,
                                 height, first_order, n_orders, format, stride, plane_stride, rgba_ptr, channels, clear_color,
                                 rgba_stride, view_stride, timings)

    def render_batch_masks_device(self, comps, masks_ptr: int, width: int, height: int, first_order: int, n_orders: int,
                                  format: str = "f32", stride: Optional[int] = None, plane_stride: Optional[int] = None,
                                  rgba_ptr: Optional[int] = None, channels=RGBA, clear_color: Color = Color(1.0, 1.0, 1.0, 1.0),
                                  rgba_stride: Optional[int] = None, frame_stride: Optional[int] = None,
                                  timings: bool = True) -> Optional[Timings]:
        """The masks (see render_masks) of every frame of render_batch_device, in one pass: frame c's
        planes hold comps[c]'s own orders [first_order, first_order + n_orders). Layout as for
        render_views_masks_device; chunked like render_batch."""
        n, args = self._batch_args(comps)
        return self._stack_masks(self._api.renderer_render_batch_masks_device, "Renderer::render_batch_masks_device", args, n, masks_ptr, width,
                                 height, first_order, n_orders, format, stride, plane_stride, rgba_ptr, channels, clear_color,
                                 rgba_stride, frame_stride, timings)

    def render_stats(self, composition: Composition, width: int, height: int, first_order: int, n_orders: int,
                     min_coverage: float = 0.0, crop: Optional[Rect] = None, out: Optional[np.ndarray] = None) -> np.ndarray:
        """Layer statistics into a host array (see include/forma_b200.h: forma_renderer_render_stats):
        per order o of [first_order, first_order + n_orders) its amodal area (sum of mask values x 2^18),
        the pixels its mask exceeds min_coverage on and their box, and the pixels its ID owns and
        their box. Returns the [n_orders] STATS_DTYPE array (`out`, if given)."""
        if out is None:
            out = np.zeros(n_orders, STATS_DTYPE)
        assert out.dtype == STATS_DTYPE and out.flags["C_CONTIGUOUS"] and out.size >= n_orders
        s = _CStats(out.ctypes.data, first_order, n_orders, min_coverage)
        _, _, rect = self._common(RGBA, Color(), crop)
        st = self._api.renderer_render_stats(self._h, composition._h, C.byref(s), width, height,
                                             C.byref(rect) if rect is not None else None, None)
        self._api.check(st, "Renderer::render_stats")
        return out

    def render_stats_device(self, composition: Composition, stats_ptr: int, width: int, height: int, first_order: int,
                            n_orders: int, min_coverage: float = 0.0, crop: Optional[Rect] = None, rgba_ptr: Optional[int] = None,
                            channels=RGBA, clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), rgba_stride: Optional[int] = None,
                            timings: bool = True) -> Optional[Timings]:
        """render_stats into device memory: the data_ptr() of a contiguous [n_orders, 12] int32 CUDA
        tensor (split_stats reads its fields). With `rgba_ptr` the frame of render_device (no layer
        cache; default stride 4 * width) is written as well, from the same pass."""
        s = _CStats(int(stats_ptr), first_order, n_orders, min_coverage)
        ch, cc, rect = self._common(channels, clear_color, crop)
        t = _CTimings() if timings else None
        st = self._api.renderer_render_stats_device(self._h, composition._h, C.byref(s), width, height,
                                                    C.byref(rect) if rect is not None else None,
                                                    None if rgba_ptr is None else C.c_void_p(int(rgba_ptr)),
                                                    4 * width if rgba_stride is None else rgba_stride, ch, cc,
                                                    C.byref(t) if t is not None else None)
        self._api.check(st, "Renderer::render_stats_device")
        return _timings(t)

    def _stack_stats(self, fn, what, first_args, n, stats_ptr, width, height, first_order, n_orders, min_coverage, rgba_ptr, channels,
                     clear_color, rgba_stride, frame_stride, timings, chunk=None):
        """Calls `fn`, the statistics entry point of views or batches, on chunks of at most
        max_views(height) frames (see _stack)."""
        rgba_stride, frame_stride = self._strides(width, height, rgba_stride, frame_stride)
        ch, cc, _ = self._common(channels, clear_color, None)
        chunk = max(min(self.max_views(height), chunk or self.max_views(height)), 1)
        t = None
        for first in range(0, max(n, 1), chunk):
            s = _CStats(int(stats_ptr) + first * n_orders * STATS_DTYPE.itemsize, first_order, n_orders, min_coverage)
            rgba = None if rgba_ptr is None else C.c_void_p(int(rgba_ptr) + first * frame_stride)
            t = _CTimings() if timings else None
            st = fn(self._h, *first_args(first, min(chunk, n - first)), C.byref(s), width, height, rgba, rgba_stride, frame_stride, ch, cc,
                    C.byref(t) if t is not None else None)
            self._api.check(st, what)
        return _timings(t)

    def render_views_stats_device(self, composition: Composition, views, stats_ptr: int, width: int, height: int, first_order: int,
                                  n_orders: int, min_coverage: float = 0.0, rgba_ptr: Optional[int] = None, channels=RGBA,
                                  clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), rgba_stride: Optional[int] = None,
                                  view_stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """The statistics (see render_stats) of every view of render_views_device, in one pass: the
        data_ptr() of a contiguous [N, n_orders, 12] int32 CUDA tensor; every view reports the same
        orders. With `rgba_ptr` the frames of render_views_device are written as well. Chunked like
        render_views."""
        n, args = self._view_args(composition, views)
        return self._stack_stats(self._api.renderer_render_views_stats_device, "Renderer::render_views_stats_device", args, n, stats_ptr,
                                 width, height, first_order, n_orders, min_coverage, rgba_ptr, channels, clear_color, rgba_stride,
                                 view_stride, timings)

    def render_batch_stats_device(self, comps, stats_ptr: int, width: int, height: int, first_order: int, n_orders: int,
                                  min_coverage: float = 0.0, rgba_ptr: Optional[int] = None, channels=RGBA,
                                  clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), rgba_stride: Optional[int] = None,
                                  frame_stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """The statistics (see render_stats) of every frame of render_batch_device, in one pass: frame
        c's records are comps[c]'s own orders [first_order, first_order + n_orders). Layout as for
        render_views_stats_device; chunked like render_batch."""
        n, args = self._batch_args(comps)
        return self._stack_stats(self._api.renderer_render_batch_stats_device, "Renderer::render_batch_stats_device", args, n, stats_ptr,
                                 width, height, first_order, n_orders, min_coverage, rgba_ptr, channels, clear_color, rgba_stride,
                                 frame_stride, timings)

    def render_poses(self, composition: Composition, poses: Poses, buffer: np.ndarray, width: int, height: int, channels=RGBA,
                     clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), stride: Optional[int] = None,
                     view_stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """One frame per pose (see Poses and include/forma_b200.h: forma_renderer_render_poses): frame b
        is the composition with the window's layers set to pose b, which the call itself leaves
        unchanged. Layout as for render_views; chunked like render_views."""
        n, args = self._pose_args(composition, poses)
        stride, view_stride = self._strides(width, height, stride, view_stride)
        assert buffer.dtype == np.uint8 and buffer.flags["C_CONTIGUOUS"]
        assert n == 0 or buffer.size >= (n - 1) * view_stride + (height - 1) * stride + 4 * width
        return self._stack(self._api.renderer_render_poses, "Renderer::render_poses", args, n, width, height,
                           (buffer.ctypes.data, stride, view_stride, channels, clear_color), None, timings)

    def render_poses_device(self, composition: Composition, poses: Poses, device_ptr: int, width: int, height: int, channels=RGBA,
                            clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), stride: Optional[int] = None,
                            view_stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """render_poses into device memory: with the defaults, the data_ptr() of a contiguous
        [N, height, width, 4] uint8 CUDA tensor."""
        n, args = self._pose_args(composition, poses)
        return self._stack(self._api.renderer_render_poses_device, "Renderer::render_poses_device", args, n, width, height,
                           (int(device_ptr), stride, view_stride, channels, clear_color), None, timings)

    def render_poses_ids(self, composition: Composition, poses: Poses, ids: np.ndarray, width: int, height: int,
                         ids_stride: Optional[int] = None, ids_view_stride: Optional[int] = None, min_coverage: float = 0.0,
                         timings: bool = True) -> Optional[Timings]:
        """The ID frame (see render_ids) of every pose, in one pass; layout as for render_views_ids."""
        n, args = self._pose_args(composition, poses)
        s, fs = self._strides(width, height, ids_stride, ids_view_stride)
        assert ids.dtype == np.uint32 and ids.flags["C_CONTIGUOUS"]
        assert n == 0 or ids.size * 4 >= (n - 1) * fs + (height - 1) * s + 4 * width
        return self._stack(self._api.renderer_render_poses_ids, "Renderer::render_poses_ids", args, n, width, height, None,
                           (ids.ctypes.data, s, fs, min_coverage), timings)

    def render_poses_ids_device(self, composition: Composition, poses: Poses, ids_device_ptr: int, width: int, height: int,
                                rgba_ptr: Optional[int] = None, channels=RGBA, clear_color: Color = Color(1.0, 1.0, 1.0, 1.0),
                                stride: Optional[int] = None, view_stride: Optional[int] = None, ids_stride: Optional[int] = None,
                                ids_view_stride: Optional[int] = None, min_coverage: float = 0.0,
                                timings: bool = True) -> Optional[Timings]:
        """render_poses_ids into device memory, with the frames of render_poses_device as well when
        `rgba_ptr` is given; layout as for render_views_ids_device."""
        n, args = self._pose_args(composition, poses)
        return self._stack(self._api.renderer_render_poses_ids_device, "Renderer::render_poses_ids_device", args, n, width, height,
                           (None if rgba_ptr is None else int(rgba_ptr), stride, view_stride, channels, clear_color),
                           (int(ids_device_ptr), ids_stride, ids_view_stride, min_coverage), timings)

    def render_poses_masks_device(self, composition: Composition, poses: Poses, masks_ptr: int, width: int, height: int,
                                  first_order: int, n_orders: int, format: str = "f32", stride: Optional[int] = None,
                                  plane_stride: Optional[int] = None, rgba_ptr: Optional[int] = None, channels=RGBA,
                                  clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), rgba_stride: Optional[int] = None,
                                  view_stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """The masks (see render_masks) of every pose, in one pass; layout as for
        render_views_masks_device. The mask window and the pose window are independent."""
        n, args = self._pose_args(composition, poses)
        return self._stack_masks(self._api.renderer_render_poses_masks_device, "Renderer::render_poses_masks_device", args, n, masks_ptr,
                                 width, height, first_order, n_orders, format, stride, plane_stride, rgba_ptr, channels, clear_color,
                                 rgba_stride, view_stride, timings)

    def render_poses_stats_device(self, composition: Composition, poses: Poses, stats_ptr: int, width: int, height: int,
                                  first_order: int, n_orders: int, min_coverage: float = 0.0, rgba_ptr: Optional[int] = None,
                                  channels=RGBA, clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), rgba_stride: Optional[int] = None,
                                  view_stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """The statistics (see render_stats) of every pose, in one pass; layout as for
        render_views_stats_device. The statistics window and the pose window are independent."""
        n, args = self._pose_args(composition, poses)
        return self._stack_stats(self._api.renderer_render_poses_stats_device, "Renderer::render_poses_stats_device", args, n, stats_ptr,
                                 width, height, first_order, n_orders, min_coverage, rgba_ptr, channels, clear_color, rgba_stride,
                                 view_stride, timings)

    def render_instances_device(self, composition: Composition, instances: Instances, device_ptr: int, width: int, height: int,
                                channels=RGBA, clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), stride: Optional[int] = None,
                                view_stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """One frame per row of the instance tables (see Instances and include/forma_b200.h:
        forma_renderer_render_instances_device): frame b draws its slots' copies of the composition's
        layers, which the call leaves unchanged. Layout as for render_views_device: with the
        defaults, the data_ptr() of a contiguous [N, height, width, 4] uint8 CUDA tensor. Chunked
        at max_views(height) frames and at 2^21 // M frames."""
        n, args, chunk = self._instance_args(composition, instances)
        return self._stack(self._api.renderer_render_instances_device, "Renderer::render_instances_device", args, n, width, height,
                           (int(device_ptr), stride, view_stride, channels, clear_color), None, timings, chunk=chunk)

    def render_instances_ids_device(self, composition: Composition, instances: Instances, ids_device_ptr: int, width: int,
                                    height: int, rgba_ptr: Optional[int] = None, channels=RGBA,
                                    clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), stride: Optional[int] = None,
                                    view_stride: Optional[int] = None, ids_stride: Optional[int] = None,
                                    ids_view_stride: Optional[int] = None, min_coverage: float = 0.0,
                                    timings: bool = True) -> Optional[Timings]:
        """The ID frame of every instance frame: per pixel the slot m of the topmost instance
        painted there, or ID_NONE (an instance-segmentation label); with `rgba_ptr` the frames of
        render_instances_device as well. Layout as for render_views_ids_device."""
        n, args, chunk = self._instance_args(composition, instances)
        return self._stack(self._api.renderer_render_instances_ids_device, "Renderer::render_instances_ids_device", args, n, width,
                           height, (None if rgba_ptr is None else int(rgba_ptr), stride, view_stride, channels, clear_color),
                           (int(ids_device_ptr), ids_stride, ids_view_stride, min_coverage), timings, chunk=chunk)

    def render_instances_masks_device(self, composition: Composition, instances: Instances, masks_ptr: int, width: int, height: int,
                                      first_order: int, n_orders: int, format: str = "f32", stride: Optional[int] = None,
                                      plane_stride: Optional[int] = None, rgba_ptr: Optional[int] = None, channels=RGBA,
                                      clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), rgba_stride: Optional[int] = None,
                                      view_stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """The masks (see render_masks) of every instance frame, plane k holding slot
        first_order + k; layout as for render_views_masks_device."""
        n, args, chunk = self._instance_args(composition, instances)
        return self._stack_masks(self._api.renderer_render_instances_masks_device, "Renderer::render_instances_masks_device", args, n,
                                 masks_ptr, width, height, first_order, n_orders, format, stride, plane_stride, rgba_ptr, channels,
                                 clear_color, rgba_stride, view_stride, timings, chunk=chunk)

    def render_instances_stats_device(self, composition: Composition, instances: Instances, stats_ptr: int, width: int, height: int,
                                      first_order: int, n_orders: int, min_coverage: float = 0.0, rgba_ptr: Optional[int] = None,
                                      channels=RGBA, clear_color: Color = Color(1.0, 1.0, 1.0, 1.0),
                                      rgba_stride: Optional[int] = None, view_stride: Optional[int] = None,
                                      timings: bool = True) -> Optional[Timings]:
        """The statistics (see render_stats) of every instance frame, record k of a frame for slot
        first_order + k (per-instance areas and boxes); layout as for render_views_stats_device."""
        n, args, chunk = self._instance_args(composition, instances)
        return self._stack_stats(self._api.renderer_render_instances_stats_device, "Renderer::render_instances_stats_device", args, n,
                                 stats_ptr, width, height, first_order, n_orders, min_coverage, rgba_ptr, channels, clear_color,
                                 rgba_stride, view_stride, timings, chunk=chunk)

    def render_poses_linear(self, composition: Composition, poses: Poses, buffer: np.ndarray, width: int, height: int, channels=RGBA,
                            clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), format: str = "f32", stride: Optional[int] = None,
                            view_stride: Optional[int] = None, timings: bool = True) -> Optional[Timings]:
        """render_poses as linear float frames (see render_linear); layout as for
        render_views_linear, chunked like render_poses."""
        code, bpp, dtype = pixel_format(format)
        n, args = self._pose_args(composition, poses)
        stride, view_stride = self._strides(width, height, stride, view_stride, bpp)
        if n:
            self._linear_host(buffer, dtype, (n - 1) * view_stride + (height - 1) * stride + bpp * width)
        return self._stack(self._api.renderer_render_poses_linear, "Renderer::render_poses_linear", args, n, width, height,
                           (buffer.ctypes.data, stride, view_stride, channels, clear_color), None, timings, bpp, (code,))

    def render_poses_linear_device(self, composition: Composition, poses: Poses, device_ptr: int, width: int, height: int,
                                   channels=RGBA, clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), format: str = "f32",
                                   stride: Optional[int] = None, view_stride: Optional[int] = None,
                                   timings: bool = True) -> Optional[Timings]:
        """render_poses_linear into device memory: with the defaults, the data_ptr() of a
        contiguous [N, height, width, 4] float32 / float16 CUDA tensor."""
        code, bpp, _ = pixel_format(format)
        n, args = self._pose_args(composition, poses)
        return self._stack(self._api.renderer_render_poses_linear_device, "Renderer::render_poses_linear_device", args, n, width,
                           height, (int(device_ptr), stride, view_stride, channels, clear_color), None, timings, bpp, (code,))

    def render_poses_over_device(self, composition: Composition, poses: Poses, device_ptr: int, width: int, height: int, channels=RGBA,
                                 format: str = "srgb8", stride: Optional[int] = None, view_stride: Optional[int] = None,
                                 timings: bool = True) -> Optional[Timings]:
        """render_poses over the frames already in device memory (see render_over_device): pose b
        over frame b of the [N, height, width, 4] tensor. Chunked like render_poses."""
        code, bpp, _ = over_format(format)
        n, args = self._pose_args(composition, poses)
        return self._stack(self._api.renderer_render_poses_over_device, "Renderer::render_poses_over_device", args, n, width, height,
                           (int(device_ptr), stride, view_stride, channels, None), None, timings, bpp, (code,))

    def launch_count(self) -> int:
        return int(self._api.renderer_launch_count(self._h))

    STAGES = ("upload", "line_setup", "rasterize", "sort", "paint_tables", "paint_kernel", "d2h", "total")

    def stage_times(self) -> dict:
        """Device-timeline ms of the last render, by stage."""
        out = (C.c_double * 8)()
        self._api.renderer_stage_times(self._h, out)
        return dict(zip(self.STAGES, list(out)))

    def kernel_times(self) -> dict:
        """CUDA-event ms and launch counts of single kernels in the last render."""
        ms, n = (C.c_double * 4)(), (C.c_uint32 * 4)()
        self._api.renderer_kernel_times(self._h, ms, n)
        names = ("radix_downsweep", "radix_upsweep_scan", "paint")
        return {k: {"ms": float(ms[i]), "launches": int(n[i])} for i, k in enumerate(names)}

    def counters(self) -> dict:
        out = (C.c_uint64 * 8)()
        self._api.renderer_counters(self._h, out)
        return dict(zip(("launches", "h2d_bytes", "d2h_bytes", "segments", "cells", "entries", "written_tiles",
                         "tables_mode"),  # tables_mode: 0 counts read back, 1 sync-free, 2 sync-free attempt redone
                        [int(v) for v in out]))

    def host_slices(self) -> list:
        """Device-timeline ms of every slice of the last host frame ([] = rendered as one piece)."""
        ms = (C.c_double * 16)()
        n = int(self._api.renderer_host_slices(self._h, ms, None))
        return [float(ms[i]) for i in range(n)]

    def host_slice_stages(self) -> list:
        """Stage times of every slice of the last host frame (dicts keyed like stage_times())."""
        ms, st = (C.c_double * 16)(), (C.c_double * 128)()
        n = int(self._api.renderer_host_slices(self._h, ms, st))
        return [dict(zip(self.STAGES, [float(st[8 * i + k]) for k in range(8)])) for i in range(n)]

    def row_costs(self) -> np.ndarray:
        """Per-tile-row cost of the last render (forma_renderer_row_costs)."""
        n = int(self._api.renderer_row_costs(self._h, 0, None))
        out = np.zeros(n, np.uint64)
        if n:
            self._api.renderer_row_costs(self._h, n, out.ctypes.data_as(_u64p))
        return out

    def set_stream(self, cuda_stream: int) -> None:
        self._api.renderer_set_stream(self._h, C.c_void_p(cuda_stream))

    # stage-level access ----------------------------------------------------
    def lines(self):
        n = int(self._api.renderer_lines(self._h, 0, None, None, None, None, None, None, None, None, None, None))
        orders = np.zeros(n, np.uint32)
        lengths = np.zeros(n, np.uint32)
        fl = [np.zeros(n, np.float32) for _ in range(8)]
        self._api.renderer_lines(self._h, n, orders.ctypes.data_as(_u32p), *[a.ctypes.data_as(_fp) for a in fl],
                                 lengths.ctypes.data_as(_u32p))
        names = ["x0", "y0", "dx", "dy", "a", "b", "c", "d"]
        out = {"orders": orders, "lengths": lengths}
        out.update(dict(zip(names, fl)))
        return out

    def segments(self) -> np.ndarray:
        n = int(self._api.renderer_segments(self._h, 0, None))
        out = np.zeros(n, np.uint64)
        self._api.renderer_segments(self._h, n, out.ctypes.data_as(_u64p))
        return out

    def rasterize_only(self, composition: Composition, width: int, height: int) -> np.ndarray:
        n = int(self._api.renderer_rasterize_only(self._h, composition._h, width, height, 0, None))
        out = np.zeros(n, np.uint64)
        self._api.renderer_rasterize_only(self._h, composition._h, width, height, n, out.ctypes.data_as(_u64p))
        return out

    def sort_u64(self, keys: np.ndarray) -> np.ndarray:
        out = np.ascontiguousarray(keys, dtype=np.uint64).copy()
        self._api.check(self._api.renderer_sort_u64(self._h, out.ctypes.data_as(_u64p), out.size), "sort_u64")
        return out

    def sort_pairs(self, keys: np.ndarray, vals: np.ndarray, layout: int = 0, mode: int = 0, count: Optional[int] = None,
                   cap: int = 0):
        """(keys, vals) sorted by the single-sweep pair passes (forma_renderer_sort_pairs).
        mode bit 0: `count` (default: len(keys)) goes to the kernels in device memory with `cap`
        as its bound; bit 1: the digit histogram is counted before the sort and passed in."""
        k = np.ascontiguousarray(keys, dtype=np.uint64).copy()
        v = np.ascontiguousarray(vals, dtype=np.uint32).copy()
        count = k.size if count is None else int(count)
        held = min(count, cap) if mode & 1 else count
        if k.size != held or v.size != held:
            raise ValueError(f"sort_pairs: {k.size} keys and {v.size} values for {held} elements")
        self._api.check(self._api.renderer_sort_pairs(self._h, layout, mode, k.ctypes.data_as(_u64p), v.ctypes.data_as(_u32p),
                                                      count, cap), "sort_pairs")
        return k, v

    def sort_bounds(self) -> dict:
        """The field bounds and bit count of the last frame's segment sort plan."""
        out = (C.c_uint64 * 4)()
        self._api.renderer_sort_bounds(self._h, out)
        return dict(zip(("layer", "tile_x", "tile_y", "total_bits"), [int(x) for x in out]))

    SORT_COUNT_SOURCES = ("none", "speculative_emit", "emit", "upsweep")

    def sort_mode(self) -> int:
        """How the last frame's sort learnt the segment count (forma_renderer_sort_mode): 0 read
        back, 1 checked on the device (option sync_free_sort), 2 attempted as 1 and redone as 0."""
        return int(self._api.renderer_sort_mode(self._h))

    def sort_counts(self, keep: int = -1) -> dict:
        """The last frame's segment-sort tile counts (forma_renderer_sort_counts): where pass 0's
        came from, and the kept counts as a [passes, tiles, 256] array (empty unless keep was on
        for that frame). keep: 1 / 0 turns keeping on / off for the following frames."""
        info = (C.c_uint32 * 3)()
        words = int(self._api.renderer_sort_counts(self._h, keep, info, None, 0))
        out = np.zeros(words, np.uint32)
        if words:
            got = int(self._api.renderer_sort_counts(self._h, -1, info, out.ctypes.data_as(_u32p), words))
            self._api.check(0 if got == words else -1, "sort_counts")
        return {"source": self.SORT_COUNT_SOURCES[info[0]], "passes": int(info[1]), "tiles": int(info[2]),
                "counts": out.reshape(int(info[1]), int(info[2]), 256)}

    def __del__(self):
        try:
            self._api.renderer_free(self._h)
        except Exception:
            pass


class MultiRenderer:
    """One renderer over several GPUs of the box (forma_renderer_multi_*): `render` /
    `render_device` have Renderer's arguments minus the layer cache; the frame is split into
    cost-balanced bands of tile rows, one per device."""

    def __init__(self, api: Api, devices: Sequence[int]):
        self._api = api
        arr = (C.c_int * len(devices))(*devices)
        self._h = api.renderer_multi_new(arr, len(devices))
        if not self._h:
            raise FormaError(f"MultiRenderer::new failed: {api.last_error().decode()}")
        self.n = int(api.renderer_multi_device_count(self._h))

    def _call(self, fn, what, composition, ptr, width, height, channels, clear_color, crop, stride):
        stride = width * 4 if stride is None else stride
        ch = (C.c_uint32 * 4)(*channels)
        cc = (C.c_float * 4)(clear_color.r, clear_color.g, clear_color.b, clear_color.a)
        rect = _CRect(crop.horizontal[0], crop.horizontal[1], crop.vertical[0], crop.vertical[1]) if crop is not None else None
        t = _CTimings()
        st = fn(self._h, composition._h, ptr, width, stride, height, ch, cc, C.byref(rect) if rect is not None else None, C.byref(t))
        self._api.check(st, what)
        return _timings(t)

    def render(self, composition: "Composition", buffer: np.ndarray, width: int, height: int, channels=RGBA,
               clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), crop: Optional[Rect] = None, stride: Optional[int] = None) -> Timings:
        s = width * 4 if stride is None else stride
        assert buffer.dtype == np.uint8 and buffer.flags["C_CONTIGUOUS"] and buffer.size >= height * s
        return self._call(self._api.renderer_multi_render, "MultiRenderer::render", composition,
                          buffer.ctypes.data_as(C.c_void_p), width, height, channels, clear_color, crop, stride)

    def render_device(self, composition: "Composition", device_ptr: int, width: int, height: int, channels=RGBA,
                      clear_color: Color = Color(1.0, 1.0, 1.0, 1.0), crop: Optional[Rect] = None,
                      stride: Optional[int] = None) -> Timings:
        return self._call(self._api.renderer_multi_render_device, "MultiRenderer::render_device", composition,
                          C.c_void_p(device_ptr), width, height, channels, clear_color, crop, stride)

    def bands(self):
        """(tile-row boundaries of the next frame's bands, ms of every band in the last frame)."""
        b = (C.c_uint32 * (self.n + 1))()
        ms = (C.c_double * self.n)()
        self._api.renderer_multi_bands(self._h, b, ms)
        return list(b), list(ms)

    def __del__(self):
        try:
            self._api.renderer_multi_free(self._h)
        except Exception:
            pass


# ---------------------------------------------------------------------------
# PixelSegment bit layout helpers (forma/src/cpu/pixel_segment.rs:100-138)
# ---------------------------------------------------------------------------


def unpack_segments(segs: np.ndarray):
    s = segs.astype(np.uint64)
    cover = ((s & np.uint64(0x3F)).astype(np.int64) ^ 0x20) - 0x20
    dam = ((s >> np.uint64(6)) & np.uint64(0x3F)).astype(np.int64)
    return {
        "tile_y": ((s >> np.uint64(53)) & np.uint64(0x7FF)).astype(np.int64) - 1,
        "tile_x": ((s >> np.uint64(41)) & np.uint64(0xFFF)).astype(np.int64) - 1,
        "layer_id": ((s >> np.uint64(20)) & np.uint64(0x1FFFFF)).astype(np.int64),
        "local_x": ((s >> np.uint64(16)) & np.uint64(0xF)).astype(np.int64),
        "local_y": ((s >> np.uint64(12)) & np.uint64(0xF)).astype(np.int64),
        "double_area": dam * cover,
        "cover": cover,
    }
