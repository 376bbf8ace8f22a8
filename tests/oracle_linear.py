"""The oracle's linear float frames (oracle/forma_oracle_linear.cpp, libforma_oracle_linear.so):
bound into the oracle's Api as `renderer_render_linear`, so that `Renderer.render_linear` of the
oracle binding renders the f32 frame of an oracle composition, plus `encode`, compute_srgb's
encode of such a frame into sRGB8 bytes."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import scenes
from forma_b200.binding import Color, Fill, Func, GradientBuilder, Point, Props, Style

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle")
LIB = os.path.join(ORACLE, "libforma_oracle_linear.so")
_lib = None


def _load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            subprocess.check_call(["make", "-C", ORACLE, "-f", "linear.mk"])
        _lib = C.CDLL(LIB)
        _lib.fo_linear_to_srgb8.restype = None
        _lib.fo_linear_to_srgb8.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint32), C.c_void_p,
                                            C.c_uint64]
    return _lib


def attach(oracle_api):
    if not hasattr(oracle_api, "renderer_render_linear"):
        oracle_api.attach(_load(), ("renderer_render_linear",))
    return oracle_api


HDR_W, HDR_H = 96, 64
HDR_CLEAR = Color(2.0, -0.5, 0.25, 1.0)
HDR_SOLID = Color(3.0, 0.5, -1.0, 1.0)


def hdr_scene(api, comp):
    """Colours outside [0, 1] in an HDR_W x HDR_H frame: an opaque solid HDR_SOLID over columns
    0 ... 31 (whole tiles, folded to that colour), a circle on the right filled with a linear
    gradient from (4, -2, 0.5, 1) to (-1, 8, 2, 0.5); the rest of the frame is clear."""
    comp.get_mut_or_insert_default(0).insert(scenes.custom_square(api, 0.0, 0.0, 32.0, 64.0)).set_props(
        Props(func=Func.Draw(Style(fill=Fill.Solid(HDR_SOLID)))))
    gb = GradientBuilder(Point(40.0, 0.0), Point(90.0, 0.0))
    gb.color(Color(4.0, -2.0, 0.5, 1.0)).color(Color(-1.0, 8.0, 2.0, 0.5))
    comp.get_mut_or_insert_default(1).insert(scenes.custom_circle(api, 66.0, 32.0, 24.0)).set_props(
        Props(func=Func.Draw(Style(fill=Fill.Gradient(gb.build())))))


def render(oracle_api, comp, w, h, channels, clear, crop=None):
    """The oracle's [h, w, 4] float32 frame."""
    out = np.zeros((h, w, 4), np.float32)
    attach(oracle_api).Renderer(0).render_linear(comp, out, w, h, channels, clear, crop, format="f32")
    return out


def encode(frame: np.ndarray, channels) -> np.ndarray:
    """compute_srgb's bytes of an [h, w, 4] float32 frame in the order of `channels`: [h, w, 4] uint8."""
    frame = np.ascontiguousarray(frame, np.float32)
    h, w = frame.shape[:2]
    out = np.zeros((h, w, 4), np.uint8)
    ch = (C.c_uint32 * 4)(*channels)
    _load().fo_linear_to_srgb8(frame.ctypes.data, w, 16 * w, h, ch, out.ctypes.data, 4 * w)
    return out
