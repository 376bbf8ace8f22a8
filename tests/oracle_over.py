"""The oracle's frames over a background (oracle/forma_oracle_over.cpp, libforma_oracle_over.so):
`render` draws an oracle composition over a host frame in place, sRGB8 ([h, w, 4] uint8) or
RGBA32F ([h, w, 4] float32), and `decode_table` is the sRGB8 decode table D the oracle and the
paint kernels share (forma_b200/csrc/srgb_decode.h)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from forma_b200.binding import Channel, Color, Rect

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle")
LIB = os.path.join(ORACLE, "libforma_oracle_over.so")
_lib = None


class _Rect(C.Structure):
    _fields_ = [("hor_start", C.c_uint64), ("hor_end", C.c_uint64), ("vert_start", C.c_uint64), ("vert_end", C.c_uint64)]


def _load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            subprocess.check_call(["make", "-C", ORACLE, "-f", "over.mk"])
        _lib = C.CDLL(LIB)
        _lib.fo_renderer_render_over.restype = C.c_int
        _lib.fo_renderer_render_over.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64,
                                                 C.POINTER(C.c_uint32), C.POINTER(_Rect), C.c_uint32, C.c_void_p]
        _lib.fo_srgb_decode_table.restype = None
        _lib.fo_srgb_decode_table.argtypes = [C.c_void_p]
    return _lib


def decode_table() -> np.ndarray:
    out = np.zeros(256, np.float32)
    _load().fo_srgb_decode_table(out.ctypes.data)
    return out


def render(comp, frame: np.ndarray, channels, crop: Rect | None = None) -> int:
    """Draws `comp` (an oracle composition) over `frame` in place: a C-contiguous [h, w, 4] uint8
    (sRGB8) or float32 (RGBA32F) array. Returns the oracle's status (0: rendered)."""
    assert frame.flags["C_CONTIGUOUS"] and frame.ndim == 3 and frame.shape[2] == 4
    fmt = {np.dtype(np.uint8): 0, np.dtype(np.float32): 2}[frame.dtype]
    h, w = frame.shape[:2]
    rect = None if crop is None else _Rect(crop.horizontal[0], crop.horizontal[1], crop.vertical[0], crop.vertical[1])
    ch = (C.c_uint32 * 4)(*[int(c) for c in channels])
    return _load().fo_renderer_render_over(None, comp._h, frame.ctypes.data, w, w * frame.itemsize * 4, h, ch,
                                           C.byref(rect) if rect is not None else None, fmt, None)


def decode(frame: np.ndarray, channels) -> np.ndarray:
    """The linear (r, g, b, a) of every pixel of an sRGB8 [h, w, 4] frame in the order of
    `channels` (a permutation of R, G, B, A): D for colour bytes, byte / 255 for alpha."""
    d = decode_table()
    out = np.zeros(frame.shape, np.float32)
    for k, c in enumerate(channels):
        c = int(c)
        b = frame[..., k]
        out[..., c] = (b.astype(np.float32) / np.float32(255.0)) if c == int(Channel.Alpha) else d[b]
    return out


def clear_of(pixel, channels) -> Color:
    """The clear colour a pixel (4 bytes in the order of `channels`) decodes to."""
    v = decode(np.asarray(pixel, np.uint8).reshape(1, 1, 4), channels)[0, 0]
    return Color(float(v[0]), float(v[1]), float(v[2]), float(v[3]))
