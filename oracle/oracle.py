"""ORACLE — test infrastructure only.

Loads oracle/libforma_oracle.so (built by oracle/Makefile) and exposes it
through the same binding classes as the product library, plus the small
known-answer hooks used to pin the oracle against the reference's unit tests.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from forma_b200 import binding

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "libforma_oracle.so")


def build(force: bool = False) -> str:
    if force or not os.path.exists(_LIB):
        subprocess.check_call(["make", "-C", _HERE] + (["-B"] if force else []))
    return _LIB


def load() -> binding.Api:
    lib = C.CDLL(build())
    api = binding.Api(lib, "fo_", optional=("renderer_render_device", "renderer_stage_times", "renderer_counters", "renderer_host_slices", "renderer_kernel_times", "renderer_set_stream", "path_program_stats",
                                        "path_program_records", "shared_frame_create", "shared_frame_open", "shared_frame_close", "shared_frame_free",
                                        "composition_evict", "composition_point_count", "set_option", "get_option", "debug_selftest", "renderer_row_costs", "renderer_multi_new", "renderer_multi_free", "renderer_multi_device_count",
                                        "renderer_multi_render", "renderer_multi_render_device", "renderer_multi_bands"))
    _declare_hooks(lib)
    api.hooks = lib
    return api


def _declare_hooks(lib):
    f, fp, i32, u32, u64 = C.c_float, C.POINTER(C.c_float), C.c_int32, C.c_uint32, C.c_uint64
    lib.fo_num_threads.restype = C.c_int
    lib.fo_find.restype, lib.fo_find.argtypes = f, [i32, f, f, f, f]
    lib.fo_pack_segment.restype, lib.fo_pack_segment.argtypes = u64, [u32, i32, i32, u32, u32, u32, i32]
    lib.fo_unpack_segment.restype, lib.fo_unpack_segment.argtypes = None, [u64, C.POINTER(i32)]
    lib.fo_to_srgb_bytes.restype, lib.fo_to_srgb_bytes.argtypes = None, [fp, C.POINTER(C.c_uint8)]
    lib.fo_to_byte.restype, lib.fo_to_byte.argtypes = C.c_uint8, [f]
    lib.fo_blend_scalar.restype, lib.fo_blend_scalar.argtypes = None, [u32, fp, fp, fp]
    lib.fo_blend_lane.restype, lib.fo_blend_lane.argtypes = None, [u32, fp, fp, fp]
    lib.fo_approx_atan2.restype, lib.fo_approx_atan2.argtypes = f, [f, f]
    lib.fo_coverage.restype, lib.fo_coverage.argtypes = f, [i32, u32]


def unpack(lib, seg: int):
    out = (C.c_int32 * 7)()
    lib.fo_unpack_segment(C.c_uint64(int(seg)), out)
    return dict(zip(["layer_id", "tile_x", "tile_y", "local_x", "local_y", "double_area", "cover"], list(out)))


def blend_scalar(lib, mode, dst, src):
    d = (C.c_float * 4)(*dst)
    s = (C.c_float * 4)(*src)
    o = (C.c_float * 4)()
    lib.fo_blend_scalar(mode, d, s, o)
    return np.array(list(o), np.float32)


def blend_lane(lib, mode, dst, src):
    d = (C.c_float * 3)(*dst)
    s = (C.c_float * 3)(*src)
    o = (C.c_float * 3)()
    lib.fo_blend_lane(mode, d, s, o)
    return np.array(list(o), np.float32)


def to_srgb_bytes(lib, color):
    c = (C.c_float * 4)(*color)
    o = (C.c_uint8 * 4)()
    lib.fo_to_srgb_bytes(c, o)
    return list(o)
