"""The oracle's layer coverage masks (oracle/forma_oracle_masks.cpp, libforma_oracle_masks.so):
bound into the oracle's Api as `renderer_render_masks`, so that `Renderer.render_masks` of the
oracle binding renders the mask planes of an oracle composition."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle")
LIB = os.path.join(ORACLE, "libforma_oracle_masks.so")


def attach(oracle_api):
    if not hasattr(oracle_api, "renderer_render_masks"):
        if not os.path.exists(LIB):
            subprocess.check_call(["make", "-C", ORACLE, "-f", "masks.mk"])
        oracle_api.attach(C.CDLL(LIB), ("renderer_render_masks",))
    return oracle_api


def render(oracle_api, comp, w, h, first_order, n_orders, fmt="f32", crop=None):
    """The oracle's [n_orders, h, w] planes (float32 or uint8)."""
    out = np.zeros((n_orders, h, w), np.float32 if fmt == "f32" else np.uint8)
    attach(oracle_api).Renderer(0).render_masks(comp, out, w, h, first_order, crop=crop)
    return out
