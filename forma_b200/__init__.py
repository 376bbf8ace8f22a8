"""forma_b200 — H100-native replacement for google/forma's rendering hot path.

The compute path lives in ``libforma_b200.so`` (hand-written CUDA for sm_90a,
built in-tree by ``forma_b200/csrc/Makefile``); this package is only the
ctypes stub over its C ABI (``include/forma_b200.h``). There is no CPU
fallback: importing works without a GPU (so the ABI can be inspected), but
``Renderer()`` raises when no H100 (sm_90) is present, and loading fails loudly when
the shared library has not been built.
"""
from __future__ import annotations

import ctypes as _C
import os as _os

from . import binding
from .binding import *  # noqa: F401,F403  (reference-like names: Point, Color, Props, RGBA, ...)

_HERE = _os.path.dirname(_os.path.abspath(__file__))
LIB_PATH = _os.path.join(_HERE, "libforma_b200.so")

_api = None


def load() -> binding.Api:
    """Loads libforma_b200.so and returns the typed API (cached)."""
    global _api
    if _api is None:
        if not _os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `make -C forma_b200/csrc` "
                "(or __graft_entry__.build()). forma_b200 has no CPU fallback.")
        lib = _C.CDLL(LIB_PATH)
        _api = binding.Api(lib, "forma_")
    return _api


def PathBuilder():
    return load().PathBuilder()


def Composition():
    return load().Composition()


def Renderer(device: int = 0):
    return load().Renderer(device)
