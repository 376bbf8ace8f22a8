"""The mask entry points' binding without a GPU: the header declares what the binding calls, the
library exports it, the descriptor has the header's layout, and the default strides are those of a
contiguous [K, H, W] / [N, K, H, W] array."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from forma_b200 import binding
from forma_b200.binding import MASK_SYMBOLS, Renderer, _CMasks, mask_format

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header():
    with open(os.path.join(ROOT, "include", "forma_b200.h")) as f:
        return f.read()


def test_header_declares_every_mask_symbol():
    h = header()
    for name in MASK_SYMBOLS:
        assert re.search(r"\bint forma_" + name + r"\(", h), name
    assert "FORMA_MASK_F32 = 0, FORMA_MASK_U8 = 1" in h


def test_signatures_and_optional():
    for name in MASK_SYMBOLS:
        assert name in binding.SIGNATURES
        assert name in binding._OPTIONAL_SYMBOLS


def test_descriptor_layout():
    assert C.sizeof(_CMasks) == 40
    assert [(n, getattr(_CMasks, n).offset) for n, _ in _CMasks._fields_] == [
        ("ptr", 0), ("first_order", 8), ("n_orders", 12), ("format", 16), ("stride", 24), ("plane_stride", 32)]


def test_library_exports_the_symbols():
    lib = C.CDLL(os.path.join(ROOT, "forma_b200", "libforma_b200.so"))
    for name in MASK_SYMBOLS:
        assert hasattr(lib, "forma_" + name)


@pytest.mark.parametrize("fmt,bpp,dtype", [("f32", 4, np.float32), ("u8", 1, np.uint8)])
def test_default_strides(fmt, bpp, dtype):
    code, b, dt, stride, plane_stride = Renderer._mask_layout(37, 21, 5, fmt, None, None)
    assert (b, dt, stride, plane_stride) == (bpp, dtype, 37 * bpp, 37 * 21 * bpp)
    assert code == {"f32": 0, "u8": 1}[fmt]
    a = np.zeros((5, 21, 37), dtype)
    assert a.strides[:2] == (plane_stride, stride)
    assert Renderer._mask_layout(37, 21, 5, fmt, 200, None)[3:] == (200, 200 * 21)


def test_unknown_format():
    with pytest.raises(ValueError):
        mask_format("f16")
