"""The statistics entry points' binding without a GPU: the header declares what the binding calls, the
library exports it, STATS_DTYPE is forma_layer_stats and _CStats is forma_stats as the header lays them
out, and split_stats reads the words of device records."""
import ctypes as C
import os
import re

import numpy as np

from forma_b200 import binding
from forma_b200.binding import STATS_DTYPE, STATS_SYMBOLS, _CStats, split_stats

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header():
    with open(os.path.join(ROOT, "include", "forma_b200.h")) as f:
        return f.read()


def test_header_declares_every_stats_symbol():
    h = header()
    for name in STATS_SYMBOLS:
        assert re.search(r"\bint forma_" + name + r"\(", h), name


def test_signatures_and_optional():
    for name in STATS_SYMBOLS:
        assert name in binding.SIGNATURES
        assert name in binding._OPTIONAL_SYMBOLS


def test_library_exports_the_symbols():
    lib = C.CDLL(os.path.join(ROOT, "forma_b200", "libforma_b200.so"))
    for name in STATS_SYMBOLS:
        assert hasattr(lib, "forma_" + name)


class _CLayerStats(C.Structure):  # forma_layer_stats as the header declares it
    _fields_ = [("area", C.c_uint64), ("pixels", C.c_uint32), ("visible", C.c_uint32), ("box", C.c_uint32 * 4),
                ("visible_box", C.c_uint32 * 4)]


def _header_fields(struct):
    body = re.search(r"typedef struct " + struct + r" \{(.*?)\} " + struct + ";", header(), re.S).group(1)
    return [m.group(2) for m in re.finditer(r"^\s*(\w+\*?|\w+)\s+\*?(\w+)(\[\d\])?[,;]", body, re.M)]


def test_record_layout():
    assert _header_fields("forma_layer_stats") == ["area", "pixels", "visible", "box", "visible_box"]
    assert STATS_DTYPE.itemsize == C.sizeof(_CLayerStats) == 48
    for name, _ in _CLayerStats._fields_:
        assert STATS_DTYPE.fields[name][1] == getattr(_CLayerStats, name).offset, name
    assert STATS_DTYPE["box"].shape == STATS_DTYPE["visible_box"].shape == (4,)


def test_descriptor_layout():
    assert "first_order, n_orders;" in re.search(r"typedef struct forma_stats \{(.*?)\}", header(), re.S).group(1)
    assert C.sizeof(_CStats) == 24
    assert [(n, getattr(_CStats, n).offset) for n, _ in _CStats._fields_] == [
        ("ptr", 0), ("first_order", 8), ("n_orders", 12), ("min_coverage", 16)]


def test_split_stats_reads_the_words():
    rec = np.zeros(3, STATS_DTYPE)
    rec["area"] = [0, (1 << 40) + 7, 3 << 18]
    rec["pixels"] = [0, 0xFFFFFFFF, 5]
    rec["visible"] = [0, 1, 2]
    rec["box"][1] = [1, 2, 3, 4]
    rec["visible_box"][2] = [10, 20, 4000, 0xFFFFFFFE]
    words = rec.view(np.int32).reshape(3, 12)
    got = split_stats(words)
    for name in ("area", "pixels", "visible", "box", "visible_box"):
        assert np.array_equal(got[name], rec[name].astype(np.int64)), name
