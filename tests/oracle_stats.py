"""The oracle's layer statistics (oracle/forma_oracle_stats.cpp, libforma_oracle_stats.so): bound into
the oracle's Api as `renderer_render_stats`, so that `Renderer.render_stats` of the oracle binding
gives the records of an oracle composition."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle")
LIB = os.path.join(ORACLE, "libforma_oracle_stats.so")


def attach(oracle_api):
    if not hasattr(oracle_api, "renderer_render_stats"):
        if not os.path.exists(LIB):
            subprocess.check_call(["make", "-C", ORACLE, "-f", "stats.mk"])
        oracle_api.attach(C.CDLL(LIB), ("renderer_render_stats",))
    return oracle_api


def render(oracle_api, comp, w, h, first_order, n_orders, min_coverage=0.0, crop=None):
    """The oracle's [n_orders] STATS_DTYPE records."""
    return attach(oracle_api).Renderer(0).render_stats(comp, w, h, first_order, n_orders, min_coverage, crop)


def region(w, h, crop=None):
    """(x0, x1, y0, y1): the pixels a single frame counts, the crop's tile rectangle in the frame."""
    if crop is None:
        return 0, w, 0, h
    (hs, he), (vs, ve) = crop.horizontal, crop.vertical
    return min(hs // 16 * 16, w), min(-(-he // 16) * 16, w), min(vs // 16 * 16, h), min(-(-ve // 16) * 16, h)


def _boxes(k, ys, xs, n):
    """Per record index k of the pixels (ys, xs): x0, y0, x1, y1, or 0s where there are none."""
    box = np.zeros((n, 4), np.int64)
    if len(k):
        lo = np.full((n, 2), np.iinfo(np.int64).max)
        hi = np.full((n, 2), -1)
        np.minimum.at(lo, (k, 0), xs)
        np.minimum.at(lo, (k, 1), ys)
        np.maximum.at(hi, (k, 0), xs + 1)
        np.maximum.at(hi, (k, 1), ys + 1)
        has = hi[:, 0] >= 0
        box[has, :2], box[has, 2:] = lo[has], hi[has]
    return box.astype(np.uint32)


def reduce(planes, ids, first_order, min_coverage, rect):
    """The records of a numpy reduction: area, pixels and box from the F32 mask planes [K, H, W],
    visible and visible_box from the ID frame [H, W], over the pixels of rect = (x0, x1, y0, y1)."""
    from forma_b200.binding import STATS_DTYPE
    x0, x1, y0, y1 = rect
    n = planes.shape[0]
    out = np.zeros(n, STATS_DTYPE)
    sub = planes[:, y0:y1, x0:x1]
    units = sub.astype(np.float64) * 262144.0
    assert np.all(units == np.floor(units)), "a mask value that is not a multiple of 2^-18"
    out["area"] = units.reshape(n, -1).sum(axis=1).astype(np.uint64)
    k, ys, xs = np.nonzero(sub > min_coverage)
    out["pixels"] = np.bincount(k, minlength=n)
    out["box"] = _boxes(k, ys + y0, xs + x0, n)
    idw = ids[y0:y1, x0:x1].astype(np.int64) - first_order
    ys, xs = np.nonzero((idw >= 0) & (idw < n))
    k = idw[ys, xs]
    out["visible"] = np.bincount(k, minlength=n)
    out["visible_box"] = _boxes(k, ys + y0, xs + x0, n)
    return out


def diff(got, want):
    """'' when the records are equal, else a description of the first records that differ."""
    bad = np.nonzero(got != want)[0]
    if not len(bad):
        return ""
    return f"{len(bad)} records differ, first {bad[:3].tolist()}: got {got[bad[:2]]}, want {want[bad[:2]]}"
