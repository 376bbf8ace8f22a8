"""NumPy replay of line setup (`line_setup`, `line_count_kernel`, `scan_block_sums_kernel` and the
loop bound of `raster_emit_kernel` in forma_b200/csrc/kernels_raster.cu; segment.rs:298-383) and
of the key packing of one pixel segment (rasterizer.rs:111-156).

`replay(points, layers, width, height, band)` follows one thread per point pair: the layer
affine with exact `fmaf`, the skip rules with the band cull at `band_lo - 1/16` / `band_hi`,
`x0, y0, dx, dy, a, b, c, d` and the exact length as u64 (a saturated `integers_between` counts
as 2^32 - 1, so such a length is a lower bound). `counts(lengths, cap)` derives from the lengths
what the reference and the device make of them: the reference's wrapped u32 inclusive prefix
sums (the oracle's `lines()["lengths"]`), the per-CTA sums, the true total, the status the
renderer returns, and the bound on the iterations of the emit pass for a given `cap`.

`fmaf` is exact: the product of two float32 values is exact in float64, the sum with the
addend is rounded to float64 and its rounding error recovered with TwoSum; only when that sum
falls on a midpoint between two float32 values does the error decide the direction.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

CTA = 256                      # kRasterThreads: lines per CTA of the count and emit passes
SEGMENT_LIMIT = 1 << 30        # Renderer::rasterize refuses a frame of this many pixel segments
U32_MAX = 0xFFFFFFFF
FORMA_OK, FORMA_ERR_CAPACITY = 0, 5
INT_MIN = -(1 << 31)

f32 = np.float32


def fmaf(a, b, c) -> np.ndarray:
    """float32 fma(a, b, c), correctly rounded (see the module docstring)."""
    a, b, c = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    with np.errstate(all="ignore"):
        p = a * b                                   # exact
        s = p + c
        bb = s - p
        e = (p - (s - bb)) + (c - bb)               # TwoSum: p + c == s + e exactly
        r = s.astype(np.float32)
        rd = r.astype(np.float64)
        toward = np.where(s > rd, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32)
        other = np.nextafter(r, toward).astype(np.float64)
        mid = (rd + other) * 0.5
        on_mid = np.isfinite(s) & np.isfinite(e) & (rd != s) & (s == mid) & (e != 0)
        nudged = np.nextafter(s, np.where(e > 0, np.inf, -np.inf)).astype(np.float32)
    return np.where(on_mid, nudged, r).astype(np.float32)


def sat_u32(v: np.ndarray) -> np.ndarray:
    """Rust `as u32` from f32 (d_sat_u32): NaN and v <= 0 -> 0, v >= 2^32 -> 2^32 - 1."""
    v = np.asarray(v, np.float32)
    with np.errstate(invalid="ignore"):
        out = np.where(v > 0, np.minimum(np.nan_to_num(v, nan=0.0, posinf=2.0 ** 32).astype(np.float64),
                                         2.0 ** 32 - 1), 0.0)
    return np.floor(out).astype(np.uint64)


def integers_between(u, v) -> np.ndarray:  # segment.rs:54-59
    with np.errstate(invalid="ignore"):
        mn, mx = np.fmin(u, v), np.fmax(u, v)
        return sat_u32((np.ceil(mx) - np.floor(mn)) - f32(1.0))


@dataclass
class LayerXf:
    """A layer: its order, whether it is enabled, and [ux, vx, uy, vy, tx, ty] or None."""
    order: int
    xf: Optional[Sequence[float]] = None
    enabled: bool = True


def point_buffer(inserts) -> tuple:
    """The composition's segment buffer of a list of (layer index, x, y, start_new_contour)
    inserts (composition/layer.rs:90-111 + segment.rs:181-198, restated in oracle/scene.hpp
    layer_insert): points and, per point, the layer of the line to the next point (-1: none)."""
    X: List[float] = []
    Y: List[float] = []
    ids: List[int] = []
    for li, x, y, contour in inserts:
        for i in range(len(x)):
            X.append(float(x[i]))
            Y.append(float(y[i]))
            ids.append(-1 if contour[i] else li)
        n = max(len(X) - 1, 0)
        ids = ids[:n] + [li] * (n - len(ids))
        if ids and ids[-1] != -1:
            ids.append(-1)
    return np.array(X, np.float32), np.array(Y, np.float32), np.array(ids, np.int64)


def replay(x, y, ids, layers: Sequence[LayerXf], width, height, band=(-3.0e38, 3.0e38)) -> dict:
    """Line records of every point pair (i, i + 1), as line_setup computes them."""
    n = max(len(x) - 1, 0)
    width, height = f32(width), f32(height)
    band_lo, band_hi = f32(band[0]), f32(band[1])
    lid = ids[:n]
    live = lid >= 0
    enabled = np.array([l.enabled for l in layers] + [False], bool)
    live &= enabled[np.where(live, lid, len(layers))]
    p0x, p0y, p1x, p1y = (np.asarray(v, np.float32).copy() for v in (x[:n], y[:n], x[1:n + 1], y[1:n + 1]))
    for k, lay in enumerate(layers):
        if lay.xf is None:
            continue
        ux, vx, uy, vy, tx, ty = (f32(v) for v in lay.xf)
        sel = lid == k
        for px, py in ((p0x, p0y), (p1x, p1y)):
            ax = fmaf(ux, px[sel], fmaf(vx, py[sel], tx))
            ay = fmaf(uy, px[sel], fmaf(vy, py[sel], ty))
            px[sel], py[sel] = ax, ay
    with np.errstate(all="ignore"):
        cull = f32(band_lo - f32(0.0625))
        skip = ((p0y == p1y) | ((p0y >= height) & (p1y >= height)) | ((p0x >= width) & (p1x >= width))
                | ((p0y <= 0) & (p1y <= 0)) | ((p0y >= band_hi) & (p1y >= band_hi)) | ((p0y <= cull) & (p1y <= cull)))
        keep = live & ~skip
        dx, dy = p1x - p0x, p1y - p0y
        rx, ry = f32(1.0) / dx, f32(1.0) / dy
        c = np.where(dx != 0, np.fmax((np.ceil(p0x) - p0x) * rx, (np.floor(p0x) - p0x) * rx), f32(0))
        d = np.where(dy != 0, np.fmax((np.ceil(p0y) - p0y) * ry, (np.floor(p0y) - p0y) * ry), f32(0))
        length = integers_between(p0x, p1x) + integers_between(p0y, p1y) + np.uint64(1)
        sat = (integers_between(p0x, p1x) == U32_MAX) | (integers_between(p0y, p1y) == U32_MAX)
    z = np.float32(0)
    orders = np.array([l.order for l in layers] + [0], np.uint32)[np.where(lid >= 0, lid, len(layers))]
    rec = {
        "orders": np.where(keep, orders, 0).astype(np.uint32),
        "x0": np.where(keep, p0x * f32(16), z), "y0": np.where(keep, p0y * f32(16), z),
        "dx": np.where(keep, dx * f32(16), z), "dy": np.where(keep, dy * f32(16), z),
        "a": np.where(keep, np.abs(rx), z), "b": np.where(keep, np.abs(ry), z),
        "c": np.where(keep, c, z), "d": np.where(keep, d, z),
        "length": np.where(keep, length, 0).astype(np.uint64),
        "saturated": keep & sat,
        "end_points": (p0x, p0y, p1x, p1y),
        "source_points": (np.asarray(x[:n], np.float32), np.asarray(y[:n], np.float32)),  # before the layer affine
        "keep": keep,
    }
    for k in ("x0", "y0", "dx", "dy", "a", "b", "c", "d"):
        rec[k] = rec[k].astype(np.float32)
    return rec


@dataclass
class Counts:
    prefix_u32: np.ndarray     # the reference's wrapped inclusive prefix sums
    block_sums: np.ndarray     # true per-CTA sums (u64)
    total: int                 # true total (a lower bound when a length saturated)
    status: int                # what Renderer::rasterize returns
    device_total: int          # what the device reads back: min(total, 2^32 - 1)
    emit_iterations: np.ndarray  # per CTA: the most segments the emit loop visits for `cap`


def counts(lengths: np.ndarray, n_points: int, cap: int = U32_MAX) -> Counts:
    """`lengths` per line (u64, n_points - 1 of them; the last point has no line)."""
    lengths = np.asarray(lengths, np.uint64)
    prefix = (np.cumsum(lengths.astype(object)) if lengths.size else np.zeros(0, object))
    prefix_u32 = np.array([int(v) & U32_MAX for v in prefix], np.uint32)
    nb = (n_points + CTA - 1) // CTA if n_points else 0
    per = np.zeros(nb * CTA, object)
    per[:lengths.size] = [int(v) for v in lengths]
    block = per.reshape(nb, CTA).sum(axis=1) if nb else np.zeros(0, object)
    total = int(sum(int(v) for v in lengths))
    base = np.concatenate([[0], np.cumsum(block)[:-1]]) if nb else np.zeros(0, object)
    sat = lambda v: min(int(v), U32_MAX)  # noqa: E731
    it = np.array([max(0, min(sat(bt), cap - sat(bb))) if sat(bb) < cap else 0 for bt, bb in zip(block, base)], np.int64)
    return Counts(prefix_u32, np.array([int(v) for v in block], object), total,
                  FORMA_ERR_CAPACITY if total >= SEGMENT_LIMIT else FORMA_OK, sat(total), it)


def max_tile(rec: dict) -> tuple:
    """The (biased) tile bounds line_count_kernel reports for the sort plan."""
    keep = rec["length"] > 0
    if not keep.any():
        return 0, 0
    with np.errstate(all="ignore"):
        ex = np.fmax(rec["x0"], rec["x0"] + rec["dx"])[keep]
        ey = np.fmax(rec["y0"], rec["y0"] + rec["dy"])[keep]

        def tile(e, hi):
            v = np.floor(np.fmin(e, f32(3.0e7)) + f32(0.5)).astype(np.float64)
            v = np.clip(np.nan_to_num(v, nan=0.0, neginf=INT_MIN), INT_MIN, 2 ** 31 - 1).astype(np.int64)
            return int(np.clip((v >> 8) + 2, 0, hi).max())
    return tile(ex, 4095), tile(ey, 2047)


# --- one pixel segment ---------------------------------------------------------------------

def round_sub(v: float) -> int:
    """rasterizer.rs:78-80 with the x86 semantics of `to_int_unchecked` (cvttss2si): NaN and
    values outside i32 give i32::MIN."""
    f = float(np.floor(f32(v) + f32(0.5)))
    return int(f) if -2.0 ** 31 <= f < 2.0 ** 31 else INT_MIN


def _i32(v: int) -> int:
    v &= U32_MAX
    return v - (1 << 32) if v >> 31 else v


def _i16(v: int) -> int:
    v &= 0xFFFF
    return v - (1 << 16) if v >> 15 else v


def segment_word(order: int, x0f: float, y0f: float, x1f: float, y1f: float) -> int:
    """The packed pixel segment of sub-pixel end points (rasterizer.rs:111-156,
    pixel_segment.rs:36-71)."""
    x0s, y0s, x1s, y1s = (round_sub(v) for v in (x0f, y0f, x1f, y1f))
    border_x, border_y = min(x0s, x1s) >> 4, min(y0s, y1s) >> 4
    tile_x, tile_y = _i16(border_x >> 4), _i16(border_y >> 4)
    local_x, local_y = border_x & 15, border_y & 15
    border = _i32((border_x << 4) + 16)
    dam = _i32(abs(_i32(x1s - x0s)) + 2 * _i32(border - max(x0s, x1s))) & 0xFF
    cover = _i32(y1s - y0s) & 0xFF
    ty = max(_i16(tile_y + 1), 0) & 0x7FF
    tx = max(_i16(tile_x + 1), 0) & 0xFFF
    return (ty << 53) | (tx << 41) | ((order & 0x1FFFFF) << 20) | (local_x << 16) | (local_y << 12) | ((dam & 0x3F) << 6) \
        | (cover & 0x3F)
