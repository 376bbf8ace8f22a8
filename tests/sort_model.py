"""A NumPy model of the sort's plan and digits (kernels_sort.cu, kernels.h), and a reference sort.

The sort orders u64 keys on bits [20, 64). Those 44 bits are three fields, listed here from the
least significant: layer | tile_x | tile_y for the pixel segments (layout 0), tile_x | layer |
tile_y for the painter's carry keys (layout 1). The caller gives the largest value of every field;
only the low `bit_length(bound)` bits of a field (at most the field's width) take part. The
participating bits, concatenated in field order, are the *virtual key*; it is cut into
ceil(total / 8) digits of nearly equal size, the larger ones first, and the sort is one stable
counting pass per digit from the least significant one. A digit whose bits come from two or three
fields is described by up to three runs (shift, width, lsh): `width` key bits from bit `shift` on
land at bit `lsh` of the digit.

`MUTATIONS` are deliberate errors of this model; tests/test_sort_plan.py checks that each of them
is caught, i.e. that the checks could tell a wrong plan from a right one.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np

SORT_SHIFT = 20
RADIX_BITS = 8
MAX_PASSES = 6
# (first key bit, width) of every field, least significant field first.
LAYOUTS = {0: ((20, 21), (41, 12), (53, 11)), 1: ((20, 12), (32, 21), (53, 11))}
FIELD_NAMES = {0: ("layer", "tile_x", "tile_y"), 1: ("tile_x", "layer", "tile_y")}
MUTATIONS = ("lsh_zero", "drop_run", "greedy_sizes")
U64 = np.uint64


@dataclass(frozen=True)
class Digit:
    shift: Tuple[int, int, int]
    width: Tuple[int, int, int]
    lsh: Tuple[int, int, int]
    bits: int

    @property
    def runs(self) -> int:
        return sum(w > 0 for w in self.width)


@dataclass(frozen=True)
class Plan:
    n_passes: int
    total_bits: int
    passes: Tuple[Digit, ...]

    def sizes(self) -> List[int]:
        return [d.bits for d in self.passes]

    def describe(self) -> str:
        out = []
        for k, d in enumerate(self.passes):
            runs = " + ".join(f"[{s}, {s + w})<<{l}" for s, w, l in zip(d.shift, d.width, d.lsh) if w)
            out.append(f"pass {k}: {d.bits} bits = {runs}")
        return f"{self.total_bits} bits, {self.n_passes} passes; " + "; ".join(out)


def field_widths(layout: int, bound: Sequence[int]) -> List[int]:
    return [min(int(b).bit_length(), w) for b, (_, w) in zip(bound, LAYOUTS[layout])]


def virtual_bits(layout: int, bound: Sequence[int]) -> List[Tuple[int, int]]:
    """(field, key bit) of every bit of the virtual key, least significant first."""
    return [(f, pos + k) for f, ((pos, _), w) in enumerate(zip(LAYOUTS[layout], field_widths(layout, bound))) for k in range(w)]


def make_plan(layout: int, bound: Sequence[int], mutation: Optional[str] = None) -> Plan:
    vbits = virtual_bits(layout, bound)
    total = len(vbits)
    n = -(-total // RADIX_BITS)
    if mutation == "greedy_sizes":
        sizes = [min(RADIX_BITS, total - RADIX_BITS * k) for k in range(n)]
    else:
        sizes = [total // n + (1 if k < total % n else 0) for k in range(n)] if n else []
    passes, lo = [], 0
    for bits in sizes:
        runs = []  # one run per field that has bits in [lo, lo + bits)
        for at, (f, kb) in enumerate(vbits[lo:lo + bits]):
            if runs and runs[-1][0] == f:
                runs[-1][2] += 1
            else:
                runs.append([f, kb, 1, at])
        if mutation == "drop_run" and len(runs) > 1:
            runs.pop()
        runs += [[None, 0, 0, 0]] * (3 - len(runs))
        passes.append(Digit(tuple(r[1] for r in runs), tuple(r[2] for r in runs),
                            tuple(0 if mutation == "lsh_zero" else r[3] for r in runs), bits))
        lo += bits
    return Plan(n, total, tuple(passes))


def plan_bytes(plan: Plan) -> bytes:
    """The plan as forma_debug_sort_plan writes it."""
    out = bytearray(2 + 10 * MAX_PASSES)
    out[0], out[1] = plan.n_passes, plan.total_bits
    for k, d in enumerate(plan.passes):
        out[2 + 10 * k:12 + 10 * k] = bytes(d.shift + d.width + d.lsh + (d.bits,))
    return bytes(out)


def parse_plan(raw: bytes) -> Plan:
    passes = []
    for k in range(raw[0]):
        r = raw[2 + 10 * k:12 + 10 * k]
        passes.append(Digit(tuple(r[0:3]), tuple(r[3:6]), tuple(r[6:9]), r[9]))
    return Plan(raw[0], raw[1], tuple(passes))


def digit_of(keys: np.ndarray, d: Digit) -> np.ndarray:
    """The digit of every key: each run's bits at its place."""
    keys = np.asarray(keys, U64)
    v = np.zeros(keys.shape, U64)
    for s, w, l in zip(d.shift, d.width, d.lsh):
        if w:
            v |= ((keys >> U64(s)) & U64((1 << w) - 1)) << U64(l)
    return v.astype(np.uint32)


def key_fields(keys: np.ndarray, layout: int) -> List[np.ndarray]:
    keys = np.asarray(keys, U64)
    return [(keys >> U64(pos)) & U64((1 << w) - 1) for pos, w in LAYOUTS[layout]]


def bounds_of(keys: np.ndarray, layout: int) -> List[int]:
    """The bounds a caller that sees the keys on the host passes: the OR of every field."""
    return [int(np.bitwise_or.reduce(f)) if f.size else 0 for f in key_fields(keys, layout)]


def virtual_key(keys: np.ndarray, layout: int, bound: Sequence[int]) -> np.ndarray:
    out, at = np.zeros(np.asarray(keys).shape, U64), 0
    for f, w in zip(key_fields(keys, layout), field_widths(layout, bound)):
        out |= (f & U64((1 << w) - 1)) << U64(at)
        at += w
    return out


def reference_order(keys: np.ndarray, layout: int, bound: Sequence[int]) -> np.ndarray:
    """The permutation a stable sort on the participating bits gives."""
    return np.argsort(virtual_key(keys, layout, bound), kind="stable")


def lsd_order(keys: np.ndarray, plan: Plan) -> np.ndarray:
    """The permutation of one stable counting pass per digit of `plan`, least significant first."""
    keys = np.asarray(keys, U64)
    order = np.arange(keys.size)
    for d in plan.passes:
        order = order[np.argsort(digit_of(keys[order], d), kind="stable")]
    return order


def plan_faults(plan: Plan, layout: int, bound: Sequence[int]) -> List[str]:
    """What is wrong with `plan` as a plan for `bound` (empty: nothing)."""
    vbits = virtual_bits(layout, bound)
    faults = []
    if plan.total_bits != len(vbits):
        faults.append(f"total_bits {plan.total_bits} != {len(vbits)}")
    if plan.n_passes != -(-len(vbits) // RADIX_BITS) or plan.n_passes != len(plan.passes):
        faults.append(f"n_passes {plan.n_passes}")
    sizes = plan.sizes()
    if sizes and (max(sizes) > RADIX_BITS or max(sizes) - min(sizes) > 1 or min(sizes) < 1):
        faults.append(f"digit sizes {sizes}")
    covered = []
    for k, d in enumerate(plan.passes):
        at, last_field = 0, -1
        for r, (s, w, l) in enumerate(zip(d.shift, d.width, d.lsh)):
            if w == 0:
                if any(d.width[r:]) or s or l:
                    faults.append(f"pass {k}: run {r} is unused but not blank, or a used run follows it")
                continue
            if l != at:
                faults.append(f"pass {k}: run {r} lands at bit {l}, not {at}")
            field = [f for f, (pos, fw) in enumerate(LAYOUTS[layout]) if pos <= s and s + w <= pos + fw]
            if len(field) != 1 or field[0] <= last_field:
                faults.append(f"pass {k}: run {r} [{s}, {s + w}) is not inside one field, in field order")
            else:
                last_field = field[0]
            covered += list(range(s, s + w))
            at += w
        if at != d.bits:
            faults.append(f"pass {k}: runs hold {at} bits, the digit {d.bits}")
    if covered != [kb for _, kb in vbits]:
        faults.append("the passes do not cover exactly the participating bits, least significant first")
    return faults


# ---- the sort's schedule (which kernels sort n keys, and how its tiles are spread) ------------
SMALL_TILE, BIG_TILE = 1024, 4096
MAX_CHUNKS, CHUNKS_PER_SUPER, DS_STAGES = 512, 16, 3


def key_path(n: int, big_log2: int, scan_log2: int) -> str:
    """The kernels a key-only sort of n keys runs under the two size options."""
    if n < (1 << big_log2):
        return "sweep4"
    return "wide" if n >= (1 << scan_log2) else "sweep16"


def tile_keys(path: str) -> int:
    return SMALL_TILE if path == "sweep4" else BIG_TILE


def tiles_of(n: int, tile: int) -> int:
    return -(-n // tile)


def tiles_owned(cta: int, tiles: int, grid: int) -> int:
    """Tiles of CTA `cta` of the persistent downsweep: cta, cta + grid, ... (grid = min(tiles, G))."""
    return len(range(cta, tiles, grid)) if cta < grid else 0


def scan_shape(tiles: int) -> Tuple[int, int, int]:
    """(tiles per chunk, chunks, super-chunks) of the tile scan."""
    tpc = -(-tiles // MAX_CHUNKS)
    chunks = -(-tiles // tpc)
    return tpc, chunks, -(-chunks // CHUNKS_PER_SUPER)


# ---- the tile bounds a frame's plan is built from (line_count_body, kernels_raster.cu) --------
FAR_EDGE = -8388352.0  # sub-pixels: two tiles before the int16 wrap of the tile coordinate


def tile_bound(lo: np.ndarray, hi: np.ndarray, clamp: int, far_rule: bool = True, slack: int = 2) -> int:
    """The bound of a tile field over lines whose sub-pixel extent along that axis is [lo, hi]
    (float32, NaN ignored by min / max as fminf / fmaxf do)."""
    if len(hi) == 0:
        return 0
    with np.errstate(invalid="ignore"):
        e = np.floor(np.fmin(np.asarray(hi, np.float32), np.float32(3.0e7)) + np.float32(0.5))
        e = np.where(np.isnan(e), -2.0 ** 31, e).astype(np.int64)  # a NaN converts to INT_MIN-like: clamps to 0
        t = np.clip((e >> 8) + slack, 0, clamp)
        if far_rule:
            t = np.where(~(np.asarray(lo, np.float32) >= np.float32(FAR_EDGE)), clamp, t)
    return int(t.max())
