"""Key sets for the sorts at their limits (tests/sort_model.py describes plans and schedules).

A `Case` is a pure function of its name: `keys(G)` builds the keys (G = CTAs of the persistent
downsweep's grid, 2 per SM; only the `wide_*` sizes depend on it), `opts` are the size options it
runs under, and `claims` say which condition it is there for. tests/test_sort_scenes.py proves
every claim on the CPU with the model, and that the case is within budget, before
tests/test_gpu_sort.py hands it to a kernel.

Claims (all optional):
  path            the kernels that sort it: sweep4 / sweep16 (single-sweep, 1024- / 4096-key tiles), wide
  total_bits      bits of the plan the entry point makes from the keys' OR
  sizes           the plan's digit sizes
  runs            {pass: runs of that pass's digit}
  const_passes    passes in which every key has the same digit
  const_digit     {pass: that digit}
  last_tile       real keys in the last, partial tile
  last_max_digit  pass in which every real key of the last tile carries the padding digit 2^bits - 1
                  (and so do earlier keys: the padding must rank after all of them)
  tiles           tiles of the sort
  cta0_tiles / cta_last_tiles   tiles owned by the first / last CTA of the downsweep
  tiles_per_chunk, supers       shape of the tile scan
  identity        the sort must return the input (nothing to sort on bits [20, 64))
  sorted_input / reversed_input the input's order
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np

import sort_model as sm

U64 = np.uint64
MAX_N = 1 << 27            # keys of the largest case
MAX_DEVICE_BYTES = 3 << 30  # device memory of one case
GRIDS = (264, 228)         # the grids the CPU test checks the G-dependent sizes for

SWEEP4 = {"sort_big_log2": 19, "sort_scan_log2": 22}   # the defaults: n < 2^19 runs 1024-key tiles
SWEEP16 = {"sort_big_log2": 10, "sort_scan_log2": 30}  # 4096-key single-sweep tiles from 1024 keys on
WIDE = {"sort_big_log2": 10, "sort_scan_log2": 10}     # reduce-then-scan passes from 1024 keys on
SETTINGS = {"sweep4": SWEEP4, "sweep16": SWEEP16, "wide": WIDE}


@dataclass
class Case:
    name: str
    target: str
    make: Callable[[int], object]  # G -> keys, or (keys, vals) for pairs
    opts: Dict[str, int]
    claims: Dict[str, object] = field(default_factory=dict)
    n: Optional[Callable[[int], int]] = None  # G -> key count, without building the keys
    layout: int = 0
    analytic: bool = False  # `expected(G)` gives the sorted keys (too many keys for a host sort)
    expected: Optional[Callable[[int], np.ndarray]] = None

    def keys(self, G: int = GRIDS[0]):
        return self.make(G)


def device_bytes(n: int, pairs: bool = False) -> int:
    """Device memory a sort of n keys takes: keys and their twin (one key of slack each), the
    look-back or tile-histogram scratch (sort_model.MAX_PASSES tables of 256 u32 per 1024-key
    tile at most), payloads and their twin."""
    tiles = sm.tiles_of(n, sm.SMALL_TILE)
    return 2 * 8 * (n + 1) + 4 * 256 * (sm.MAX_PASSES * (tiles + 1) + sm.MAX_PASSES * 544) + (2 * 4 * (n + 1) if pairs else 0)


def pack(f0, f1, f2, low, layout: int = 0) -> np.ndarray:
    """Keys from their three fields (least significant first) and the 20 bits below them."""
    (p0, _), (p1, _), (p2, _) = sm.LAYOUTS[layout]
    return (np.asarray(f2, U64) << U64(p2)) | (np.asarray(f1, U64) << U64(p1)) | (np.asarray(f0, U64) << U64(p0)) | np.asarray(low, U64)


def _low(rng, n):
    return rng.integers(0, 1 << 20, size=n, dtype=np.uint64)


def _seed(name: str) -> int:
    return int.from_bytes(name.encode(), "little") % (1 << 63)


def random_fields(name: str, n: int, widths, layout: int = 0) -> np.ndarray:
    """Uniform fields of the given widths, random low bits; the first key has every field bit set
    and the second none, so that the OR of the keys gives exactly `widths`."""
    rng = np.random.default_rng(_seed(name))
    f = [rng.integers(0, 1 << w, size=n, dtype=np.uint64) for w in widths]
    for k in range(3):
        if n > 0:
            f[k][0] = (1 << widths[k]) - 1
        if n > 1:
            f[k][1] = 0
    return pack(f[0], f[1], f[2], _low(rng, n), layout)


# ---- the cases -------------------------------------------------------------------------------
SHAPES = {  # total bits -> field widths (layer, tile_x, tile_y)
    1: (1, 0, 0), 7: (0, 7, 0), 8: (0, 0, 8), 9: (4, 5, 0), 15: (5, 5, 5), 16: (0, 8, 8), 17: (1, 8, 8),
    24: (8, 8, 8), 25: (21, 4, 0), 43: (21, 12, 10), 44: (21, 12, 11)}
STRADDLES = [(1, 1, 6), (3, 2, 3), (5, 12, 0), (0, 0, 11), (21, 0, 0), (2, 3, 11)]
SHAPE_N = 3 * sm.BIG_TILE + 7


def _sizes(total):
    n = -(-total // 8)
    return [total // n + (1 if k < total % n else 0) for k in range(n)]


def _shape_cases() -> List[Case]:
    out = []
    shapes = [(f"bits{t}", w) for t, w in SHAPES.items()] + [("runs_" + "_".join(map(str, w)), w) for w in STRADDLES]
    for label, w in shapes:
        claims = {"total_bits": sum(w), "sizes": _sizes(sum(w)), "last_tile": 7}
        if w == (1, 1, 6):
            claims["runs"] = {0: 3}
        if w == (3, 2, 3):
            claims["runs"] = {0: 3}
        if w == (5, 12, 0):
            claims["runs"] = {0: 2, 1: 1, 2: 1}
        if w == (2, 3, 11):
            claims["runs"] = {0: 3, 1: 1}
        for path, opts in SETTINGS.items():
            name = f"shape_{label}_{path}"
            out.append(Case(name, f"plan of widths {w} on the {path} passes",
                            (lambda nm, ww: lambda G: random_fields(nm, SHAPE_N, ww))(name, w), opts,
                            dict(claims, path=path), n=lambda G: SHAPE_N))
    return out


def _distribution(kind: str, name: str, n: int) -> np.ndarray:
    rng = np.random.default_rng(_seed(name))
    low = _low(rng, n)
    i = np.arange(n, dtype=np.uint64)
    if kind == "constant":
        return pack(5, 9, 3, low)
    if kind == "sorted":
        return np.sort(random_fields(name, n, (6, 7, 5)) >> U64(20)) << U64(20) | low
    if kind == "reversed":
        return (np.sort(random_fields(name, n, (6, 7, 5)) >> U64(20))[::-1].copy() << U64(20)) | low
    if kind == "alternating":
        return np.where(i % U64(2) == 0, pack(1000, 40, 17, 0), pack(3, 2, 900, 0)) | low
    if kind == "top_digit_only":  # 24 bits; the two low digits are 255 in every key
        return pack(0xFF, 0xFF, i % U64(251), low)
    if kind == "hot_key":  # one key value but for 31 strays
        k = np.full(n, pack(77, 300, 21, 0), U64)
        at = rng.choice(n, size=31, replace=False)
        k[at] = random_fields(name, 31, (9, 10, 6)) & ~U64(0xFFFFF)
        return k | low
    if kind == "zipf_rows":  # most keys in a few tile rows
        ty = np.minimum(rng.zipf(1.3, size=n), 135).astype(np.uint64)
        return pack(rng.integers(0, 50, size=n), rng.integers(0, 240, size=n), ty, low)
    if kind == "below_20":
        return low
    if kind == "digit_255":  # 16 bits of layer: every key has 255 in pass 0
        hi = rng.integers(0, 256, size=n, dtype=np.uint64)
        hi[0] = 255
        return pack((hi << U64(8)) | U64(255), 0, 0, low)
    raise KeyError(kind)


DISTRIBUTIONS = {
    "constant": {"total_bits": 9, "const_passes": [0, 1]},
    "sorted": {"sorted_input": True},
    "reversed": {"reversed_input": True},
    "alternating": {},
    "top_digit_only": {"total_bits": 24, "const_passes": [0, 1], "const_digit": {0: 255, 1: 255}},
    "hot_key": {},
    "zipf_rows": {},
    "below_20": {"identity": True, "total_bits": 0},
    "digit_255": {"total_bits": 16, "const_passes": [0], "const_digit": {0: 255}},
}
DIST_N = 5 * sm.BIG_TILE + 1001  # odd


def _distribution_cases() -> List[Case]:
    out = []
    for kind, claims in DISTRIBUTIONS.items():
        for path, opts in SETTINGS.items():
            name = f"dist_{kind}_{path}"
            out.append(Case(name, f"{kind} keys on the {path} passes",
                            (lambda k, nm: lambda G: _distribution(k, nm, DIST_N))(kind, name), opts, dict(claims, path=path),
                            n=lambda G: DIST_N))
    return out


def _max_digit_tail(name: str, tile: int, widths, last: int) -> np.ndarray:
    """3 tiles + 7 keys of `widths`, whose pass `last` has fewer than 8 bits; the 7 keys of the
    last tile, and every fifth key before them, carry all ones in that digit: the padding's digit."""
    n = 3 * tile + 7
    k = random_fields(name, n, widths)
    d = sm.make_plan(0, [(1 << w) - 1 for w in widths]).passes[last]
    top = U64(sum(((1 << w) - 1) << s for s, w in zip(d.shift, d.width)))
    k[3 * tile:] |= top
    k[2:3 * tile:5] |= top
    return k


def _tail_cases() -> List[Case]:
    out = []
    for path, opts in SETTINGS.items():
        tile = sm.tile_keys(path)
        for widths, last in (((0, 0, 5), 0), ((8, 0, 3), 1), ((4, 4, 7), 1)):
            name = f"tail_{'_'.join(map(str, widths))}_{path}"
            out.append(Case(name, f"the last tile's 7 real keys carry the padding digit of a {_sizes(sum(widths))[last]}-bit pass ({path})",
                            (lambda nm, t, w, l: lambda G: _max_digit_tail(nm, t, w, l))(name, tile, widths, last), opts,
                            {"path": path, "last_tile": 7, "last_max_digit": last, "sizes": _sizes(sum(widths))},
                            n=(lambda t: lambda G: 3 * t + 7)(tile)))
    return out


def _size_cases() -> List[Case]:
    out = []
    sizes = {"sweep4": [1, 2, 3, 1023, 1024, 1025, 2047, 2049],
             "sweep16": [1024, 1025, 4095, 4096, 4097, 8191, 8193],
             "wide": [1024, 1025, 4095, 4096, 4097, 8191, 8193]}
    for path, ns in sizes.items():
        for n in ns:
            name = f"size_{n}_{path}"
            out.append(Case(name, f"{n} keys on the {path} passes",
                            (lambda nm, nn: lambda G: random_fields(nm, nn, (5, 4, 3)))(name, n), SETTINGS[path],
                            {"path": path, "last_tile": n % sm.tile_keys(path) or sm.tile_keys(path)}, n=(lambda nn: lambda G: nn)(n)))
    return out


WIDE_TILES = ["1", "2", "3", "G-1", "G", "G+1", "2G", "2G+1", "3G", "3G+1", "511", "512", "513", "1024", "1025", "8193"]
WIDE_LAST = [1, 2, 4095, 4096]
WIDE_WIDTHS = [(0, 8, 8), (1, 1, 6), (5, 5, 5), (0, 0, 11)]  # 16, 8, 15, 11 bits: a host sort on 16-bit values


def _wide_tiles(spec: str, G: int) -> int:
    mult, _, rest = spec.partition("G")
    if "G" not in spec:
        return int(spec)
    return (int(mult) if mult else 1) * G + (int(rest) if rest else 0)


def _wide_cases() -> List[Case]:
    out = []
    for ti, spec in enumerate(WIDE_TILES):
        for li, last in enumerate(WIDE_LAST):
            if spec == "1" and last < sm.SMALL_TILE:
                continue  # fewer than 1024 keys never reach the wide passes
            w = WIDE_WIDTHS[(ti + li) % len(WIDE_WIDTHS)]
            name = f"wide_{spec}_last{last}"
            n_of = (lambda s, l: lambda G: (_wide_tiles(s, G) - 1) * sm.BIG_TILE + l)(spec, last)
            claims = {"path": "wide", "tiles": spec, "last_tile": last, "total_bits": sum(w)}
            out.append(Case(name, f"{spec} tiles, {last} keys in the last one, widths {w}",
                            (lambda nm, nf, ww: lambda G: random_fields(nm, nf(G), ww))(name, n_of, w), WIDE, claims, n=n_of))
    return out


# The largest case: 2^27 keys whose 24 sorted bits are a bijection of the key's index modulo 2^24,
# so the sorted array is known without a host sort.
BIG_A, BIG_BITS = 0x9E3779, 24  # odd multiplier


def _big_pack(v: np.ndarray, i: np.ndarray) -> np.ndarray:
    return pack(v & U64(0xFF), (v >> U64(8)) & U64(0xFF), v >> U64(16), i >> U64(7))


def _big_keys(G: int = 0, lo: int = 0, hi: int = MAX_N) -> np.ndarray:
    i = np.arange(lo, hi, dtype=np.uint64)
    return _big_pack((i * U64(BIG_A)) & U64((1 << BIG_BITS) - 1), i)


def _big_expected(G: int = 0, lo: int = 0, hi: int = MAX_N) -> np.ndarray:
    """Sorted position p holds the (p % 8)-th key (in input order) of value p // 8."""
    p = np.arange(lo, hi, dtype=np.uint64)
    v, j = p >> U64(3), p & U64(7)
    inv = pow(BIG_A, -1, 1 << BIG_BITS)
    i = ((v * U64(inv)) & U64((1 << BIG_BITS) - 1)) + (j << U64(BIG_BITS))
    return _big_pack(v, i)


def _big_case() -> Case:
    return Case("big_2p27", "2^27 keys, 3 passes, 64 tiles per chunk of the tile scan", _big_keys, SWEEP4,
                {"path": "wide", "total_bits": 24, "sizes": [8, 8, 8], "tiles_per_chunk": 64}, n=lambda G: MAX_N,
                analytic=True, expected=_big_expected)


CASES: Dict[str, Case] = {c.name: c for c in
                          _shape_cases() + _distribution_cases() + _tail_cases() + _size_cases() + _wide_cases() + [_big_case()]}


# ---- pairs -----------------------------------------------------------------------------------
PAIR_TILES = {4: {"sort_big_log2": 19}, 16: {"sort_big_log2": 10}}  # keys per thread -> option
PAIR_N = 6 * sm.BIG_TILE + 333
PAIR_KINDS = {  # kind -> field widths per layout (least significant field first)
    "random": {0: (9, 8, 7), 1: (8, 9, 7)},
    "straddle": {0: (3, 2, 3), 1: (5, 12, 2)},
    "full": {0: (21, 12, 11), 1: (12, 21, 11)},
}


def pair_keys(kind: str, layout: int, n: int = PAIR_N) -> np.ndarray:
    name = f"pair_{kind}_{layout}_{n}"
    if kind in PAIR_KINDS:
        return random_fields(name, n, PAIR_KINDS[kind][layout], layout)
    k = _distribution(kind, name, n)  # built as segment keys: reuse the words under either layout
    return k


PAIR_DISTRIBUTIONS = ["constant", "sorted", "reversed", "top_digit_only", "hot_key", "digit_255", "below_20"]
PAIR_MAX_N = 1 << 21  # the painter's pair sorts stay below a few million entries


# ---- verification of the claims (CPU) --------------------------------------------------------
def plan_of(keys: np.ndarray, layout: int = 0) -> sm.Plan:
    return sm.make_plan(layout, sm.bounds_of(keys, layout))


def check_claims(case: Case, keys: np.ndarray, G: int) -> List[str]:
    """The claims of `case` that `keys` do not meet (empty: all met)."""
    c, bad = case.claims, []
    n = keys.size
    big, scan = case.opts["sort_big_log2"], case.opts["sort_scan_log2"]
    path = sm.key_path(n, big, scan)
    plan = plan_of(keys, case.layout)
    tile = sm.tile_keys(path)
    tiles = sm.tiles_of(n, tile)

    def claim(key, got, want=None):
        want = c[key] if want is None else want
        if got != want:
            bad.append(f"{key}: {got!r}, claimed {want!r}")

    if "path" in c:
        claim("path", path)
    if "total_bits" in c:
        claim("total_bits", plan.total_bits)
    if "sizes" in c:
        claim("sizes", plan.sizes())
    for p, runs in c.get("runs", {}).items():
        claim("runs", plan.passes[p].runs, runs)
    digits = [sm.digit_of(keys, d) for d in plan.passes] if any(k in c for k in ("const_passes", "const_digit", "last_max_digit")) else []
    for p in c.get("const_passes", []):
        if p >= len(digits) or np.unique(digits[p]).size != 1:
            bad.append(f"const_passes: pass {p} has several digits (or does not exist)")
    for p, d in c.get("const_digit", {}).items():
        if not np.all(digits[p] == d):
            bad.append(f"const_digit: pass {p} is not all {d}")
    if "last_tile" in c:
        claim("last_tile", n - (tiles - 1) * tile)
    if "last_max_digit" in c:
        p = c["last_max_digit"]
        top = (1 << plan.passes[p].bits) - 1
        tail = digits[p][(tiles - 1) * tile:]
        if plan.passes[p].bits >= 8 or not np.all(tail == top) or not np.any(digits[p][:(tiles - 1) * tile] == top) or \
                np.all(digits[p] == top):
            bad.append(f"last_max_digit: pass {p} ({plan.passes[p].bits} bits)")
    if "tiles" in c:
        claim("tiles", tiles, _wide_tiles(c["tiles"], G))
    if "tiles_per_chunk" in c:
        claim("tiles_per_chunk", sm.scan_shape(tiles)[0])
    if c.get("identity") and plan.n_passes != 0:
        bad.append("identity: the plan has passes")
    v = keys >> U64(20)
    if c.get("sorted_input") and not (np.all(v[1:] >= v[:-1]) and v[0] != v[-1]):
        bad.append("sorted_input")
    if c.get("reversed_input") and not (np.all(v[1:] <= v[:-1]) and v[0] != v[-1]):
        bad.append("reversed_input")
    return bad


def ring_facts(tiles: int, G: int) -> Dict[str, int]:
    """How the persistent downsweep spreads `tiles` over its grid of min(tiles, G) CTAs."""
    grid = min(tiles, G)
    tpc, chunks, supers = sm.scan_shape(tiles)
    return {"grid": grid, "cta0_tiles": sm.tiles_owned(0, tiles, grid), "cta_last_tiles": sm.tiles_owned(grid - 1, tiles, grid),
            "rounds": -(-tiles // grid), "tiles_per_chunk": tpc, "chunks": chunks, "supers": supers}


def host_sorted(keys: np.ndarray, layout: int = 0) -> Tuple[np.ndarray, np.ndarray]:
    """(sorted keys, the permutation) of a stable sort on the fields: by 16-bit radix passes when
    the participating bits fit 16, by a stable sort of the virtual key otherwise."""
    bound = sm.bounds_of(keys, layout)
    v = sm.virtual_key(keys, layout, bound)
    if sum(sm.field_widths(layout, bound)) <= 16:
        v = v.astype(np.uint16)
    order = np.argsort(v, kind="stable")
    return keys[order], order
