"""Every key set of tests/sort_scenes.py meets the condition it declares and stays within budget,
proved on the CPU with tests/sort_model.py before tests/test_gpu_sort.py gives it to a kernel."""
import numpy as np
import pytest

import sort_model as sm
import sort_scenes as ss

U64 = np.uint64
SMALL = [n for n, c in ss.CASES.items() if not c.analytic]


@pytest.mark.parametrize("G", ss.GRIDS)
def test_every_case_is_within_budget(G):
    for name, c in ss.CASES.items():
        n = c.n(G)
        assert 0 < n <= ss.MAX_N < (1 << 30), name
        assert ss.device_bytes(n) <= ss.MAX_DEVICE_BYTES, name
        assert set(c.opts) == {"sort_big_log2", "sort_scan_log2"}, name
    assert ss.device_bytes(ss.PAIR_MAX_N, pairs=True) <= ss.MAX_DEVICE_BYTES
    assert sum(c.n(G) for c in ss.CASES.values()) < 3 * ss.MAX_N  # what one run of the GPU test sorts


@pytest.mark.parametrize("G", ss.GRIDS)
def test_every_case_meets_its_claims(G):
    for name in SMALL:
        c = ss.CASES[name]
        if G != ss.GRIDS[0] and "G" not in str(c.claims.get("tiles", "")):
            continue  # only the wide sizes depend on the grid
        keys = c.keys(G)
        assert keys.dtype == np.uint64 and keys.size == c.n(G), name
        if keys.size <= 1 << 20:
            assert np.array_equal(keys, c.keys(G)), f"{name} is not a pure function of its name"
        assert not ss.check_claims(c, keys, G), (name, ss.check_claims(c, keys, G))
        # Bits [0, 20) must travel untouched and in stable order: they are never constant.
        low = keys[:65536] & U64(0xFFFFF)
        assert keys.size < 64 or np.unique(low).size > low.size // 4, name


def test_all_conditions_are_present():
    claims = [c.claims for c in ss.CASES.values()]
    for total in (1, 7, 8, 9, 15, 16, 17, 24, 25, 43, 44, 0):
        assert any(c.get("total_bits") == total for c in claims), total
    for path in ss.SETTINGS:
        assert any(c.get("path") == path and 3 in c.get("runs", {}).values() for c in claims), path
        assert any(c.get("path") == path and 2 in c.get("runs", {}).values() for c in claims), path
        assert any(c.get("path") == path and "last_max_digit" in c for c in claims), path
        assert any(c.get("path") == path and c.get("identity") for c in claims), path
        assert any(c.get("path") == path and c.get("const_digit") for c in claims), path
    # odd and even pass counts (the sorted keys end in either buffer), odd and even n
    passes = {len(c["sizes"]) for c in claims if "sizes" in c}
    assert {1, 2, 3, 4, 6} <= passes
    assert {c.n(264) % 2 for c in ss.CASES.values()} == {0, 1}


@pytest.mark.parametrize("G", ss.GRIDS)
def test_the_ring_and_the_tile_scan_are_run_at_their_edges(G):
    """What the wide sizes make of the persistent downsweep (CTA c owns tiles c, c + grid, ...;
    sort_model.DS_STAGES - 1 = 2 copies are issued up front) and of the tile scan."""
    facts = {spec: ss.ring_facts(ss._wide_tiles(spec, G), G) for spec in ss.WIDE_TILES}
    assert sm.DS_STAGES - 1 == 2
    assert facts["1"]["grid"] == 1 and facts["1"]["cta0_tiles"] == 1         # one copy up front, nothing after
    assert facts["2"]["grid"] == 2 and facts["3"]["cta_last_tiles"] == 1
    assert facts["G-1"]["grid"] == G - 1 and facts["G-1"]["cta0_tiles"] == 1   # a grid smaller than G
    assert facts["G"]["cta0_tiles"] == facts["G"]["cta_last_tiles"] == 1
    assert facts["G+1"]["cta0_tiles"] == 2 and facts["G+1"]["cta_last_tiles"] == 1  # exactly the up-front copies
    assert facts["2G"]["cta0_tiles"] == facts["2G"]["cta_last_tiles"] == 2
    assert facts["2G+1"]["cta0_tiles"] == 3 and facts["2G+1"]["cta_last_tiles"] == 2  # first copy issued inside the loop
    assert facts["3G"]["cta_last_tiles"] == 3 and facts["3G+1"]["cta0_tiles"] == 4   # a stage reused
    assert facts["8193"]["rounds"] >= 2 * sm.DS_STAGES * 2  # every stage's phase bit flips several times
    # tile scan: tiles per chunk 1 -> 2 at 513 tiles, 2 -> 3 at 1025; super-chunks every 16 chunks
    assert [facts[s]["tiles_per_chunk"] for s in ("511", "512", "513", "1024", "1025", "8193")] == [1, 1, 2, 2, 3, 17]
    assert facts["512"]["chunks"] == 512 and facts["512"]["supers"] == 32
    assert facts["513"]["chunks"] == 257 and facts["513"]["supers"] == 17  # chunk rows past the last are read as zeros
    assert facts["1025"]["chunks"] == 342 and facts["8193"]["chunks"] == 482
    assert facts["G"]["supers"] == -(-G // 16) and facts["G+1"]["supers"] == -(-(G + 1) // 16)
    for last in ss.WIDE_LAST:  # every size exists with each last tile
        for spec in ss.WIDE_TILES[1:]:
            c = ss.CASES[f"wide_{spec}_last{last}"]
            assert c.n(G) == (ss._wide_tiles(spec, G) - 1) * sm.BIG_TILE + last
            assert sm.key_path(c.n(G), c.opts["sort_big_log2"], c.opts["sort_scan_log2"]) == "wide"


def test_the_largest_case_and_its_expected_order():
    c = ss.CASES["big_2p27"]
    assert c.n(0) == 1 << 27 and sm.key_path(c.n(0), 19, 22) == "wide"
    assert sm.scan_shape(sm.tiles_of(c.n(0), sm.BIG_TILE))[0] == c.claims["tiles_per_chunk"] == 64
    # The keys' OR over a window that holds every value of the 24 sorted bits once.
    k = ss._big_keys(lo=0, hi=1 << 18)
    assert sm.make_plan(0, sm.bounds_of(k, 0)).sizes() == c.claims["sizes"]
    assert ss.BIG_A % 2 == 1  # odd: index -> value is a bijection modulo 2^24, every value 8 times in 2^27 keys
    # The analytic order is the stable order: checked in full on the same construction at 2^20
    # keys of 17 sorted bits, and on windows of the real one.
    A, bits, n = ss.BIG_A, 17, 1 << 20
    i = np.arange(n, dtype=np.uint64)
    small = ((i * U64(A)) & U64((1 << bits) - 1)) << U64(20) | (i >> U64(7))
    p = np.arange(n, dtype=np.uint64)
    inv = pow(A, -1, 1 << bits)
    src = (((p >> U64(3)) * U64(inv)) & U64((1 << bits) - 1)) + ((p & U64(7)) << U64(bits))
    assert np.array_equal(small[np.argsort(small >> U64(20), kind="stable")], small[src.astype(np.int64)])
    for lo in (0, (1 << 26) - 5, (1 << 27) - 4096):
        e = ss._big_expected(lo=lo, hi=lo + 4096)
        v = e >> U64(20)
        assert np.all(v[1:] >= v[:-1])
        # each expected key is the input key of the index packed into its low bits and value
        val = ((e >> U64(20)) & U64(0xFF)) | (((e >> U64(41)) & U64(0xFF)) << U64(8)) | ((e >> U64(53)) << U64(16))
        inv24 = pow(A, -1, 1 << 24)
        idx = ((val * U64(inv24)) & U64((1 << 24) - 1)) + (np.arange(lo, lo + 4096, dtype=np.uint64) & U64(7)) * U64(1 << 24)
        assert np.array_equal(e, np.concatenate([ss._big_keys(lo=int(j), hi=int(j) + 1) for j in idx[:64]] +
                                                [ss._big_keys(lo=int(j), hi=int(j) + 1) for j in idx[64:]]))


def test_pair_key_sets():
    for layout in (0, 1):
        for kind, widths in ss.PAIR_KINDS.items():
            k = ss.pair_keys(kind, layout)
            assert sm.field_widths(layout, sm.bounds_of(k, layout)) == list(widths[layout]), (kind, layout)
            plan = ss.plan_of(k, layout)
            if kind == "straddle":
                assert max(d.runs for d in plan.passes) >= 2 + (layout == 0)
        for kind in ss.PAIR_DISTRIBUTIONS:
            k = ss.pair_keys(kind, layout)
            assert k.size == ss.PAIR_N and k.size % 2 == 1
        assert ss.plan_of(ss.pair_keys("below_20", layout), layout).n_passes == 0
    assert sm.tiles_of(ss.PAIR_N, sm.SMALL_TILE) > 4 and sm.tiles_of(ss.PAIR_N, sm.BIG_TILE) > 4


def test_host_sorted_is_the_stable_sort_on_bits_20_up():
    for name in ("shape_bits16_wide", "shape_bits44_sweep4", "wide_3_last2", "dist_hot_key_sweep16", "tail_0_0_5_wide"):
        k = ss.CASES[name].keys()
        out, order = ss.host_sorted(k)
        assert np.array_equal(order, np.argsort(k >> U64(20), kind="stable")), name
        assert np.array_equal(out, k[order])


# ---- the checks bite ---------------------------------------------------------------------------
def test_a_wrong_claim_is_caught():
    c = ss.CASES["tail_0_0_5_wide"]
    k = c.keys()
    assert not ss.check_claims(c, k, 264)
    assert ss.check_claims(c, k[:-1], 264)                       # 6 real keys in the last tile
    k2 = k.copy()
    k2[-3] &= U64((1 << 53) - 1)                                   # one tail key without the padding digit
    assert ss.check_claims(c, k2, 264)
    c = ss.CASES["shape_runs_1_1_6_sweep16"]
    assert ss.check_claims(c, c.keys() & ~U64(1 << 41), 264)     # the tile_x bit gone: two runs, 7 bits
    c = ss.CASES["wide_G+1_last1"]
    assert not ss.check_claims(c, c.keys(228), 228) and ss.check_claims(c, c.keys(228), 264)


def test_the_tile_bound_model_and_its_mutations():
    """The bound of a tile field (line_count_body): the largest biased tile any segment of the
    lines can carry fits the bit length of the bound; without the two tiles of slack, or without
    the far rule, it does not."""
    f32 = np.float32
    # sub-pixel extents of lines along one axis: [lo, hi]
    hi = np.array([255.4, 255.5, 4095.0, 16.0 * 1920, 3.1e7, -50.0], f32)
    lo = np.array([0.0, 100.0, -300.0, 0.0, 0.0, -4000.0], f32)
    true_tile = [1 + 1, 1 + 1, 15 + 1, 120 + 1, None, 0]  # biased tile of round(hi) (None: clamped)
    for k in range(len(hi)):
        b = sm.tile_bound(lo[k:k + 1], hi[k:k + 1], 4095)
        if true_tile[k] is None:
            assert b == 4095
        else:
            assert true_tile[k] <= b <= true_tile[k] + 1
    assert sm.tile_bound(lo[:1], np.array([255.5], f32), 4095) == 3            # rounds up into tile 1, biased 2, + 1 slack
    assert sm.tile_bound(lo[:1], np.array([255.5], f32), 4095, slack=0) == 1   # "+ 2 -> + 0": biased 2 does not fit 1 bit
    assert (1).bit_length() < (2).bit_length()
    # a line from inside the frame to 2^20 px left (or above): every bit of the field can be set
    far_lo = np.array([-16.0 * 2 ** 20], f32)
    assert sm.tile_bound(far_lo, np.array([160.0], f32), 4095) == 4095 and sm.tile_bound(far_lo, np.array([160.0], f32), 2047) == 2047
    assert sm.tile_bound(far_lo, np.array([160.0], f32), 4095, far_rule=False) == 2
    # the rule starts two tiles before the int16 wrap (tile -32769 is the first to wrap)
    assert sm.tile_bound(np.array([-32767.0 * 256 - 1], f32), np.array([160.0], f32), 4095) == 4095
    assert sm.tile_bound(np.array([-32767.0 * 256], f32), np.array([160.0], f32), 4095) == 2
    def biased(tile):  # the emit pass: `as i16` of the tile, + 1, `as i16` again, negative -> 0, 12 bits
        t16 = int(np.array(tile).astype(np.int16))
        return max(int(np.array(t16 + 1).astype(np.int16)), 0) & 0xFFF
    assert [biased(t) for t in (-1, 0, -32768, -32769)] == [0, 1, 0, 0] and biased(-32770) == 4095 and biased(-65536 + 4) == 5
    assert -32770 * 256.0 < sm.FAR_EDGE < -32766 * 256.0
    assert sm.tile_bound(np.array([np.nan], f32), np.array([np.nan], f32), 4095) == 4095  # NaN: fminf gives 3e7
