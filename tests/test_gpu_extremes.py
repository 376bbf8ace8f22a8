"""Parity at the limits of the painter and its tables (scenes: tests/extremes.py): cells of
thousands of segments and cells across CTA tiles of the cells pass, pixel areas beyond i16,
windings that wrap the i8 covers, tiles with up to 5000 entries and clips across 32-entry
groups, lines of 12 k segments and geometry far outside the frame, and non-separable blends
whose channels become NaN (encoded as byte 0, like the reference on a CPU; also in BGRA order).

For every scene the CUDA library and the oracle must agree on the frame (byte for byte), the
pixel-segment count and the sorted segments (as multisets), and the cell / entry counts of the
painter tables must equal both the GPU's counters and tests/tables_model.py, a second
reference computed from the oracle's segments. Each scene is rendered by one fresh renderer
twice (tables built with count read-backs, then sync-free), once with one copy band and once
into device memory; the crowds then run three frames with a layer cache while a layer deep in
the stack moves."""
import numpy as np
import pytest

import extremes
import tables_model as tm
from forma_b200.binding import BGRA, RGBA, Color

pytestmark = pytest.mark.gpu

CLEAR = Color(1.0, 1.0, 1.0, 0.0)


def _diff_report(got, want, sc, tc, what):
    if np.array_equal(got, want):
        return
    w, h = sc.width, sc.height
    a4, b4 = got.reshape(h, w, 4).astype(int), want.reshape(h, w, 4).astype(int)
    d = np.abs(a4 - b4).max(axis=2)
    ys, xs = np.nonzero(d)
    y, x = int(ys[0]), int(xs[0])
    ty, tx = y // 16, x // 16
    in_tile = (tc.cell_keys[:, 0] == ty) & (tc.cell_keys[:, 1] == tx)
    tiles = sorted({(int(v) // 16, int(u) // 16) for v, u in zip(ys[:2000], xs[:2000])})
    raise AssertionError(
        f"{what}: {len(ys)} pixels differ (max channel diff {d.max()}), first at x={x} y={y} (tile x={tx} y={ty}): "
        f"cuda {a4[y, x].tolist()} oracle {b4[y, x].tolist()}; that tile has {int(in_tile.sum())} cells "
        f"(largest {int(tc.cell_sizes[in_tile].max()) if in_tile.any() else 0} segments) and "
        f"{tc.gaps_per_tile.get((ty, tx), 0)} carry-only entries in the model; "
        f"{len(tiles)} tiles among the first 2000 differing pixels, e.g. {tiles[:6]}")


@pytest.fixture(scope="module")
def expected(oracle_api):
    """Oracle frame, sorted segments and model counts per scene (built on first use)."""
    memo = {}

    def get(name):
        if name not in memo:
            comp, built, sc = extremes.build(oracle_api, name)
            r = oracle_api.Renderer(0)
            buf = np.zeros(sc.width * sc.height * 4, np.uint8)
            t = r.render(comp, buf, sc.width, sc.height, RGBA, CLEAR, sc.crop)
            segs = r.segments()
            raster = r.rasterize_only(comp, sc.width, sc.height) if sc.raster else None
            tc = tm.table_counts(segs, sc.width, sc.height, built.rules, sc.crop)
            memo.clear()  # one scene at a time: the 8K and far-geometry scenes are large
            memo[name] = (buf, int(t.n_segments), np.sort(segs), raster, tc)
        return memo[name]
    return get


@pytest.fixture()
def copy_bands_restored(cuda_api):
    saved = cuda_api.get_option("copy_bands")
    yield
    cuda_api.set_option("copy_bands", saved)


@pytest.mark.parametrize("name", list(extremes.SCENES))
def test_extreme_scene_matches_oracle_and_table_model(cuda_api, oracle_api, expected, unsliced, copy_bands_restored, name):
    want, n_want, segs_want, raster_want, tc = expected(name)
    oracle_comp = extremes.build(oracle_api, name)[0] if "nan" in extremes.SCENES[name].tags else None
    comp, built, sc = extremes.build(cuda_api, name)
    w, h = sc.width, sc.height
    r = cuda_api.Renderer(0)
    modes = []
    for attempt in range(2):  # frame 1: counts read back (tables_mode 0); frame 2: sync-free (1)
        buf = np.zeros(w * h * 4, np.uint8)
        t = r.render(comp, buf, w, h, RGBA, CLEAR, sc.crop)
        c = r.counters()
        modes.append(c["tables_mode"])
        _diff_report(buf, want, sc, tc, f"{name} frame {attempt + 1}")
        assert int(t.n_segments) == n_want, f"{name}: {t.n_segments} pixel segments on the device, {n_want} in the oracle"
        assert (c["cells"], c["entries"]) == (tc.cells, tc.entries), \
            f"{name} frame {attempt + 1}: device cells/entries {c['cells']}/{c['entries']}, model {tc.cells}/{tc.entries}"
        segs = r.segments()
        assert segs.size == segs_want.size
        assert np.array_equal(np.sort(segs), segs_want), f"{name}: sorted segments differ from the oracle's"
        del segs
    assert modes == [0, 1], modes

    cuda_api.set_option("copy_bands", 1)
    buf = np.zeros(w * h * 4, np.uint8)
    r.render(comp, buf, w, h, RGBA, CLEAR, sc.crop)
    _diff_report(buf, want, sc, tc, f"{name} with one copy band")

    import torch
    dev = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda:0")
    r.render_device(comp, dev.data_ptr(), w, h, RGBA, CLEAR, sc.crop)
    torch.cuda.synchronize()
    _diff_report(dev.cpu().numpy(), want, sc, tc, f"{name} into device memory")
    del dev

    if "nan" in sc.tags:  # the encoder of other channel orders (and of solid tiles) as well
        frames = []
        for api, rr, cc in ((cuda_api, r, comp), (oracle_api, oracle_api.Renderer(0), oracle_comp)):
            b2 = np.zeros(w * h * 4, np.uint8)
            rr.render(cc, b2, w, h, BGRA, CLEAR, sc.crop)
            frames.append(b2)
        _diff_report(frames[0], frames[1], sc, tc, f"{name} in BGRA order")

    if sc.raster:
        got = r.rasterize_only(comp, w, h)
        assert got.shape == raster_want.shape, f"{name}: {got.size} vs {raster_want.size} unsorted segments"
        assert np.array_equal(got, raster_want), f"{name}: unsorted segments differ (emission order)"


@pytest.mark.parametrize("name", [n for n, s in extremes.SCENES.items() if "crowd" in s.tags])
def test_crowd_with_layer_cache_while_a_deep_layer_moves(cuda_api, oracle_api, name):
    """One frame without a cache, then three with one; a layer a third of the way up the stack
    moves between the cached frames on both sides."""
    sides = []
    for api in (cuda_api, oracle_api):
        comp, built, sc = extremes.build(api, name)
        r = api.Renderer(0)
        sides.append((comp, built, r, r.create_buffer_layer_cache(), np.zeros(sc.width * sc.height * 4, np.uint8)))
    w, h = sc.width, sc.height
    for comp, built, r, cache, buf in sides:
        r.render(comp, buf, w, h, RGBA, CLEAR)
    tc = tm.table_counts(sides[1][2].segments(), w, h, sides[1][1].rules)
    _diff_report(sides[0][4], sides[1][4], sc, tc, f"{name} without cache")
    for frame in range(1, 4):
        for comp, built, r, cache, buf in sides:
            if frame > 1:
                built.animate(frame)
            r.render(comp, buf, w, h, RGBA, CLEAR, None, cache)
        tc = tm.table_counts(sides[1][2].segments(), w, h, sides[1][1].rules)
        _diff_report(sides[0][4], sides[1][4], sc, tc, f"{name} cached frame {frame}")
