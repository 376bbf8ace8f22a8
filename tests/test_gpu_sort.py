"""The sorts on the device against a host sort, at tolerance 0 and in order (not as multisets).

- Every key set of tests/sort_scenes.py (each proved on the CPU by tests/test_sort_scenes.py to
  meet the condition it is there for) through Renderer.sort_u64 under the size options that send
  it to the 1024-key single-sweep passes, the 4096-key ones, or the reduce-then-scan passes.
- The pair sorts of the painter tables through Renderer.sort_pairs: payload = original index, so
  the expected payload is the stable argsort itself; both key layouts, both tile sizes, the count
  on the host or in device memory, the histogram counted by the sort or before it.
- Frames: the segments a frame leaves behind are in order on bits [20, 64) as returned, and the
  bounds its plan was built from cover every field without sorting bits nobody needs.
"""
import numpy as np
import pytest

import batch_scenes as bs
import line_scenes as ls
import scenes
import sort_model as sm
import sort_scenes as ss
import view_scenes as vs
from forma_b200.binding import RGBA, Color, FormaError, Rect

pytestmark = pytest.mark.gpu
U64 = np.uint64
CLEAR = Color(1.0, 1.0, 1.0, 0.0)
SORT_OPTIONS = ("sort_big_log2", "sort_scan_log2", "sort_full_key")


@pytest.fixture()
def sort_options(cuda_api):
    """set(**options) for the test; the three sort options are put back afterwards."""
    saved = {k: cuda_api.get_option(k) for k in SORT_OPTIONS}

    def set_options(**opts):
        for k, v in opts.items():
            assert k in SORT_OPTIONS
            cuda_api.set_option(k, v)
    yield set_options
    for k, v in saved.items():
        cuda_api.set_option(k, v)


@pytest.fixture(scope="module")
def grid():
    """CTAs of the persistent downsweep: two per SM."""
    import torch
    return 2 * torch.cuda.get_device_properties(0).multi_processor_count


def explain(got, want, keys, case_opts, layout=0):
    """Where and how two key arrays differ: index, tiles, the plan and both keys' digits."""
    if got.shape != want.shape:
        return f"{got.size} keys came back for {want.size}"
    at = int(np.flatnonzero(got != want)[0])
    plan = ss.plan_of(keys, layout)
    n_bad = int(np.count_nonzero(got != want))
    dg = [int(sm.digit_of(got[at:at + 1], d)[0]) for d in plan.passes]
    dw = [int(sm.digit_of(want[at:at + 1], d)[0]) for d in plan.passes]
    is_input = "is" if np.any(keys == got[at]) else "is NOT"
    return (f"first difference at index {at} of {want.size} ({n_bad} differ): 4096-key tile {at // 4096} slot {at % 4096}, "
            f"1024-key tile {at // 1024} slot {at % 1024}; options {case_opts}; plan: {plan.describe()}; "
            f"got {int(got[at]):#018x} digits {dg} (this key {is_input} one of the input's), "
            f"want {int(want[at]):#018x} digits {dw}")


def _run_case(r, sort_options, name, G):
    c = ss.CASES[name]
    keys = c.keys(G)
    assert keys.size == c.n(G) <= ss.MAX_N and not ss.check_claims(c, keys, G), name
    sort_options(**c.opts)
    got = r.sort_u64(keys)
    want, _ = ss.host_sorted(keys)
    assert np.array_equal(got, want), f"{name} ({c.target}): " + explain(got, want, keys, c.opts)
    if c.claims.get("identity"):
        assert np.array_equal(got, keys)


GROUPS = {g: [n for n in ss.CASES if n.startswith(g + "_")] for g in ("shape", "dist", "tail", "size")}


@pytest.mark.parametrize("group", sorted(GROUPS))
def test_key_sets_sort_like_a_stable_host_sort(cuda_renderer, sort_options, grid, group):
    assert GROUPS[group]
    for name in GROUPS[group]:
        _run_case(cuda_renderer, sort_options, name, grid)


@pytest.mark.parametrize("spec", ss.WIDE_TILES)
def test_downsweep_ring_and_tile_scan_sizes(cuda_renderer, sort_options, grid, spec):
    """Tile counts around the grid of the persistent downsweep (read from the device) and around
    the steps of the tile scan, each with a last tile of 1, 2, 4095 and 4096 keys."""
    names = [f"wide_{spec}_last{last}" for last in ss.WIDE_LAST if f"wide_{spec}_last{last}" in ss.CASES]
    assert len(names) >= 2
    for name in names:
        _run_case(cuda_renderer, sort_options, name, grid)


def test_the_largest_sort(cuda_renderer, sort_options):
    c = ss.CASES["big_2p27"]
    sort_options(**c.opts)
    got = cuda_renderer.sort_u64(c.keys(0))
    step = 1 << 24
    for lo in range(0, ss.MAX_N, step):
        want = c.expected(0, lo, lo + step)
        if not np.array_equal(got[lo:lo + step], want):
            at = lo + int(np.flatnonzero(got[lo:lo + step] != want)[0])
            pytest.fail(f"big_2p27: first difference at index {at}: 4096-key tile {at // 4096} (chunk {at // 4096 // 64}) slot "
                        f"{at % 4096}; got {int(got[at]):#018x}, want {int(want[at - lo]):#018x}")


def test_refused_and_trivial_sizes(cuda_renderer, cuda_api):
    import ctypes as C
    one = np.array([123 << 20], np.uint64)
    st = cuda_api.renderer_sort_u64(cuda_renderer._h, one.ctypes.data_as(C.POINTER(C.c_uint64)), 1 << 30)
    assert st == 5 and one[0] == 123 << 20  # FORMA_ERR_CAPACITY, refused before the array is read
    assert cuda_renderer.sort_u64(np.zeros(0, np.uint64)).size == 0
    assert np.array_equal(cuda_renderer.sort_u64(one), one)


# ---- pairs -------------------------------------------------------------------------------------
def _pairs(r, keys, layout, mode, count=None, cap=0):
    vals = np.arange(keys.size, dtype=np.uint32)
    return r.sort_pairs(keys, vals, layout=layout, mode=mode, count=count, cap=cap)


def _check_pairs(got, keys, layout, what):
    want_k, order = ss.host_sorted(keys, layout)
    gk, gv = got
    assert np.array_equal(gk, want_k), f"{what}: keys: " + explain(gk, want_k, keys, what, layout)
    if not np.array_equal(gv, order.astype(np.uint32)):
        at = int(np.flatnonzero(gv != order)[0])
        pytest.fail(f"{what}: payload differs first at {at} (1024-key tile {at // 1024}, 4096-key tile {at // 4096}): "
                    f"got {int(gv[at])}, want {int(order[at])}; plan: {ss.plan_of(keys, layout).describe()}")


@pytest.mark.parametrize("items", sorted(ss.PAIR_TILES))
@pytest.mark.parametrize("layout", [0, 1])
def test_pair_sorts(cuda_renderer, sort_options, layout, items):
    sort_options(**ss.PAIR_TILES[items])
    for kind in list(ss.PAIR_KINDS) + ss.PAIR_DISTRIBUTIONS:
        keys = ss.pair_keys(kind, layout)
        for mode in range(4):
            cap = keys.size + (0 if mode == 1 else 5000)  # a bound above the count too
            got = _pairs(cuda_renderer, keys, layout, mode, cap=cap)
            _check_pairs(got, keys, layout, f"{kind} layout {layout} mode {mode} {items} keys/thread")
            if kind == "below_20":
                assert np.array_equal(got[1], np.arange(keys.size))


@pytest.mark.parametrize("items", sorted(ss.PAIR_TILES))
@pytest.mark.parametrize("mode", [1, 3])
def test_pair_sorts_with_a_device_count(cuda_renderer, sort_options, mode, items):
    """count = 0, 1, cap - 1, cap; cap + 1 and far above (nothing is sorted, nothing is changed);
    a cap far above the count (the tiles past the count return early, nobody waits for them)."""
    sort_options(**ss.PAIR_TILES[items])
    cap = 3 * 4096 + 17
    full = ss.pair_keys("random", 1, cap)
    for count in (0, 1, cap - 1, cap):
        keys = full[:count]
        got = _pairs(cuda_renderer, keys, 1, mode, count=count, cap=cap)
        if count:
            _check_pairs(got, keys, 1, f"count {count} cap {cap} mode {mode}")
    for count in (cap + 1, 5 * cap, (1 << 30) - 1):
        gk, gv = _pairs(cuda_renderer, full, 1, mode, count=count, cap=cap)
        assert np.array_equal(gk, full) and np.array_equal(gv, np.arange(cap)), f"count {count} > cap {cap}: changed"
    keys = full[:1500]
    _check_pairs(_pairs(cuda_renderer, keys, 1, mode, count=1500, cap=200 * 4096), keys, 1, f"cap >> count, mode {mode}")
    with pytest.raises(FormaError):
        cuda_renderer.sort_pairs(full[:1], np.zeros(1, np.uint32), layout=2)


@pytest.mark.parametrize("layout", [0, 1])
def test_two_million_pairs(cuda_renderer, sort_options, layout):
    sort_options(sort_big_log2=19)
    keys = ss.pair_keys("random", layout, ss.PAIR_MAX_N)
    for mode in (0, 3):
        _check_pairs(_pairs(cuda_renderer, keys, layout, mode, cap=keys.size), keys, layout, f"2^21 pairs mode {mode}")


# ---- frames ------------------------------------------------------------------------------------
TY, TX, LAYER = (53, 11), (41, 12), (20, 21)


def _field(segs, f):
    return (segs >> U64(f[0])) & U64((1 << f[1]) - 1)


def check_frame_sorted(r, what, tile_y_rule="frame", far=False):
    """The last frame's segments, as returned, are in order on bits [20, 64); every field that
    took part fits the bit length of its bound; and a tile bound is no more than one bit wider
    than the largest value needs, except:
      - clamp: a bound at the field's maximum (4095 / 2047) says nothing about the values;
      - far: a line reaches more than 32767 tiles left of (or above) the frame: the field's maximum;
      - stacked: a views / batch call's tile_y bound is (last frame with lines + 1) * rows, whatever
        its lines reach.
    One exception to the order: stacked row 0 (biased tile_y 0) gathers the out-of-view segments of
    every frame of a views / batch call; when the layer digits are left to the emission order it
    is ordered by tile only (no painted tile reads that row)."""
    segs = r.segments()
    b = r.sort_bounds()
    v = segs >> U64(20)
    if tile_y_rule == "stacked" and b["layer"] == 0:
        v = np.where(_field(segs, TY) == 0, v & ~U64((1 << 21) - 1), v)
    if segs.size > 1 and not np.all(v[1:] >= v[:-1]):
        at = int(np.flatnonzero(v[1:] < v[:-1])[0])
        plan = sm.make_plan(0, [b["layer"], b["tile_x"], b["tile_y"]])
        pytest.fail(f"{what}: segments {at} and {at + 1} of {segs.size} are out of order: {int(segs[at]):#018x} > "
                    f"{int(segs[at + 1]):#018x} (tile_y, tile_x, layer = "
                    f"{[int(_field(segs[at:at + 2], f)[0]) for f in (TY, TX, LAYER)]} then "
                    f"{[int(_field(segs[at:at + 2], f)[1]) for f in (TY, TX, LAYER)]}); bounds {b}; plan {plan.describe()}")
    if segs.size == 0:
        return b
    mx = {"tile_y": int(_field(segs, TY).max()), "tile_x": int(_field(segs, TX).max()), "layer": int(_field(segs, LAYER).max())}
    widths = sm.field_widths(0, [b["layer"], b["tile_x"], b["tile_y"]])
    assert b["total_bits"] == sum(widths), what
    for name, w in zip(("layer", "tile_x", "tile_y"), widths):
        if name == "layer" and b["layer"] == 0:
            continue  # inserts in layer order: the layer digits are left to the emission order
        assert mx[name] <= (1 << w) - 1, f"{what}: {name} reaches {mx[name]}, its bound {b[name]} sorts {w} bits"
    for name, top in (("tile_x", 4095), ("tile_y", 2047)):
        if b[name] == top or far or (name == "tile_y" and tile_y_rule == "stacked"):
            continue
        # the bound is the biased tile of the lines' largest end point + 1: at most one more than
        # the largest tile a segment can lie in, which the frame's own segments reach or come close to
        assert b[name].bit_length() <= (mx[name] + 1).bit_length() + 1, f"{what}: {name} bound {b[name]} for a maximum of {mx[name]}"
    return b


def _render_device(r, comp, w, h, crop=None):
    import torch
    t = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda:0")
    r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR, crop)
    torch.cuda.synchronize()
    return t.cpu().numpy()


FAR_LINE_SCENES = ("far_up", "far_left_line", "translations", "nan", "tile_wrap")


@pytest.mark.parametrize("full_key", [0, 1])
@pytest.mark.parametrize("name", ls.IN_LIMIT)
def test_line_scene_frames_are_sorted(cuda_api, sort_options, unsliced, name, full_key):
    sc = ls.SCENES[name]
    sort_options(sort_full_key=full_key)
    comp, _, _ = ls.build(cuda_api, sc.layers)
    r = cuda_api.Renderer(0)
    _render_device(r, comp, sc.width, sc.height)
    b = check_frame_sorted(r, f"{name} full_key {full_key}", far=name in FAR_LINE_SCENES)
    if name == "far_up":
        assert b["tile_y"] == 2047  # by the rows' rule: the lines' largest y is 20 px
    if name == "far_left_line":
        assert b["tile_x"] == 4095  # by the columns' rule: the lines' largest x is 20 px
    for crop in sc.crops:
        _render_device(r, comp, sc.width, sc.height, Rect(crop[0:2], crop[2:4]))
        check_frame_sorted(r, f"{name} crop {crop}", far=name in FAR_LINE_SCENES)


def test_inserts_out_of_layer_order_sort_their_layer_digits(cuda_api, sort_options, unsliced):
    specs = [ls.LayerSpec(o, None, [ls.star(60 + 7 * k, 60, 10, 40, 5)]) for k, o in enumerate((9, 2, 300, 5, 0, 77))]
    comp, _, _ = ls.build(cuda_api, specs)
    r = cuda_api.Renderer(0)
    for full_key in (0, 1):
        sort_options(sort_full_key=full_key)
        _render_device(r, comp, 256, 128)
        b = check_frame_sorted(r, f"out of order, full_key {full_key}")
        assert b["layer"] == 300
    ordered = [ls.LayerSpec(o, None, [ls.star(60 + 7 * o, 60, 10, 40, 5)]) for o in range(6)]
    comp, _, _ = ls.build(cuda_api, ordered)
    for full_key, want in ((0, 0), (1, 5)):
        sort_options(sort_full_key=full_key)
        _render_device(r, comp, 256, 128)
        assert check_frame_sorted(r, f"in order, full_key {full_key}")["layer"] == want


VIEW_NAMES = [n for n in vs.IN_LIMIT if n not in vs.LIMIT_SCENES]


@pytest.mark.parametrize("name", VIEW_NAMES)
def test_view_frames_are_sorted(cuda_api, sort_options, name):
    import torch
    sc = vs.SCENES[name]
    w, h, n = sc.width, sc.height, len(sc.views)
    comp, xf = vs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    far = name in ("far_left", "inf_points") or name.startswith("e2e_")  # e2e_views ends with a -2^20 px translation
    for full_key in (0, 1):
        sort_options(sort_full_key=full_key)
        t = torch.zeros(n * w * h * 4, dtype=torch.uint8, device="cuda:0")
        r.render_views_device(comp, sc.views, t.data_ptr(), w, h, RGBA, CLEAR)
        torch.cuda.synchronize()
        b = check_frame_sorted(r, f"{name} views full_key {full_key}", tile_y_rule="stacked", far=far)
        assert b["tile_y"] <= n * vs.rows(h)
    # the same views as single frames (the view applied as layer transforms)
    if name.startswith("paris"):
        return
    for k, v in list(enumerate(sc.views))[-3:]:
        vs.set_view(comp, xf, v)
        _render_device(r, comp, w, h)
        check_frame_sorted(r, f"{name} view {k} as a single frame", far=True)


def test_far_left_single_frame_sorts_its_tile_columns(cuda_api, unsliced):
    """Every line 2^20 px left of the frame: the tile columns wrap into 1 ... 5 and must be sorted."""
    sc = vs.SCENES["far_left"]
    comp, xf = vs.build(cuda_api, sc)
    vs.set_view(comp, xf, sc.views[0])
    r = cuda_api.Renderer(0)
    _render_device(r, comp, sc.width, sc.height)
    b = check_frame_sorted(r, "far_left", far=True)
    segs = r.segments()
    assert b["tile_x"] == 4095 and segs.size > 0 and int(_field(segs, TX).max()) > 1


@pytest.mark.parametrize("name", [n for n in bs.IN_LIMIT if n not in bs.LIMIT_SCENES])
def test_batch_frames_are_sorted(cuda_api, sort_options, name):
    import torch
    sc = bs.SCENES[name]
    _, frames = bs.build(cuda_api, sc)
    r = cuda_api.Renderer(0)
    for full_key in (0, 1):
        sort_options(sort_full_key=full_key)
        t = torch.zeros(len(frames) * sc.width * sc.height * 4, dtype=torch.uint8, device="cuda:0")
        r.render_batch_device(frames, t.data_ptr(), sc.width, sc.height, RGBA, CLEAR)
        torch.cuda.synchronize()
        b = check_frame_sorted(r, f"{name} batch full_key {full_key}", tile_y_rule="stacked")
        assert b["tile_y"] <= len(frames) * vs.rows(sc.height)


@pytest.mark.parametrize("name", sorted(scenes.E2E))
def test_e2e_frames_are_sorted(cuda_api, sort_options, unsliced, name):
    comp = cuda_api.Composition()
    scenes.E2E[name](cuda_api, comp)
    r = cuda_api.Renderer(0)
    for full_key in (0, 1):
        sort_options(sort_full_key=full_key)
        _render_device(r, comp, 64, 64)
        check_frame_sorted(r, f"e2e {name} full_key {full_key}")
    _render_device(r, comp, 64, 64, Rect((0, 64), (16, 48)))
    check_frame_sorted(r, f"e2e {name} crop band")
