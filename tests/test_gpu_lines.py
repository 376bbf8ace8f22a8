"""Line setup and rasterization on the device at their limits, at tolerance 0 against the oracle
(scenes: tests/line_scenes.py; model: tests/line_model.py). Every scene is first replayed by the
model: in-limit scenes must equal the oracle's records and fit the budget; over-limit scenes must
reach a total the renderer refuses, with an emit pass bounded by the buffer.

- In-limit scenes: `lines()` records, `rasterize_only` segments in emission order, frames and
  sorted segments in table modes 0 and 1, crops, `render_device`, `render_ids` and
  `MultiRenderer([0])`; sync-free frames whose counts grow.
- Host slices: a 1024-row frame without layer transforms rendered in four slices (checked with
  `host_slices()`), in limit and refused.
- Out-of-range sub-pixels: `rasterize_only` at width 2^31 equals the oracle's words.
- Frame sequences: a layer transform set, changed and cleared under a layer cache, so that the
  layer records switch between 4 and 36 bytes; compared frame by frame.
- Over-limit scenes: every entry point returns FORMA_ERR_CAPACITY, and the next frame on the same
  renderer and cache equals the oracle's frame for the same edits.
"""
import numpy as np
import pytest

import flatten_model as fm
import line_model as lm
import line_scenes as ls
import oracle_ids
from forma_b200.binding import RGBA, Color, FormaError, Rect

pytestmark = pytest.mark.gpu

CLEAR = Color(1.0, 1.0, 1.0, 0.0)


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float32:
        na, nb = np.isnan(a), np.isnan(b)
        return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))
    return np.array_equal(a, b)


def _checked(oracle_api, name):
    sc = ls.SCENES[name]
    rec = ls.model(oracle_api, sc)
    c = rec["counts"]
    if sc.over:
        assert c.status == lm.FORMA_ERR_CAPACITY
        assert int(lm.counts(rec["length"], rec["n_points"], 2 ** 26).emit_iterations.sum()) <= 2 ** 26
    else:
        assert sc.reached(rec) and c.status == lm.FORMA_OK and c.total <= fm.SEGMENT_CAP, name
    return sc, rec


def _oracle_frame(oracle_api, sc, crop=None):
    comp, _, _ = ls.build(oracle_api, sc.layers)
    r = oracle_api.Renderer(0)
    buf = np.zeros(sc.width * sc.height * 4, np.uint8)
    r.render(comp, buf, sc.width, sc.height, RGBA, CLEAR, crop)
    return buf, np.sort(r.segments())


@pytest.mark.parametrize("name", ls.IN_LIMIT)
def test_lines_and_segments_match_oracle(cuda_api, oracle_api, unsliced, name):
    sc, rec = _checked(oracle_api, name)
    w, h = sc.width, sc.height
    ocomp, _, _ = ls.build(oracle_api, sc.layers)
    ro = oracle_api.Renderer(0)
    want_segs = ro.rasterize_only(ocomp, w, h)
    want_lines = ro.lines()
    comp, _, _ = ls.build(cuda_api, sc.layers)
    r = cuda_api.Renderer(0)
    got = r.rasterize_only(comp, w, h)
    assert np.array_equal(got, want_segs), f"{name}: rasterize_only differs ({got.size} vs {want_segs.size})"
    lines = r.lines()
    for k in ("orders", "x0", "y0", "dx", "dy", "a", "b", "c", "d", "lengths"):
        assert _same(lines[k], want_lines[k]), f"{name}: lines()[{k}] differs"
    want, want_sorted = _oracle_frame(oracle_api, sc)
    modes = []
    for attempt in range(2):
        buf = np.zeros(w * h * 4, np.uint8)
        r.render(comp, buf, w, h, RGBA, CLEAR)
        modes.append(r.counters()["tables_mode"])
        assert np.array_equal(buf, want), f"{name}: frame {attempt + 1} differs"
        assert np.array_equal(np.sort(r.segments()), want_sorted), f"{name}: sorted segments differ"
    assert modes == [0, 1], modes
    for crop in sc.crops:
        rect = Rect(crop[0:2], crop[2:4])
        cw, _ = _oracle_frame(oracle_api, sc, rect)
        buf = np.zeros(w * h * 4, np.uint8)
        r.render(comp, buf, w, h, RGBA, CLEAR, rect)
        assert np.array_equal(buf, cw), f"{name}: crop {crop} differs"


@pytest.mark.parametrize("name", ["rotations", "subnormal", "translations", "nan", "edges", "layer_and_path"])
def test_device_entry_points_match_oracle(cuda_api, oracle_api, name):
    import torch
    sc, _ = _checked(oracle_api, name)
    w, h = sc.width, sc.height
    want, _ = _oracle_frame(oracle_api, sc)
    comp, _, _ = ls.build(cuda_api, sc.layers)
    r = cuda_api.Renderer(0)
    t = torch.zeros(h * w * 4, dtype=torch.uint8, device="cuda:0")
    r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR)
    torch.cuda.synchronize()
    assert np.array_equal(t.cpu().numpy(), want), f"{name}: render_device differs"
    ids = np.zeros(w * h, np.uint32)
    r.render_ids(comp, ids, w, h)
    ocomp, _, _ = ls.build(oracle_api, sc.layers)
    oids = np.zeros(w * h, np.uint32)
    oracle_ids.attach(oracle_api).Renderer(0).render_ids(ocomp, oids, w, h)
    assert np.array_equal(ids, oids), f"{name}: render_ids differs"
    m = cuda_api.MultiRenderer([0])
    buf = np.zeros(w * h * 4, np.uint8)
    m.render(comp, buf, w, h, RGBA, CLEAR)
    assert np.array_equal(buf, want), f"{name}: MultiRenderer([0]) differs"


def test_out_of_range_sub_pixels_match_oracle(cuda_api, oracle_api):
    comp, _, _ = ls.build(cuda_api, ls.origin_layers())
    ocomp, _, _ = ls.build(oracle_api, ls.origin_layers())
    for width in (2 ** 27, 2 ** 31):
        want = oracle_api.Renderer(0).rasterize_only(ocomp, width, 64)
        got = cuda_api.Renderer(0).rasterize_only(comp, width, 64)
        assert np.array_equal(got, want), f"width {width}: rasterize_only differs from the oracle's words"


def _sequence(api):
    """Frames under a layer cache while a layer transform is set, changed and cleared."""
    sc = ls.SCENES["rotations"]
    comp, _, _ = ls.build(api, sc.layers[:2])
    r = api.Renderer(0)
    cache = r.create_buffer_layer_cache()
    w, h = sc.width, sc.height
    frames = []

    def shot():
        buf = np.full(w * h * 4, 9, np.uint8) if not frames else frames[-1].copy()
        r.render(comp, buf, w, h, RGBA, CLEAR, None, cache)
        frames.append(buf)

    shot()
    layer = comp.get(0)
    layer.set_transform([1, 0, 0, 1, 3.5, -2.25])          # 4-byte -> 36-byte layer records
    shot()
    layer.set_transform(ls._about(0.0, 1.0, w / 2, h / 2))
    shot()
    layer.set_transform([1, 0, 0, 1, 0, 0])                # back to 4-byte records
    shot()
    comp.get(1).set_transform([0.6, 0.8, -0.8, 0.6, 100, 20])
    shot()
    return frames, r


def test_frame_sequence_with_layer_cache(cuda_api, oracle_api, unsliced):
    want, _ = _sequence(oracle_api)
    got, r = _sequence(cuda_api)
    for i, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a, b), f"frame {i} differs"


def test_sync_free_frames_follow_growing_counts(cuda_api, oracle_api, unsliced):
    """Counts that grow between sync-free frames (150 stars added before the third): every frame
    equals the oracle's."""
    sc = ls.SCENES["rotations"]
    w, h = sc.width, sc.height
    stars = [ls.star(40 + 29 * (i % 15), 40 + 30 * (i // 15), 8 + i % 40, 60 + i % 90, 30 + i % 20, 0.01 * i) for i in range(150)]
    frames, modes = {}, []
    for api in (oracle_api, cuda_api):
        comp, _, _ = ls.build(api, sc.layers[:2])
        big = comp.get_mut_or_insert_default(40).set_props(ls.Props())
        r = api.Renderer(0)
        out = []
        for k in range(3):
            if k == 2:
                for pts in stars:
                    big.insert(ls.build_path(api, pts))
            buf = np.zeros(w * h * 4, np.uint8)
            r.render(comp, buf, w, h, RGBA, CLEAR)
            out.append(buf)
            if api is cuda_api:
                modes.append(r.counters()["tables_mode"])
        frames[api is cuda_api] = out
    for k, (a, b) in enumerate(zip(frames[True], frames[False])):
        assert np.array_equal(a, b), f"frame {k} differs"
    assert modes[:2] == [0, 1], modes



SLICED_H = 1024  # 64 tile rows: four slices of 16


def _sliced_base():
    """Layers without transforms (a layer transform turns slicing off) over 1024 rows."""
    edges = ls.SCENES["edges"].layers[0].paths
    stars = [ls.star(60 + 45 * (i % 10), 60 + 100 * (i // 10), 15, 40, 5 + i % 4, 0.1 * i) for i in range(90)]
    return [ls.LayerSpec(0, None, edges), ls.LayerSpec(1, None, stars, even_odd=True),
            ls.LayerSpec(2, None, [[(3.5, 2.0), (500.25, 1000.5), (10.0, 1020.0)]])]


@pytest.fixture()
def four_slices(cuda_api):
    names = ("host_slices", "slice_min_points")
    saved = {n: cuda_api.get_option(n) for n in names}
    cuda_api.set_option("slice_min_points", 0)
    cuda_api.set_option("host_slices", 4)
    yield
    for n, v in saved.items():
        cuda_api.set_option(n, v)


def _oracle_sliced(oracle_api, layers):
    comp, _, _ = ls.build(oracle_api, layers)
    buf = np.zeros(ls.W * SLICED_H * 4, np.uint8)
    oracle_api.Renderer(0).render(comp, buf, ls.W, SLICED_H, RGBA, CLEAR)
    return buf


def test_host_slices_match_oracle(cuda_api, oracle_api, four_slices):
    want = _oracle_sliced(oracle_api, _sliced_base())
    comp, _, _ = ls.build(cuda_api, _sliced_base())
    r = cuda_api.Renderer(0)
    for frame in range(2):
        buf = np.zeros(ls.W * SLICED_H * 4, np.uint8)
        r.render(comp, buf, ls.W, SLICED_H, RGBA, CLEAR)
        assert len(r.host_slices()) == 4
        assert np.array_equal(buf, want), f"sliced frame {frame} differs"


@pytest.mark.parametrize("name", ["span_3e38", "scan_wrap"])
def test_host_slices_refuse_over_limit_frames(cuda_api, oracle_api, four_slices, name):
    """span_3e38 reaches the top slice only (the others may paint their bands before the frame is
    refused, see INTEGRATION.md); scan_wrap reaches all four."""
    sc, _ = _checked(oracle_api, name)
    base = _sliced_base()
    comp, _, _ = ls.build(cuda_api, base)
    r = cuda_api.Renderer(0)
    buf = np.zeros(ls.W * SLICED_H * 4, np.uint8)
    r.render(comp, buf, ls.W, SLICED_H, RGBA, CLEAR)
    assert len(r.host_slices()) == 4
    layer = comp.get_mut_or_insert_default(50)
    for spec in sc.layers:
        for pts in spec.paths:
            layer.insert(ls.build_path(cuda_api, pts))
    _refused(lambda: r.render(comp, buf, ls.W, SLICED_H, RGBA, CLEAR))
    assert r.host_slices() == [] and r.counters()["segments"] == 0 and r.row_costs().size == 0
    layer.disable()
    buf = np.zeros(ls.W * SLICED_H * 4, np.uint8)
    r.render(comp, buf, ls.W, SLICED_H, RGBA, CLEAR)
    assert len(r.host_slices()) == 4
    assert np.array_equal(buf, _oracle_sliced(oracle_api, base)), f"{name}: the sliced frame after the refusal differs"


def _refused(fn):
    with pytest.raises(FormaError, match="status 5"):
        fn()


@pytest.mark.parametrize("name", ls.OVER_LIMIT)
def test_over_limit_scenes_are_refused_and_leave_nothing_behind(cuda_api, oracle_api, unsliced, name):
    import torch
    sc, _ = _checked(oracle_api, name)
    w, h = ls.W, ls.H
    base = ls.SCENES["rotations"].layers[:2]
    # The same edits on both sides; the device renders a frame between them that fails.
    comp, _, _ = ls.build(cuda_api, base)
    ocomp, _, _ = ls.build(oracle_api, base)
    r = cuda_api.Renderer(0)
    cache = r.create_buffer_layer_cache()
    ro = oracle_api.Renderer(0)
    ocache = ro.create_buffer_layer_cache()
    buf = np.full(w * h * 4, 9, np.uint8)
    obuf = buf.copy()
    r.render(comp, buf, w, h, RGBA, CLEAR, None, cache)
    ro.render(ocomp, obuf, w, h, RGBA, CLEAR, None, ocache)
    assert np.array_equal(buf, obuf)
    for c in (comp, ocomp):
        api = cuda_api if c is comp else oracle_api
        layer = c.get_mut_or_insert_default(50)
        for spec in sc.layers:
            for pts in spec.paths:
                layer.insert(ls.build_path(api, pts))
            if spec.xf is not None:
                layer.set_transform(spec.xf)
    t = torch.zeros(h * w * 4, dtype=torch.uint8, device="cuda:0")
    ti = torch.zeros(h * w, dtype=torch.int32, device="cuda:0")
    failed = buf.copy()
    _refused(lambda: r.render(comp, failed, w, h, RGBA, CLEAR, None, cache))
    assert np.array_equal(failed, buf), "a refused frame wrote to the buffer"
    # A refused frame leaves no segment count behind for the inspection calls to read.
    assert r.counters()["segments"] == 0 and r.segments().size == 0
    assert r.row_costs().size == 0
    _refused(lambda: r.render_device(comp, t.data_ptr(), w, h, RGBA, CLEAR, None, cache))
    _refused(lambda: r.render_ids_device(comp, ti.data_ptr(), w, h))
    _refused(lambda: r.render_device_with_ids(comp, t.data_ptr(), ti.data_ptr(), w, h))
    _refused(lambda: r.render_ids(comp, np.zeros(w * h, np.uint32), w, h))
    assert r.rasterize_only(comp, w, h).size == 0
    assert "exceed" in cuda_api.last_error().decode()
    _refused(lambda: cuda_api.MultiRenderer([0]).render(comp, np.zeros(w * h * 4, np.uint8), w, h, RGBA, CLEAR))
    # Back in limit: the next frame on the same renderer and cache is the oracle's.
    comp.get(50).disable()
    ocomp.get(50).disable()
    r.render(comp, buf, w, h, RGBA, CLEAR, None, cache)
    ro.render(ocomp, obuf, w, h, RGBA, CLEAR, None, ocache)
    assert np.array_equal(buf, obuf), f"{name}: the frame after the refused ones differs"
