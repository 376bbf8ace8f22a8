"""Parity of stage 1 at its limits (scenes: tests/flatten_scenes.py; model and budget:
tests/flatten_model.py). Every test first runs the scene's pre-flight check itself: the model
replays the kernel's indexing in range and agrees with the reference's quad walk, and the point
(and, for rendered scenes, pixel-segment) counts fit the budget, with no surviving line that has a
non-finite end point. Only then does the device see the scene.

- Points: x and y bits (NaN compared as a class: the device's canonical NaN is not the CPU's) and
  contour flags equal the oracle's for every path, plain and through every transform.
- Rendered scenes: frames, pixel-segment counts and sorted segments equal the oracle's, with the
  tables built from read-back counts and then sync-free.
- Band filter: inserts whose bounds sit 0 ... 1 px from a band edge (shallow zig-zags whose
  segments round onto the edge's row, rotated by geometry-preserving path transforms, rational
  quads whose control point lies beyond the curve, inserts without a bound) rendered through sequences of bands, narrowing, widening, layer transforms, appends,
  compaction and eviction. Every frame equals the oracle's with the same crop, the band's rows of
  the sorted segments equal the whole frame's, and a narrowing uploads no geometry."""
import numpy as np
import pytest

import flatten_model as fm
import flatten_scenes as fs
from forma_b200.binding import RGBA, Color, Rect
from test_band_counts_model import row_counts

pytestmark = pytest.mark.gpu

CLEAR = Color(1.0, 1.0, 1.0, 0.0)


def _same(a, b):
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def _cases(sc, pc, po):
    yield "plain", pc, po
    if sc.transforms:
        for tn, m in fs.TRANSFORMS.items():
            yield tn, pc.transform(m), po.transform(m)
        for a, b in fs.CHAINS:
            ma, mb = fs.TRANSFORMS[a], fs.TRANSFORMS[b]
            yield f"{a}+{b}", pc.transform(ma).transform(mb), po.transform(ma).transform(mb)
    if not sc.finite or sc.transforms:
        for tn, m in fs.DEGENERATE_TRANSFORMS.items():
            yield tn, pc.transform(m), po.transform(m)


@pytest.mark.parametrize("name", [n for n, s in fs.PATHS.items() if s.device])
def test_flatten_points_bit_exact_at_the_limits(cuda_api, oracle_api, cuda_renderer, name):
    sc = fs.PATHS[name]
    for i, (pc, po) in enumerate(zip(sc.build(cuda_api), sc.build(oracle_api))):
        for tn, a, b in _cases(sc, pc, po):
            what = f"{name} path {i} {tn}"
            prog = a.program()
            r = fm.check_program(prog)
            assert r["mismatch"] is None, f"{what}: {r['mismatch']}"
            fm.assert_preflight(fm.preflight(prog["stats"]["points"]), what)
            xc, yc, cc = a.segments()
            xo, yo, co = b.segments()
            assert xc.shape == xo.shape, f"{what}: {xc.size} vs {xo.size} points"
            assert _same(xc, xo) and _same(yc, yo), f"{what}: points differ from the oracle's"
            assert np.array_equal(cc, co), f"{what}: contour flags differ"


def _budget(cuda_api, oracle_api, oracle_renderer, build, w, h, what):
    """Pre-flight of a whole scene: (cuda comp, oracle comp), built and checked before rendering."""
    rec = []

    class Rec:  # records the inserts for the model
        def get_mut_or_insert_default(self, order):
            return self

        def insert(self, p):
            rec.append(p)
            return self

        def set_props(self, props):
            return self
    build(cuda_api, Rec())
    progs = [p.program() for p in rec]
    b = fm.layout(progs)
    r = fm.replay(b)
    mm = fm.reference_walk_mismatch(b, r)
    assert mm is None, f"{what}: {mm}"
    ocomp = oracle_api.Composition()
    build(oracle_api, ocomp)
    fm.assert_preflight(fm.preflight(b.n_points, oracle_renderer, ocomp, w, h), what)
    comp = cuda_api.Composition()
    build(cuda_api, comp)
    return comp, ocomp


def _frame_diff(got, want, what):
    if not np.array_equal(got, want):
        d = np.abs(got.astype(int) - want.astype(int)).reshape(-1, 4).max(axis=1)
        ys = np.nonzero(d)[0]
        raise AssertionError(f"{what}: {len(ys)} pixels differ, first at pixel {ys[0]} (row {ys[0] // fs.W})")


@pytest.mark.parametrize("name", list(fs.RENDER))
def test_render_scene_matches_oracle_in_both_table_modes(cuda_api, oracle_api, oracle_renderer, unsliced, name):
    sc = fs.RENDER[name]
    w, h = sc.width, sc.height
    comp, ocomp = _budget(cuda_api, oracle_api, oracle_renderer, sc.build, w, h, name)
    want = np.zeros(w * h * 4, np.uint8)
    ro = oracle_api.Renderer(0)
    t = ro.render(ocomp, want, w, h, RGBA, CLEAR)
    segs_want, n_want = np.sort(ro.segments()), int(t.n_segments)
    r = cuda_api.Renderer(0)
    modes = []
    for attempt in range(2):
        buf = np.zeros(w * h * 4, np.uint8)
        t = r.render(comp, buf, w, h, RGBA, CLEAR)
        modes.append(r.counters()["tables_mode"])
        _frame_diff(buf, want, f"{name} frame {attempt + 1}")
        assert int(t.n_segments) == n_want
        assert np.array_equal(np.sort(r.segments()), segs_want), f"{name}: sorted segments differ"
    assert modes == [0, 1], modes


class _Band:
    """One band scene on both sides: every render is compared with the oracle's with the same crop."""

    def __init__(self, cuda_api, oracle_api, oracle_renderer, name):
        sc = fs.BANDS[name]
        self.name, self.cuda_api, self.oracle_api = name, cuda_api, oracle_api
        self.comp, self.ocomp = _budget(cuda_api, oracle_api, oracle_renderer, sc.build, fs.W, fs.H, name)
        self.ro = oracle_api.Renderer(0)
        self.tiles_y = (fs.H + 15) // 16

    def oracle(self, crop):
        buf = np.full(fs.W * fs.H * 4, 7, np.uint8)
        self.ro.render(self.ocomp, buf, fs.W, fs.H, RGBA, CLEAR, crop)
        return buf

    def whole_rows(self):
        self.ro.render(self.ocomp, np.zeros(fs.W * fs.H * 4, np.uint8), fs.W, fs.H, RGBA, CLEAR)
        return row_counts(np.sort(self.ro.segments()), self.tiles_y)

    def check(self, renderer, crop, what, rows=True):
        buf = np.full(fs.W * fs.H * 4, 7, np.uint8)
        renderer.render(self.comp, buf, fs.W, fs.H, RGBA, CLEAR, crop)
        _frame_diff(buf, self.oracle(crop), f"{self.name}: {what}")
        if rows and crop is not None and hasattr(renderer, "segments"):
            t0, t1 = crop.vertical[0] // 16, (crop.vertical[1] + 15) // 16
            got = row_counts(np.sort(renderer.segments()), self.tiles_y)[t0:t1]
            want = self.whole_rows()[t0:t1]
            assert np.array_equal(got, want), f"{self.name}: {what}: band rows {got.tolist()} vs the frame's {want.tolist()}"

    def preflight(self, oracle_renderer):
        fm.assert_preflight(fm.preflight(self.comp.point_count(), oracle_renderer, self.ocomp, fs.W, fs.H), self.name)

    def both(self, fn):
        fn(self.comp)
        fn(self.ocomp)


@pytest.mark.parametrize("name", list(fs.BANDS))
def test_band_filter_sequences_match_oracle(cuda_api, oracle_api, oracle_renderer, unsliced, name):
    s = _Band(cuda_api, oracle_api, oracle_renderer, name)
    r = cuda_api.Renderer(0)
    h2d = lambda: r.counters()["h2d_bytes"]  # noqa: E731
    s.check(r, fs.BAND, "band")
    b0 = h2d()
    s.check(r, fs.INNER_BAND, "narrower band inside it")
    assert h2d() - b0 < 4096, "a narrowing inside the resident band uploads no geometry"
    s.check(r, fs.OUTER_BAND, "band outside it")
    s.check(r, None, "whole frame")
    s.check(r, fs.BAND, "band after the whole frame")
    # a layer that gains a transform (the filter is off while one exists), then loses it
    s.both(lambda c: c.get(0).set_transform([1.0, 0.0, 0.0, 1.0, 0.5, 3.25]))
    s.check(r, fs.BAND, "band with a layer transform")
    s.both(lambda c: c.get(0).set_transform([1.0, 0.0, 0.0, 1.0, 0.0, 0.0]))
    s.check(r, fs.BAND, "band after the transform is reset")
    s.check(r, fs.INNER_BAND, "narrower band after the transform is reset")
    # inserts appended between band renders
    for api, c in ((cuda_api, s.comp), (oracle_api, s.ocomp)):
        lay = c.get_mut_or_insert_default(1).set_props(fs.solid(Color(0.5, 0.5, 0.1, 0.6)))
        pb = api.PathBuilder()
        pb.move_to(fs.P(10.0, 63.99)).line_to(fs.P(240.0, 63.99)).line_to(fs.P(120.0, 40.0))
        lay.insert(pb.build())
        pb = api.PathBuilder()
        pb.move_to(fs.P(10.0, 127.6)).line_to(fs.P(240.0, 128.5)).line_to(fs.P(120.0, 150.0))
        lay.insert(pb.build())
    s.preflight(oracle_renderer)
    s.check(r, fs.BAND, "band after appended inserts")
    s.check(r, fs.INNER_BAND, "narrower band after appended inserts")
    # a compaction between band renders: a large layer is cleared (its points become garbage)
    for api, c in ((cuda_api, s.comp), (oracle_api, s.ocomp)):
        xy = np.stack([np.linspace(5.0, 250.0, 70_000), 200.0 + 20.0 * (np.arange(70_000) % 2)], 1).astype(np.float32)
        cmds = np.ones(len(xy), np.uint8)
        cmds[0] = 0
        c.get_mut_or_insert_default(2).set_props(fs.solid(Color(0.1, 0.1, 0.9, 0.4))).insert(
            api.PathBuilder().extend(cmds, xy.ravel()).build())
    s.preflight(oracle_renderer)
    s.check(r, fs.BAND, "band with the large layer")
    s.both(lambda c: c.get(2).clear())
    s.check(r, fs.BAND, "band after the large layer is cleared (compaction)")
    s.check(r, fs.OUTER_BAND, "band outside after compaction")
    # evict, then a different band
    s.comp.evict()
    s.check(r, fs.OUTER_BAND, "band outside after evict")
    s.comp.evict()
    s.check(r, fs.BAND, "band after a second evict")
    s.check(r, None, "whole frame at the end")


@pytest.mark.parametrize("name", list(fs.BANDS))
def test_band_scenes_through_multi_renderer_and_host_slices(cuda_api, oracle_api, oracle_renderer, name):
    s = _Band(cuda_api, oracle_api, oracle_renderer, name)
    m = cuda_api.MultiRenderer([0])
    for crop, what in ((None, "whole frame"), (fs.BAND, "band"), (fs.INNER_BAND, "narrower band"),
                       (fs.OUTER_BAND, "band outside")):
        s.check(m, crop, f"MultiRenderer([0]) {what}", rows=False)
    saved = cuda_api.get_option("host_slices")
    cuda_api.set_option("host_slices", 4)
    try:
        r = cuda_api.Renderer(0)
        for crop, what in ((None, "whole frame"), (fs.BAND, "band"), (Rect((0, fs.W), (40, 200)), "wide band")):
            s.check(r, crop, f"host_slices = 4 {what}", rows=False)
    finally:
        cuda_api.set_option("host_slices", saved)
