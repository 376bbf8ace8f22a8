"""The device's layer cache at its limits: every named edit sequence of tests/cache_sequences.py, frame by
frame at tolerance 0, against the oracle's frames and against the write set of the model in
tests/cache_model.py, which the marker tiles reveal. Host frames (packed written tiles and the host
scatter; `written_tiles` equals the model's count) and device frames (torch buffers: the tiles a frame
does not write keep the caller's bytes, and so do the bytes between rows), with padded strides, crops,
widths and heights that are not multiples of 16, and every paint build and table mode.

The sync-free redo in the field: a scene that grows past the renderer's bounds between two cached
device frames, and a cached device frame right after a small ID frame. The same calls without a cache
take the redo (tables_mode 2); a cached device frame builds its tables with the counts read back
(tables_mode 0) and writes only what the oracle writes.

Every expectation is computed on the CPU, through the oracle and the model, before the device is
touched."""
import numpy as np
import pytest

import cache_model
import cache_sequences as cq
from forma_b200.binding import RGBA

pytestmark = pytest.mark.gpu

PAD = 12          # bytes between a padded stride's rows, beyond 4 * width
PAD_BYTE = 0xE7
OPTIONS = ("paint_solid", "paint_wide", "sync_free", "test_fast_shrink", "host_slices")


@pytest.fixture()
def options(cuda_api):
    saved = {n: cuda_api.get_option(n) for n in OPTIONS}
    yield cuda_api
    for n, v in saved.items():
        cuda_api.set_option(n, v)


_expected = {}


def expected(oracle_api, name, pad):
    """The oracle's frames of a sequence and the model's ops per frame, checked against each other."""
    key = (name, pad)
    if key not in _expected:
        s = cq.run(name, oracle_api, record=True, pad=pad)
        m = cache_model.CacheModel()
        ops = []
        for k, (f, (before, after)) in enumerate(zip(s.inputs, s.frames)):
            want, o = m.frame(f, before)
            assert np.array_equal(want, after), f"{name} frame {k}: the model and the oracle differ"
            ops.append(o)
        _expected[key] = (s, ops)
    return _expected[key]


def small_comp(api):
    comp = api.Composition()
    comp.insert(0, comp.create_layer().insert(cq.rect(api, 1.0, 1.0, 5.0, 6.0)).set_props(cq.solid(0.5, 0.2, 0.1)))
    return comp


def between(kind, s, **kw):
    """Uncached calls of the session's first renderer (the device side's Session.between hook)."""
    import torch
    api, r, comp = s.api, s.renderers[0], s.comp
    w, h = 40, 24
    if kind == "evict":
        comp.evict()
    elif kind == "rgba":
        r.render(comp, np.zeros(w * h * 4, np.uint8), w, h, RGBA, cq.CLEAR)
    elif kind == "ids":
        r.render_ids(comp, np.zeros(w * h, np.uint32), w, h)
    elif kind == "masks":
        r.render_masks(comp, np.zeros(4 * w * h, np.float32), w, h, 0, 4)
    elif kind == "stats":
        r.render_stats(comp, w, h, 0, 8)
    elif kind == "linear":
        r.render_linear(comp, np.zeros(w * h * 4, np.float32), w, h, RGBA, cq.CLEAR)
    elif kind == "over":
        buf = torch.full((h, w, 4), 0x40, dtype=torch.uint8, device="cuda:0")
        r.render_over_device(comp, buf.data_ptr(), w, h)
        torch.cuda.synchronize()
    elif kind == "views":
        r.render_views(comp, [[1.0, 0.0, 0.0, 1.0, 0.0, 0.0], [1.0, 0.0, 0.0, 1.0, 5.0, 3.0]], np.zeros(2 * w * h * 4, np.uint8),
                       w, h, RGBA, cq.CLEAR)
    elif kind == "batch":
        r.render_batch([comp, small_comp(api)], np.zeros(2 * w * h * 4, np.uint8), w, h, RGBA, cq.CLEAR)
    elif kind == "small":
        r.render(small_comp(api), np.zeros(8 * 8 * 4, np.uint8), 8, 8, RGBA, cq.CLEAR)
    elif kind == "small_ids":
        r.render_ids(small_comp(api), np.zeros(8 * 8, np.uint32), 8, 8)
    else:
        raise AssertionError(kind)


class DeviceFrames:
    """Session.render for device frames: the session's buffer goes to a torch buffer with the same
    stride, the frame is rendered there and the whole buffer comes back."""

    def __init__(self):
        self.modes = []

    def __call__(self, r, comp, buf, w, h, stride, channels, clear, crop, cache):
        import torch
        dev = torch.from_numpy(buf.copy()).to("cuda:0")
        torch.cuda.synchronize()
        r.render_device(comp, dev.data_ptr(), w, h, channels, clear, crop, cache, stride=stride)
        torch.cuda.synchronize()
        buf[:] = dev.cpu().numpy()
        self.modes.append(r.counters()["tables_mode"])


class HostFrames:
    def __init__(self):
        self.written = []

    def __call__(self, r, comp, buf, w, h, stride, channels, clear, crop, cache):
        cq.host_render(r, comp, buf, w, h, stride, channels, clear, crop, cache)
        self.written.append(r.counters()["written_tiles"])


def run_device(cuda_api, oracle_api, name, device, pad):
    s_ref, ops = expected(oracle_api, name, pad)
    sink = DeviceFrames() if device else HostFrames()
    pads = []

    def render(r, comp, buf, w, h, stride, *rest):
        if stride > 4 * w:  # the bytes between rows carry a pattern of their own
            buf.reshape(h, stride)[:, 4 * w:] = PAD_BYTE
        sink(r, comp, buf, w, h, stride, *rest)
        pads.append(buf.reshape(h, stride)[:, 4 * w:].copy())

    s = cq.run(name, cuda_api, render=render, between=between, pad=pad)
    assert len(s.frames) == len(s_ref.frames)
    for k, ((_, got), (_, want), o) in enumerate(zip(s.frames, s_ref.frames, ops)):
        bad = np.argwhere((got != want).any(axis=2))
        if len(bad):
            y, x = bad[0].tolist()
            tiles = sorted({(int(b[1]) // 16, int(b[0]) // 16) for b in bad})
            pytest.fail(f"{name} frame {k}: {len(bad)} pixels in {len(tiles)} tiles differ, first (x {x}, y {y}): device "
                        f"{got[y, x].tolist()}, oracle {want[y, x].tolist()}, model op {o.get((x // 16, y // 16))}; "
                        f"tiles {tiles[:8]}")
        assert not pads[k].size or (pads[k] == PAD_BYTE).all(), f"{name} frame {k}: bytes between rows written"
        if not device:
            written = cache_model.count(o, cache_model.SOLID) + cache_model.count(o, cache_model.PAINT)
            assert sink.written[k] == written, f"{name} frame {k}: {sink.written[k]} tiles copied back, the model writes {written}"
    return sink


@pytest.mark.parametrize("name", sorted(cq.SEQUENCES))
@pytest.mark.parametrize("device,pad", [(False, 0), (True, 0), (True, PAD), (False, PAD)])
def test_sequence(cuda_api, oracle_api, name, device, pad):
    run_device(cuda_api, oracle_api, name, device, pad)


@pytest.mark.parametrize("name", ["decision_edges", "frame_state", "between_frames", "random_12"])
@pytest.mark.parametrize("setting", [("paint_solid", 0), ("paint_wide", 1), ("sync_free", 0), ("test_fast_shrink", 1),
                                     ("host_slices", 3)])
@pytest.mark.parametrize("device", [False, True])
def test_sequence_options(options, oracle_api, name, setting, device):
    """A cached host frame is never sliced (host_slices), and every paint build and table mode keeps
    the cache's decisions."""
    options.set_option(*setting)
    run_device(options, oracle_api, name, device, PAD if device else 0)


@pytest.mark.parametrize("name", cq.REDO)
def test_redo_in_the_field(options, oracle_api, name):
    """The frames that set up a sync-free redo: uncached, the same calls of a renderer take the redo;
    cached, the frame is counted and equals the oracle's (on device frames before this rule, the
    first attempt wrote the clear colour into the caller's buffer and recorded it, and the redo then
    skipped every tile under an unchanged opaque layer)."""
    options.set_option("sync_free", 1)
    options.set_option("test_fast_shrink", 0)
    sink = run_device(options, oracle_api, name, True, PAD)
    # The frame after the growth or after the small ID frame is frame 2 in both sequences.
    assert sink.modes[2] == 0, f"tables_mode {sink.modes}"

    def uncached(r, comp, buf, w, h, stride, channels, clear, crop, cache):
        sink(r, comp, buf, w, h, stride, channels, clear, crop, None)

    sink = DeviceFrames()
    cq.run(name, options, render=uncached, between=between, pad=PAD)
    assert sink.modes[2] == 2, f"uncached tables_mode {sink.modes}: the sequence no longer reaches the redo"


def test_fast_shrink_unchanged_scene(options):
    """An unchanged scene under a full-frame opaque layer in three cached device frames, the third with
    test_fast_shrink: it writes nothing, as the oracle's does (the reference writes no tile of an
    unchanged frame). The same three frames without a cache take the redo."""
    import torch
    w, h = cq.RW, cq.RH
    s = cq.Session(options)
    s.mixed(1000, w, h, 5)
    s.add(1000, [cq.rect(options, -2.0, -2.0, w + 2.0, h + 2.0)], cq.solid(0.7, 0.1, 0.3))
    options.set_option("sync_free", 1)
    dev = torch.full((h, w, 4), 0x11, dtype=torch.uint8, device="cuda:0")
    modes = []
    for cached in (True, False):
        r = s.renderers[0] if cached else options.Renderer(0)
        cache = s.cache().h if cached else None
        options.set_option("test_fast_shrink", 0)
        for k in range(3):
            if k == 2:
                options.set_option("test_fast_shrink", 1)
                dev.fill_(0x22)
            torch.cuda.synchronize()
            r.render_device(s.comp, dev.data_ptr(), w, h, RGBA, cq.CLEAR, None, cache)
            torch.cuda.synchronize()
        modes.append(r.counters()["tables_mode"])
        if cached:
            assert bool((dev == 0x22).all()), "the unchanged frame wrote tiles"
    assert modes == [0, 2], f"tables_mode cached / uncached: {modes}"
