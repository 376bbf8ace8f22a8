"""The binding of the ID frames of views and batches, without a GPU: default strides and chunking
(the library calls replaced by recorders), the declarations in the header, and the oracle
library, which has none of the four entry points, still loading through the same binding."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from forma_b200 import binding
from forma_b200.binding import RGBA, Color, Renderer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H = 10, 7


class _Handle:
    def __init__(self, h):
        self._h = h


class _Recorder:
    """Stands in for an Api: the four entry points record their arguments and succeed."""

    def __init__(self, max_views):
        self.calls = []
        self._max_views = max_views
        for name in binding.STACK_ID_SYMBOLS:
            setattr(self, name, self._entry(name))

    def _entry(self, name):
        def call(*args):
            self.calls.append((name, [a.value if isinstance(a, C.c_void_p) else a for a in args]))
            return 0
        return call

    def renderer_max_views(self, height):
        return self._max_views

    def renderer_free(self, h):
        pass

    def check(self, status, what):
        assert status == 0, what


def _renderer(max_views):
    r = object.__new__(Renderer)
    r._api, r._h = _Recorder(max_views), 77
    return r


def _views(n):
    return [[1.0, 0.0, 0.0, 1.0, float(k), 0.0] for k in range(n)]


def test_batch_ids_device_defaults_and_chunks():
    r = _renderer(2)
    comps = [_Handle(100 + k) for k in range(5)]
    r.render_batch_ids_device(comps, 1 << 20, W, H, rgba_ptr=1 << 30, clear_color=Color(0.0, 0.0, 0.0, 1.0), min_coverage=0.25,
                              timings=False)
    calls = r._api.calls
    assert [c[0] for c in calls] == ["renderer_render_batch_ids_device"] * 3
    for k, (_, a) in enumerate(calls):
        first, count = 2 * k, min(2, 5 - 2 * k)
        handle, arr, n, rgba, w, stride, h, frame_stride, ch, cc, ids, ids_stride, ids_frame_stride, mc, t = a
        assert (handle, n, w, h, mc, t) == (77, count, W, H, 0.25, None)
        assert [arr[i] for i in range(count)] == [100 + first + i for i in range(count)]
        assert (stride, frame_stride, ids_stride, ids_frame_stride) == (4 * W, 4 * W * H, 4 * W, 4 * W * H)
        assert rgba == (1 << 30) + first * 4 * W * H and ids == (1 << 20) + first * 4 * W * H
        assert list(ch) == list(RGBA) and list(cc) == [0.0, 0.0, 0.0, 1.0]


def test_batch_ids_device_without_rgba_and_with_strides():
    r = _renderer(3)
    comps = [_Handle(k) for k in range(1, 5)]
    r.render_batch_ids_device(comps, 4096, W, H, ids_stride=48, ids_frame_stride=400, timings=False)
    (_, a), (_, b) = r._api.calls
    assert a[3] is None and b[3] is None           # no RGBA frames
    assert (a[2], b[2]) == (3, 1)
    assert (a[10], b[10]) == (4096, 4096 + 3 * 400)
    assert a[11:13] == [48, 400] and b[11:13] == [48, 400]
    r = _renderer(3)
    r.render_batch_ids_device(comps, 4096, W, H, rgba_ptr=8192, stride=44, ids_stride=48, timings=False)
    (_, a), (_, b) = r._api.calls
    assert a[5:8] == [44, H, 44 * H] and a[11:13] == [48, 48 * H]
    assert (b[3], b[10]) == (8192 + 3 * 44 * H, 4096 + 3 * 48 * H)


def test_views_ids_defaults_and_chunks():
    r = _renderer(2)
    comp = _Handle(5)
    r.render_views_ids_device(comp, _views(3), 1 << 20, W, H, rgba_ptr=1 << 30, timings=False)
    (n0, a), (n1, b) = r._api.calls
    assert n0 == n1 == "renderer_render_views_ids_device"
    assert (a[0], a[1], a[3], b[3]) == (77, 5, 2, 1)
    assert [a[2][i] for i in range(12)] == sum(_views(3)[:2], []) and [b[2][i] for i in range(6)] == _views(3)[2]
    assert a[4:9] == [1 << 30, W, 4 * W, H, 4 * W * H] and a[11:15] == [1 << 20, 4 * W, 4 * W * H, 0.0]
    assert (b[4], b[11]) == ((1 << 30) + 2 * 4 * W * H, (1 << 20) + 2 * 4 * W * H)
    # the host call: IDs only, the array's own address
    r = _renderer(2)
    ids = np.zeros((3, H, W), np.uint32)
    r.render_views_ids(comp, _views(3), ids, W, H, min_coverage=0.5, timings=False)
    (n0, a), (n1, b) = r._api.calls
    assert n0 == n1 == "renderer_render_views_ids"
    assert a[3:] == [2, ids.ctypes.data, W, 4 * W, H, 4 * W * H, 0.5, None]
    assert b[3:] == [1, ids.ctypes.data + 2 * 4 * W * H, W, 4 * W, H, 4 * W * H, 0.5, None]


def test_batch_ids_host_defaults_and_size_check():
    r = _renderer(8)
    comps = [_Handle(k) for k in range(1, 4)]
    ids = np.zeros((3, H, W), np.uint32)
    r.render_batch_ids(comps, ids, W, H, timings=False)
    (name, a), = r._api.calls
    assert name == "renderer_render_batch_ids"
    assert a[2:] == [3, ids.ctypes.data, W, 4 * W, H, 4 * W * H, 0.0, None]
    with pytest.raises(AssertionError):
        r.render_batch_ids(comps, np.zeros((2, H, W), np.uint32), W, H)
    with pytest.raises(AssertionError):
        r.render_views_ids(_Handle(1), _views(3), np.zeros((3, H, W), np.int32), W, H)


def test_the_header_declares_the_four_entry_points():
    with open(os.path.join(ROOT, "include", "forma_b200.h")) as f:
        header = f.read()
    for name in binding.STACK_ID_SYMBOLS:
        assert name in binding.SIGNATURES
        m = re.search(r"\bint forma_%s\(([^;]*)\);" % name, header)
        assert m, name
        params = [p for p in m.group(1).split(",") if p.strip()]
        assert len(params) == len(binding.SIGNATURES[name][1]), name
    assert set(binding.STACK_ID_SYMBOLS).isdisjoint(binding.ID_FRAME_SYMBOLS + binding.VIEW_SYMBOLS + binding.BATCH_SYMBOLS)


def test_the_oracle_loads_without_them(oracle_api):
    for name in binding.STACK_ID_SYMBOLS:
        assert not hasattr(oracle_api, name)
    assert hasattr(oracle_api, "renderer_render")
