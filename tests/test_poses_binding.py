"""The binding of poses, without a GPU: the Poses value, default strides and chunking with the pose
tables sliced per chunk (the library calls replaced by recorders), the declarations in the header,
and the oracle library, which has none of the entry points, still loading through the binding."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from forma_b200 import binding
from forma_b200.binding import RGBA, Color, Poses, Renderer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H = 10, 7


class _Handle:
    def __init__(self, h):
        self._h = h


class _Recorder:
    """Stands in for an Api: the pose entry points record their arguments (the forma_poses
    descriptor read out at call time) and succeed."""

    def __init__(self, max_views):
        self.calls = []
        self._max_views = max_views
        for name in binding.POSE_SYMBOLS:
            setattr(self, name, self._entry(name))

    def _entry(self, name):
        def call(*args):
            out = []
            for a in args:
                if isinstance(a, C.c_void_p):
                    out.append(a.value)
                elif type(a).__name__ == "CArgObject":
                    d = a._obj
                    if isinstance(d, binding._CPoses):
                        out.append(self._read(d, args[3]))
                    else:
                        out.append(d)
                else:
                    out.append(a)
            self.calls.append((name, out))
            return 0
        return call

    @staticmethod
    def _read(d, n):
        k = d.n_orders
        t = None if not d.transforms else np.ctypeslib.as_array((C.c_float * (n * k * 6)).from_address(d.transforms)).reshape(n, k, 6).copy()
        v = None if not d.visible else np.ctypeslib.as_array((C.c_uint8 * (n * k)).from_address(d.visible)).reshape(n, k).copy()
        return (d.first_order, k, t, v)

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


def _poses(n, k, first=3, transforms=True, visible=True):
    t = np.arange(n * k * 6, dtype=np.float32).reshape(n, k, 6) if transforms else None
    v = (np.arange(n * k).reshape(n, k) % 2).astype(bool) if visible else None
    return Poses(first, t, v)


def test_poses_value_checks_its_tables():
    p = _poses(5, 4)
    assert (p.n, p.n_orders, p.first_order, len(p)) == (5, 4, 3, 5)
    assert p.transforms.dtype == np.float32 and p.visible.dtype == np.uint8
    assert Poses(0, visible=[[True, False]]).n_orders == 2
    with pytest.raises(ValueError):
        Poses(0)
    with pytest.raises(ValueError):
        Poses(0, np.zeros((2, 3, 6)), np.zeros((2, 4), bool))  # K disagrees
    with pytest.raises(ValueError):
        Poses(0, np.zeros((3, 3, 6)), np.zeros((2, 3), bool))  # n disagrees
    with pytest.raises(ValueError):
        Poses(0, np.zeros((2, 3, 4)))


def test_poses_device_defaults_and_sliced_chunks():
    r = _renderer(2)
    p = _poses(5, 4)
    r.render_poses_device(_Handle(5), p, 1 << 30, W, H, RGBA, Color(0.0, 0.0, 0.0, 1.0), timings=False)
    calls = r._api.calls
    assert [c[0] for c in calls] == ["renderer_render_poses_device"] * 3
    for j, (_, a) in enumerate(calls):
        first, count = 2 * j, min(2, 5 - 2 * j)
        handle, comp, (fo, k, t, v), n, ptr, w, stride, h, view_stride, ch, cc, tm = a
        assert (handle, comp, fo, k, n, w, h, tm) == (77, 5, 3, 4, count, W, H, None)
        assert np.array_equal(t, p.transforms[first:first + count]) and np.array_equal(v, p.visible[first:first + count])
        assert (stride, view_stride) == (4 * W, 4 * W * H) and ptr == (1 << 30) + first * 4 * W * H
        assert list(ch) == list(RGBA) and list(cc) == [0.0, 0.0, 0.0, 1.0]


def test_poses_host_and_one_table_only():
    r = _renderer(8)
    p = _poses(3, 2, first=0, transforms=False)
    buf = np.zeros(3 * H * W * 4, np.uint8)
    r.render_poses(_Handle(1), p, buf, W, H, timings=False)
    (name, a), = r._api.calls
    assert name == "renderer_render_poses"
    fo, k, t, v = a[2]
    assert (fo, k, t) == (0, 2, None) and np.array_equal(v, p.visible)
    assert a[3:9] == [3, buf.ctypes.data, W, 4 * W, H, 4 * W * H]
    with pytest.raises(AssertionError):
        r.render_poses(_Handle(1), p, np.zeros(2 * H * W * 4, np.uint8), W, H)


def test_poses_ids_masks_stats_chunks():
    r = _renderer(2)
    p = _poses(3, 2, transforms=True, visible=False)
    r.render_poses_ids_device(_Handle(5), p, 1 << 20, W, H, rgba_ptr=1 << 30, timings=False)
    (_, a), (_, b) = r._api.calls
    assert (a[3], b[3]) == (2, 1) and b[2][2].shape == (1, 2, 6) and np.array_equal(b[2][2][0], p.transforms[2])
    assert (a[11], b[11]) == (1 << 20, (1 << 20) + 2 * 4 * W * H) and (a[4], b[4]) == (1 << 30, (1 << 30) + 2 * 4 * W * H)
    r = _renderer(2)
    ids = np.zeros((3, H, W), np.uint32)
    r.render_poses_ids(_Handle(5), p, ids, W, H, min_coverage=0.5, timings=False)
    (_, a), (_, b) = r._api.calls
    assert a[3:] == [2, ids.ctypes.data, W, 4 * W, H, 4 * W * H, 0.5, None]
    assert b[3:] == [1, ids.ctypes.data + 2 * 4 * W * H, W, 4 * W, H, 4 * W * H, 0.5, None]
    r = _renderer(2)
    r.render_poses_masks_device(_Handle(5), p, 4096, W, H, 1, 3, format="u8", timings=False)
    (_, a), (_, b) = r._api.calls
    assert (a[4].ptr, b[4].ptr) == (4096, 4096 + 2 * 3 * W * H) and (a[4].first_order, a[4].n_orders) == (1, 3)
    r = _renderer(2)
    r.render_poses_stats_device(_Handle(5), p, 8192, W, H, 0, 4, timings=False)
    (_, a), (_, b) = r._api.calls
    assert (a[4].ptr, b[4].ptr) == (8192, 8192 + 2 * 4 * 48)


def test_the_header_declares_the_pose_entry_points():
    with open(os.path.join(ROOT, "include", "forma_b200.h")) as f:
        header = f.read()
    for name in binding.POSE_SYMBOLS:
        assert name in binding.SIGNATURES
        m = re.search(r"\bint forma_%s\(([^;]*)\);" % name, header)
        assert m, name
        params = [p for p in re.sub(r"/\*.*?\*/", "", m.group(1)).split(",") if p.strip()]
        assert len(params) == len(binding.SIGNATURES[name][1]), name
        assert "const forma_poses* poses" in params[2]
    m = re.search(r"typedef struct forma_poses \{(.*?)\} forma_poses;", header, re.S)
    fields = re.findall(r"(\w+)\s*;", re.sub(r"/\*.*?\*/", "", m.group(1)).replace("first_order,", "first_order; "))
    assert fields == [f for f, _ in binding._CPoses._fields_]


def test_the_oracle_loads_without_them(oracle_api):
    for name in binding.POSE_SYMBOLS:
        assert not hasattr(oracle_api, name)
    assert hasattr(oracle_api, "renderer_render")
