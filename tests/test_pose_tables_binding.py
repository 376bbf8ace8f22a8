"""Pose tables in device memory without a GPU: Poses takes objects with __cuda_array_interface__
(fakes here) as it takes arrays, checks their type, shape and contiguity without copying them, and
passes each chunk of frames the address of its first row; the library's recorder reads the
descriptors. Importing the binding does not import torch."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from forma_b200 import binding
from forma_b200.binding import Poses, Renderer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H = 10, 7


class FakeCuda:
    """An object exposing only a __cuda_array_interface__ dict (version 3)."""

    def __init__(self, shape, typestr, ptr=1 << 32, strides=None, **extra):
        self.__cuda_array_interface__ = dict(shape=tuple(shape), typestr=typestr, data=(ptr, False), strides=strides, version=3,
                                             **extra)


def _c_strides(shape, itemsize):
    out, step = [], itemsize
    for n in reversed(shape):
        out.append(step)
        step *= n
    return tuple(reversed(out))


class _Handle:
    def __init__(self, h):
        self._h = h


class _Recorder:
    """Stands in for an Api: every pose entry point records its chunk's descriptor (addresses, not
    contents: the fakes point at no memory) and succeeds."""

    def __init__(self, max_views, read_visible=False):
        self.calls = []
        self.visible = []  # with read_visible: each call's host visibility rows, read at call time
        self._max_views = max_views
        self._read_visible = read_visible
        for name in binding.POSE_SYMBOLS:
            setattr(self, name, self._entry(name))

    def _entry(self, name):
        def call(*args):
            d = args[2]._obj
            if self._read_visible:
                rows = (C.c_uint8 * (args[3] * d.n_orders)).from_address(d.visible)
                self.visible.append(np.ctypeslib.as_array(rows).reshape(args[3], d.n_orders).copy())
            self.calls.append((name, (d.first_order, d.n_orders, d.transforms, d.visible, d.colors), args[3]))
            return 0
        return call

    def renderer_max_views(self, height):
        return self._max_views

    def renderer_free(self, h):
        pass

    def check(self, status, what):
        assert status == 0, what


def _renderer(max_views, read_visible=False):
    r = object.__new__(Renderer)
    r._api, r._h = _Recorder(max_views, read_visible), 77
    return r


@pytest.mark.parametrize("strided", [False, True])
@pytest.mark.parametrize("vis_type", ["|u1", "|b1"])
def test_cuda_tables_are_accepted(strided, vis_type):
    n, k = 5, 3
    st = (lambda shape, size: _c_strides(shape, size)) if strided else (lambda shape, size: None)
    t = FakeCuda((n, k, 6), "<f4", 4096, st((n, k, 6), 4))
    v = FakeCuda((n, k), vis_type, 8192, st((n, k), 1))
    c = FakeCuda((n, k, 4), "<f4", 16384, st((n, k, 4), 4))
    p = Poses(2, t, v, c)
    assert (p.n, p.n_orders, p.first_order) == (n, k, 2)
    assert (p.transforms.ptr, p.visible.ptr, p.colors.ptr) == (4096, 8192, 16384)
    assert (p.transforms.row_bytes, p.visible.row_bytes, p.colors.row_bytes) == (24 * k, k, 16 * k)
    assert p.transforms.owner is t  # kept alive, not copied
    for one in (Poses(0, transforms=t), Poses(0, visible=v), Poses(0, colors=c)):
        assert (one.n, one.n_orders) == (n, k)


def test_size_one_dimensions_may_have_any_stride():
    p = Poses(0, FakeCuda((1, 3, 6), "<f4", strides=(999, 24, 4)))
    assert (p.n, p.n_orders) == (1, 3)


@pytest.mark.parametrize("kw, table", [
    ("transforms", FakeCuda((4, 3, 6), "<f4", strides=(3 * 6 * 4 * 2, 24, 4))),  # every other frame
    ("transforms", FakeCuda((4, 3, 6), "<f4", strides=(4, 16, 48 * 4))),          # Fortran order
    ("visible", FakeCuda((4, 3), "|u1", strides=(1, 4))),                          # transposed
    ("colors", FakeCuda((4, 3, 4), "<f4", strides=(48, 16, 8))),                   # every other channel
])
def test_non_contiguous_cuda_tables_are_refused(kw, table):
    with pytest.raises(ValueError, match="contiguous"):
        Poses(0, **{kw: table})


@pytest.mark.parametrize("kw, table", [
    ("transforms", FakeCuda((4, 3, 6), "<f8")), ("transforms", FakeCuda((4, 3, 6), "<f2")), ("transforms", FakeCuda((4, 3, 6), "<i4")),
    ("visible", FakeCuda((4, 3), "<i4")), ("visible", FakeCuda((4, 3), "<f4")), ("visible", FakeCuda((4, 3), "|i1")),
    ("colors", FakeCuda((4, 3, 4), "<f8")), ("colors", FakeCuda((4, 3, 4), "|u1")),
])
def test_wrong_cuda_types_are_refused(kw, table):
    with pytest.raises(ValueError, match="type"):
        Poses(0, **{kw: table})


@pytest.mark.parametrize("tables", [
    dict(transforms=FakeCuda((4, 3, 5), "<f4")), dict(transforms=FakeCuda((4, 3), "<f4")), dict(visible=FakeCuda((4, 3, 1), "|u1")),
    dict(colors=FakeCuda((4, 3, 3), "<f4")),
    dict(transforms=FakeCuda((4, 3, 6), "<f4"), visible=FakeCuda((4, 2), "|u1")),
    dict(transforms=FakeCuda((4, 3, 6), "<f4"), colors=FakeCuda((5, 3, 4), "<f4")),
    dict(transforms=np.zeros((4, 3, 6), np.float32), visible=FakeCuda((3, 3), "|b1")),
    dict(visible=np.ones((4, 3), bool), colors=FakeCuda((4, 4, 4), "<f4")),
])
def test_wrong_shapes_are_refused(tables):
    with pytest.raises(ValueError):
        Poses(0, **tables)


def test_masked_cuda_arrays_are_refused():
    with pytest.raises(ValueError, match="masked"):
        Poses(0, visible=FakeCuda((4, 3), "|u1", mask=FakeCuda((4, 3), "|b1")))


def test_refusals_come_before_any_library_call():
    r = _renderer(8)
    with pytest.raises(ValueError):
        r.render_poses_device(_Handle(5), Poses(0, FakeCuda((4, 3, 6), "<f8")), 1 << 30, W, H, timings=False)
    assert r._api.calls == []


def test_host_and_cuda_tables_mix():
    n, k = 3, 4
    xf = np.tile(np.array([1, 0, 0, 1, 2, 3], np.float32), (n, k, 1))
    p = Poses(1, xf, FakeCuda((n, k), "|b1", 777), np.ones((n, k, 4), np.float32))
    assert isinstance(p.transforms, np.ndarray) and isinstance(p.colors, np.ndarray) and p.visible.ptr == 777
    r = _renderer(8)
    r.render_poses_device(_Handle(5), p, 1 << 30, W, H, timings=False)
    (name, (fo, kk, t, v, c), count), = r._api.calls
    assert (fo, kk, v, count) == (1, k, 777, n)
    assert t == p.transforms.ctypes.data and c == p.colors.ctypes.data


@pytest.mark.parametrize("method", ["render_poses_device", "render_poses_linear_device", "render_poses_over_device"])
def test_chunks_pass_offsets_into_the_cuda_tables(method):
    """max_views 2: the chunk [f, f + c) gets ptr + 24 f K, ptr + f K and ptr + 16 f K."""
    n, k = 5, 3
    pt, pv, pc = 1 << 32, 1 << 33, (1 << 33) + (1 << 20)
    p = Poses(7, FakeCuda((n, k, 6), "<f4", pt), FakeCuda((n, k), "|u1", pv), FakeCuda((n, k, 4), "<f4", pc))
    r = _renderer(2)
    getattr(r, method)(_Handle(5), p, 1 << 30, W, H, timings=False)
    calls = r._api.calls
    assert len(calls) == 3
    for j, (_, (fo, kk, t, v, c), count) in enumerate(calls):
        f = 2 * j
        assert (fo, kk, count) == (7, k, min(2, n - f))
        assert (t, v, c) == (pt + 24 * f * k, pv + f * k, pc + 16 * f * k)


def test_chunks_mix_offsets_and_host_slices():
    n, k = 5, 2
    vis = (np.arange(n * k) % 3 != 0).reshape(n, k)
    p = Poses(0, FakeCuda((n, k, 6), "<f4", 4096), vis)
    r = _renderer(2, read_visible=True)
    r.render_poses_ids_device(_Handle(5), p, 1 << 30, W, H, timings=False)
    assert len(r._api.calls) == 3
    for j, (_, (_, _, t, _, _), count) in enumerate(r._api.calls):
        f = 2 * j
        assert t == 4096 + 24 * f * k
        assert np.array_equal(r._api.visible[j], vis[f:f + count])


def test_importing_the_binding_does_not_import_torch():
    code = "import sys; import forma_b200.binding; assert 'torch' not in sys.modules, 'torch imported'"
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    subprocess.run([sys.executable, "-s", "-c", code], check=True, cwd=ROOT, env=env)
