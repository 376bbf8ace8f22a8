"""Instances in the binding without a GPU: the descriptor's layout against include/forma_b200.h,
the validation of Instances (host and CUDA tables, fakes here), the chunking of the four instance
methods (at max_views(height) and at 2^21 // M frames, each chunk handed its rows of the tables;
the library's recorder reads the descriptors), and the oracle library still loading without the
instance entry points."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from forma_b200 import binding
from forma_b200.binding import Instances, NO_INSTANCE, Renderer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H = 10, 7


class FakeCuda:
    """An object exposing only a __cuda_array_interface__ dict (version 3)."""

    def __init__(self, shape, typestr, ptr=1 << 32, strides=None):
        self.__cuda_array_interface__ = dict(shape=tuple(shape), typestr=typestr, data=(ptr, False), strides=strides, version=3)


def test_descriptor_matches_the_header():
    header = open(os.path.join(ROOT, "include", "forma_b200.h")).read()
    body = re.search(r"typedef struct forma_instances \{(.*?)\} forma_instances;", header, re.S).group(1)
    fields = re.findall(r"^\s*(?:const\s+)?(\w+)\*?\s+\*?(\w+);", body, re.M)
    assert [f for _, f in fields] == [name for name, _ in binding._CInstances._fields_]
    assert [t for t, _ in fields] == ["uint32_t", "uint32_t", "float", "float"]
    assert [getattr(binding._CInstances, f).offset for f, _ in binding._CInstances._fields_] == [0, 8, 16, 24]
    assert C.sizeof(binding._CInstances) == 32
    assert int(re.search(r"#define FORMA_NO_INSTANCE (0x[0-9A-Fa-f]+)u", header).group(1), 16) == NO_INSTANCE
    for name in binding.INSTANCE_SYMBOLS:
        assert f"forma_{name}(" in header


def test_host_tables():
    i = Instances([[0, -1, 3], [NO_INSTANCE, 7, 7]], np.zeros((2, 3, 6)), np.zeros((2, 3, 4), np.float32))
    assert (i.n, i.n_instances, len(i)) == (2, 3, 2)
    assert i.prototypes.dtype == np.uint32 and i.prototypes.tolist() == [[0, NO_INSTANCE, 3], [NO_INSTANCE, 7, 7]]
    assert i.transforms.dtype == np.float32 and i.transforms.flags["C_CONTIGUOUS"]
    assert Instances(np.array([[1, 2]], np.int32)).transforms is None


@pytest.mark.parametrize("kw, msg", [
    (dict(prototypes=None), "required"),
    (dict(prototypes=[[0.5, 1.0]]), "integers"),
    (dict(prototypes=[[-2, 0]]), "orders"),
    (dict(prototypes=[[1 << 32, 0]]), "orders"),
    (dict(prototypes=[0, 1, 2]), "shape"),
    (dict(prototypes=np.zeros((2, 0), np.uint32)), "M = 0"),
    (dict(prototypes=[[0, 1]], transforms=np.zeros((1, 3, 6), np.float32)), "disagree"),
    (dict(prototypes=[[0, 1]], transforms=np.zeros((1, 2, 4), np.float32)), "transforms"),
    (dict(prototypes=[[0, 1]], colors=np.zeros((1, 2, 4), np.float64)), "colors"),
    (dict(prototypes=[[0, 1]], colors=np.zeros((2, 2, 4), np.float32)), "disagree"),
])
def test_host_refusals(kw, msg):
    with pytest.raises(ValueError, match=msg):
        Instances(**kw)


def test_cuda_tables():
    p = FakeCuda((5, 3), "<i4", 4096)
    t = FakeCuda((5, 3, 6), "<f4", 8192)
    c = FakeCuda((5, 3, 4), "<f4", 16384)
    i = Instances(p, t, c)
    assert (i.n, i.n_instances) == (5, 3)
    assert (i.prototypes.ptr, i.transforms.ptr, i.colors.ptr) == (4096, 8192, 16384)
    assert (i.prototypes.row_bytes, i.transforms.row_bytes, i.colors.row_bytes) == (12, 72, 48)
    assert Instances(FakeCuda((2, 4), "<u4")).n_instances == 4
    mixed = Instances(FakeCuda((2, 3), "<u4"), np.zeros((2, 3, 6), np.float32))
    assert isinstance(mixed.transforms, np.ndarray)


@pytest.mark.parametrize("kw, table, msg", [
    ("prototypes", FakeCuda((4, 3), "<f4"), "type"), ("prototypes", FakeCuda((4, 3), "<i8"), "type"),
    ("prototypes", FakeCuda((4, 3), "<i4", strides=(4, 16)), "contiguous"),
    ("transforms", FakeCuda((4, 3, 6), "<f8"), "type"), ("colors", FakeCuda((4, 3, 4), "|u1"), "type"),
    ("colors", FakeCuda((4, 3, 4), "<f4", strides=(96, 32, 4)), "contiguous"),
])
def test_cuda_refusals(kw, table, msg):
    args = dict(prototypes=FakeCuda((4, 3), "<u4"))
    args[kw] = table
    with pytest.raises(ValueError, match=f"Instances: .*{msg}"):
        Instances(**args)


class _Recorder:
    """Stands in for an Api: every instance entry point records its chunk's descriptor and the
    host rows it points at (read at call time), and its target pointers, and succeeds."""

    def __init__(self, max_views):
        self.calls = []
        self._max_views = max_views
        for name in binding.INSTANCE_SYMBOLS:
            setattr(self, name, self._entry(name))

    def _entry(self, name):
        def call(*args):
            d, n = args[2]._obj, args[3]
            rows = None
            if d.prototypes and d.prototypes < (1 << 32):  # (host tables; the fakes' addresses start at 2^32)
                rows = np.ctypeslib.as_array((C.c_uint32 * (n * d.n_instances)).from_address(d.prototypes)).reshape(n, -1).copy()
            target = args[4]
            target = target._obj.ptr if hasattr(target, "_obj") else (target.value if target is not None else None)
            self.calls.append((name, d.n_instances, n, d.prototypes, d.transforms, d.colors, rows, target))
            return 0
        return call

    def renderer_max_views(self, height):
        return self._max_views

    def check(self, status, what):
        assert status == 0, what


def _renderer(max_views):
    r = object.__new__(Renderer)
    r._api, r._h = _Recorder(max_views), 77
    return r


def _composition():
    comp = object.__new__(binding.Composition)
    comp._h = 5
    return comp


def test_chunks_at_max_views_slice_host_tables():
    n, m = 7, 3
    protos = np.arange(n * m, dtype=np.uint32).reshape(n, m)
    tr = np.zeros((n, m, 6), np.float32)
    r = _renderer(3)
    r.render_instances_device(_composition(), Instances(protos, tr), 1 << 40, W, H)
    calls = r._api.calls
    assert [c[2] for c in calls] == [3, 3, 1]
    for k, c in enumerate(calls):
        assert np.array_equal(c[6], protos[3 * k:3 * k + c[2]])
        assert c[7] == (1 << 40) + 3 * k * 4 * W * H, "each chunk writes its own frames"


def test_chunks_at_the_layer_field():
    """n M <= 2^21 per call: with M = 2^19 slots a call takes 4 frames, whatever max_views allows;
    CUDA tables are passed the address of each chunk's first row."""
    n, m = 9, 1 << 19
    p = FakeCuda((n, m), "<i4", 1 << 36)
    t = FakeCuda((n, m, 6), "<f4", 1 << 37)
    c = FakeCuda((n, m, 4), "<f4", 1 << 38)
    r = _renderer(100)
    comp = _composition()
    r.render_instances_device(comp, Instances(p, t, c), 1 << 40, W, H)
    calls = r._api.calls
    assert [c[2] for c in calls] == [4, 4, 1]
    assert all(c[1] == m and c[2] * m <= 1 << 21 for c in calls)
    for k, call in enumerate(calls):
        assert call[3:6] == ((1 << 36) + 4 * k * 4 * m, (1 << 37) + 4 * k * 24 * m, (1 << 38) + 4 * k * 16 * m)


def test_ids_masks_stats_chunks():
    n, m = 5, 2
    inst = Instances(np.zeros((n, m), np.uint32))
    comp = _composition()
    r = _renderer(2)
    r.render_instances_ids_device(comp, inst, 1 << 40, W, H, rgba_ptr=1 << 41)
    r.render_instances_masks_device(comp, inst, 1 << 42, W, H, 0, 3)
    r.render_instances_stats_device(comp, inst, 1 << 43, W, H, 0, 3)
    by = {}
    for c in r._api.calls:
        by.setdefault(c[0], []).append(c)
    assert [c[2] for c in by["renderer_render_instances_ids_device"]] == [2, 2, 1]
    assert [c[7] for c in by["renderer_render_instances_ids_device"]] == [(1 << 41) + k * 4 * W * H for k in (0, 2, 4)]
    assert [c[7] for c in by["renderer_render_instances_masks_device"]] == [(1 << 42) + k * 3 * 4 * W * H for k in (0, 2, 4)]
    assert [c[7] for c in by["renderer_render_instances_stats_device"]] == [(1 << 43) + k * 3 * 48 for k in (0, 2, 4)]


def test_oracle_library_loads_without_instance_symbols(oracle_api):
    assert not any(hasattr(oracle_api, name) for name in binding.INSTANCE_SYMBOLS)
    assert hasattr(oracle_api, "renderer_render")
