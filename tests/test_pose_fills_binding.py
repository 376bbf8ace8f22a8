"""Pose fills without a GPU: the Poses value with colours, the colours sliced per chunk (the
library calls replaced by recorders), the header's declarations of the float and over pose calls
and the forma_poses layout, the oracle library loading without the new entry points, and the
scenes' recorded props and set_pose_fill on the oracle."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import pose_fill_scenes as pfs
from forma_b200 import binding
from forma_b200.binding import Color, Poses, Renderer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H = 10, 7
NEW_SYMBOLS = ("renderer_render_poses_linear", "renderer_render_poses_linear_device", "renderer_render_poses_over_device")


class _Handle:
    def __init__(self, h):
        self._h = h


class _Recorder:
    """Stands in for an Api: the pose entry points record their arguments, with the forma_poses
    descriptor's tables read out at call time, and succeed."""

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
                elif type(a).__name__ == "CArgObject" and isinstance(a._obj, binding._CPoses):
                    out.append(self._read(a._obj, args[3]))
                else:
                    out.append(a)
            self.calls.append((name, out))
            return 0
        return call

    @staticmethod
    def _read(d, n):
        k = d.n_orders

        def table(ptr, ctype, shape):
            if not ptr:
                return None
            return np.ctypeslib.as_array((ctype * int(np.prod(shape))).from_address(ptr)).reshape(shape).copy()
        return (d.first_order, k, table(d.transforms, C.c_float, (n, k, 6)), table(d.visible, C.c_uint8, (n, k)),
                table(d.colors, C.c_float, (n, k, 4)))

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


def _colors(n, k):
    return np.arange(n * k * 4, dtype=np.float32).reshape(n, k, 4)


def test_poses_value_takes_colours():
    p = Poses(2, colors=_colors(5, 3))
    assert (p.n, p.n_orders, p.first_order, p.transforms, p.visible) == (5, 3, 2, None, None)
    assert p.colors.dtype == np.float32 and p.colors.flags["C_CONTIGUOUS"]
    p = Poses(0, np.zeros((4, 2, 6), np.float32), np.ones((4, 2), bool), _colors(4, 2))
    assert (p.n, p.n_orders) == (4, 2)
    assert Poses(0, colors=_colors(3, 4)[:, ::2]).colors.flags["C_CONTIGUOUS"]
    with pytest.raises(ValueError):
        Poses(0)
    with pytest.raises(ValueError):
        Poses(0, colors=_colors(2, 3).astype(np.float64))  # not float32
    with pytest.raises(ValueError):
        Poses(0, colors=[[[0.0, 0.0, 0.0, 1.0]]])  # not an array
    with pytest.raises(ValueError):
        Poses(0, colors=np.zeros((2, 3, 3), np.float32))  # not [n, K, 4]
    with pytest.raises(ValueError):
        Poses(0, colors=np.zeros((2, 3), np.float32))
    with pytest.raises(ValueError):
        Poses(0, np.zeros((2, 3, 6), np.float32), colors=_colors(2, 4))  # K disagrees
    with pytest.raises(ValueError):
        Poses(0, visible=np.ones((3, 3), bool), colors=_colors(2, 3))  # n disagrees


@pytest.mark.parametrize("method, symbol, bpp", [("render_poses_linear_device", "renderer_render_poses_linear_device", 16),
                                                 ("render_poses_over_device", "renderer_render_poses_over_device", 4),
                                                 ("render_poses_device", "renderer_render_poses_device", 4)])
def test_colours_are_sliced_per_chunk(method, symbol, bpp):
    r = _renderer(2)
    p = Poses(3, np.arange(5 * 4 * 6, dtype=np.float32).reshape(5, 4, 6), None, _colors(5, 4))
    getattr(r, method)(_Handle(5), p, 1 << 30, W, H, timings=False)
    calls = r._api.calls
    assert [c[0] for c in calls] == [symbol] * 3
    for j, (_, a) in enumerate(calls):
        first, count = 2 * j, min(2, 5 - 2 * j)
        handle, comp, (fo, k, t, v, c), n, ptr, w, stride, h, view_stride = a[:9]
        assert (handle, comp, fo, k, n, w, h, v) == (77, 5, 3, 4, count, W, H, None)
        assert np.array_equal(c, p.colors[first:first + count]) and np.array_equal(t, p.transforms[first:first + count])
        assert (stride, view_stride) == (bpp * W, bpp * W * H) and ptr == (1 << 30) + first * bpp * W * H


def test_linear_host_and_formats():
    r = _renderer(8)
    p = Poses(0, colors=_colors(3, 2))
    buf = np.zeros((3, H, W, 4), np.float16)
    r.render_poses_linear(_Handle(1), p, buf, W, H, format="f16", timings=False)
    (name, a), = r._api.calls
    assert name == "renderer_render_poses_linear"
    assert a[2][:4] == (0, 2, None, None) and np.array_equal(a[2][4], p.colors)
    assert a[3:9] == [3, buf.ctypes.data, W, 8 * W, H, 8 * W * H] and a[11] == 1  # FORMA_PIXEL_RGBA16F
    with pytest.raises(AssertionError):
        r.render_poses_linear(_Handle(1), p, np.zeros((2, H, W, 4), np.float16), W, H, format="f16")
    r = _renderer(8)
    r.render_poses_over_device(_Handle(1), p, 4096, W, H, format="f32", timings=False)
    (name, a), = r._api.calls
    assert a[8] == 16 * W * H and a[10] == 2 and len(a) == 12  # no clear colour; FORMA_PIXEL_RGBA32F


def test_the_header_declares_the_new_calls_and_the_field():
    with open(os.path.join(ROOT, "include", "forma_b200.h")) as f:
        header = f.read()
    for name in NEW_SYMBOLS:
        assert name in binding.POSE_SYMBOLS and name in binding.SIGNATURES
        m = re.search(r"\bint forma_%s\(([^;]*)\);" % name, header)
        assert m, name
        params = [q.strip() for q in re.sub(r"/\*.*?\*/", "", m.group(1)).split(",") if q.strip()]
        assert len(params) == len(binding.SIGNATURES[name][1]), name
        assert params[2] == "const forma_poses* poses" and params[3] == "uint32_t n"
        twin = re.search(r"\bint forma_%s\(([^;]*)\);" % name.replace("poses", "views"), header)
        twin_params = [q.strip() for q in re.sub(r"/\*.*?\*/", "", twin.group(1)).split(",") if q.strip()]
        assert params[4:] == twin_params[4:], name
    m = re.search(r"typedef struct forma_poses \{(.*?)\} forma_poses;", header, re.S)
    assert re.sub(r"/\*.*?\*/", "", m.group(1)).split()[-2:] == ["float*", "colors;"]


def test_descriptor_layout():
    """colors is the last member: the earlier members keep their offsets, and a zeroed descriptor
    has no colours."""
    assert [f for f, _ in binding._CPoses._fields_] == ["first_order", "n_orders", "transforms", "visible", "colors"]
    assert binding._CPoses.transforms.offset == 8 and binding._CPoses.visible.offset == 16
    assert binding._CPoses.colors.offset == 24 and C.sizeof(binding._CPoses) == 32
    assert binding._CPoses(0, 4, None, None).colors is None


def test_the_oracle_loads_without_them(oracle_api):
    for name in NEW_SYMBOLS:
        assert not hasattr(oracle_api, name)
    assert hasattr(oracle_api, "renderer_render")


@pytest.mark.parametrize("name", ["e2e_texture", "e2e_clipping", "e2e_blend_modes__Hue", "alpha_flips", "window_gaps_filled",
                                  "fill_window_top"])
def test_scenes_record_every_layers_props(oracle_api, name):
    """The recorded props are those the layers were built with: the frame of set_pose_fill with each
    layer's recorded colour is the untouched frame."""
    sc = pfs.SCENES[name]
    comp, orders = sc.build(oracle_api)
    props = pfs.props_of(comp)
    assert sorted(props) == orders
    r = oracle_api.Renderer()
    before = np.zeros(sc.width * sc.height * 4, np.uint8)
    r.render(comp, before, sc.width, sc.height)
    for o, p in props.items():
        if p.func.draw is not None and p.func.draw.fill.solid is not None:
            c = p.func.draw.fill.solid
            comp.get(o).set_props(pfs.filled(p, (c.r, c.g, c.b, c.a)))
    after = np.zeros_like(before)
    r.render(comp, after, sc.width, sc.height)
    assert np.array_equal(before, after)


def test_scene_tables_are_consistent():
    for sc in pfs.SCENES.values():
        tables = [t for t in (sc.colors, sc.transforms, sc.visible) if t is not None]
        assert {t.shape[:2] for t in tables} == {(sc.n, sc.n_orders)}, sc.name
        assert sc.colors is None or sc.colors.dtype == np.float32
        assert sc.first_order + sc.n_orders <= 1 << 21
    assert len([n for n in pfs.SCENES if n.startswith("blend_top_")]) == 16


def test_set_pose_fill_changes_what_it_should(oracle_api):
    """Frames of the flips scene differ from each other; the clip layer's garbage colour changes
    nothing (frame 0 of clip_ignored equals the frame with a sane colour at the clip's slot)."""
    sc = pfs.SCENES["alpha_flips"]
    comp, orders = sc.build(oracle_api)
    r = oracle_api.Renderer()
    frames = []
    for b in range(sc.n):
        pfs.set_pose_fill(comp, sc, orders, b)
        buf = np.zeros(sc.width * sc.height * 4, np.uint8)
        r.render(comp, buf, sc.width, sc.height, clear_color=Color(1.0, 1.0, 1.0, 0.0))
        frames.append(buf)
    assert all(not np.array_equal(frames[a], frames[b]) for a in range(sc.n) for b in range(a))
    sc = pfs.SCENES["clip_ignored"]
    out = []
    for clip_colour in (None, [0.5, 0.5, 0.5, 1.0]):
        comp, orders = sc.build(oracle_api)
        if clip_colour is not None:
            sc = pfs.FillScene(sc.name, sc.build, sc.width, sc.height, sc.first_order, sc.colors.copy())
            sc.colors[0, 1] = clip_colour
        pfs.set_pose_fill(comp, sc, orders, 0)
        buf = np.zeros(sc.width * sc.height * 4, np.uint8)
        r.render(comp, buf, sc.width, sc.height)
        out.append(buf)
    assert np.array_equal(out[0], out[1])
