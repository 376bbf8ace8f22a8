"""The painter's per-pixel styling on the device against the oracle, at tolerance 0, for every
scene of tests/style_scenes.py: sRGB8 bytes, and RGBA16F / RGBA32F bits (a NaN matches any
NaN). Scenes run in RGBA and BGRA order (all six orders for the encoder sweep), into host and
device memory, with paint_wide 0 and 1 (sRGB8), with a crop and a padded stride (a subset),
and through render_views* / render_batch* (a subset, direct and repacked). A mismatch reports
the first differing pixel, the paths of its tile's entries from the path model, and the device
and oracle values with their float bits."""
import numpy as np
import pytest

import oracle_linear
import style_scenes as ss
from forma_b200.binding import BGR0, BGR1, BGRA, RGB0, RGB1, RGBA, Rect

pytestmark = pytest.mark.gpu

ORDERS = {"RGBA": RGBA, "BGRA": BGRA, "RGB0": RGB0, "BGR0": BGR0, "RGB1": RGB1, "BGR1": BGR1}
DTYPES = {"f32": np.float32, "f16": np.float16}
BPP = {"f32": 16, "f16": 8}
SENTINEL = 0xA5
NAMES = list(ss.SCENES)
SUBSET = ["matrix_lin4", "matrix_tex", "hostile_nan_r", "gradient_edges", "gradient_stack", "encoder_sweep"]
VIEWS = [[1.0, 0.0, 0.0, 1.0, 0.0, 0.0], [1.0, 0.0, 0.0, 1.0, 0.0, 16.0], [1.0, 0.0, 0.0, 1.0, 3.5, -7.25],
         [0.0, -1.0, 1.0, 0.0, 32.0, 0.0]]
BATCH = ["matrix_lin4", "matrix_tex", "matrix_lin4", "matrix_rad4", "matrix_solid"]  # all 512 x 256

_ORACLE, _MODEL = {}, {}


@pytest.fixture(autouse=True)
def _oracle_linear(oracle_api):
    oracle_linear.attach(oracle_api)


@pytest.fixture()
def paint_wide_restored(cuda_api):
    saved = cuda_api.get_option("paint_wide")
    yield
    cuda_api.set_option("paint_wide", saved)


def oracle_frames(oracle_api, name, order="RGBA", xf=None):
    """(sRGB8 [h, w, 4], f32 [h, w, 4]) of the oracle; xf: a transform set on every layer."""
    key = (name, order, tuple(xf) if xf else None)
    if key not in _ORACLE:
        comp, built, sc = ss.build(oracle_api, name)
        if xf is not None:
            for o in built.layers:
                comp.get(o).set_transform(list(xf))
        ch = ORDERS[order]
        buf = np.zeros(sc.width * sc.height * 4, np.uint8)
        oracle_api.Renderer(0).render(comp, buf, sc.width, sc.height, ch, sc.clear)
        f = oracle_linear.render(oracle_api, comp, sc.width, sc.height, ch, sc.clear)
        _ORACLE[key] = (buf.reshape(sc.height, sc.width, 4), f)
        if xf is None and order == "RGBA":
            r = oracle_api.Renderer(0)
            r.render(comp, np.zeros(sc.width * sc.height * 4, np.uint8), sc.width, sc.height, RGBA, sc.clear)
            _MODEL[name] = ss.PathModel(r.segments(), sc.width, sc.height, built.layers)
    return _ORACLE[key]


def _bits(v):
    v = np.asarray(v)
    return [f"{x!r}/0x{int(b):0{2 * v.itemsize}x}" for x, b in
            zip(v.tolist(), v.view({4: np.uint32, 2: np.uint16}[v.itemsize]).tolist())] if v.dtype.kind == "f" else v.tolist()


def check(got, want32, fmt, what, name, oracle_api):
    """got [h, w, 4] (uint8 for fmt "srgb8", else the format's dtype) against the oracle."""
    if fmt == "srgb8":
        g, w = np.asarray(got, np.uint8), want32
        bad = (g != w)
    else:
        w = want32.astype(DTYPES[fmt])
        bits = np.uint32 if fmt == "f32" else np.uint16
        g = np.ascontiguousarray(got, DTYPES[fmt])
        bad = (g.view(bits) != w.view(bits)) & ~(np.isnan(g) & np.isnan(w))
    if not bad.any():
        return
    px = bad.any(axis=-1)
    ys, xs = np.nonzero(px)
    y, x = int(ys[0]), int(xs[0])
    if name not in _MODEL:
        oracle_frames(oracle_api, name)
    model = _MODEL[name]
    raise AssertionError(f"{name} {what} ({fmt}): {len(ys)} pixels differ, first at x={x} y={y} (tile {x // 16}, {y // 16}; "
                         f"entries {model.path_at(x % model.w, y % model.h)}): cuda {_bits(g[y, x])} oracle {_bits(w[y, x])}")


def _dev(n, dtype):
    import torch
    return torch.zeros(n, dtype=dtype, device="cuda:0")


@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("order", ["RGBA", "BGRA"])
@pytest.mark.parametrize("name", NAMES)
def test_srgb8(cuda_api, oracle_api, paint_wide_restored, name, order, where):
    import torch
    want, _ = oracle_frames(oracle_api, name, order)
    comp, _, sc = ss.build(cuda_api, name)
    r = cuda_api.Renderer(0)
    for wide in (0, 1):
        cuda_api.set_option("paint_wide", wide)
        if where == "host":
            buf = np.zeros(sc.width * sc.height * 4, np.uint8)
            r.render(comp, buf, sc.width, sc.height, ORDERS[order], sc.clear)
        else:
            t = _dev(sc.width * sc.height * 4, torch.uint8)
            r.render_device(comp, t.data_ptr(), sc.width, sc.height, ORDERS[order], sc.clear)
            torch.cuda.synchronize()
            buf = t.cpu().numpy()
        check(buf.reshape(sc.height, sc.width, 4), want, "srgb8", f"{order} {where} paint_wide {wide}", name, oracle_api)


@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("fmt", ["f32", "f16"])
@pytest.mark.parametrize("name", NAMES)
def test_linear(cuda_api, oracle_api, name, fmt, where):
    import torch
    comp, _, sc = ss.build(cuda_api, name)
    r = cuda_api.Renderer(0)
    for order in ("RGBA", "BGRA"):
        _, want = oracle_frames(oracle_api, name, order)
        if where == "host":
            out = np.zeros((sc.height, sc.width, 4), DTYPES[fmt])
            r.render_linear(comp, out, sc.width, sc.height, ORDERS[order], sc.clear, format=fmt)
        else:
            t = torch.zeros((sc.height, sc.width, 4), dtype=torch.float32 if fmt == "f32" else torch.float16, device="cuda:0")
            r.render_linear_device(comp, t.data_ptr(), sc.width, sc.height, ORDERS[order], sc.clear, format=fmt)
            torch.cuda.synchronize()
            out = t.cpu().numpy()
        check(out, want, fmt, f"{order} {where}", name, oracle_api)


@pytest.mark.parametrize("order", list(ORDERS))
def test_encoder_sweep_every_order(cuda_api, oracle_api, order):
    name = "encoder_sweep"
    comp, built, sc = ss.build(cuda_api, name)
    r = cuda_api.Renderer(0)
    want8, want32 = oracle_frames(oracle_api, name, order)
    buf = np.zeros(sc.width * sc.height * 4, np.uint8)
    r.render(comp, buf, sc.width, sc.height, ORDERS[order], sc.clear)
    got8 = buf.reshape(sc.height, sc.width, 4)
    check(got8, want8, "srgb8", order, name, oracle_api)
    for fmt in ("f32", "f16"):
        out = np.zeros((sc.height, sc.width, 4), DTYPES[fmt])
        r.render_linear(comp, out, sc.width, sc.height, ORDERS[order], sc.clear, format=fmt)
        check(out, want32, fmt, order, name, oracle_api)
    for ty, _ in built.notes["solid_rows"]:  # folded tiles 0-7 and painted tiles 8-15: the same bytes
        rows = got8[16 * ty:16 * ty + 16]
        assert (rows == rows[0, 0]).all(), f"{order} tile row {ty}: folded and painted tiles encode differently"


@pytest.mark.parametrize("name", SUBSET)
def test_crop_and_padded_stride(cuda_api, oracle_api, name):
    import torch
    comp, _, sc = ss.build(cuda_api, name)
    w, h = sc.width, sc.height
    crop = Rect((min(20, w - 1), w - 3), (min(5, h - 1), h))
    x0, y0 = (crop.horizontal[0] // 16) * 16, (crop.vertical[0] // 16) * 16
    x1, y1 = min(w, -(-crop.horizontal[1] // 16) * 16), min(h, -(-crop.vertical[1] // 16) * 16)
    r = cuda_api.Renderer(0)
    want8, want32 = oracle_frames(oracle_api, name, "BGRA")
    for fmt, bpp in (("srgb8", 4), ("f32", 16), ("f16", 8)):
        for where in ("host", "device"):
            stride = bpp * w + 36 if fmt == "srgb8" else bpp * w + 4
            n = h * stride
            if where == "host":
                raw = np.full(n, SENTINEL, np.uint8)
                if fmt == "srgb8":
                    r.render(comp, raw, w, h, BGRA, sc.clear, crop, stride=stride)
                else:
                    r.render_linear(comp, raw.view(DTYPES[fmt]), w, h, BGRA, sc.clear, crop, format=fmt, stride=stride)
            else:
                t = torch.full((n,), SENTINEL, dtype=torch.uint8, device="cuda:0")
                if fmt == "srgb8":
                    r.render_device(comp, t.data_ptr(), w, h, BGRA, sc.clear, crop, stride=stride)
                else:
                    r.render_linear_device(comp, t.data_ptr(), w, h, BGRA, sc.clear, crop, format=fmt, stride=stride)
                torch.cuda.synchronize()
                raw = t.cpu().numpy()
            grid = raw.reshape(h, stride)
            inside = grid[y0:y1, x0 * bpp:x1 * bpp].copy()
            got = inside.reshape(y1 - y0, x1 - x0, 4) if fmt == "srgb8" else inside.view(DTYPES[fmt]).reshape(y1 - y0, x1 - x0, 4)
            check(got, (want8 if fmt == "srgb8" else want32)[y0:y1, x0:x1], fmt, f"crop, padded stride, {where}", name, oracle_api)
            mask = np.ones(grid.shape, bool)
            mask[y0:y1, x0 * bpp:x1 * bpp] = False
            assert (grid[mask] == SENTINEL).all(), f"{name} {fmt} {where}: bytes outside the crop's tile rectangle written"


def _stack_out(n, w, h, fmt, where, padded):
    bpp = 4 if fmt == "srgb8" else BPP[fmt]
    stride = bpp * w + (16 if padded else 0)
    frame_stride = stride * h + (48 if padded else 0)
    size = (n - 1) * frame_stride + h * stride
    if where == "device":
        import torch
        t = torch.full((size,), SENTINEL, dtype=torch.uint8, device="cuda:0")
        return t, t.data_ptr(), stride, frame_stride
    raw = np.full(size, SENTINEL, np.uint8)
    return raw, raw if fmt == "srgb8" else raw.view(DTYPES[fmt]), stride, frame_stride


def _unstack(raw, n, w, h, fmt, stride, frame_stride):
    if not isinstance(raw, np.ndarray):
        import torch
        torch.cuda.synchronize()
        raw = raw.cpu().numpy()
    bpp = 4 if fmt == "srgb8" else BPP[fmt]
    out = []
    for b in range(n):
        rows = np.stack([raw[b * frame_stride + y * stride:b * frame_stride + y * stride + bpp * w] for y in range(h)])
        out.append(rows.reshape(h, w, 4) if fmt == "srgb8" else rows.copy().view(DTYPES[fmt]).reshape(h, w, 4))
    return out


@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("fmt", ["srgb8", "f32", "f16"])
@pytest.mark.parametrize("name", ["matrix_lin4", "matrix_tex", "gradient_edges", "hostile_nan_r"])
def test_views(cuda_api, oracle_api, name, fmt, where, padded):
    """Gradients and textures are sampled at the rows of their view: views 1-3 put them on
    stacked tile rows other than the view's first."""
    comp, _, sc = ss.build(cuda_api, name)
    n, w, h = len(VIEWS), sc.width, sc.height
    buf, arg, stride, fs = _stack_out(n, w, h, fmt, where, padded)
    r = cuda_api.Renderer(0)
    if fmt == "srgb8":
        (r.render_views_device if where == "device" else r.render_views)(comp, VIEWS, arg, w, h, RGBA, sc.clear, stride, fs)
    else:
        (r.render_views_linear_device if where == "device" else r.render_views_linear)(
            comp, VIEWS, arg, w, h, RGBA, sc.clear, format=fmt, stride=stride, view_stride=fs)
    got = _unstack(buf, n, w, h, fmt, stride, fs)
    for b, v in enumerate(VIEWS):
        want8, want32 = oracle_frames(oracle_api, name, "RGBA", v)
        check(got[b], want8 if fmt == "srgb8" else want32, fmt, f"view {b} {where} padded {padded}", name, oracle_api)


@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("fmt", ["srgb8", "f32", "f16"])
def test_batch(cuda_api, oracle_api, fmt, where, padded):
    distinct = {nm: ss.build(cuda_api, nm) for nm in dict.fromkeys(BATCH)}
    comps = [distinct[nm][0] for nm in BATCH]
    sc = distinct[BATCH[0]][2]
    w, h = sc.width, sc.height
    assert all(d[2].width == w and d[2].height == h and d[2].clear == sc.clear for d in distinct.values())
    n = len(comps)
    buf, arg, stride, fs = _stack_out(n, w, h, fmt, where, padded)
    r = cuda_api.Renderer(0)
    if fmt == "srgb8":
        (r.render_batch_device if where == "device" else r.render_batch)(comps, arg, w, h, RGBA, sc.clear, stride, fs)
    else:
        (r.render_batch_linear_device if where == "device" else r.render_batch_linear)(
            comps, arg, w, h, RGBA, sc.clear, format=fmt, stride=stride, frame_stride=fs)
    got = _unstack(buf, n, w, h, fmt, stride, fs)
    for b, nm in enumerate(BATCH):
        want8, want32 = oracle_frames(oracle_api, nm)
        check(got[b], want8 if fmt == "srgb8" else want32, fmt, f"batch frame {b} {where} padded {padded}", nm, oracle_api)
