"""The oracle's layer coverage masks (fo_renderer_render_masks, tests/oracle_masks.py), pinned without a
GPU to the oracles already pinned: each layer's F32 plane is the alpha of a linear oracle frame of the
composition with every other Draw layer disabled and the layer made solid white, opaque and Over
(clear colour 0, so no Alpha -> One upgrade: alpha = coverage x clip mask exactly); its U8 plane is
that frame's sRGB8 alpha byte; on clip-free scenes the ID oracle is the top-most mask above its
threshold. tests/test_gpu_masks.py then holds the device to these planes."""
import numpy as np
import pytest

import extremes
import oracle_ids
import oracle_linear
import oracle_masks
import scenes
import synth
from forma_b200.binding import ID_NONE, RGBA, BlendMode, Color, Fill, FormaError, Func, Layer, Props, Rect, Style

WHITE = Color(1.0, 1.0, 1.0, 1.0)
CLEAR = Color(0.0, 0.0, 0.0, 0.0)
MAX_ORDER_SCAN = 8192


class Recorder:
    """The props every layer was given while a scene was built (the binding cannot read them back)."""

    def __init__(self, monkeypatch):
        self.props = {}
        orig = Layer.set_props

        def set_props(layer, p):
            self.props[layer._h] = p
            return orig(layer, p)
        monkeypatch.setattr(Layer, "set_props", set_props)

    def build(self, api, build):
        self.props.clear()
        comp = api.Composition()
        build(api, comp)
        layers, n = {}, len(comp)
        for o in range(MAX_ORDER_SCAN):
            if len(layers) == n:
                break
            layer = comp.get(o)
            if layer is not None:
                layers[o] = (self.props.get(layer._h, Props()), layer.is_enabled())
        return comp, layers


@pytest.fixture
def recorder(monkeypatch, oracle_api):
    oracle_masks.attach(oracle_api)
    oracle_linear.attach(oracle_api)
    oracle_ids.attach(oracle_api)
    return Recorder(monkeypatch)


def isolated(api, recorder, build, order, layers):
    """The composition with every Draw layer but `order` disabled and `order` made solid white,
    opaque and Over (a clip layer becomes an unclipped Draw layer)."""
    comp, _ = recorder.build(api, build)
    for o, (p, _) in layers.items():
        if o != order and p.func.draw is not None:
            comp.get(o).set_is_enabled(False)
    p = layers[order][0]
    clipped = p.func.draw is not None and p.func.draw.is_clipped
    comp.get(order).set_props(Props(fill_rule=p.fill_rule,
                                    func=Func.Draw(Style(is_clipped=clipped, fill=Fill.Solid(WHITE), blend_mode=BlendMode.Over))))
    return comp


def check_layers(api, recorder, build, w, h, crop=None, limit=None):
    comp, layers = recorder.build(api, build)
    n = max(layers) + 1 if layers else 1
    f32 = oracle_masks.render(api, comp, w, h, 0, n, "f32", crop)
    u8 = oracle_masks.render(api, comp, w, h, 0, n, "u8", crop)
    orders = sorted(layers)
    if limit is not None and len(orders) > limit:  # clips and clipped layers first, then a spread of the rest
        clipish = [o for o in orders if layers[o][0].func.draw is None or layers[o][0].func.draw.is_clipped]
        rest = [o for o in orders if o not in clipish]
        orders = sorted(set(clipish[:limit // 2] + rest[::max(1, len(rest) // (limit - min(len(clipish), limit // 2)))]))
    checked = 0
    for o in orders:
        iso = isolated(api, recorder, build, o, layers)
        alpha = oracle_linear.render(api, iso, w, h, RGBA, CLEAR, crop)[..., 3]
        assert np.array_equal(alpha.view(np.uint32), f32[o].view(np.uint32)), \
            f"order {o}: {int((alpha != f32[o]).sum())} pixels differ from the isolated linear frame"
        buf = np.zeros(w * h * 4, np.uint8)
        api.Renderer(0).render(iso, buf, w, h, RGBA, CLEAR, crop)
        assert np.array_equal(buf.reshape(h, w, 4)[..., 3], u8[o]), f"order {o}: U8 plane != sRGB8 alpha"
        checked += 1
    return f32, layers, checked


@pytest.mark.parametrize("name", sorted(scenes.E2E))
def test_layers_e2e(oracle_api, recorder, name):
    f32, layers, checked = check_layers(oracle_api, recorder, scenes.E2E[name], 64, 64)
    assert checked == len(layers)
    assert all(((f32 * 512) % 1 == 0).ravel()) or any(layers[o][0].func.draw is not None and layers[o][0].func.draw.is_clipped
                                                      for o in layers)


def test_layers_random_mixed(oracle_api, recorder):
    _, layers, checked = check_layers(oracle_api, recorder, lambda a, c: synth.random_mixed(a, c, 40, 120, 90, 5), 120, 90)
    assert checked == len(layers) == 40


@pytest.mark.parametrize("name", sorted(extremes.SCENES))
def test_layers_extremes(oracle_api, recorder, name):
    sc = extremes.SCENES[name]
    big = sc.width * sc.height > 1 << 18
    _, layers, checked = check_layers(oracle_api, recorder, sc.build, sc.width, sc.height, sc.crop, limit=3 if big else 8)
    assert checked >= min(len(layers), 3)


def clip_free(layers):
    return all(p.func.draw is not None and not p.func.draw.is_clipped for p, _ in layers.values())


@pytest.mark.parametrize("name", [n for n in sorted(scenes.E2E) if n not in scenes.NON_SEPARABLE] + ["random_mixed"])
@pytest.mark.parametrize("threshold", [0.0, 0.5])
def test_ids_are_the_top_most_mask(oracle_api, recorder, name, threshold):
    # Only scenes without clip-ish layers: the painter never paints a clipped layer above its first
    # opaque layer (so it never hits there), while its amodal mask keeps it.
    build = scenes.E2E.get(name) or (lambda a, c: synth.random_mixed(a, c, 60, 120, 90, 9))
    w, h = (64, 64) if name in scenes.E2E else (120, 90)
    comp, layers = recorder.build(oracle_api, build)
    if not clip_free(layers):
        pytest.skip("clip-ish layers")
    n = max(layers) + 1
    m = oracle_masks.render(oracle_api, comp, w, h, 0, n)
    ids = np.zeros(w * h, np.uint32)
    oracle_api.Renderer(0).render_ids(comp, ids, w, h, min_coverage=threshold)
    want = np.full((h, w), ID_NONE, np.uint32)
    for o in range(n):
        want[m[o] > threshold] = o
    assert np.array_equal(ids.reshape(h, w), want)


def test_windows(oracle_api, recorder):
    w, h = 100, 70
    build = lambda a, c: synth.random_mixed(a, c, 30, w, h, 4)  # noqa: E731
    comp, layers = recorder.build(oracle_api, build)
    n = max(layers) + 1
    full = oracle_masks.render(oracle_api, comp, w, h, 0, n)
    assert sum(bool(full[o].any()) for o in range(n)) > n // 2  # (some layers lie off the frame)
    for first, k in ((0, 1), (7, 1), (0, 5), (n - 3, 6), (n, 4), (n + 100, 2), ((1 << 21) - 2, 2)):
        got = oracle_masks.render(oracle_api, comp, w, h, first, k)
        for j in range(k):
            want = full[first + j] if first + j < n else np.zeros((h, w), np.float32)
            assert np.array_equal(got[j], want), (first, k, j)
    u8 = oracle_masks.render(oracle_api, comp, w, h, 0, n, "u8")
    assert np.array_equal(u8, np.rint(np.float32(255.0) * full).astype(np.uint8))  # to_byte: 255 v, rounded half to even


@pytest.mark.parametrize("fmt,bpp", [("f32", 4), ("u8", 1)])
def test_crop_and_padded_strides(oracle_api, recorder, fmt, bpp):
    w, h, k, pad, gap = 100, 70, 5, 12, 40
    comp, _ = recorder.build(oracle_api, lambda a, c: synth.random_mixed(a, c, 12, w, h, 6))
    full = oracle_masks.render(oracle_api, comp, w, h, 2, k, fmt)
    stride = bpp * w + pad
    plane_stride = stride * h + gap
    buf = np.full(k * plane_stride, 0xAB, np.uint8)
    arr = buf.view(np.float32) if fmt == "f32" else buf
    oracle_api.Renderer(0).render_masks(comp, arr, w, h, 2, n_orders=k, crop=Rect((20, 50), (17, 40)), stride=stride,
                                        plane_stride=plane_stride)
    for j in range(k):
        plane = buf[j * plane_stride:j * plane_stride + h * stride].reshape(h, stride)
        inside = np.zeros(plane.shape, bool)
        inside[16:48, 16 * bpp:64 * bpp] = True
        got = plane[inside].reshape(32, 48 * bpp).view(full.dtype)
        assert np.array_equal(got, full[j, 16:48, 16:64])
        assert (plane[~inside] == 0xAB).all()
        assert (buf[j * plane_stride + h * stride:(j + 1) * plane_stride] == 0xAB).all()


@pytest.mark.parametrize("case", ["k0", "past_field", "format", "stride", "plane_stride", "unaligned"])
def test_invalid_arguments_leave_the_buffer(oracle_api, recorder, case):
    w, h = 64, 64
    comp, _ = recorder.build(oracle_api, scenes.E2E["clipping"])
    buf = np.full(4 * (4 * w * h + 64), 0x5A, np.uint8)
    kw = dict(first_order=0, n_orders=2, stride=4 * w, plane_stride=4 * w * h)
    arr = buf.view(np.float32)
    if case == "k0":
        kw["n_orders"] = 0
    elif case == "past_field":
        kw["first_order"] = (1 << 21) - 1
    elif case == "stride":
        kw["stride"] = 4 * w - 4
    elif case == "plane_stride":
        kw["plane_stride"] = 4 * w * h - 4
    elif case == "unaligned":
        kw["stride"] = 4 * w + 2
        kw["plane_stride"] = (4 * w + 2) * h
    if case == "format":
        from forma_b200.binding import _CMasks
        import ctypes as C
        m = _CMasks(buf.ctypes.data, 0, 2, 7, 4 * w, 4 * w * h)
        r = oracle_api.Renderer(0)
        assert oracle_api.renderer_render_masks(r._h, comp._h, C.byref(m), w, h, None, None) != 0
    else:
        with pytest.raises(FormaError):
            oracle_api.Renderer(0).render_masks(comp, arr, w, h, **kw)
    assert (buf == 0x5A).all()
