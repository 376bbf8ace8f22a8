"""Frames over a background without a GPU: the decode table D, the over oracle
(tests/oracle_over.py) and the binding of the three over entry points.

- D: every byte round-trips through the project's encoder (the oracle's compute_srgb encode),
  alpha too; D[b] is the f32 of the sRGB EOTF of b / 255 where that value round-trips and the
  nearest round-tripping f32 where it does not (byte 11); D is strictly increasing.
- With a uniform background the over oracle is libforma_oracle.so (sRGB8) and
  libforma_oracle_linear.so (f32) with that clear colour, on every e2e golden scene, every scene
  of tests/extremes.py and tests/style_scenes.py and random_mixed in RGBA and BGRA order, for
  backgrounds of alpha 0, alpha 1 (the Alpha -> One upgrade) and in between.
- Pixels no layer covers keep a random background.
- The header declares the entry points and the binding knows them (OVER_SYMBOLS)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import extremes
import oracle_linear
import oracle_over
import scenes
import style_scenes as ss
import synth
from forma_b200 import binding
from forma_b200.binding import BGRA, RGBA, BlendMode, Color, Fill, Func, Props, Rect, Renderer, Style

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORDERS = {"RGBA": RGBA, "BGRA": BGRA}
# Background pixels (bytes in RGBA order): alpha 0, alpha 1 and in between; byte 11 is D's corrected entry.
BG_BYTES = {"a0": (200, 11, 90, 0), "a1": (30, 140, 250, 255), "mid": (64, 128, 11, 77)}
# Float backgrounds (r, g, b, a).
BG_FLOATS = {"a0": (0.75, 0.125, 0.5, 0.0), "a1": (0.2, 0.4, 0.6, 1.0), "mid": (1.5, -0.25, 0.3, 0.4)}


@pytest.fixture(autouse=True)
def _recip_mode_0(oracle_api):
    oracle_api.hooks.fo_set_recip_mode(0)


def eotf(b: int) -> float:
    c = b / 255.0
    return c / 12.92 if c <= 0.04045 else ((c + 0.055) / 1.055) ** 2.4


def encode_colour(values) -> np.ndarray:
    """compute_srgb's byte of each value as a colour channel (the oracle's encoder)."""
    v = np.asarray(values, np.float32).reshape(-1, 1)
    frame = np.concatenate([v, v, v, np.zeros_like(v)], axis=1).reshape(1, -1, 4)
    return oracle_linear.encode(frame, RGBA)[0, :, 0]


# --- the decode table ----------------------------------------------------------------------------
def test_decode_table_round_trips_every_byte():
    d = oracle_over.decode_table()
    assert (encode_colour(d) == np.arange(256)).all()
    alpha = np.arange(256, dtype=np.float32) / np.float32(255.0)
    frame = np.stack([np.zeros(256, np.float32)] * 3 + [alpha], axis=1).reshape(1, 256, 4)
    assert (oracle_linear.encode(frame, RGBA)[0, :, 3] == np.arange(256)).all()
    assert (np.diff(d.astype(np.float64)) > 0).all()


def test_decode_table_is_the_eotf_where_it_round_trips():
    d = oracle_over.decode_table()
    nearest = np.array([np.float32(eotf(b)) for b in range(256)], np.float32)
    trips = encode_colour(nearest) == np.arange(256)
    assert (d[trips] == nearest[trips]).all()
    assert list(np.nonzero(~trips)[0]) == [11]
    assert abs(float(d[11]) - 0.0033159761) < 1e-9
    # The nearest f32 that round-trips: D[11]'s neighbour towards the EOTF does not, and nothing
    # between the EOTF and D[11] does (D[11] < EOTF: the f32s above it up to the EOTF encode to 12).
    e = eotf(11)
    assert float(d[11]) < e
    above = np.nextafter(d[11], np.float32(1.0))
    assert encode_colour([above])[0] == 12
    lo, hi = d[11].view(np.int32), np.float32(e).view(np.int32)
    between = np.arange(lo + 1, hi + 1, dtype=np.int32).view(np.float32)
    assert (encode_colour(between) != 11).all()
    # ... and on the other side the nearest round-tripping f32 is farther from the EOTF.
    assert (encode_colour(np.array([np.float32(e)], np.float32)) == 12).all()


def test_decode_table_matches_its_header():
    text = open(os.path.join(ROOT, "forma_b200", "csrc", "srgb_decode.h")).read()
    body = text[text.index("{"):text.rindex("}")]
    vals = [float.fromhex(v.rstrip("f")) for v in re.findall(r"-?0x[0-9a-fA-F.]+p[-+]\d+f", body)]
    assert np.array_equal(np.array(vals, np.float32), oracle_over.decode_table())


# --- uniform backgrounds ---------------------------------------------------------------------------
def srgb_twin(oracle_api, comp, w, h, channels, clear, crop, bg):
    out = np.ascontiguousarray(np.broadcast_to(np.asarray(bg, np.uint8), (h, w, 4)))
    oracle_api.Renderer(0).render(comp, out.reshape(-1), w, h, channels, clear, crop)
    return out


def f32_twin(oracle_api, comp, w, h, channels, clear, crop, bg):
    out = np.ascontiguousarray(np.broadcast_to(np.asarray(bg, np.float32), (h, w, 4)))
    oracle_linear.attach(oracle_api).Renderer(0).render_linear(comp, out, w, h, channels, clear, crop, format="f32")
    return out


def check_uniform(oracle_api, comp, w, h, crop, orders, what):
    for order in orders:
        ch = ORDERS[order]
        for name, rgba in BG_BYTES.items():
            px = [rgba[int(c)] for c in ch]  # the pixel's bytes in channel order
            frame = np.ascontiguousarray(np.broadcast_to(np.asarray(px, np.uint8), (h, w, 4)))
            assert oracle_over.render(comp, frame, ch, crop) == 0
            want = srgb_twin(oracle_api, comp, w, h, ch, oracle_over.clear_of(px, ch), crop, px)
            assert np.array_equal(frame, want), f"{what} sRGB8 {order} {name}: {(frame != want).any(axis=2).sum()} pixels differ"
        for name, c in BG_FLOATS.items():
            vals = [c[int(k)] for k in ch]
            frame = np.ascontiguousarray(np.broadcast_to(np.asarray(vals, np.float32), (h, w, 4)))
            assert oracle_over.render(comp, frame, ch, crop) == 0
            want = f32_twin(oracle_api, comp, w, h, ch, Color(*c), crop, vals)
            assert np.array_equal(frame.view(np.uint32), want.view(np.uint32)), f"{what} f32 {order} {name}"


@pytest.mark.parametrize("name", list(scenes.E2E))
def test_e2e_scene_over_uniform_background_is_the_twin(oracle_api, name):
    comp = oracle_api.Composition()
    scenes.E2E[name](oracle_api, comp)
    check_uniform(oracle_api, comp, 64, 64, None, ORDERS, name)


@pytest.mark.parametrize("name", list(extremes.SCENES))
def test_extreme_scene_over_uniform_background_is_the_twin(oracle_api, name):
    comp, _, sc = extremes.build(oracle_api, name)
    check_uniform(oracle_api, comp, sc.width, sc.height, sc.crop, ("RGBA",), name)


@pytest.mark.parametrize("name", list(ss.SCENES))
def test_style_scene_over_uniform_background_is_the_twin(oracle_api, name):
    comp, _, sc = ss.build(oracle_api, name)
    check_uniform(oracle_api, comp, sc.width, sc.height, None, ("RGBA",), name)


def test_random_mixed_over_uniform_background_is_the_twin(oracle_api):
    w, h = 200, 120
    comp = oracle_api.Composition()
    synth.random_mixed(oracle_api, comp, 150, w, h, 11)
    check_uniform(oracle_api, comp, w, h, None, ORDERS, "random_mixed")
    check_uniform(oracle_api, comp, w, h, Rect((20, 150), (17, 90)), ("BGRA",), "random_mixed crop")


# --- random backgrounds ------------------------------------------------------------------------------
def test_uncovered_pixels_keep_a_random_background(oracle_api):
    """A transparent layer over the whole frame reaches every tile; a few shapes cover part of it.
    Pixels that the shapes leave alone in two renders with different clear colours have zero
    coverage; over a random background they keep their bytes (sRGB8) and bits (f32)."""
    w, h = 96, 80
    comp = oracle_api.Composition()
    comp.get_mut_or_insert_default(0).insert(scenes.custom_square(oracle_api, 0.0, 0.0, float(w), float(h))).set_props(
        Props(func=Func.Draw(Style(fill=Fill.Solid(Color(0.3, 0.6, 0.9, 0.0))))))
    comp.get_mut_or_insert_default(1).insert(scenes.custom_circle(oracle_api, 30.0, 30.0, 17.0)).set_props(
        Props(func=Func.Draw(Style(fill=Fill.Solid(Color(0.9, 0.1, 0.2, 0.7)), blend_mode=BlendMode.Multiply))))
    comp.get_mut_or_insert_default(2).insert(scenes.custom_square(oracle_api, 50.0, 41.0, 77.5, 70.25)).set_props(
        Props(func=Func.Draw(Style(fill=Fill.Solid(Color(0.1, 0.8, 0.3, 1.0))))))
    a = srgb_twin(oracle_api, comp, w, h, RGBA, Color(1.0, 0.0, 0.0, 1.0), None, (255, 0, 0, 255))
    b = srgb_twin(oracle_api, comp, w, h, RGBA, Color(0.0, 0.0, 1.0, 0.0), None, (0, 0, 255, 0))
    free = (a == [255, 0, 0, 255]).all(axis=2) & (b == [0, 0, 255, 0]).all(axis=2)
    assert 0.3 < free.mean() < 0.9
    rng = np.random.default_rng(5)
    bg = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    frame = bg.copy()
    assert oracle_over.render(comp, frame, RGBA) == 0
    assert np.array_equal(frame[free], bg[free]) and not np.array_equal(frame[~free], bg[~free])
    bgf = rng.normal(0.0, 2.0, (h, w, 4)).astype(np.float32)
    framef = bgf.copy()
    assert oracle_over.render(comp, framef, BGRA) == 0
    assert np.array_equal(framef[free].view(np.uint32), bgf[free].view(np.uint32))


def test_oracle_refuses_orders_it_cannot_decode(oracle_api):
    comp = oracle_api.Composition()
    scenes.E2E["clipping"](oracle_api, comp)
    frame = np.full((64, 64, 4), 7, np.uint8)
    for ch in (binding.RGB1, binding.RGB0, (0, 0, 1, 3)):
        assert oracle_over.render(comp, frame, ch) != 0
    assert (frame == 7).all()


# --- declarations and binding ----------------------------------------------------------------------
def test_header_declares_the_over_entry_points():
    text = open(os.path.join(ROOT, "include", "forma_b200.h")).read()
    for name in binding.OVER_SYMBOLS:
        assert re.search(r"\bint forma_" + name + r"\(", text), name
        assert name in binding.SIGNATURES
    assert "FORMA_PIXEL_SRGB8 = 0" in text
    assert binding.over_format("srgb8") == (0, 4, np.uint8)
    with pytest.raises(ValueError):
        binding.over_format("u8")


def test_oracle_library_loads_without_the_over_entry_points(oracle_api):
    assert not any(hasattr(oracle_api, n) for n in binding.OVER_SYMBOLS)


class _Handle:
    def __init__(self, h):
        self._h = h


class _Recorder:
    def __init__(self, max_views):
        self.calls, self._max_views = [], max_views
        for name in binding.OVER_SYMBOLS:
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


@pytest.mark.parametrize("fmt,bpp,code", [("srgb8", 4, 0), ("f16", 8, 1), ("f32", 16, 2)])
def test_binding_passes_channels_without_a_clear_colour(fmt, bpp, code):
    W, H = 10, 7
    r = _renderer(2)
    r.render_over_device(_Handle(5), 1 << 20, W, H, BGRA, format=fmt, timings=False)
    name, a = r._api.calls[-1]
    assert name == "renderer_render_over_device" and a[:6] == [77, 5, 1 << 20, W, bpp * W, H]
    assert list(a[6]) == list(BGRA) and a[7] is None and a[8] == code and a[9] is None and len(a) == 10
    r.render_views_over_device(_Handle(5), np.zeros((3, 6), np.float32), 1 << 20, W, H, format=fmt, timings=False)
    views = [c for c in r._api.calls if c[0] == "renderer_render_views_over_device"]
    assert [c[1][3] for c in views] == [2, 1]  # chunked by max_views
    a = views[1][1]
    assert a[4] == (1 << 20) + 2 * bpp * W * H and a[5:9] == [W, bpp * W, H, bpp * W * H]
    assert list(a[9]) == list(RGBA) and a[10] == code and len(a) == 12
    r.render_batch_over_device([_Handle(1), _Handle(2)], 1 << 20, W, H, format=fmt, frame_stride=bpp * W * H + 64, timings=False)
    name, a = r._api.calls[-1]
    assert name == "renderer_render_batch_over_device" and a[2] == 2 and a[4:8] == [W, bpp * W, H, bpp * W * H + 64]
    assert a[9] == code and len(a) == 11
