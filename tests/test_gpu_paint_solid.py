"""The paint kernel's lean build for frames whose layers are all solid `Over` fills without clips
(option paint_solid, Composition::solid_over_only): such frames must come out byte for byte as
the general build paints them and as the oracle renders them, and every other frame must stay
on the general build.

Frames: the paris-30k and 100 k-cubic workloads at 4K, every scene of tests/style_scenes.py and
tests/extremes.py (non-finite colours, a -0 clear, even-odd and deep windings, crowded tiles,
crops), in all six channel orders, with a crop and a padded stride, into host and device
memory, as views and as batches, and over several frames with a layer cache while layers move.
Which kernel painted a frame is read from torch.profiler's kernel names."""
import numpy as np
import pytest

import extremes
import style_scenes as ss
import synth
import workloads
from forma_b200.binding import (BGR0, BGR1, BGRA, RGB0, RGB1, RGBA, BlendMode, Color, Fill, FillRule, Func, GradientBuilder, Point,
                                Props, Rect, Style)

pytestmark = pytest.mark.gpu

CLEAR = Color(1.0, 1.0, 1.0, 0.0)
ORDERS = (RGBA, BGRA, RGB0, BGR0, RGB1, BGR1)


@pytest.fixture()
def paint_solid_restored(cuda_api):
    saved = cuda_api.get_option("paint_solid")
    yield
    cuda_api.set_option("paint_solid", saved)


def painters(fn):
    """The paint kernels (lean "solid" / "general") that ran during fn(). fn is called again when
    the profiler delivered no paint kernel at all (its activity records of a short session can go
    missing); every call renders the same frame."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    out = set()
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        for n in {e.key for e in prof.key_averages()}:
            if "paint_solid_kernel" in n or "paint_views_solid_kernel" in n:
                out.add("solid")
            elif "paint_kernel<" in n or "paint_views_kernel<" in n:
                out.add("general")
        if out:
            return out
    return out


def is_solid_over(props: Props) -> bool:
    d = props.func.draw
    return d is not None and d.fill.solid is not None and d.blend_mode == BlendMode.Over and not d.is_clipped


def render_both(cuda_api, comp, w, h, fn):
    """fn(renderer, comp) -> frame, with paint_solid 1 then 0: (frames, painters of each)."""
    frames, used = [], []
    r = cuda_api.Renderer(0)
    for v in (1, 0):
        cuda_api.set_option("paint_solid", v)
        box = []
        used.append(painters(lambda: box.append(fn(r, comp))))
        frames.append(box[0])
    return frames, used


def host_frame(w, h, channels=RGBA, crop=None, stride=None, clear=CLEAR):
    def fn(r, comp):
        s = stride or w * 4
        buf = np.full(h * s, 0xA5, np.uint8)
        r.render(comp, buf, w, h, channels, clear, crop, stride=s)
        return buf
    return fn


def device_frame(w, h, channels=RGBA, clear=CLEAR):
    def fn(r, comp):
        import torch
        t = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda:0")
        r.render_device(comp, t.data_ptr(), w, h, channels, clear)
        torch.cuda.synchronize()
        return t.cpu().numpy()
    return fn


def oracle_frame(oracle_api, comp, w, h, channels=RGBA, crop=None, stride=None, clear=CLEAR):
    s = stride or w * 4
    buf = np.full(h * s, 0xA5, np.uint8)
    oracle_api.Renderer(0).render(comp, buf, w, h, channels, clear, crop, stride=s)
    return buf


def check(frames, used, want, solid, what):
    lean, general = frames
    assert used[0] == ({"solid"} if solid else {"general"}), f"{what}: paint_solid 1 ran {used[0]}"
    assert used[1] == {"general"}, f"{what}: paint_solid 0 ran {used[1]}"
    assert np.array_equal(lean, general), f"{what}: the lean and the general build differ"
    if want is not None:
        assert np.array_equal(lean, want), f"{what}: differs from the oracle"


@pytest.mark.parametrize("name", ["paris4k", "cubics100k"])
def test_workloads(cuda_api, oracle_api, paint_solid_restored, name):
    comp, w, h = workloads.build_scene(cuda_api, name)
    ocomp, _, _ = workloads.build_scene(oracle_api, name)
    want = oracle_frame(oracle_api, ocomp, w, h)
    for where, fn in (("host", host_frame(w, h)), ("device", device_frame(w, h))):
        frames, used = render_both(cuda_api, comp, w, h, fn)
        check(frames, used, want, True, f"{name} {where}")


@pytest.mark.parametrize("name", list(ss.SCENES))
def test_style_scenes(cuda_api, oracle_api, paint_solid_restored, name):
    comp, built, sc = ss.build(cuda_api, name)
    ocomp, _, _ = ss.build(oracle_api, name)
    solid = all(is_solid_over(p) for p in built.layers.values())
    for ch in (RGBA, BGRA):
        want = oracle_frame(oracle_api, ocomp, sc.width, sc.height, ch, clear=sc.clear)
        frames, used = render_both(cuda_api, comp, sc.width, sc.height, host_frame(sc.width, sc.height, ch, clear=sc.clear))
        check(frames, used, want, solid, f"{name} channels {ch}")


def test_style_scenes_include_solid_over_frames():
    """The scenes above exercise the lean build: the defects (non-finite colours, a -0 clear)
    are solid `Over` frames, and most other scenes are not."""
    from oracle import oracle
    api = oracle.load()
    solid = {n for n in ss.SCENES if all(is_solid_over(p) for p in ss.build(api, n)[1].layers.values())}
    assert {"defect_nan_r", "defect_inf_r", "defect_inf_a", "defect_neg_zero_clear"} <= solid, sorted(solid)
    assert solid != set(ss.SCENES)


# extremes.py: the crowds hold clips and clipped layers, nan_blends non-separable modes, textures and
# a gradient; every other scene is solid `Over` fills (both fill rules).
EXTREME_SOLID = {n for n in extremes.SCENES if not n.startswith("crowd_") and n != "nan_blends"}


@pytest.mark.parametrize("name", list(extremes.SCENES))
def test_extreme_scenes(cuda_api, oracle_api, paint_solid_restored, name):
    comp, built, sc = extremes.build(cuda_api, name)
    ocomp, _, _ = extremes.build(oracle_api, name)
    want = oracle_frame(oracle_api, ocomp, sc.width, sc.height, crop=sc.crop)
    frames, used = render_both(cuda_api, comp, sc.width, sc.height, host_frame(sc.width, sc.height, crop=sc.crop))
    check(frames, used, want, name in EXTREME_SOLID, name)


W, H = 640, 360


def _cubics(api, seed, opaque=False):
    comp = api.Composition()
    synth.random_cubics(api, comp, 300, W, H, seed, extent=(10.0, 120.0), opaque=opaque)
    return comp


@pytest.mark.parametrize("channels", ORDERS)
def test_channel_orders_crop_and_stride(cuda_api, oracle_api, paint_solid_restored, channels):
    comp, ocomp = _cubics(cuda_api, 5), _cubics(oracle_api, 5)
    crop, stride = Rect((37, 600), (9, 333)), W * 4 + 52
    for crop_, stride_ in ((None, None), (crop, stride)):
        want = oracle_frame(oracle_api, ocomp, W, H, channels, crop_, stride_)
        frames, used = render_both(cuda_api, comp, W, H, host_frame(W, H, channels, crop_, stride_))
        check(frames, used, want, True, f"channels {channels} crop {crop_} stride {stride_}")
    want = oracle_frame(oracle_api, ocomp, W, H, channels)
    frames, used = render_both(cuda_api, comp, W, H, device_frame(W, H, channels))
    check(frames, used, want, True, f"channels {channels} device")


def test_views(cuda_api, paint_solid_restored):
    import torch
    comp = _cubics(cuda_api, 9)
    views = [[1.0, 0.0, 0.0, 1.0, 0.0, 0.0], [0.5, -0.25, 0.25, 0.5, 100.0, 20.0], [1.0, 0.0, 0.0, 1.0, 3.5, -7.25],
             [0.0, -1.0, 1.0, 0.0, 360.0, 0.0]]

    def fn(r, c):
        out = torch.zeros((len(views), H, W, 4), dtype=torch.uint8, device="cuda:0")
        r.render_views_device(c, views, out.data_ptr(), W, H, RGBA, CLEAR)
        torch.cuda.synchronize()
        host = np.zeros(len(views) * H * W * 4, np.uint8)
        r.render_views(c, views, host, W, H, BGRA, CLEAR)
        return np.concatenate([out.cpu().numpy().ravel(), host])
    frames, used = render_both(cuda_api, comp, W, H, fn)
    check(frames, used, None, True, "views")


def test_batches(cuda_api, paint_solid_restored):
    import torch
    comps = [_cubics(cuda_api, s, opaque=(s % 2 == 0)) for s in (11, 12, 13)]

    def fn(r, _):
        out = torch.zeros((len(comps) + 1, H, W, 4), dtype=torch.uint8, device="cuda:0")
        r.render_batch_device(comps + comps[:1], out.data_ptr(), W, H, RGBA, CLEAR)
        torch.cuda.synchronize()
        host = np.zeros(len(comps) * H * W * 4, np.uint8)
        r.render_batch(comps, host, W, H, RGBA, CLEAR)
        return np.concatenate([out.cpu().numpy().ravel(), host])
    frames, used = render_both(cuda_api, None, W, H, fn)
    check(frames, used, None, True, "batch")
    # One composition with a gradient layer sends the whole batch to the general build.
    mixed = _cubics(cuda_api, 14)
    mixed.get_mut_or_insert_default(50).set_props(_gradient_props())
    comps.append(mixed)
    frames, used = render_both(cuda_api, None, W, H, fn)
    check(frames, used, None, False, "batch with a gradient layer")


def test_layer_cache_over_frames(cuda_api, oracle_api, paint_solid_restored):
    """Frames with a layer cache while layers move, disappear and change colour: the lean build
    reads and writes the cache the way the general one does."""
    def step(c, k):
        c.get_mut_or_insert_default(7).set_transform([1.0, 0.0, 0.0, 1.0, 3.0 * k, -2.0 * k])
        c.get_mut_or_insert_default(150).set_props(Props(func=Func.Draw(Style(fill=Fill.Solid(Color(0.1 * k, 0.5, 0.2, 1.0))))))
        if k == 2:
            c.get_mut_or_insert_default(200).disable()

    for v in (1, 0):
        cuda_api.set_option("paint_solid", v)
        comp, ocomp = _cubics(cuda_api, 21, opaque=True), _cubics(oracle_api, 21, opaque=True)
        r = cuda_api.Renderer(0)
        cache = r.create_buffer_layer_cache()
        buf = np.zeros(W * H * 4, np.uint8)
        for k in range(4):
            step(comp, k)
            step(ocomp, k)
            used = painters(lambda: r.render(comp, buf, W, H, RGBA, CLEAR, layer_cache=cache))
            assert used == ({"solid"} if v else {"general"}), (v, k, used)
            assert np.array_equal(buf, oracle_frame(oracle_api, ocomp, W, H)), f"paint_solid {v}: cached frame {k} differs"


def _gradient_props(clipped=False):
    gb = GradientBuilder(Point(0.0, 0.0), Point(float(W), float(H)))
    gb.color(Color(1.0, 0.0, 0.0, 1.0))
    gb.color(Color(0.0, 0.0, 1.0, 0.5))
    return Props(func=Func.Draw(Style(fill=Fill.Gradient(gb.build()), is_clipped=clipped)))


FALLBACKS = {
    "gradient": lambda: _gradient_props(),
    "blend_multiply": lambda: Props(func=Func.Draw(Style(fill=Fill.Solid(Color(0.5, 0.2, 0.9, 0.8)), blend_mode=BlendMode.Multiply))),
    "clip": lambda: Props(func=Func.Clip(3)),
    "clipped": lambda: Props(func=Func.Draw(Style(fill=Fill.Solid(Color(0.5, 0.2, 0.9, 0.8)), is_clipped=True))),
    "even_odd_only": lambda: Props(fill_rule=FillRule.EvenOdd, func=Func.Draw(Style(fill=Fill.Solid(Color(0.5, 0.2, 0.9, 0.8))))),
}


@pytest.mark.parametrize("kind", list(FALLBACKS))
def test_one_other_layer_keeps_the_general_build(cuda_api, oracle_api, paint_solid_restored, kind):
    """A single layer that is not a solid `Over` fill, or a clip, or a clipped layer sends the frame to
    the general build (an even-odd solid `Over` layer does not); the frame stays the oracle's."""
    frames_used = []
    for api in (cuda_api, oracle_api):
        c = _cubics(api, 31)
        c.get_mut_or_insert_default(120).set_props(FALLBACKS[kind]())
        frames_used.append(c)
    comp, ocomp = frames_used
    want = oracle_frame(oracle_api, ocomp, W, H)
    frames, used = render_both(cuda_api, comp, W, H, host_frame(W, H))
    check(frames, used, want, kind == "even_odd_only", kind)
