// Per-pixel arithmetic of the painter: coverage, fills, the 16 blend modes in
// both of the reference's forms, and the sRGB encoder.
//
// Every expression keeps the reference's operation order; `fmaf` appears
// exactly where the Rust source says `mul_add` (files are built with
// --fmad=false). Vector code of the reference (f32x8) is evaluated per lane
// following the portable SIMD shim forma/src/utils/simd/auto.rs.
#pragma once

#include "cuda_common.cuh"

namespace forma {

struct Rgba {
    float r, g, b, a;
};

// cpu/painter/mod.rs:76-94 (doubled_area_to_coverage); PIXEL_DOUBLE_AREA = 512.
__device__ __forceinline__ float coverage_of(int32_t doubled_area, uint32_t fill_rule) {
    if (fill_rule == 0u) return d_clamp(fabsf((float)doubled_area * (1.0f / 512.0f)), 0.0f, 1.0f);
    int32_t v = 512 - abs((doubled_area & 1023) - 512);
    return (float)v * (1.0f / 512.0f);
}

// cpu/painter/mod.rs:98-112
__device__ __forceinline__ float linear_to_srgb(float l) {
    float s = sqrtf(l);
    float s3 = l * s;
    float m = l * 12.92f;
    float n = fmaf(0.20101772f, s3, fmaf(-0.51280147f, l, fmaf(1.344401f, s, -0.030656587f)));
    return l <= 0.0031308f ? m : n;
}

// cpu/painter/mod.rs:135-143 (to_u32x8 + low byte). A NaN channel (e.g. clip_color! dividing by
// x - l = 0 for a colour outside [0, 1]) passes the clamp, and its byte is the low byte of the
// NaN's bits. On the CPUs the reference runs on, arithmetic produces the default NaN (x86
// 0xFFC00000, Arm 0x7FC00000) and propagates its payload, so the byte is 0; the GPU's canonical
// NaN 0x7FFFFFFF would give 255.
__device__ __forceinline__ uint32_t to_byte(float v) {
    float scaled = d_clamp(v * 255.0f, 0.0f, 255.0f);
    float val = scaled + __uint_as_float(0x4B000000u);
    return val != val ? 0u : __float_as_uint(val) & 0xFFu;
}

__device__ __forceinline__ float channel_of(const Rgba& c, uint32_t ch) {  // cpu/painter/styling.rs:46-55
    switch (ch) {
        case 0: return c.r;
        case 1: return c.g;
        case 2: return c.b;
        case 3: return c.a;
        case 4: return 0.0f;
        default: return 1.0f;
    }
}

// to_srgb_bytes(channels.map(|c| color.channel(c))) — the Solid tile path,
// cpu/painter/mod.rs:156-162,691-692. Packed little-endian (byte 0 first).
__device__ __forceinline__ uint32_t solid_to_srgb_bytes(const Rgba& c, const uint32_t ch[4]) {
    uint32_t b0 = to_byte(linear_to_srgb(channel_of(c, ch[0])));
    uint32_t b1 = to_byte(linear_to_srgb(channel_of(c, ch[1])));
    uint32_t b2 = to_byte(linear_to_srgb(channel_of(c, ch[2])));
    uint32_t b3 = to_byte(channel_of(c, ch[3]));
    return b0 | (b1 << 8) | (b2 << 16) | (b3 << 24);
}

// compute_srgb for one pixel, cpu/painter/mod.rs:466-483.
__device__ __forceinline__ uint32_t pixel_to_srgb_bytes(float r, float g, float b, float a, const uint32_t ch[4]) {
    Rgba s{linear_to_srgb(r), linear_to_srgb(g), linear_to_srgb(b), a};
    return to_byte(channel_of(s, ch[0])) | (to_byte(channel_of(s, ch[1])) << 8) | (to_byte(channel_of(s, ch[2])) << 16) |
           (to_byte(channel_of(s, ch[3])) << 24);
}

// The same for the RGBA channel order (no channel selection).
__device__ __forceinline__ uint32_t pixel_to_srgb_bytes_rgba(float r, float g, float b, float a) {
    return to_byte(linear_to_srgb(r)) | (to_byte(linear_to_srgb(g)) << 8) | (to_byte(linear_to_srgb(b)) << 16) |
           (to_byte(a) << 24);
}

// ---------------------------------------------------------------------------
// Scalar blend: BlendMode::blend (cpu/painter/styling.rs:195-339). Used when a
// tile folds to one solid colour (skip_fully_covered_layers.rs:103-113).
// ---------------------------------------------------------------------------
namespace sblend {
__device__ __forceinline__ float ch3(const Rgba& c, int i) { return i == 0 ? c.r : (i == 1 ? c.g : c.b); }
__device__ __forceinline__ float lum(const Rgba& c) { return fmaf(c.r, 0.3f, fmaf(c.g, 0.59f, c.b * 0.11f)); }
__device__ __forceinline__ float cmax(const Rgba& c) { return fmaxf(c.r, fmaxf(c.g, c.b)); }
__device__ __forceinline__ float cmin(const Rgba& c) { return fminf(c.r, fminf(c.g, c.b)); }
__device__ __forceinline__ float multiply(float d, float s) { return d * s; }
__device__ __forceinline__ float screen(float d, float s) { return d + s - (d * s); }
__device__ __forceinline__ float hard_light(float d, float s) {
    return s <= 0.5f ? multiply(d, 2.0f * s) : screen(d, 2.0f * s - 1.0f);
}
__device__ __forceinline__ float clip_color(int i, const Rgba& color) {
    float l = lum(color), n = cmin(color), x = cmax(color);
    float c = ch3(color, i);
    if (n < 0.0f) {
        float k = d_rcp(l - n) * l;
        c = fmaf(k, c - l, l);
    }
    if (x > 1.0f) {
        float l_1 = l - 1.0f;
        float k = d_rcp(x - l);
        c = fmaf(k, fmaf(l, l_1 - c, c), l);
    }
    return c;
}
__device__ __forceinline__ float set_lum(int i, Rgba color, float l) {
    float d = l - lum(color);
    color.r += d;
    color.g += d;
    color.b += d;
    return clip_color(i, color);
}
__device__ __forceinline__ float sat(const Rgba& c) { return cmax(c) - cmin(c); }
__device__ __forceinline__ Rgba set_sat(Rgba color, float s) {
    // Color::sorted, cpu/painter/styling.rs:33-44 -> indices of (min, mid, max)
    bool a = color.r < color.g, b = color.r < color.b, c = color.g < color.b;
    int imin, imid, imax;
    if (a && b && c) { imin = 0; imid = 1; imax = 2; }
    else if (a && b && !c) { imin = 0; imid = 2; imax = 1; }
    else if (a && !b) { imin = 2; imid = 0; imax = 1; }
    else if (!a && b && c) { imin = 1; imid = 0; imax = 2; }
    else if (!a && !c) { imin = 2; imid = 1; imax = 0; }
    else { imin = 1; imid = 2; imax = 0; }
    float v[3] = {color.r, color.g, color.b};
    float vmin = v[imin], vmid = v[imid], vmax = v[imax];
    float nmid, nmax;
    if (vmax > vmin) {
        nmid = fmaf(s, vmid, -s * vmin) / (vmax - vmin);
        nmax = s;
    } else {
        nmid = 0.0f;
        nmax = 0.0f;
    }
    float o[3];
    o[imin] = 0.0f;
    o[imid] = nmid;
    o[imax] = nmax;
    // When two indices coincide in value order the assignment order of the
    // reference is (mid, max) then min; indices are always distinct here.
    color.r = o[0];
    color.g = o[1];
    color.b = o[2];
    return color;
}
__device__ __forceinline__ float soft_d(float d) {
    return d <= 0.25f ? ((16.0f * d - 12.0f) * d + 4.0f) * d : sqrtf(d);
}
__device__ inline float blend_channel(uint32_t mode, int i, const Rgba& dst, const Rgba& src) {
    float d = ch3(dst, i), s = ch3(src, i);
    switch (mode) {
        case 0: return s;
        case 1: return multiply(d, s);
        case 2: return screen(d, s);
        case 3: return hard_light(s, d);
        case 4: return fminf(d, s);
        case 5: return fmaxf(d, s);
        case 6: return d == 0.0f ? 0.0f : (s == 1.0f ? 1.0f : fminf(1.0f, d / (1.0f - s)));
        case 7: return d == 1.0f ? 1.0f : (s == 0.0f ? 0.0f : 1.0f - fminf(1.0f, (1.0f - d) / s));
        case 8: return hard_light(d, s);
        case 9: return s <= 0.5f ? d - (1.0f - 2.0f * s) * d * (1.0f - d) : d + (2.0f * s - 1.0f) * (soft_d(d) - d);
        case 10: return fabsf(d - s);
        case 11: return d + s - 2.0f * d * s;
        case 12: return set_lum(i, set_sat(src, sat(dst)), lum(dst));   // Hue
        case 13: return set_lum(i, set_sat(dst, sat(src)), lum(dst));   // Saturation
        case 14: return set_lum(i, src, lum(dst));                      // Color
        default: return set_lum(i, dst, lum(src));                      // Luminosity
    }
}
__device__ inline Rgba blend(uint32_t mode, const Rgba& dst, const Rgba& src) {
    float inv_dst_a = 1.0f - dst.a;
    float inv_dst_a_src_a = inv_dst_a * src.a;
    float inv_src_a = 1.0f - src.a;
    float dst_a_src_a = dst.a * src.a;
    float cr = fmaf(src.r, inv_dst_a_src_a, blend_channel(mode, 0, dst, src) * dst_a_src_a);
    float cg = fmaf(src.g, inv_dst_a_src_a, blend_channel(mode, 1, dst, src) * dst_a_src_a);
    float cb = fmaf(src.b, inv_dst_a_src_a, blend_channel(mode, 2, dst, src) * dst_a_src_a);
    Rgba o;
    o.r = fmaf(dst.r, inv_src_a, cr);
    o.g = fmaf(dst.g, inv_src_a, cg);
    o.b = fmaf(dst.b, inv_src_a, cb);
    o.a = fmaf(dst.a, inv_src_a, src.a);
    return o;
}
}  // namespace sblend

// ---------------------------------------------------------------------------
// Per-lane form of the vector macro blend_function! (styling.rs:342-594): this
// is what per-pixel painting uses (op order differs from the scalar form).
// ---------------------------------------------------------------------------
namespace vblend {
__device__ __forceinline__ float lum(float r, float g, float b) { return fmaf(r, 0.3f, fmaf(g, 0.59f, b * 0.11f)); }
__device__ __forceinline__ float sat(float r, float g, float b) {
    return fmaxf(r, fmaxf(g, b)) - fminf(r, fminf(g, b));
}
__device__ __forceinline__ void clip_color(float r, float g, float b, float o[3]) {
    float l = lum(r, g, b);
    float n = fminf(r, fminf(g, b));
    float x = fmaxf(r, fmaxf(g, b));
    float l_1 = l - 1.0f;
    float x_l_recip = d_rcp(x - l);
    float l_n_recip_l = d_rcp(l - n) * l;
    float in[3] = {r, g, b};
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        float c = in[i];
        float hi = fmaf(x_l_recip, fmaf(l, l_1 - c, c), l);
        float lo = n < 0.0f ? fmaf(l_n_recip_l, c - l, l) : c;
        o[i] = 1.0f < x ? hi : lo;
    }
}
__device__ __forceinline__ void set_lum(float r, float g, float b, float l, float o[3]) {
    float d = l - lum(r, g, b);
    r += d;
    g += d;
    b += d;
    clip_color(r, g, b, o);
}
__device__ __forceinline__ void set_sat(float sat_dst, float sr, float sg, float sb, float o[3]) {
    float src_min = fminf(sr, fminf(sg, sb));
    float src_max = fmaxf(sr, fmaxf(sg, sb));
    float src_mid = sr + sg + sb - src_min - src_max;
    bool lt = src_min < src_max;
    float sat_mid = lt ? (fmaf(sat_dst, -src_min, sat_dst * src_mid) / (src_max - src_min)) : 0.0f;
    float sat_max = lt ? sat_dst : 0.0f;
    float in[3] = {sr, sg, sb};
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        float inner = in[i] == src_min ? 0.0f : sat_mid;
        o[i] = in[i] == src_max ? sat_max : inner;
    }
}
__device__ __forceinline__ float hard(float d, float s, float sel) {
    return sel <= 0.5f ? d * s * 2.0f : 2.0f * (d + s - fmaf(d, s, 0.5f));
}
__device__ __forceinline__ void blend(uint32_t mode, float dr, float dg, float db, float sr, float sg, float sb,
                                      float o[3]) {
    float d[3] = {dr, dg, db}, s[3] = {sr, sg, sb};
    switch (mode) {
        case 0:
#pragma unroll
            for (int i = 0; i < 3; ++i) o[i] = s[i];
            return;
        case 1:
#pragma unroll
            for (int i = 0; i < 3; ++i) o[i] = d[i] * s[i];
            return;
        case 2:
#pragma unroll
            for (int i = 0; i < 3; ++i) o[i] = fmaf(d[i], -s[i], d[i]) + s[i];
            return;
        case 3:
#pragma unroll
            for (int i = 0; i < 3; ++i) o[i] = hard(d[i], s[i], d[i]);
            return;
        case 4:
#pragma unroll
            for (int i = 0; i < 3; ++i) o[i] = fminf(d[i], s[i]);
            return;
        case 5:
#pragma unroll
            for (int i = 0; i < 3; ++i) o[i] = fmaxf(d[i], s[i]);
            return;
        case 6:
#pragma unroll
            for (int i = 0; i < 3; ++i) o[i] = s[i] == 1.0f ? 1.0f : fminf(1.0f, d[i] / (1.0f - s[i]));
            return;
        case 7:
#pragma unroll
            for (int i = 0; i < 3; ++i) o[i] = s[i] == 0.0f ? 0.0f : 1.0f - fminf(1.0f, (1.0f - d[i]) / s[i]);
            return;
        case 8:
#pragma unroll
            for (int i = 0; i < 3; ++i) o[i] = hard(d[i], s[i], s[i]);
            return;
        case 9:
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                float dd = d[i] <= 0.25f ? fmaf(fmaf(16.0f, d[i], -12.0f), d[i], 4.0f) * d[i] : sqrtf(d[i]);
                float k = fmaf(2.0f, s[i], -1.0f);
                o[i] = s[i] <= 0.5f ? fmaf(d[i] * (1.0f - d[i]), k, d[i]) : fmaf(dd - d[i], k, d[i]);
            }
            return;
        case 10:
#pragma unroll
            for (int i = 0; i < 3; ++i) o[i] = fabsf(d[i] - s[i]);
            return;
        case 11:
#pragma unroll
            for (int i = 0; i < 3; ++i) o[i] = fmaf(-2.0f * d[i], s[i], d[i]) + s[i];
            return;
        case 12: {
            float t[3];
            set_sat(sat(dr, dg, db), sr, sg, sb, t);
            set_lum(t[0], t[1], t[2], lum(dr, dg, db), o);
            return;
        }
        case 13: {
            float t[3];
            set_sat(sat(sr, sg, sb), dr, dg, db, t);
            set_lum(t[0], t[1], t[2], lum(dr, dg, db), o);
            return;
        }
        case 14:
            set_lum(sr, sg, sb, lum(dr, dg, db), o);
            return;
        default:
            set_lum(dr, dg, db, lum(sr, sg, sb), o);
            return;
    }
}
}  // namespace vblend

// Gradient::color_at for one lane (cpu/painter/styling.rs:58-144). `x` is the
// pixel column, `y_base` the y of lane 0 of the reference's f32x8 (a multiple
// of 8), `lane` in 0..8.
__device__ inline void gradient_at(const StyleRec& st, const StopRec* __restrict__ stops, float x, float y_base,
                                   int lane, float out[4]) {
    float dx = st.end[0] - st.start[0];
    float dy = st.end[1] - st.start[1];
    float dot = dx * dx + dy * dy;
    float dot_recip = d_rcp(dot);
    float t;
    if (st.gradient_type == 0u) {
        float tx = (x - st.start[0]) * dx * dot_recip;
        float ty = y_base - st.start[1];
        t = fmaf(((float)lane + ty) * dy, dot_recip, tx);
    } else {
        float px = x - st.start[0];
        float px2 = px * px;
        float py = (float)lane + (y_base - st.start[1]);
        t = sqrtf(fmaf(py, py, px2) * dot_recip);
    }
    const StopRec* sp = stops + st.stop_first;
    uint32_t bits[4] = {0u, 0u, 0u, 0u};
    StopRec first = sp[0];
    bool acc = t <= first.stop;
    if (acc) {
#pragma unroll
        for (int k = 0; k < 4; ++k) bits[k] |= __float_as_uint(first.color[k]);
    }
    float start_stop = 0.0f;
    float sc[4] = {first.color[0], first.color[1], first.color[2], first.color[3]};
    for (uint32_t i = 1; i < st.stop_count; ++i) {
        StopRec cur = sp[i];
        bool mask = acc != (t < cur.stop);
        if (mask) {
            float d = cur.stop - start_stop;
            float local_t = (t - start_stop) * d_rcp(d);
#pragma unroll
            for (int k = 0; k < 4; ++k)
                bits[k] |= __float_as_uint(fmaf(local_t, cur.color[k], fmaf(-local_t, sc[k], sc[k])));
            acc = true;
        }
        start_stop = cur.stop;
#pragma unroll
        for (int k = 0; k < 4; ++k) sc[k] = cur.color[k];
    }
    if (!acc) {
        StopRec last = sp[st.stop_count - 1];
#pragma unroll
        for (int k = 0; k < 4; ++k) bits[k] |= __float_as_uint(last.color[k]);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) out[k] = __uint_as_float(bits[k]);
}

// The same function for gradients of at most four stops whose stops (and the
// per-gradient terms dx, dy, 1 / dot) were loaded once per layer: the pixel loop
// then runs out of registers. Identical operations in identical order.
struct GradientSetup {
    float dx, dy, dot_recip;
    StopRec c[4];
    uint32_t count;
};
__device__ __forceinline__ GradientSetup gradient_setup(const StyleRec& st, const StopRec* __restrict__ stops) {
    GradientSetup g;
    g.dx = st.end[0] - st.start[0];
    g.dy = st.end[1] - st.start[1];
    float dot = g.dx * g.dx + g.dy * g.dy;
    g.dot_recip = d_rcp(dot);
    g.count = st.stop_count;
    const StopRec* sp = stops + st.stop_first;
#pragma unroll
    for (uint32_t i = 0; i < 4u; ++i) g.c[i] = sp[i < g.count ? i : g.count - 1u];
    return g;
}
__device__ __forceinline__ void gradient_at_small(const StyleRec& st, const GradientSetup& g, float x, float y_base, int lane,
                                                  float out[4]) {
    float t;
    if (st.gradient_type == 0u) {
        float tx = (x - st.start[0]) * g.dx * g.dot_recip;
        float ty = y_base - st.start[1];
        t = fmaf(((float)lane + ty) * g.dy, g.dot_recip, tx);
    } else {
        float px = x - st.start[0];
        float px2 = px * px;
        float py = (float)lane + (y_base - st.start[1]);
        t = sqrtf(fmaf(py, py, px2) * g.dot_recip);
    }
    uint32_t bits[4] = {0u, 0u, 0u, 0u};
    bool acc = t <= g.c[0].stop;
    if (acc) {
#pragma unroll
        for (int k = 0; k < 4; ++k) bits[k] |= __float_as_uint(g.c[0].color[k]);
    }
    float start_stop = 0.0f;
#pragma unroll
    for (uint32_t i = 1; i < 4u; ++i) {
        if (i < g.count) {
            bool mask = acc != (t < g.c[i].stop);
            if (mask) {
                float d = g.c[i].stop - start_stop;
                float local_t = (t - start_stop) * d_rcp(d);
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    bits[k] |= __float_as_uint(fmaf(local_t, g.c[i].color[k], fmaf(-local_t, g.c[i - 1].color[k], g.c[i - 1].color[k])));
                acc = true;
            }
            start_stop = g.c[i].stop;
        }
    }
    if (!acc) {  // g.c[3] is the last stop (padding repeats it)
#pragma unroll
        for (int k = 0; k < 4; ++k) bits[k] |= __float_as_uint(g.c[3].color[k]);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) out[k] = __uint_as_float(bits[k]);
}

// gradient_at_small with the style's start point and type passed in registers (the painter's
// pixel-pair loop); identical operations in identical order.
__device__ __forceinline__ void gradient_at_small_xy(const GradientSetup& g, uint32_t gradient_type, float sx, float sy, float x,
                                                     float y_base, int lane, float out[4]) {
    float t;
    if (gradient_type == 0u) {
        float tx = (x - sx) * g.dx * g.dot_recip;
        float ty = y_base - sy;
        t = fmaf(((float)lane + ty) * g.dy, g.dot_recip, tx);
    } else {
        float px = x - sx;
        float px2 = px * px;
        float py = (float)lane + (y_base - sy);
        t = sqrtf(fmaf(py, py, px2) * g.dot_recip);
    }
    uint32_t bits[4] = {0u, 0u, 0u, 0u};
    bool acc = t <= g.c[0].stop;
    if (acc) {
#pragma unroll
        for (int k = 0; k < 4; ++k) bits[k] |= __float_as_uint(g.c[0].color[k]);
    }
    float start_stop = 0.0f;
#pragma unroll
    for (uint32_t i = 1; i < 4u; ++i) {
        if (i < g.count) {
            bool mask = acc != (t < g.c[i].stop);
            if (mask) {
                float d = g.c[i].stop - start_stop;
                float local_t = (t - start_stop) * d_rcp(d);
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    bits[k] |= __float_as_uint(fmaf(local_t, g.c[i].color[k], fmaf(-local_t, g.c[i - 1].color[k], g.c[i - 1].color[k])));
                acc = true;
            }
            start_stop = g.c[i].stop;
        }
    }
    if (!acc) {  // g.c[3] is the last stop (padding repeats it)
#pragma unroll
        for (int k = 0; k < 4; ++k) bits[k] |= __float_as_uint(g.c[3].color[k]);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) out[k] = __uint_as_float(bits[k]);
}

// Texture::color_at for one lane (cpu/painter/styling.rs:146-193).
__device__ inline void texture_at(const StyleRec& st, const uint16_t* __restrict__ texels, float x, float y_base,
                                  int lane, float out[4]) {
    float y = y_base + (float)lane;
    float tx = fmaf(x, st.tex_xf[0], fmaf(st.tex_xf[2], y, st.tex_xf[4]));
    float ty = fmaf(x, st.tex_xf[1], fmaf(st.tex_xf[3], y, st.tex_xf[5]));
    uint32_t ix = d_sat_u32(fminf(tx, st.tex_max_x));
    uint32_t iy = d_sat_u32(fminf(ty, st.tex_max_y));
    uint32_t off = iy * st.tex_width + ix;
    const uint16_t* p = texels + 4ull * ((uint64_t)st.tex_first + off);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        uint16_t h = p[k];  // styling.rs:231-238 f16::to_f32
        out[k] = h != 0 ? __uint_as_float(0x38000000u + ((uint32_t)h << 13)) : 0.0f;
    }
}

}  // namespace forma
