// Stage 4b: the painter — one warp per 16x16 tile. Replaces
// LayerWorkbench::drive_tile_painting + the optimiser passes
// (cpu/painter/layer_workbench/mod.rs:280-342, passes/*.rs),
// Painter::paint_layer / blend_at / clip_at / compute_srgb
// (cpu/painter/mod.rs:290-483) and LinearLayout::write
// (cpu/buffer/layout/mod.rs:265-282).
//
// Lane l owns eight horizontally consecutive pixels: row r = l / 2, columns 8 (l % 2) .. +8.
//   * the winding cover of a pixel is the carry-in of its row plus the covers of the
//     segments left of it in the same row: a running sum inside the lane and one shuffle
//     for the right half (the reference sweeps its columns left to right,
//     cpu/painter/mod.rs:388-404);
//   * the lane's eight cells are two 16-byte words of shared memory and its eight output
//     pixels one 32-byte run of the frame buffer;
//   * an entry without segments has one coverage value per lane.
// The reference's f32x8 is eight rows of one column; its "skip when all eight coverages
// are zero" (mod.rs:317-319) is kept on every path: from eight ballots for the pair and
// generic paths, and from three shuffles of a per-lane 8-bit mask for a solid `Over` layer.
// Blending at zero coverage is not the identity there either: a non-finite colour or alpha
// makes the pixel NaN, and a -0 plane becomes +0.
//
// Per (tile, layer) entry the segments are scatter-added into packed cells — area in the
// high and cover in the low 16 bits of one word, one shared-memory atomic per segment —
// one entry ahead of the blend: while entry k is blended from one cell buffer, entry k + 1
// is accumulated into the other and the segments of entry k + 2 are in flight.
//
// Blend arithmetic is written on pixel pairs (f2). sm_90 has no packed fp32 instructions,
// so each half is one scalar IEEE operation, the one the reference performs; additions and
// subtractions are written as fma(x, +-1, y), which is the same single rounding, so that no
// product is ever contracted into a sum.
//
// Warps are persistent and take tiles by ticket. Tiles with many entries come first
// (tile_index_kernel sorts them into four classes by entry count): a tile is painted by
// one warp from its first to its last layer, so the heaviest tile bounds the kernel's
// tail unless it starts early (longest-processing-time order).
#include <cuda_fp16.h>

#include <map>
#include <mutex>

#include "paint_common.cuh"
#include "paint_math.cuh"
#include "srgb_decode.h"

namespace forma {

struct PaintInputs {
    const uint64_t* segs;
    const EntryRec* recs;        // sorted entries (kernels_tables.cu: merge_entries_kernel)
    const uint2* tile_range;     // per tile: [begin, end) of its entries
    const uint32_t* heavy;       // kHeavyClasses lists of heavy tiles (linear ids), n_tiles_total each
    const uint32_t* heavy_count; // their lengths
    uint32_t n_tiles_total;
    uint8_t* eflags;             // per sorted entry: optimizer flags, initialised with EntryRec::flags0
    uint8_t* framebuffer;
    uint32_t* tile_counter;
};

__device__ __forceinline__ uint32_t meta_fill_rule(uint32_t m) { return m & 1u; }
__device__ __forceinline__ uint32_t meta_func(uint32_t m) { return (m >> 1) & 1u; }
__device__ __forceinline__ bool meta_is_clipped(uint32_t m) { return (m >> 2) & 1u; }
__device__ __forceinline__ uint32_t meta_fill_type(uint32_t m) { return (m >> 3) & 3u; }
__device__ __forceinline__ uint32_t meta_blend(uint32_t m) { return (m >> 5) & 15u; }

// ---------------------------------------------------------------------------
// Packed fp32 pairs
// ---------------------------------------------------------------------------
struct f2 {
    float x, y;
};
__device__ __forceinline__ f2 f2_splat(float v) { return f2{v, v}; }
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) { return f2{__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)}; }
__device__ __forceinline__ f2 mul2(f2 a, f2 b) { return f2{__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)}; }
// a + b and a - b as one fused operation each (exact product, one rounding: the IEEE sum).
__device__ __forceinline__ f2 add2(f2 a, f2 b) { return fma2(a, f2_splat(1.0f), b); }
__device__ __forceinline__ f2 sub2(f2 a, f2 b) { return fma2(b, f2_splat(-1.0f), a); }
__device__ __forceinline__ f2 neg2(f2 a) { return f2{-a.x, -a.y}; }
__device__ __forceinline__ f2 min2(f2 a, f2 b) { return f2{fminf(a.x, b.x), fminf(a.y, b.y)}; }
__device__ __forceinline__ f2 max2(f2 a, f2 b) { return f2{fmaxf(a.x, b.x), fmaxf(a.y, b.y)}; }
// The blended pair where bit 0 (x) / bit 1 (y) of `act` is set, the old pair elsewhere.
__device__ __forceinline__ f2 keep2(uint32_t act, f2 blended, f2 old) { return f2{act & 1u ? blended.x : old.x, act & 2u ? blended.y : old.y}; }

// The 12 separable blend modes of the vector macro blend_function! (styling.rs:438-592) on a
// pixel pair, same operation order as vblend::blend (paint_math.cuh). `mode` is uniform.
__device__ __forceinline__ f2 hard2(f2 d, f2 s, f2 sel) {
    // sel <= 0.5 ? d * s * 2 : 2 * (d + s - fma(d, s, 0.5))
    const f2 lo = mul2(mul2(d, s), f2_splat(2.0f));
    const f2 hi = mul2(f2_splat(2.0f), sub2(add2(d, s), fma2(d, s, f2_splat(0.5f))));
    return f2{sel.x <= 0.5f ? lo.x : hi.x, sel.y <= 0.5f ? lo.y : hi.y};
}
__device__ __forceinline__ float soft1(float d, float s) {
    float dd = d <= 0.25f ? fmaf(fmaf(16.0f, d, -12.0f), d, 4.0f) * d : sqrtf(d);
    float k = fmaf(2.0f, s, -1.0f);
    return s <= 0.5f ? fmaf(d * (1.0f - d), k, d) : fmaf(dd - d, k, d);
}
__device__ __forceinline__ f2 blend_sep2(uint32_t mode, f2 d, f2 s) {
    switch (mode) {
        case 0: return s;
        case 1: return mul2(d, s);
        case 2: return add2(fma2(d, neg2(s), d), s);
        case 3: return hard2(d, s, d);
        case 4: return min2(d, s);
        case 5: return max2(d, s);
        case 6: return f2{s.x == 1.0f ? 1.0f : fminf(1.0f, d.x / (1.0f - s.x)), s.y == 1.0f ? 1.0f : fminf(1.0f, d.y / (1.0f - s.y))};
        case 7:
            return f2{s.x == 0.0f ? 0.0f : 1.0f - fminf(1.0f, (1.0f - d.x) / s.x),
                      s.y == 0.0f ? 0.0f : 1.0f - fminf(1.0f, (1.0f - d.y) / s.y)};
        case 8: return hard2(d, s, s);
        case 9: return f2{soft1(d.x, s.x), soft1(d.y, s.y)};
        case 10: {
            const f2 t = sub2(d, s);
            return f2{fabsf(t.x), fabsf(t.y)};
        }
        default: return add2(fma2(mul2(f2_splat(-2.0f), d), s, d), s);  // 11 Exclusion
    }
}

// blend_at's composition (cpu/painter/mod.rs:434-446) for a pixel pair and one channel:
//   current = fma(src, inv_dst_a * src_a, blended * (dst_a * src_a)); dst = fma(dst, 1 - src_a, current)
__device__ __forceinline__ f2 compose2(f2 dst, f2 src, f2 blended, f2 inv_dst_a_src_a, f2 dst_a_src_a, f2 inv_src_a) {
    const f2 cur = fma2(src, inv_dst_a_src_a, mul2(blended, dst_a_src_a));
    return fma2(dst, inv_src_a, cur);
}

// ---------------------------------------------------------------------------
// Out-of-line helpers for the rare paths (kept out of the kernel's instruction stream)
// ---------------------------------------------------------------------------
// One pixel of blend_at for any fill / blend mode.
__device__ __noinline__ float4 blend_pixel_generic(const StyleRec* __restrict__ st, const StopRec* __restrict__ stops,
                                                   const uint16_t* __restrict__ texels, float fx, float fy_base, int l,
                                                   float coverage, float clip, float4 dst) {
    float fill[4];
    if (st->fill_type == 0u) {
        fill[0] = st->color[0]; fill[1] = st->color[1]; fill[2] = st->color[2]; fill[3] = st->color[3];
    } else if (st->fill_type == 1u) {
        gradient_at(*st, stops, fx, fy_base, l, fill);
    } else {
        texture_at(*st, texels, fx, fy_base, l, fill);
    }
    float sa = fill[3] * coverage;
    if (clip >= 0.0f) sa *= clip;  // clip < 0: no mask applies
    float bl[3];
    vblend::blend(st->blend_mode, dst.x, dst.y, dst.z, fill[0], fill[1], fill[2], bl);
    float inv_dst_a = 1.0f - dst.w;
    float inv_dst_a_src_a = inv_dst_a * sa;
    float inv_src_a = 1.0f - sa;
    float dst_a_src_a = dst.w * sa;
    float cr = fmaf(fill[0], inv_dst_a_src_a, bl[0] * dst_a_src_a);
    float cg = fmaf(fill[1], inv_dst_a_src_a, bl[1] * dst_a_src_a);
    float cb = fmaf(fill[2], inv_dst_a_src_a, bl[2] * dst_a_src_a);
    return make_float4(fmaf(dst.x, inv_src_a, cr), fmaf(dst.y, inv_src_a, cg), fmaf(dst.z, inv_src_a, cb),
                       fmaf(dst.w, inv_src_a, sa));
}

__device__ __noinline__ uint32_t srgb_bytes_any_order(float r, float g, float b, float a, const uint32_t* ch) {
    return pixel_to_srgb_bytes(r, g, b, a, ch);
}

// The scalar blend of the solid-tile fold (all 16 modes) stays out of line too.
__device__ __noinline__ Rgba blend_solid(uint32_t mode, Rgba dst, Rgba src) { return sblend::blend(mode, dst, src); }

// sRGB encode of a pixel pair (compute_srgb, mod.rs:466-483), RGBA order.
__device__ __forceinline__ f2 srgb2(f2 l) {
    const f2 s = f2{sqrtf(l.x), sqrtf(l.y)};
    const f2 s3 = mul2(l, s);
    const f2 m = mul2(l, f2_splat(12.92f));
    const f2 n = fma2(f2_splat(0.20101772f), s3,
                      fma2(f2_splat(-0.51280147f), l, fma2(f2_splat(1.344401f), s, f2_splat(-0.030656587f))));
    return f2{l.x <= 0.0031308f ? m.x : n.x, l.y <= 0.0031308f ? m.y : n.y};
}
__device__ __forceinline__ void to_byte2(f2 v, uint32_t& b0, uint32_t& b1) {
    f2 sc = mul2(v, f2_splat(255.0f));
    sc.x = d_clamp(sc.x, 0.0f, 255.0f);
    sc.y = d_clamp(sc.y, 0.0f, 255.0f);
    const f2 val = add2(sc, f2_splat(__uint_as_float(0x4B000000u)));
    b0 = val.x != val.x ? 0u : __float_as_uint(val.x) & 0xFFu;  // NaN: see to_byte (paint_math.cuh)
    b1 = val.y != val.y ? 0u : __float_as_uint(val.y) & 0xFFu;
}

__device__ __forceinline__ void store_tile_solid(const PaintScene& S, uint8_t* fb, uint32_t tx, uint32_t ty, uint32_t lane,
                                                 uint32_t rgba, bool vec_ok) {
    const uint32_t py = ty * 16u + (lane >> 1);
    const uint32_t px0 = tx * 16u + (lane & 1u) * 8u;
    if (py >= S.height || px0 >= S.width) return;
    uint8_t* row = fb + (size_t)py * S.stride + (size_t)px0 * 4u;
    if (vec_ok && px0 + 8u <= S.width) {
        const uint4 v = make_uint4(rgba, rgba, rgba, rgba);
        reinterpret_cast<uint4*>(row)[0] = v;
        reinterpret_cast<uint4*>(row)[1] = v;
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (px0 + (uint32_t)j < S.width) reinterpret_cast<uint32_t*>(row)[j] = rgba;
    }
}

// Gradient::color_at (cpu/painter/styling.rs:58-144) for the pixel pair (x, x + 1) of one row,
// from the per-style record in shared memory (read as eight 16-byte words). Same operations
// in the same order as gradient_at (paint_math.cuh); d.recip() of every stop interval comes
// precomputed.
__device__ __forceinline__ void gradient_pair(const GradRec* gp, float x, float y_base, int lane_in_f32x8, f2& r, f2& gg, f2& b, f2& a) {
    const float4* gv = reinterpret_cast<const float4*>(gp);
    const float4 geo = gv[0];                                      // sx, sy, dx, dy
    const float4 hdr = gv[1];                                      // dot_recip, type, count, -
    const uint32_t type = __float_as_uint(hdr.y), count = __float_as_uint(hdr.z);
    const float4 st4 = gv[6], rc4 = gv[7];
    const float stop[4] = {st4.x, st4.y, st4.z, st4.w}, rcp_d[3] = {rc4.x, rc4.y, rc4.z};
    f2 t;
    const f2 xs = f2{x, x + 1.0f};
    if (type == 0u) {
        // tx = (x - sx) * dx * dot_recip; t = fma((lane + (y_base - sy)) * dy, dot_recip, tx)
        const f2 tx = mul2(mul2(sub2(xs, f2_splat(geo.x)), f2_splat(geo.z)), f2_splat(hdr.x));
        const float ty = y_base - geo.y;
        t = fma2(f2_splat(((float)lane_in_f32x8 + ty) * geo.w), f2_splat(hdr.x), tx);
    } else {
        const f2 px = sub2(xs, f2_splat(geo.x));
        const f2 px2 = mul2(px, px);
        const float py = (float)lane_in_f32x8 + (y_base - geo.y);
        const f2 q = mul2(fma2(f2_splat(py), f2_splat(py), px2), f2_splat(hdr.x));
        t = f2{sqrtf(q.x), sqrtf(q.y)};
    }
    float4 c_prev = gv[2];
    const float cp0[4] = {c_prev.x, c_prev.y, c_prev.z, c_prev.w};
    uint32_t bx[4], by[4];
    bool accx = t.x <= stop[0], accy = t.y <= stop[0];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        bx[k] = accx ? __float_as_uint(cp0[k]) : 0u;
        by[k] = accy ? __float_as_uint(cp0[k]) : 0u;
    }
    float start = 0.0f;
#pragma unroll
    for (uint32_t i = 1; i < 4u; ++i) {
        if (i < count) {
            const float4 c_cur = gv[2 + i];
            const bool mx = accx != (t.x < stop[i]), my = accy != (t.y < stop[i]);
            if (mx || my) {
                const f2 local_t = mul2(sub2(t, f2_splat(start)), f2_splat(rcp_d[i - 1]));
                const f2 neg_t = neg2(local_t);
                const float c0[4] = {c_prev.x, c_prev.y, c_prev.z, c_prev.w}, c1[4] = {c_cur.x, c_cur.y, c_cur.z, c_cur.w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const f2 s0 = f2_splat(c0[k]);
                    const f2 v = fma2(local_t, f2_splat(c1[k]), fma2(neg_t, s0, s0));
                    if (mx) bx[k] |= __float_as_uint(v.x);
                    if (my) by[k] |= __float_as_uint(v.y);
                }
                accx = accx || mx;
                accy = accy || my;
            }
            start = stop[i];
            c_prev = c_cur;
        }
    }
    {
        const float4 c_last = gv[5];  // color[3] is the last stop (padding repeats it)
        const float cl[4] = {c_last.x, c_last.y, c_last.z, c_last.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (!accx) bx[k] |= __float_as_uint(cl[k]);
            if (!accy) by[k] |= __float_as_uint(cl[k]);
        }
    }
    r = f2{__uint_as_float(bx[0]), __uint_as_float(by[0])};
    gg = f2{__uint_as_float(bx[1]), __uint_as_float(by[1])};
    b = f2{__uint_as_float(bx[2]), __uint_as_float(by[2])};
    a = f2{__uint_as_float(bx[3]), __uint_as_float(by[3])};
}

// blend_at (cpu/painter/mod.rs:406-447) for one pixel pair of a layer with a separable blend mode
// and a solid or small-gradient fill. One out-of-line copy for the whole kernel: the twelve modes
// and the gradient, inlined per pair, do not fit the instruction cache. Arguments and result
// travel in registers.
//   ctl: blend mode | apply_clip << 8 | gradient fill << 9 | blend pixel x << 16 | blend pixel y << 17
struct PairPlanes {
    f2 r, g, b, a;
};
__device__ __noinline__ PairPlanes blend_pair_separable(PairPlanes d, f2 cov, f2 clip, uint32_t ctl, float x, float y_base,
                                                       int lane_in_f32x8, const GradRec* grad, float4 solid) {
    f2 fr = f2_splat(solid.x), fg = f2_splat(solid.y), fb = f2_splat(solid.z), fa = f2_splat(solid.w);
    if (ctl & 0x200u) gradient_pair(grad, x, y_base, lane_in_f32x8, fr, fg, fb, fa);
    f2 sa = mul2(fa, cov);
    if (ctl & 0x100u) sa = mul2(sa, clip);
    const uint32_t mode = ctl & 15u;
    const f2 br = blend_sep2(mode, d.r, fr), bg = blend_sep2(mode, d.g, fg), bb = blend_sep2(mode, d.b, fb);
    const f2 inv_dst_a = sub2(f2_splat(1.0f), d.a);
    const f2 inv_dst_a_src_a = mul2(inv_dst_a, sa);
    const f2 inv_src_a = sub2(f2_splat(1.0f), sa);
    const f2 dst_a_src_a = mul2(d.a, sa);
    const f2 nr = compose2(d.r, fr, br, inv_dst_a_src_a, dst_a_src_a, inv_src_a);
    const f2 ng = compose2(d.g, fg, bg, inv_dst_a_src_a, dst_a_src_a, inv_src_a);
    const f2 nb = compose2(d.b, fb, bb, inv_dst_a_src_a, dst_a_src_a, inv_src_a);
    const f2 na = fma2(d.a, inv_src_a, sa);
    if (ctl & 0x10000u) {
        d.r.x = nr.x; d.g.x = ng.x; d.b.x = nb.x; d.a.x = na.x;
    }
    if (ctl & 0x20000u) {
        d.r.y = nr.y; d.g.y = ng.y; d.b.y = nb.y; d.a.y = na.y;
    }
    return d;
}

constexpr int kPaintWarpsPerBlock = 2;

struct WarpSmem {
    uint32_t cells[2][256];  // packed (area << 16) + cover, double-buffered by entry parity
    float clip[256];         // clip mask, same layout
    EntryRec hdr[32];        // the 32 entry records of the current group (pad = current optimizer flags)
    GradRec grad;            // gradient of the entry being blended
};

template <int kMinBlocks>
__global__ void __launch_bounds__(kPaintWarpsPerBlock * 32, kMinBlocks) paint_kernel(PaintScene S, PaintInputs in, uint32_t n_tiles) {
    chain_begin();
#define FORMA_PAINT_FRAME_TY(ty) (ty)
#include "paint_kernel_body.cuh"
#undef FORMA_PAINT_FRAME_TY
}
// S is a stack of views of `view_rows` tile rows each (see ViewArgs): gradients and textures are
// sampled at the tile row inside its view.
template <int kMinBlocks>
__global__ void __launch_bounds__(kPaintWarpsPerBlock * 32, kMinBlocks)
    paint_views_kernel(PaintScene S, PaintInputs in, uint32_t n_tiles, uint32_t view_rows) {
    chain_begin();
#define FORMA_PAINT_FRAME_TY(ty) ((ty) % view_rows)
#include "paint_kernel_body.cuh"
#undef FORMA_PAINT_FRAME_TY
}
// paint_kernel / paint_views_kernel for a frame whose layers are all solid `Over` fills without clips
// (Composition::solid_over_only): the same body without the code of other styles and clips. Built
// for 8 CTAs / SM it needs 96 registers and no spills, so 10 CTAs fit an SM; the bounds 10 and 12
// (95 registers; 80 with 74 B of spills) were no faster on paris4k and slower on cubics100k.
#define FORMA_PAINT_SOLID_OVER
template <int kMinBlocks>
__global__ void __launch_bounds__(kPaintWarpsPerBlock * 32, kMinBlocks) paint_solid_kernel(PaintScene S, PaintInputs in, uint32_t n_tiles) {
    chain_begin();
#define FORMA_PAINT_FRAME_TY(ty) (ty)
#include "paint_kernel_body.cuh"
#undef FORMA_PAINT_FRAME_TY
}
template <int kMinBlocks>
__global__ void __launch_bounds__(kPaintWarpsPerBlock * 32, kMinBlocks)
    paint_views_solid_kernel(PaintScene S, PaintInputs in, uint32_t n_tiles, uint32_t view_rows) {
    chain_begin();
#define FORMA_PAINT_FRAME_TY(ty) ((ty) % view_rows)
#include "paint_kernel_body.cuh"
#undef FORMA_PAINT_FRAME_TY
}
#undef FORMA_PAINT_SOLID_OVER

// ---------------------------------------------------------------------------
// Linear float frames: the painter's planes as they are, RGBA16F (8-byte pixels, each value
// __float2half_rn) or RGBA32F (16-byte pixels), in channel order
// ---------------------------------------------------------------------------
// The four values of a pixel in channel order: what compute_srgb encodes, not encoded.
__device__ __forceinline__ float4 linear_pixel(float r, float g, float b, float a, const uint32_t ch[4]) {
    const Rgba c{r, g, b, a};
    return make_float4(channel_of(c, ch[0]), channel_of(c, ch[1]), channel_of(c, ch[2]), channel_of(c, ch[3]));
}
__device__ __forceinline__ uint32_t half2_bits(float lo, float hi) {
    return (uint32_t)__half_as_ushort(__float2half_rn(lo)) | ((uint32_t)__half_as_ushort(__float2half_rn(hi)) << 16);
}
// Stores the pixel pair (p0, p1) whose first pixel is at `dst`; `both`: p1 lies inside the frame.
// vec: the frame and its stride are 16-byte aligned (a pair is 16 or 32 bytes at a 16-byte
// offset); otherwise 4-byte stores, which the 4-byte alignment of float frames allows.
__device__ __forceinline__ void store_linear_pair(uint8_t* dst, float4 p0, float4 p1, bool both, bool vec, uint32_t bpp) {
    if (bpp == 8u) {
        const uint4 h = make_uint4(half2_bits(p0.x, p0.y), half2_bits(p0.z, p0.w), half2_bits(p1.x, p1.y), half2_bits(p1.z, p1.w));
        uint32_t* w = reinterpret_cast<uint32_t*>(dst);
        if (vec && both) {
            *reinterpret_cast<uint4*>(dst) = h;
        } else {
            w[0] = h.x;
            w[1] = h.y;
            if (both) {
                w[2] = h.z;
                w[3] = h.w;
            }
        }
    } else if (vec) {
        float4* v = reinterpret_cast<float4*>(dst);
        v[0] = p0;
        if (both) v[1] = p1;
    } else {
        float* f = reinterpret_cast<float*>(dst);
        f[0] = p0.x; f[1] = p0.y; f[2] = p0.z; f[3] = p0.w;
        if (both) {
            f[4] = p1.x; f[5] = p1.y; f[6] = p1.z; f[7] = p1.w;
        }
    }
}
// The lane's eight pixels of row py from column x0 (planes in pixel pairs, as the painter holds them).
__device__ __forceinline__ void store_linear_run(const PaintScene& S, uint8_t* fb, uint32_t py, uint32_t x0, const f2 (&r)[4],
                                                 const f2 (&g)[4], const f2 (&b)[4], const f2 (&a)[4], bool vec, uint32_t bpp) {
    if (py >= S.height || x0 >= S.width) return;
    uint8_t* row = fb + (size_t)py * S.stride + (size_t)x0 * bpp;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const uint32_t x = x0 + 2u * (uint32_t)q;
        if (x < S.width)
            store_linear_pair(row + (size_t)(2 * q) * bpp, linear_pixel(r[q].x, g[q].x, b[q].x, a[q].x, S.channels),
                              linear_pixel(r[q].y, g[q].y, b[q].y, a[q].y, S.channels), x + 1u < S.width, vec, bpp);
    }
}
// store_tile_solid for a linear frame: the folded colour (BlendMode::blend's result) in every pixel.
__device__ __forceinline__ void store_tile_solid_linear(const PaintScene& S, uint8_t* fb, uint32_t tx, uint32_t ty, uint32_t lane,
                                                        const Rgba& c, bool vec, uint32_t bpp) {
    const f2 r[4] = {f2_splat(c.r), f2_splat(c.r), f2_splat(c.r), f2_splat(c.r)};
    const f2 g[4] = {f2_splat(c.g), f2_splat(c.g), f2_splat(c.g), f2_splat(c.g)};
    const f2 b[4] = {f2_splat(c.b), f2_splat(c.b), f2_splat(c.b), f2_splat(c.b)};
    const f2 a[4] = {f2_splat(c.a), f2_splat(c.a), f2_splat(c.a), f2_splat(c.a)};
    store_linear_run(S, fb, ty * 16u + (lane >> 1), tx * 16u + (lane & 1u) * 8u, r, g, b, a, vec, bpp);
}

// paint_kernel / paint_views_kernel storing a linear frame of `bpp` (8: RGBA16F, 16: RGBA32F)
// bytes per pixel. Built for 8 CTAs / SM only. A float frame takes no layer cache, so the
// solid-tile hook has no cached colour to compare with.
#define FORMA_PAINT_STORE_SOLID(c) store_tile_solid_linear(S, in.framebuffer, tx, ty, lane, c, vec_ok, bpp)
#define FORMA_PAINT_STORE_PIXELS() \
    (void)rgba_order;              \
    store_linear_run(S, in.framebuffer, ty * 16u + row, x0, dr, dg, db, da, vec_ok, bpp)
__global__ void __launch_bounds__(kPaintWarpsPerBlock * 32, 8)
    paint_linear_kernel(PaintScene S, PaintInputs in, uint32_t n_tiles, uint32_t bpp) {
    chain_begin();
#define FORMA_PAINT_FRAME_TY(ty) (ty)
#include "paint_kernel_body.cuh"
#undef FORMA_PAINT_FRAME_TY
}
__global__ void __launch_bounds__(kPaintWarpsPerBlock * 32, 8)
    paint_views_linear_kernel(PaintScene S, PaintInputs in, uint32_t n_tiles, uint32_t view_rows, uint32_t bpp) {
    chain_begin();
#define FORMA_PAINT_FRAME_TY(ty) ((ty) % view_rows)
#include "paint_kernel_body.cuh"
#undef FORMA_PAINT_FRAME_TY
}
#undef FORMA_PAINT_STORE_SOLID
#undef FORMA_PAINT_STORE_PIXELS

// ---------------------------------------------------------------------------
// Frames over a background (forma_renderer_render_over_device): the frame's own pixels are each
// pixel's clear colour. sRGB8 bytes decode through the table D (srgb_decode.h: every byte
// round-trips through compute_srgb's encode) and alpha as byte / 255; RGBA16F through
// __half2float; RGBA32F as stored. The channel order is a permutation of R, G, B, A (for sRGB8
// with A last, see check_request).
// ---------------------------------------------------------------------------
__device__ const float kSrgbDecode[256] = FORMA_SRGB_DECODE_TABLE;

// The byte (sRGB8) or value (float) position of each of R, G, B, A in a pixel: 2 bits each.
__device__ __forceinline__ uint32_t channel_positions(const uint32_t ch[4]) {
    uint32_t pos = 0;
#pragma unroll
    for (uint32_t k = 0; k < 4u; ++k) pos |= k << (2u * (ch[k] & 3u));
    return pos;
}
__device__ __forceinline__ uint32_t pos_of(uint32_t pos, uint32_t c) { return (pos >> (2u * c)) & 3u; }

// One background pixel into element `h` (0: x, 1: y) of the pair planes; its opaque bit at `bit`.
__device__ __forceinline__ void put_pixel(f2& r, f2& g, f2& b, f2& a, uint32_t h, float vr, float vg, float vb, float va,
                                          uint32_t& opaque, uint32_t bit) {
    if (h == 0u) {
        r.x = vr; g.x = vg; b.x = vb; a.x = va;
    } else {
        r.y = vr; g.y = vg; b.y = vb; a.y = va;
    }
    if (va == 1.0f) opaque |= 1u << bit;
}

// The lane's eight sRGB8 pixels of row py from column x0 (pixels outside the frame read as 0).
__device__ __forceinline__ void load_srgb_run(const PaintScene& S, const uint8_t* fb, uint32_t py, uint32_t x0, bool vec,
                                              const float* dec, uint32_t pos, f2 (&r)[4], f2 (&g)[4], f2 (&b)[4], f2 (&a)[4],
                                              uint32_t& opaque) {
    uint32_t w[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
    if (py < S.height && x0 < S.width) {
        const uint8_t* rowp = fb + (size_t)py * S.stride + (size_t)x0 * 4u;
        if (vec && x0 + 8u <= S.width) {
            const uint4 v0 = reinterpret_cast<const uint4*>(rowp)[0], v1 = reinterpret_cast<const uint4*>(rowp)[1];
            w[0] = v0.x; w[1] = v0.y; w[2] = v0.z; w[3] = v0.w; w[4] = v1.x; w[5] = v1.y; w[6] = v1.z; w[7] = v1.w;
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (x0 + (uint32_t)j < S.width) w[j] = reinterpret_cast<const uint32_t*>(rowp)[j];
        }
    }
    const uint32_t sr = 8u * pos_of(pos, 0), sg = 8u * pos_of(pos, 1), sb = 8u * pos_of(pos, 2), sa = 8u * pos_of(pos, 3);
    opaque = 0u;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const uint32_t v = w[j];
        put_pixel(r[j >> 1], g[j >> 1], b[j >> 1], a[j >> 1], (uint32_t)j & 1u, dec[(v >> sr) & 0xFFu], dec[(v >> sg) & 0xFFu],
                  dec[(v >> sb) & 0xFFu], (float)((v >> sa) & 0xFFu) / 255.0f, opaque, (uint32_t)j);
    }
}

// The same for a float frame of `bpp` bytes per pixel (8: RGBA16F, 16: RGBA32F).
__device__ __forceinline__ void load_linear_run(const PaintScene& S, const uint8_t* fb, uint32_t py, uint32_t x0, bool vec, uint32_t bpp,
                                                uint32_t pos, f2 (&r)[4], f2 (&g)[4], f2 (&b)[4], f2 (&a)[4], uint32_t& opaque) {
    opaque = 0u;
    const bool row_in = py < S.height;
    const uint8_t* rowp = fb + (size_t)py * S.stride + (size_t)x0 * bpp;
    const uint32_t pr = pos_of(pos, 0), pg = pos_of(pos, 1), pb = pos_of(pos, 2), pa = pos_of(pos, 3);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        float v[4] = {0.0f, 0.0f, 0.0f, 0.0f};
        if (row_in && x0 + (uint32_t)j < S.width) {
            const uint8_t* px = rowp + (size_t)j * bpp;
            if (bpp == 8u) {
                uint2 h;
                if (vec) {
                    h = *reinterpret_cast<const uint2*>(px);
                } else {
                    h.x = reinterpret_cast<const uint32_t*>(px)[0];
                    h.y = reinterpret_cast<const uint32_t*>(px)[1];
                }
                v[0] = __half2float(__ushort_as_half((unsigned short)(h.x & 0xFFFFu)));
                v[1] = __half2float(__ushort_as_half((unsigned short)(h.x >> 16)));
                v[2] = __half2float(__ushort_as_half((unsigned short)(h.y & 0xFFFFu)));
                v[3] = __half2float(__ushort_as_half((unsigned short)(h.y >> 16)));
            } else if (vec) {
                const float4 f = *reinterpret_cast<const float4*>(px);
                v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
            } else {
                const float* f = reinterpret_cast<const float*>(px);
                v[0] = f[0]; v[1] = f[1]; v[2] = f[2]; v[3] = f[3];
            }
        }
        put_pixel(r[j >> 1], g[j >> 1], b[j >> 1], a[j >> 1], (uint32_t)j & 1u, v[pr], v[pg], v[pb], v[pa], opaque, (uint32_t)j);
    }
}

// The per-pixel Alpha -> One upgrade (renderer.rs:87-92 with the pixel's background as clear colour):
// an opaque background gives alpha 1 whatever was painted. The channel order is a permutation, so
// storing alpha 1 is storing ONE.
__device__ __forceinline__ void upgrade_alpha(f2 (&a)[4], uint32_t opaque) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        if ((opaque >> (2 * q)) & 1u) a[q].x = 1.0f;
        if ((opaque >> (2 * q + 1)) & 1u) a[q].y = 1.0f;
    }
}

// compute_srgb + LinearLayout::write of the lane's eight pixels, as the body stores them. With A the
// last channel, a solid tile's to_srgb_bytes (position 3 unencoded) is this encode of its colour.
__device__ __forceinline__ void store_srgb_run(const PaintScene& S, uint8_t* fb, uint32_t py, uint32_t x0, const f2 (&dr)[4],
                                               const f2 (&dg)[4], const f2 (&db)[4], const f2 (&da)[4], bool vec, bool rgba_order) {
    if (py >= S.height || x0 >= S.width) return;
    uint32_t out[8];
    if (rgba_order) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            uint32_t r0, r1, g0, g1, b0, b1, a0, a1;
            to_byte2(srgb2(dr[q]), r0, r1);
            to_byte2(srgb2(dg[q]), g0, g1);
            to_byte2(srgb2(db[q]), b0, b1);
            to_byte2(da[q], a0, a1);
            out[2 * q] = r0 | (g0 << 8) | (b0 << 16) | (a0 << 24);
            out[2 * q + 1] = r1 | (g1 << 8) | (b1 << 16) | (a1 << 24);
        }
    } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            out[2 * q] = srgb_bytes_any_order(dr[q].x, dg[q].x, db[q].x, da[q].x, S.channels);
            out[2 * q + 1] = srgb_bytes_any_order(dr[q].y, dg[q].y, db[q].y, da[q].y, S.channels);
        }
    }
    uint8_t* rowp = fb + (size_t)py * S.stride + (size_t)x0 * 4u;
    if (vec && x0 + 8u <= S.width) {
        reinterpret_cast<uint4*>(rowp)[0] = make_uint4(out[0], out[1], out[2], out[3]);
        reinterpret_cast<uint4*>(rowp)[1] = make_uint4(out[4], out[5], out[6], out[7]);
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (x0 + (uint32_t)j < S.width) reinterpret_cast<uint32_t*>(rowp)[j] = out[j];
    }
}

// paint_kernel / paint_views_kernel over the frame's own sRGB8 pixels, and their linear twins over
// float pixels. The general build at 8 CTAs / SM whatever paint_wide and paint_solid say. D is
// copied to shared memory once per CTA: the eight bytes of a lane index it at random, which the
// constant cache would serialise.
#define FORMA_PAINT_OVER_SRGB_PROLOGUE                                          \
    __shared__ float s_decode[256];                                             \
    for (uint32_t i = threadIdx.x; i < 256u; i += blockDim.x) s_decode[i] = kSrgbDecode[i]; \
    __syncthreads();                                                            \
    const uint32_t over_pos = channel_positions(S.channels);
#define FORMA_PAINT_LOAD_PIXELS() load_srgb_run(S, in.framebuffer, ty * 16u + row, x0, vec_ok, s_decode, over_pos, dr, dg, db, da, bg_opaque)
#define FORMA_PAINT_STORE_PIXELS()   \
    upgrade_alpha(da, bg_opaque); \
    store_srgb_run(S, in.framebuffer, ty * 16u + row, x0, dr, dg, db, da, vec_ok, rgba_order)
__global__ void __launch_bounds__(kPaintWarpsPerBlock * 32, 8) paint_over_kernel(PaintScene S, PaintInputs in, uint32_t n_tiles) {
    chain_begin();
    FORMA_PAINT_OVER_SRGB_PROLOGUE
#define FORMA_PAINT_FRAME_TY(ty) (ty)
#include "paint_kernel_body.cuh"
#undef FORMA_PAINT_FRAME_TY
}
__global__ void __launch_bounds__(kPaintWarpsPerBlock * 32, 8)
    paint_views_over_kernel(PaintScene S, PaintInputs in, uint32_t n_tiles, uint32_t view_rows) {
    chain_begin();
    FORMA_PAINT_OVER_SRGB_PROLOGUE
#define FORMA_PAINT_FRAME_TY(ty) ((ty) % view_rows)
#include "paint_kernel_body.cuh"
#undef FORMA_PAINT_FRAME_TY
}
#undef FORMA_PAINT_LOAD_PIXELS
#undef FORMA_PAINT_STORE_PIXELS
#undef FORMA_PAINT_OVER_SRGB_PROLOGUE

#define FORMA_PAINT_LOAD_PIXELS() load_linear_run(S, in.framebuffer, ty * 16u + row, x0, vec_ok, bpp, over_pos, dr, dg, db, da, bg_opaque)
#define FORMA_PAINT_STORE_PIXELS()   \
    (void)rgba_order;                \
    upgrade_alpha(da, bg_opaque); \
    store_linear_run(S, in.framebuffer, ty * 16u + row, x0, dr, dg, db, da, vec_ok, bpp)
__global__ void __launch_bounds__(kPaintWarpsPerBlock * 32, 8)
    paint_over_linear_kernel(PaintScene S, PaintInputs in, uint32_t n_tiles, uint32_t bpp) {
    chain_begin();
    const uint32_t over_pos = channel_positions(S.channels);
#define FORMA_PAINT_FRAME_TY(ty) (ty)
#include "paint_kernel_body.cuh"
#undef FORMA_PAINT_FRAME_TY
}
__global__ void __launch_bounds__(kPaintWarpsPerBlock * 32, 8)
    paint_views_over_linear_kernel(PaintScene S, PaintInputs in, uint32_t n_tiles, uint32_t view_rows, uint32_t bpp) {
    chain_begin();
    const uint32_t over_pos = channel_positions(S.channels);
#define FORMA_PAINT_FRAME_TY(ty) ((ty) % view_rows)
#include "paint_kernel_body.cuh"
#undef FORMA_PAINT_FRAME_TY
}
#undef FORMA_PAINT_LOAD_PIXELS
#undef FORMA_PAINT_STORE_PIXELS

// The inverse of repack_views_kernel: rows [0, height) of every frame of the caller's stack (frame b
// at src + b * view_stride, row r at + r * stride) to the stacked frame (frame b's first row at
// dst + b * view_rows_px * dst_stride), so that a stack painted in scratch starts from its
// background. One thread per 4-byte word, `width` words per row.
__global__ void __launch_bounds__(256) unpack_views_kernel(const uint8_t* __restrict__ src, uint64_t stride, uint64_t view_stride,
                                                           uint8_t* __restrict__ dst, uint64_t dst_stride, uint32_t view_rows_px,
                                                           uint32_t width, uint32_t height) {
    chain_begin();
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t r = blockIdx.y, b = blockIdx.z;
    if (x >= width) return;
    const uint8_t* s = src + (uint64_t)b * view_stride + (uint64_t)r * stride + (uint64_t)x * 4u;
    uint8_t* d = dst + ((uint64_t)b * view_rows_px + r) * dst_stride + (uint64_t)x * 4u;
    *reinterpret_cast<uint32_t*>(d) = *reinterpret_cast<const uint32_t*>(s);
}
void launch_unpack_views(const uint8_t* src, uint64_t stride, uint64_t view_stride, uint8_t* dst, uint64_t dst_stride,
                         uint32_t view_rows_px, uint32_t width, uint32_t height, uint32_t n_views, cudaStream_t st) {
    if (!width || !height || !n_views) return;
    launch_chained(unpack_views_kernel, dim3((width + 255u) / 256u, height, n_views), 256, 0, st, src, stride, view_stride, dst, dst_stride,
                                                                                      view_rows_px, width, height);
}

// Rows [0, height) of every view of a stacked frame (view b at src + b * view_rows_px * src_stride)
// to dst + b * view_stride + row * stride: padding rows and the bytes between views stay untouched.
// One thread per pixel, 4 bytes apart in every row.
__global__ void __launch_bounds__(256) repack_views_kernel(const uint8_t* __restrict__ src, uint64_t src_stride, uint32_t view_rows_px,
                                                           uint8_t* __restrict__ dst, uint64_t stride, uint64_t view_stride,
                                                           uint32_t width, uint32_t height, bool aligned) {
    chain_begin();
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t r = blockIdx.y, b = blockIdx.z;
    if (x >= width) return;
    const uint8_t* s = src + ((uint64_t)b * view_rows_px + r) * src_stride + (uint64_t)x * 4u;
    uint8_t* d = dst + (uint64_t)b * view_stride + (uint64_t)r * stride + (uint64_t)x * 4u;
    if (aligned) {
        *reinterpret_cast<uint32_t*>(d) = *reinterpret_cast<const uint32_t*>(s);
    } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) d[k] = s[k];
    }
}
void launch_repack_views(const uint8_t* src, uint64_t src_stride, uint32_t view_rows_px, uint8_t* dst, uint64_t stride,
                         uint64_t view_stride, uint32_t width, uint32_t height, uint32_t n_views, cudaStream_t st) {
    if (!width || !height || !n_views) return;
    const bool aligned = (((uintptr_t)dst | stride | view_stride | (uintptr_t)src | src_stride) & 3u) == 0u;
    launch_chained(repack_views_kernel, dim3((width + 255u) / 256u, height, n_views), 256, 0, st, src, src_stride, view_rows_px, dst, stride,
                                                                                     view_stride, width, height, aligned);
}

// Packs the tiles named in `list` (written by paint_kernel) into 1 KB records,
// row-major 16x16 RGBA8, so that a damaged frame costs a device->host copy
// proportional to the damage. One warp per tile.
__global__ void __launch_bounds__(256) gather_tiles_kernel(const uint8_t* __restrict__ fb, uint32_t stride, uint32_t width,
                                                           uint32_t height, uint32_t tiles_x,
                                                           const uint32_t* __restrict__ list,
                                                           const uint32_t* __restrict__ count, uint32_t* __restrict__ out) {
    chain_begin();
    const uint32_t n = *count;
    const uint32_t lane = threadIdx.x & 31u;
    for (uint32_t i = blockIdx.x * 8u + (threadIdx.x >> 5); i < n; i += gridDim.x * 8u) {
        const uint32_t tid = list[i];
        const uint32_t x0 = (tid % tiles_x) * 16u, y0 = (tid / tiles_x) * 16u;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const uint32_t p = (uint32_t)k * 32u + lane;  // pixel index in the tile, row-major
            const uint32_t x = x0 + (p & 15u), y = y0 + (p >> 4);
            uint32_t v = 0;
            if (x < width && y < height) v = *reinterpret_cast<const uint32_t*>(fb + (size_t)y * stride + (size_t)x * 4u);
            out[(size_t)i * 256u + p] = v;
        }
    }
}

void launch_gather_tiles(const PaintScene& S, const uint8_t* framebuffer, uint32_t* packed, cudaStream_t st) {
    launch_chained(gather_tiles_kernel, device_sm_count() * 4, 256, 0, st, framebuffer, S.stride, S.width, S.height, S.tiles_x, S.written_list,
                                                               S.written_count, packed);
}

// One thread per style slot: the GradRec of a gradient of up to four stops, with the very
// operations Gradient::get_t / color_at perform per call (styling.rs:59-66,107-108).
__global__ void grad_setup_kernel(const StyleRec* __restrict__ styles, const StopRec* __restrict__ stops, uint32_t n,
                                  GradRec* __restrict__ grads) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const StyleRec st = styles[i];
    GradRec g;
    g.pad = 0u;
    if (st.fill_type != 1u || st.stop_count < 2u || st.stop_count > 4u) {
        g.sx = g.sy = g.dx = g.dy = g.dot_recip = 0.0f;
        g.type = 0u;
        g.count = 0xFFFFFFFFu;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            g.stop[k] = g.rcp_d[k] = 0.0f;
#pragma unroll
            for (int c = 0; c < 4; ++c) g.color[k][c] = 0.0f;
        }
        grads[i] = g;
        return;
    }
    g.sx = st.start[0];
    g.sy = st.start[1];
    g.dx = st.end[0] - st.start[0];
    g.dy = st.end[1] - st.start[1];
    const float dot = g.dx * g.dx + g.dy * g.dy;
    g.dot_recip = d_rcp(dot);
    g.type = st.gradient_type;
    g.count = st.stop_count;
    const StopRec* sp = stops + st.stop_first;
    float start_stop = 0.0f;
#pragma unroll
    for (uint32_t k = 0; k < 4u; ++k) {
        const StopRec s = sp[k < st.stop_count ? k : st.stop_count - 1u];
#pragma unroll
        for (int c = 0; c < 4; ++c) g.color[k][c] = s.color[c];
        g.stop[k] = s.stop;
        if (k >= 1u) {
            g.rcp_d[k - 1u] = d_rcp(s.stop - start_stop);
            start_stop = s.stop;
        }
    }
    g.rcp_d[3] = 0.0f;
    grads[i] = g;
}
void launch_grad_setup(const StyleRec* styles, const StopRec* stops, uint32_t n_styles, GradRec* grads, cudaStream_t st) {
    if (n_styles) grad_setup_kernel<<<(n_styles + 127) / 128, 128, 0, st>>>(styles, stops, n_styles, grads);
}

// Self-test of the pair arithmetic (forma_debug_selftest): every pair helper against the
// scalar IEEE operation it stands for, on `n` operand triples. Returns mismatches in out[0].
__global__ void f32x2_selftest_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ c,
                                      uint32_t n, uint32_t* __restrict__ out) {
    const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) * 2u;
    if (i + 1u >= n) return;
    const f2 x{a[i], a[i + 1]}, y{b[i], b[i + 1]}, z{c[i], c[i + 1]};
    uint32_t bad = 0;
    auto same = [](float p, float q) { return __float_as_uint(p) == __float_as_uint(q) || (p != p && q != q); };
    const f2 f = fma2(x, y, z), m = mul2(x, y), s = add2(x, y), d = sub2(x, y);
    const f2 ms = add2(mul2(x, y), z);  // a product followed by a sum must stay two roundings
    bad += !same(f.x, fmaf(x.x, y.x, z.x)) + !same(f.y, fmaf(x.y, y.y, z.y));
    bad += !same(m.x, x.x * y.x) + !same(m.y, x.y * y.y);
    bad += !same(s.x, x.x + y.x) + !same(s.y, x.y + y.y);
    bad += !same(d.x, x.x - y.x) + !same(d.y, x.y - y.y);
    bad += !same(ms.x, (x.x * y.x) + z.x) + !same(ms.y, (x.y * y.y) + z.y);
    if (bad) atomicAdd(out, bad);
}
void launch_f32x2_selftest(const float* a, const float* b, const float* c, uint32_t n, uint32_t* out, cudaStream_t st) {
    f32x2_selftest_kernel<<<(n / 2 + 255) / 256, 256, 0, st>>>(a, b, c, n, out);
}

// Several host threads may render on one device, and paint_kernel<8> and paint_kernel<6> share a
// type: the occupancy cache is keyed by the kernel's address and the device, under one lock.
TileGrid tile_grid(const PaintScene& S, const void* kernel, uint32_t warps, uint32_t* tile_counter, cudaStream_t st,
                   bool counter_zeroed) {
    if (S.tx_hi <= S.tx_lo || S.ty_hi <= S.ty_lo) return TileGrid{0u, 0u};
    const uint32_t n_tiles = (S.tx_hi - S.tx_lo) * (S.ty_hi - S.ty_lo);
    if (!counter_zeroed) cudaMemsetAsync(tile_counter, 0, sizeof(uint32_t), st);
    static std::mutex mu;
    static std::map<std::pair<const void*, int>, int> blocks_per_sm;
    int per_sm = 0;
    {
        std::lock_guard<std::mutex> lk(mu);
        int& slot = blocks_per_sm[{kernel, current_device_index()}];
        if (!slot) {
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&slot, kernel, (int)warps * 32, 0);
            if (slot < 1) slot = 1;
        }
        per_sm = slot;
    }
    return TileGrid{n_tiles, min((uint32_t)(per_sm * device_sm_count()), (n_tiles + warps - 1u) / warps)};
}

static PaintInputs paint_inputs(const PaintScene& S, const TileTables& t, uint8_t* eflags, uint8_t* framebuffer,
                                uint32_t* tile_counter) {
    return PaintInputs{t.segs, t.recs, t.tile_range, t.heavy, t.heavy_count, S.tiles_x * S.tiles_y, eflags, framebuffer, tile_counter};
}

void launch_paint(const PaintScene& S, const TileTables& t, uint8_t* eflags, uint8_t* framebuffer, uint32_t* tile_counter,
                  cudaStream_t st, uint32_t view_rows, bool solid_over, bool counter_zeroed) {
    // Build 0: the general kernel at 128 registers (8 CTAs / SM); 1: option paint_wide = 1, up to 168
    // registers (6 CTAs / SM); 2: a solid `Over` frame (option paint_solid = 1), the lean build at 96
    // registers (10 CTAs / SM).
    const int build = solid_over && options().paint_solid ? 2 : options().paint_wide ? 1 : 0;
    void (*const frame[3])(PaintScene, PaintInputs, uint32_t) = {paint_kernel<8>, paint_kernel<6>, paint_solid_kernel<8>};
    void (*const views[3])(PaintScene, PaintInputs, uint32_t, uint32_t) = {paint_views_kernel<8>, paint_views_kernel<6>,
                                                                            paint_views_solid_kernel<8>};
    const void* kernel = view_rows ? (const void*)views[build] : (const void*)frame[build];
    const TileGrid g = tile_grid(S, kernel, kPaintWarpsPerBlock, tile_counter, st, counter_zeroed);
    if (!g.n_tiles) return;
    const PaintInputs in = paint_inputs(S, t, eflags, framebuffer, tile_counter);
    if (view_rows) launch_chained(views[build], g.ctas, kPaintWarpsPerBlock * 32, 0, st, S, in, g.n_tiles, view_rows);
    else launch_chained(frame[build], g.ctas, kPaintWarpsPerBlock * 32, 0, st, S, in, g.n_tiles);
}

void launch_paint_linear(const PaintScene& S, const TileTables& t, uint8_t* eflags, uint8_t* framebuffer, uint32_t* tile_counter,
                         cudaStream_t st, uint32_t view_rows, uint32_t bpp, bool counter_zeroed) {
    const void* kernel = view_rows ? (const void*)paint_views_linear_kernel : (const void*)paint_linear_kernel;
    const TileGrid g = tile_grid(S, kernel, kPaintWarpsPerBlock, tile_counter, st, counter_zeroed);
    if (!g.n_tiles) return;
    const PaintInputs in = paint_inputs(S, t, eflags, framebuffer, tile_counter);
    if (view_rows) launch_chained(paint_views_linear_kernel, g.ctas, kPaintWarpsPerBlock * 32, 0, st, S, in, g.n_tiles, view_rows, bpp);
    else launch_chained(paint_linear_kernel, g.ctas, kPaintWarpsPerBlock * 32, 0, st, S, in, g.n_tiles, bpp);
}

void launch_paint_over(const PaintScene& S, const TileTables& t, uint8_t* eflags, uint8_t* framebuffer, uint32_t* tile_counter,
                       cudaStream_t st, uint32_t view_rows, uint32_t bpp, bool counter_zeroed) {
    const bool linear = bpp != 4u;
    const void* kernel = view_rows ? (linear ? (const void*)paint_views_over_linear_kernel : (const void*)paint_views_over_kernel)
                                   : (linear ? (const void*)paint_over_linear_kernel : (const void*)paint_over_kernel);
    const TileGrid g = tile_grid(S, kernel, kPaintWarpsPerBlock, tile_counter, st, counter_zeroed);
    if (!g.n_tiles) return;
    const PaintInputs in = paint_inputs(S, t, eflags, framebuffer, tile_counter);
    const uint32_t block = kPaintWarpsPerBlock * 32;
    if (view_rows) {
        if (linear) launch_chained(paint_views_over_linear_kernel, g.ctas, block, 0, st, S, in, g.n_tiles, view_rows, bpp);
        else launch_chained(paint_views_over_kernel, g.ctas, block, 0, st, S, in, g.n_tiles, view_rows);
    } else {
        if (linear) launch_chained(paint_over_linear_kernel, g.ctas, block, 0, st, S, in, g.n_tiles, bpp);
        else launch_chained(paint_over_kernel, g.ctas, block, 0, st, S, in, g.n_tiles);
    }
}

}  // namespace forma
