// Helpers shared by the painter-table kernels (kernels_tables.cu), the painter itself
// (kernels_painter.cu) and the ID kernel (kernels_ids.cu): key field access, packed 16 x i8
// covers, the per-entry accumulation of segments into packed cells and the coverage rules.
#pragma once

#include "cuda_common.cuh"
#include "kernels.h"

namespace forma {

// --- key helpers (keys keep the segment layout; low 20 bits are zero) ---------
__device__ __forceinline__ uint32_t key_ty(uint64_t k) { return (uint32_t)(k >> 53) & 0x7FFu; }   // biased (+1)
__device__ __forceinline__ uint32_t key_tx(uint64_t k) { return (uint32_t)(k >> 41) & 0xFFFu; }   // biased (+1)
__device__ __forceinline__ uint32_t key_layer(uint64_t k) { return (uint32_t)(k >> 20) & 0x1FFFFFu; }
// (tile_y, layer, tile_x) ordering key in the same [20, 64) bit window.
__device__ __forceinline__ uint64_t make_key2(uint64_t k) {
    return ((uint64_t)key_ty(k) << 53) | ((uint64_t)key_layer(k) << 32) | ((uint64_t)key_tx(k) << 20);
}
__device__ __forceinline__ uint32_t key2_tx(uint64_t k2) { return (uint32_t)(k2 >> 20) & 0xFFFu; }
__device__ __forceinline__ uint32_t key2_layer(uint64_t k2) { return (uint32_t)(k2 >> 32) & 0x1FFFFFu; }

// --- packed 16 x i8 covers -----------------------------------------------------
__device__ __forceinline__ uint4 cover_add(uint4 a, uint4 b) {
    return make_uint4(__vadd4(a.x, b.x), __vadd4(a.y, b.y), __vadd4(a.z, b.z), __vadd4(a.w, b.w));
}
// Cover::is_empty / is_full, cpu/painter/mod.rs:187-214.
__device__ __forceinline__ bool cover_is_empty(uint4 c, uint32_t fill_rule) {
    uint32_t any = c.x | c.y | c.z | c.w;
    return fill_rule == 0u ? any == 0u : (any & 0x1F1F1F1Fu) == 0u;
}
__device__ __forceinline__ bool cover_is_full(uint4 c, uint32_t fill_rule) {
    if (fill_rule == 0u) {
        const uint32_t k = 0x10101010u;
        return __vabs4(c.x) == k && __vabs4(c.y) == k && __vabs4(c.z) == k && __vabs4(c.w) == k;
    }
    const uint32_t m = 0x1F1F1F1Fu, k = 0x10101010u;
    return (c.x & m) == k && (c.y & m) == k && (c.z & m) == k && (c.w & m) == k;
}

// --- per-entry optimizer flags (layer_workbench passes) -----------------------------
constexpr uint32_t kFlagHasSegs = 1, kFlagFull = 2, kFlagMaskedOut = 4, kFlagSkipClip = 8, kFlagUnchanged = 16;
constexpr uint32_t kFlagClipish = 32;      // Func::Clip, or a Draw layer with is_clipped
constexpr uint32_t kFlagOpaque = 64;       // Draw, solid fill, BlendMode::Over, alpha == 1
constexpr uint32_t kFlagClippedDraw = 128; // Draw layer with is_clipped

// Tiles with at least kHeavyMin entries are listed by class (class c: 2^(c+4) <= entries <
// 2^(c+5), the last class open-ended) so that the painter starts them first.
constexpr int kHeavyClasses = kHeavyListClasses;
constexpr uint32_t kHeavyMin = 16;
__device__ __forceinline__ int heavy_class(uint32_t entries) {
    const int c = 27 - __clz((int)entries);  // floor(log2) - 4
    return c > kHeavyClasses - 1 ? kHeavyClasses - 1 : c;
}

// packed style: fill_rule | func<<1 | is_clipped<<2 | fill_type<<3 | blend_mode<<5 | unchanged<<9 |
//               small gradient (<= 4 stops: the painter uses its GradRec)<<10
constexpr uint32_t kMetaSmallGradient = 1u << 10;
__device__ __forceinline__ uint32_t pack_style_meta(const StyleRec& st, bool unchanged) {
    return (st.fill_rule & 1u) | ((st.func & 1u) << 1) | ((st.is_clipped ? 1u : 0u) << 2) | ((st.fill_type & 3u) << 3) |
           ((st.blend_mode & 15u) << 5) | (unchanged ? (1u << 9) : 0u) |
           ((st.fill_type == 1u && st.stop_count >= 2u && st.stop_count <= 4u) ? kMetaSmallGradient : 0u);
}

__device__ __forceinline__ uint32_t fill_rule_of(const PaintScene& S, uint32_t layer) {
    int32_t slot = layer < S.n_orders ? S.order_to_style[layer] : -1;
    return slot >= 0 ? S.styles[slot].fill_rule : 0u;
}


// --- per-entry accumulation of the painter and the ID kernel -------------------------
// Shared-memory word of pixel (local_x, local_y): row-major, ly * 16 + lx, i.e. the segment's
// (local_x, local_y) byte with its nibbles swapped. Lane l = 2 ly + lx / 8 owns the eight
// consecutive words l * 8 .. + 8 (two 16-byte accesses, two-way bank conflict: negligible
// next to the index arithmetic a swizzle would cost per segment).
__device__ __forceinline__ uint32_t cell_index_of(uint64_t s) {
    const uint32_t t = (uint32_t)(s >> 12);  // bits 7..4 local_x, 3..0 local_y
    return ((t & 15u) << 4) | ((t >> 4) & 15u);
}

// doubled_area_to_coverage (cpu/painter/mod.rs:76-94) by fill rule. The clamp of the
// non-zero rule only ever sees a non-negative, non-NaN value: min(v, 1) is the same result.
__device__ __forceinline__ float coverage_non_zero(int32_t doubled_area) {
    return fminf(fabsf((float)doubled_area * (1.0f / 512.0f)), 1.0f);
}
__device__ __forceinline__ float coverage_even_odd(int32_t doubled_area) {
    return (float)(512 - abs((doubled_area & 1023) - 512)) * (1.0f / 512.0f);
}

constexpr uint32_t kPackedSegLimit = 2016u;  // segments per normalisation round of the packed cells (< 2048)

// acc_segment (cpu/painter/mod.rs:257-271) for one segment: area and cover into the packed cell.
__device__ __forceinline__ void scatter_one(uint32_t* cells, uint64_t s) {
    const int32_t cv = (int32_t)(((uint32_t)s & 0x3Fu) ^ 0x20u) - 0x20;
    const int32_t dam = (int32_t)((uint32_t)(s >> 6) & 0x3Fu);
    atomicAdd(&cells[cell_index_of(s)], (uint32_t)((dam * cv) * 65536 + cv));
}

// Segments 64.. of a long entry (about one entry in ten has more than 64). Every
// kPackedSegLimit segments the low halves are folded back to i8 so that they cannot overflow
// 16 bits (areas wrap at i16, covers at i8, exactly like the reference's lanes).
__device__ __noinline__ inline void scatter_rest(const uint64_t* __restrict__ segs, uint32_t from, uint32_t s1, uint32_t* cells,
                                                 uint32_t lane) {
    uint32_t done = 64u;
    for (uint32_t i0 = from; i0 < s1; i0 += 32u) {
        if (i0 + lane < s1) scatter_one(cells, segs[i0 + lane]);
        done += 32u;
        if (done >= kPackedSegLimit && i0 + 32u < s1) {
            __syncwarp();
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const uint32_t w = cells[k * 32 + lane];
                const int32_t lo = (int32_t)(int16_t)(w & 0xFFFFu);
                const uint32_t area = (w - (uint32_t)lo) & 0xFFFF0000u;
                cells[k * 32 + lane] = area + (uint32_t)(int32_t)(int8_t)lo;
            }
            __syncwarp();
            done = 0;
        }
    }
}

// Scatter-adds the segments [s0, s1) of one entry into `cells`. `pre0` / `pre1` hold the
// first two 32-segment chunks (requested one entry earlier).
__device__ __forceinline__ void scatter_entry(const uint64_t* __restrict__ segs, uint32_t s0, uint32_t s1, uint64_t pre0,
                                              uint64_t pre1, uint32_t* cells, uint32_t lane) {
    const uint32_t n = s1 - s0;
    if (lane < n) scatter_one(cells, pre0);
    if (lane + 32u < n) scatter_one(cells, pre1);
    if (n > 64u) scatter_rest(segs, s0 + 64u, s1, cells, lane);
}

// The grid of a persistent tile kernel (paint, ID, mask and statistics kernels) over the tile
// rectangle of S: n_tiles = 0 for an empty rectangle (launch nothing); otherwise `tile_counter` is
// reset on `st` and ctas = min(resident CTAs x SMs, ceil(n_tiles / warps)), the kernel's occupancy
// at `warps` warps per CTA being queried once per kernel and device (kernels_painter.cu).
struct TileGrid {
    uint32_t n_tiles, ctas;
};
// counter_zeroed: the counter is already zero (a kernel earlier in the chain cleared it), no memset.
TileGrid tile_grid(const PaintScene& S, const void* kernel, uint32_t warps, uint32_t* tile_counter, cudaStream_t st,
                   bool counter_zeroed = false);

// Cells that cannot influence a painted tile (rows outside the painted band,
// columns right of it) get this key in both pair sorts: it sorts last and keeps
// the sort keys inside host-known bounds (tile_y field = tiles_y + 1).
__device__ __host__ __forceinline__ uint64_t sentinel_key(uint32_t tiles_y) { return (uint64_t)(tiles_y + 1u) << 53; }

}  // namespace forma
