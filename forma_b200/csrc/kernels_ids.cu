// ID frames: the order of the topmost Func::Draw layer that hits each pixel, from the painter
// tables (build_tables) in place of the paint kernel. One warp per 16x16 tile, persistent warps
// taking tiles by ticket (heavy-tile lists first, like paint_kernel); lane l owns the painter's
// eight pixels (row l / 2, columns 8 (l % 2) .. + 8).
//
// A layer L hits pixel p where the painter would run blend_at for L at p with
// coverage x clip mask > min_coverage (the mask only where the painter applies a clip to L).
// Coverages are k / 512 and the product of two of them is exact in f32, so the result is
// integer-exact. Colour, alpha, fill and blend mode play no part.
//
// Tiles without clip-ish entries (no Func::Clip, no clipped Draw) are walked top-down: the
// first hit settles a pixel, and the warp stops as soon as a ballot finds all 256 settled. A
// full entry (kFlagFull: no segments, a full carried cover) settles every open pixel without
// reading anything. The painter's skip_fully_covered_layers pass needs no counterpart here:
// the layer it starts from is full, so the top-down walk never passes it.
//
// Tiles with clips follow the painter's own order bottom-up, with its clip state, and the
// last hit wins. The entry flags start from EntryRec::flags0 (paint_kernel rewrites `eflags`
// in place, and the combined call runs this kernel after it): skip_trivial_clips runs again
// from flags0 into `id_flags`, and the walk starts at the same top-most full opaque layer
// as the painter (a clipped layer above it whose clip lies below it is never painted).
//
// Stacked frames: a tile row belongs to one frame and the walk never looks at another tile, so
// the views of one composition need nothing else. The frames of a batch carry base + order in
// their entries (BatchFrame::order_base), and the walk compares layers and clip ranges in that
// shifted space; paint_ids_stacked_kernel, the same body, takes the frame's base off every ID it
// stores (one look-up per tile).
#include <mutex>

#include "../../include/forma_b200.h"
#include "paint_common.cuh"

namespace forma {

struct IdInputs {
    const uint64_t* segs;
    const EntryRec* recs;
    const uint2* tile_range;
    const uint32_t* heavy;        // kHeavyClasses lists of heavy tiles (linear ids), n_tiles_total each; may be null
    const uint32_t* heavy_count;
    uint32_t n_tiles_total;
    uint8_t* id_flags;            // per sorted entry: the flags after skip_trivial_clips (clip tiles only)
    uint32_t* ids;                // the ID frame
    size_t ids_stride;            // bytes
    float min_coverage;
    uint32_t* tile_counter;
};

constexpr int kIdWarpsPerBlock = 2;

struct IdWarpSmem {
    uint32_t cells[256];  // packed (area << 16) + cover
    float clip[256];      // clip mask, same layout
    uint32_t ids[256];    // the tile's IDs so far, same layout (kept out of registers: they would be spilled
                          // around the out-of-line scatter_rest)
    EntryRec hdr[32];     // the current group of entry records (pad = the entry's flags)
};

// Coverage of the lane's eight pixels for entry h (segments accumulated into W.cells, which
// are left zeroed). Called by the whole warp.
__device__ __forceinline__ void entry_coverage(IdWarpSmem& W, const EntryRec& h, const uint64_t* __restrict__ segs,
                                               uint32_t lane, float cov[8]) {
    const uint32_t row = lane >> 1, hx = lane & 1u;
    const uint32_t fill_rule = h.meta & 1u;
    const uint32_t cw = reinterpret_cast<const uint32_t*>(&h.carry)[row >> 2];
    int32_t run = (int32_t)(int8_t)((cw >> (8u * (row & 3u))) & 0xFFu);
    const uint32_t s0 = h.seg0, s1 = h.seg1;
    if (s1 == s0) {
        const float c = fill_rule == 0u ? coverage_non_zero(32 * run) : coverage_even_odd(32 * run);
#pragma unroll
        for (int j = 0; j < 8; ++j) cov[j] = c;
        return;
    }
    const uint64_t pre0 = s0 + lane < s1 ? segs[s0 + lane] : 0ull;
    const uint64_t pre1 = s0 + 32u + lane < s1 ? segs[s0 + 32u + lane] : 0ull;
    scatter_entry(segs, s0, s1, pre0, pre1, W.cells, lane);
    __syncwarp();
    uint4* c4 = reinterpret_cast<uint4*>(W.cells);
    const uint4 w0 = c4[2u * lane], w1 = c4[2u * lane + 1u];
    c4[2u * lane] = make_uint4(0u, 0u, 0u, 0u);
    c4[2u * lane + 1u] = make_uint4(0u, 0u, 0u, 0u);
    // The painter's unpacking (paint_kernel inlines the same arithmetic).
    const uint32_t w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
    int32_t area[8], cv[8], total = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        cv[j] = (int32_t)(int16_t)(w[j] & 0xFFFFu);
        area[j] = (int32_t)(w[j] + 0x8000u) >> 16;
        total += cv[j];
    }
    const int32_t left = __shfl_xor_sync(kFullMask, total, 1);
    if (hx) run += left;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int32_t dbl = 32 * (int32_t)(int8_t)run + area[j];
        run += cv[j];
        cov[j] = fill_rule == 0u ? coverage_non_zero(dbl) : coverage_even_odd(dbl);
    }
}

// Stages the records [lo, lo + cnt) in W.hdr, with the flags the walk uses in `pad`.
__device__ __forceinline__ void stage_group(IdWarpSmem& W, const IdInputs& in, uint32_t lo, uint32_t cnt, bool clip_tile,
                                            uint32_t lane) {
    __syncwarp();  // the previous group's records are no longer read
    if (lane < cnt) {
        const uint4* src = reinterpret_cast<const uint4*>(in.recs + lo + lane);
        uint4* dst = reinterpret_cast<uint4*>(&W.hdr[lane]);
        uint4 q3 = src[3];
        q3.w = clip_tile ? (uint32_t)in.id_flags[lo + lane] : q3.z;  // pad <- flags (q3.z = flags0)
        dst[0] = src[0]; dst[1] = src[1]; dst[2] = src[2]; dst[3] = q3;
    }
    __syncwarp();
}

// skip_trivial_clips (passes/skip_trivial_clips.rs:27-112) from flags0 into id_flags, as
// paint_kernel's pass B does it into eflags. One lane.
__device__ __forceinline__ void skip_trivial_clips_ids(const EntryRec* __restrict__ recs, uint8_t* __restrict__ out, uint32_t b,
                                                    uint32_t e) {
    bool has_clip = false, clip_full = false, clip_used = false;
    uint32_t clip_last = 0, clip_i = 0;
    for (uint32_t p = b; p < e; ++p) {
        uint32_t f = recs[p].flags0;
        const uint32_t id = recs[p].layer;
        if (!(f & kFlagClipish)) {
            out[p] = (uint8_t)f;
            if (has_clip && id > clip_last) {
                has_clip = false;
                if (!clip_used) out[clip_i] |= (uint8_t)kFlagMaskedOut;
            }
            continue;
        }
        if (!(f & kFlagClippedDraw)) {  // Func::Clip
            clip_full = (f & kFlagFull) != 0;
            clip_last = id + recs[p].clip_layers;
            clip_i = p;
            clip_used = false;
            has_clip = true;
            if (clip_full) f |= kFlagMaskedOut;
        } else {
            if (has_clip && id <= clip_last) {
                if (clip_full) f |= kFlagSkipClip;
                else clip_used = true;
            } else {
                f |= kFlagMaskedOut;
            }
        }
        out[p] = (uint8_t)f;
        if (has_clip && id > clip_last) {
            has_clip = false;
            if (!clip_used) out[clip_i] |= (uint8_t)kFlagMaskedOut;
        }
    }
    if (has_clip && !clip_used) out[clip_i] |= (uint8_t)kFlagMaskedOut;
}

// The lane's eight IDs of a batch frame's tile (base + order) as the frame's own orders.
__device__ __forceinline__ void rebase_ids(uint32_t* out, uint32_t base) {
#pragma unroll
    for (int j = 0; j < 8; ++j)
        if (out[j] != FORMA_ID_NONE) out[j] -= base;
}

__global__ void __launch_bounds__(kIdWarpsPerBlock * 32) paint_ids_kernel(PaintScene S, IdInputs in, uint32_t n_tiles) {
#define FORMA_IDS_REBASE(out, ty)
#include "paint_ids_body.cuh"
#undef FORMA_IDS_REBASE
}
// S stacks the frames of a batch, `rows` tile rows each; frame c's entries carry
// frames[c].order_base + order, and the IDs stored are the frame's own orders.
__global__ void __launch_bounds__(kIdWarpsPerBlock * 32) paint_ids_stacked_kernel(PaintScene S, IdInputs in, uint32_t n_tiles,
                                                                                  uint32_t rows, const BatchFrame* __restrict__ frames) {
#define FORMA_IDS_REBASE(out, ty) rebase_ids(out, frames[(ty) / rows].order_base)
#include "paint_ids_body.cuh"
#undef FORMA_IDS_REBASE
}

// CTAs of `kernel` that fill the device (one occupancy query per device and kernel).
template <class Kernel>
static uint32_t id_grid_limit(Kernel kernel, int (&blocks_per_sm)[kMaxDevices]) {
    static std::mutex config_mu;
    std::lock_guard<std::mutex> lk(config_mu);
    int& slot = blocks_per_sm[current_device_index()];
    if (!slot) {
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&slot, kernel, kIdWarpsPerBlock * 32, 0);
        if (slot < 1) slot = 1;
    }
    return (uint32_t)(slot * device_sm_count());
}

void launch_paint_ids(const PaintScene& S, const uint64_t* segs, const EntryRec* recs, const uint2* tile_range,
                      const uint32_t* heavy, const uint32_t* heavy_count, uint8_t* id_flags, uint32_t* ids, size_t ids_stride,
                      float min_coverage, uint32_t* tile_counter, cudaStream_t st, uint32_t rows, const BatchFrame* frames) {
    if (S.tx_hi <= S.tx_lo || S.ty_hi <= S.ty_lo) return;
    const uint32_t n_tiles = (S.tx_hi - S.tx_lo) * (S.ty_hi - S.ty_lo);
    cudaMemsetAsync(tile_counter, 0, sizeof(uint32_t), st);
    IdInputs in{segs, recs, tile_range, heavy, heavy_count, S.tiles_x * S.tiles_y, id_flags, ids, ids_stride, min_coverage,
                tile_counter};
    static int blocks_per_sm[2][kMaxDevices] = {{0}};
    const uint32_t need = (n_tiles + kIdWarpsPerBlock - 1) / kIdWarpsPerBlock;
    if (frames) {
        const uint32_t want = id_grid_limit(paint_ids_stacked_kernel, blocks_per_sm[1]);
        paint_ids_stacked_kernel<<<min(want, need), kIdWarpsPerBlock * 32, 0, st>>>(S, in, n_tiles, rows, frames);
    } else {
        const uint32_t want = id_grid_limit(paint_ids_kernel, blocks_per_sm[0]);
        paint_ids_kernel<<<min(want, need), kIdWarpsPerBlock * 32, 0, st>>>(S, in, n_tiles);
    }
}

}  // namespace forma
