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
#include <algorithm>
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

// ---------------------------------------------------------------------------
// Layer coverage masks (forma_renderer_render_masks): plane k of a frame holds, per pixel, the
// coverage of order o = first_order + k as paint_layer computes it, times the clip mask where a
// clip applies to o. Amodal: every layer of the tile is walked, none is skipped below an opaque
// one. The same warp scheme as the ID kernel (tickets, heavy lists first, lane = the painter's
// eight pixels), with entry_coverage, stage_group and skip_trivial_clips_ids reused as they are.
//
// Tiles without clip-ish entries: the entries are sorted by layer, so the walk bisects to the
// window's first entry and stops at its end; nothing outside the window is read. Tiles with
// clips walk bottom-up from their first entry with the painter's clip state after
// skip_trivial_clips (as in the ID kernel's clip tiles, without the skip below the first opaque
// layer). A clip below the window is only accumulated when its mask can still apply to a window
// entry (the clip state's last layer reaches the window); other entries below the window are
// skipped without reading their segments.
//
// Only tiles with window entries are stored, and each such entry stores its own plane: the zero
// fill before the kernel (zero_masks_kernel) gives every other pixel its 0.
// ---------------------------------------------------------------------------
struct MaskInputs {
    IdInputs t;  // tables, id_flags and ticket counter (t.ids, t.ids_stride and t.min_coverage unused)
    uint8_t* out;
    uint64_t stride, plane_stride;
    uint32_t first_order, n_orders;
    uint32_t height;  // rows of one frame
    uint32_t rows;    // stacks: tile rows per frame; 0: a single frame
    bool u8;
};

// compute_srgb's alpha encode (paint_math.cuh: to_byte) of a coverage in [0, 1].
__device__ __forceinline__ uint32_t mask_byte(float v) {
    const float scaled = fminf(fmaxf(v * 255.0f, 0.0f), 255.0f);
    return __float_as_uint(scaled + __uint_as_float(0x4B000000u)) & 0xFFu;
}

// The lane's eight values at `p` (its first pixel of plane row), n <= 8 of them inside the frame.
__device__ __forceinline__ void store_mask(uint8_t* p, const float cov[8], uint32_t n, bool u8, bool vec_ok) {
    if (u8) {
        uint32_t lo = 0, hi = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            lo |= mask_byte(cov[j]) << (8 * j);
            hi |= mask_byte(cov[4 + j]) << (8 * j);
        }
        if (vec_ok && n == 8u) {
            *reinterpret_cast<uint2*>(p) = make_uint2(lo, hi);
        } else {
#pragma unroll
            for (uint32_t j = 0; j < 8u; ++j)
                if (j < n) p[j] = (uint8_t)((j < 4u ? lo >> (8u * j) : hi >> (8u * (j - 4u))) & 0xFFu);
        }
        return;
    }
    float* f = reinterpret_cast<float*>(p);
    if (vec_ok && n == 8u) {
        reinterpret_cast<float4*>(f)[0] = make_float4(cov[0], cov[1], cov[2], cov[3]);
        reinterpret_cast<float4*>(f)[1] = make_float4(cov[4], cov[5], cov[6], cov[7]);
    } else {
#pragma unroll
        for (uint32_t j = 0; j < 8u; ++j)
            if (j < n) f[j] = cov[j];
    }
}

// ---------------------------------------------------------------------------
// Layer statistics (forma_renderer_render_stats): per frame and window order one
// forma_layer_stats record, reduced from the walks of the mask kernel (amodal: area, pixels, box)
// and of the ID kernel (visible, visible_box) instead of stored planes. Each (tile, entry) of the
// amodal walk and each distinct window ID of a tile in the visible walk is one warp reduction and
// one set of integer atomics on its record, so the result is exact and does not depend on the
// order of the atomics. Boxes start as {~0, ~0, 0, 0} (min / max sentinels) and
// fix_stats_kernel turns the box of an empty set into {0, 0, 0, 0} at the end.
// ---------------------------------------------------------------------------
struct StatsOut {
    forma_layer_stats* rec;  // n_frames x n_orders records
    uint32_t first_order, n_orders;
    uint32_t height;  // rows of one frame
    uint32_t rows;    // stacks: tile rows per frame; 0: a single frame
    float min_cov;
};

// Widens `box` (x0, y0, x1, y1) to hold [x0, x1) x [y0, y1). Bounds only move outwards, so a
// relaxed read that finds one already as wide skips its atomic (a stale read only costs an atomic).
__device__ __forceinline__ void widen_box(uint32_t* box, uint32_t x0, uint32_t y0, uint32_t x1, uint32_t y1) {
    const uint2 lo = __ldcg(reinterpret_cast<const uint2*>(box)), hi = __ldcg(reinterpret_cast<const uint2*>(box + 2));
    if (x0 < lo.x) atomicMin(box, x0);
    if (y0 < lo.y) atomicMin(box + 1, y0);
    if (x1 > hi.x) atomicMax(box + 2, x1);
    if (y1 > hi.y) atomicMax(box + 3, y1);
}

// The amodal statistics of one (tile, entry): the lane's eight values cov (n_px of them in the
// frame, from column x0 of frame row py) into `r`. `full`: a kFlagFull entry that no clip mask
// scales, 1 on the tile's whole in-frame rectangle [tx0, tx0 + tw) x [ty0, ty0 + th), taken without
// a reduction. Called by the whole warp.
__device__ __forceinline__ void add_amodal(forma_layer_stats* r, const float cov[8], bool full, uint32_t n_px, uint32_t x0,
                                           uint32_t py, uint32_t tx0, uint32_t tw, uint32_t ty0, uint32_t th, float min_cov,
                                           uint32_t lane) {
    if (full) {
        if (lane == 0 && tw && th) {
            atomicAdd(reinterpret_cast<unsigned long long*>(&r->area), (unsigned long long)(tw * th) << 18);
            atomicAdd(&r->pixels, tw * th);
            widen_box(r->box, tx0, ty0, tx0 + tw, ty0 + th);
        }
        return;
    }
    uint32_t units = 0, cnt = 0, xl = ~0u, xh = 0;
#pragma unroll
    for (uint32_t j = 0; j < 8u; ++j) {
        if (j >= n_px) continue;
        units += (uint32_t)(cov[j] * 262144.0f);  // exact: v x 2^18 is an integer <= 2^18
        if (cov[j] > min_cov) {
            ++cnt;
            xl = min(xl, x0 + j);
            xh = x0 + j + 1u;
        }
    }
    units = __reduce_add_sync(kFullMask, units);  // <= 256 x 2^18
    const uint32_t n = __reduce_add_sync(kFullMask, cnt);
    if (n) {
        xl = __reduce_min_sync(kFullMask, xl);
        xh = __reduce_max_sync(kFullMask, xh);
    }
    const uint32_t yl = n ? __reduce_min_sync(kFullMask, cnt ? py : ~0u) : 0u;
    const uint32_t yh = n ? __reduce_max_sync(kFullMask, cnt ? py + 1u : 0u) : 0u;
    if (lane == 0) {
        if (units) atomicAdd(reinterpret_cast<unsigned long long*>(&r->area), (unsigned long long)units);
        if (n) {
            atomicAdd(&r->pixels, n);
            widen_box(r->box, xl, yl, xh, yh);
        }
    }
}

// The visible statistics of one tile (tile row ty, column tx) from the ID walk's eight IDs `out` of
// each lane (tile row `row`, half hx): one reduction per distinct window ID of the tile. `frames`: a batch, whose IDs carry
// the frame's order base. Called by the whole warp.
__device__ __forceinline__ void add_visible(const PaintScene& S, const StatsOut& so, const uint32_t* out, uint32_t ty, uint32_t tx,
                                            uint32_t row, uint32_t hx, uint32_t lane, const BatchFrame* __restrict__ frames) {
    const uint32_t frame = so.rows ? ty / so.rows : 0u, fty = so.rows ? ty - frame * so.rows : ty;
    const uint32_t lo_w = (frames ? frames[frame].order_base : 0u) + so.first_order;
    const uint32_t py = fty * 16u + row, x0 = tx * 16u + hx * 8u;
    const uint32_t n_px = py < so.height && x0 < S.width ? min(8u, S.width - x0) : 0u;
    uint32_t k[8], pend = 0;  // window indices; the lane's pixels not reduced yet
#pragma unroll
    for (uint32_t j = 0; j < 8u; ++j) {
        k[j] = out[j] - lo_w;  // (FORMA_ID_NONE and orders outside the window land at >= n_orders)
        if (j < n_px && k[j] < so.n_orders) pend |= 1u << j;
    }
    forma_layer_stats* rec = so.rec + (size_t)frame * so.n_orders;
    for (;;) {
        const uint32_t any = __ballot_sync(kFullMask, pend != 0u);
        if (!any) break;
        uint32_t mine = 0, seen = 0;
#pragma unroll
        for (uint32_t j = 0; j < 8u; ++j)
            if (((pend >> j) & 1u) && !seen) {
                mine = k[j];
                seen = 1;
            }
        const uint32_t id = __shfl_sync(kFullMask, mine, __ffs(any) - 1);
        uint32_t cnt = 0, xl = ~0u, xh = 0;
#pragma unroll
        for (uint32_t j = 0; j < 8u; ++j)
            if (((pend >> j) & 1u) && k[j] == id) {
                ++cnt;
                xl = min(xl, x0 + j);
                xh = x0 + j + 1u;
                pend &= ~(1u << j);
            }
        const uint32_t n = __reduce_add_sync(kFullMask, cnt);
        xl = __reduce_min_sync(kFullMask, xl);
        xh = __reduce_max_sync(kFullMask, xh);
        const uint32_t yl = __reduce_min_sync(kFullMask, cnt ? py : ~0u), yh = __reduce_max_sync(kFullMask, cnt ? py + 1u : 0u);
        if (lane == 0) {
            atomicAdd(&rec[id].visible, n);
            widen_box(rec[id].visible_box, xl, yl, xh, yh);
        }
    }
}

// kStats: the amodal statistics (add_amodal into so) in place of the planes; `in` then only
// gives the tables and the window.
template <bool kBatch, bool kStats = false>
__device__ __forceinline__ void paint_masks_body(const PaintScene& S, const MaskInputs& in, uint32_t n_tiles,
                                                 const BatchFrame* __restrict__ frames, const StatsOut& so = StatsOut{}) {
    __shared__ __align__(16) IdWarpSmem s_warp[kIdWarpsPerBlock];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    IdWarpSmem& W = s_warp[warp];
    const IdInputs& T = in.t;
    const uint32_t ntx = S.tx_hi - S.tx_lo;
    const uint32_t row = lane >> 1, hx = lane & 1u;
    const uint32_t bpp = in.u8 ? 1u : 4u;
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(in.out) | (uintptr_t)in.stride | (uintptr_t)in.plane_stride) &
                         (in.u8 ? 7u : 15u)) == 0u;
#pragma unroll
    for (int k = 0; k < 8; ++k) W.cells[k * 32 + lane] = 0u;
    __syncwarp();

    uint32_t hcount[kHeavyClasses], H = 0;
#pragma unroll
    for (int c = 0; c < kHeavyClasses; ++c) {
        hcount[c] = T.heavy ? T.heavy_count[c] : 0u;
        H += hcount[c];
    }
    const uint32_t n_tickets = H + n_tiles;
    for (;;) {
        uint32_t ticket = 0;
        if (lane == 0) ticket = atomicAdd(T.tile_counter, 1u);
        ticket = __shfl_sync(kFullMask, ticket, 0);
        if (ticket >= n_tickets) break;
        uint32_t tid;
        if (ticket < H) {  // the heavy lists, largest class first (as in the ID kernel)
            uint32_t t = ticket;
            int c = kHeavyClasses - 1;
#pragma unroll
            for (int q = kHeavyClasses - 1; q > 0; --q)
                if (c == q && t >= hcount[q]) {
                    t -= hcount[q];
                    c = q - 1;
                }
            tid = T.heavy[(size_t)c * T.n_tiles_total + t];
            const uint32_t ty = tid / S.tiles_x, tx = tid - ty * S.tiles_x;
            if (ty < S.ty_lo || ty >= S.ty_hi || tx < S.tx_lo || tx >= S.tx_hi) continue;
        } else {
            const uint32_t lin = ticket - H;
            tid = (S.ty_lo + lin / ntx) * S.tiles_x + S.tx_lo + lin % ntx;
        }
        const uint2 range = T.tile_range[tid];
        const uint32_t b = range.x, e = range.y;
        if (ticket >= H && T.heavy && e - b >= kHeavyMin) continue;  // done from its list
        if (e == b) continue;
        const uint32_t ty = tid / S.tiles_x, tx = tid - ty * S.tiles_x;
        const uint32_t frame = in.rows ? ty / in.rows : 0u, fty = in.rows ? ty - frame * in.rows : ty;
        const uint32_t base = kBatch ? frames[frame].order_base : 0u;
        const uint32_t lo_w = base + in.first_order, hi_w = lo_w + in.n_orders;  // the window in the entries' layer space
        const uint32_t py = fty * 16u + row, x0 = tx * 16u + hx * 8u;
        const bool inside = py < in.height && x0 < S.width;
        const uint32_t n_px = inside ? min(8u, S.width - x0) : 0u;
        uint8_t* const px = in.out + ((size_t)frame * in.n_orders) * in.plane_stride + (size_t)py * in.stride + (size_t)x0 * bpp;
        float cov[8];
        bool full = false;  // cov is a kFlagFull entry's 1 everywhere (kStats)
        auto put = [&](uint32_t layer) {
            if constexpr (kStats) {
                const uint32_t tx0 = tx * 16u, ty0 = fty * 16u;
                const uint32_t tw = tx0 < S.width ? min(16u, S.width - tx0) : 0u, th = ty0 < in.height ? min(16u, in.height - ty0) : 0u;
                add_amodal(so.rec + (size_t)frame * in.n_orders + (layer - lo_w), cov, full, n_px, x0, py, tx0, tw, ty0, th,
                           so.min_cov, lane);
            } else if (inside) {
                store_mask(px + (size_t)(layer - lo_w) * in.plane_stride, cov, n_px, in.u8, vec_ok);
            }
        };
        auto coverage = [&](const EntryRec& h) {
            full = (h.pad & kFlagFull) != 0u;
            if (h.pad & kFlagFull) {  // no segments, a full carried cover: coverage 1 without reading anything
#pragma unroll
                for (int j = 0; j < 8; ++j) cov[j] = 1.0f;
            } else {
                entry_coverage(W, h, T.segs, lane, cov);
            }
        };

        bool clip_tile = false;
        for (uint32_t p0 = b; p0 < e && !clip_tile; p0 += 32u) {
            const uint32_t p = p0 + lane;
            clip_tile = __any_sync(kFullMask, p < e && (T.recs[p].flags0 & kFlagClipish) != 0u);
        }

        if (!clip_tile) {
            uint32_t lo = b, hi = e;  // the first entry of the window
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (T.recs[mid].layer < lo_w) lo = mid + 1u;
                else hi = mid;
            }
            bool done = false;
            for (uint32_t p0 = lo; p0 < e && !done; p0 += 32u) {
                const uint32_t cnt = min(32u, e - p0);
                stage_group(W, T, p0, cnt, false, lane);
                for (uint32_t k = 0; k < cnt; ++k) {
                    const EntryRec& h = W.hdr[k];
                    if (h.layer >= hi_w) {
                        done = true;
                        break;
                    }
                    if (h.pad & kFlagMaskedOut) continue;  // a layer without props
                    coverage(h);
                    put(h.layer);
                }
            }
        } else {
            if (lane == 0) skip_trivial_clips_ids(T.recs, T.id_flags, b, e);
            __syncwarp();
            bool clip_active = false, done = false;
            uint32_t clip_last = 0;
            for (uint32_t p0 = b; p0 < e && !done; p0 += 32u) {
                const uint32_t cnt = min(32u, e - p0);
                stage_group(W, T, p0, cnt, true, lane);
                for (uint32_t k = 0; k < cnt; ++k) {
                    const EntryRec& h = W.hdr[k];
                    const uint32_t flags = h.pad, layer = h.layer, meta = h.meta;
                    if (layer >= hi_w) {
                        done = true;
                        break;
                    }
                    const bool is_clip = ((meta >> 1) & 1u) != 0u, in_window = layer >= lo_w;
                    if (flags & kFlagMaskedOut) {
                        // Not painted, no clip state. A clip's plane is its own coverage all the
                        // same (a layer without props has meta 0: no clip).
                        if (is_clip && in_window) {
                            coverage(h);
                            put(layer);
                        }
                        continue;
                    }
                    if (clip_active && clip_last < layer) clip_active = false;  // mod.rs:302-306
                    if (is_clip) {  // clip_at, mod.rs:449-464
                        if (!clip_active) {
                            clip_active = true;
                            clip_last = layer + h.clip_layers;
                        }
                        const bool mask_used = clip_last >= lo_w;
                        if (!mask_used && !in_window) continue;
                        coverage(h);
                        if (mask_used) {
                            float4* m4 = reinterpret_cast<float4*>(W.clip);
                            m4[2u * lane] = make_float4(cov[0], cov[1], cov[2], cov[3]);
                            m4[2u * lane + 1u] = make_float4(cov[4], cov[5], cov[6], cov[7]);
                            __syncwarp();
                        }
                        if (in_window) put(layer);
                        continue;
                    }
                    if (!in_window) continue;
                    const bool apply_clip = ((meta >> 2) & 1u) && !(flags & kFlagSkipClip);
                    if (apply_clip && !clip_active) continue;  // mod.rs:317-323: never painted, 0
                    coverage(h);
                    if (apply_clip) {
                        const float4* m4 = reinterpret_cast<const float4*>(W.clip);
                        const float4 m0 = m4[2u * lane], m1 = m4[2u * lane + 1u];
                        const float m[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
#pragma unroll
                        for (int j = 0; j < 8; ++j) cov[j] = __fmul_rn(cov[j], m[j]);
                        full = false;
                    }
                    put(layer);
                }
            }
        }
    }
}

__global__ void __launch_bounds__(kIdWarpsPerBlock * 32) paint_masks_kernel(PaintScene S, MaskInputs in, uint32_t n_tiles) {
    paint_masks_body<false>(S, in, n_tiles, nullptr);
}
// S stacks the frames of a batch; frame c's entries carry frames[c].order_base + order, and its
// planes hold the frame's own orders.
__global__ void __launch_bounds__(kIdWarpsPerBlock * 32) paint_masks_stacked_kernel(PaintScene S, MaskInputs in, uint32_t n_tiles,
                                                                                    const BatchFrame* __restrict__ frames) {
    paint_masks_body<true>(S, in, n_tiles, frames);
}

// Zeroes `row_bytes` bytes from byte x0 of rows [y0, y0 + n_rows) of n_planes planes: one warp per
// row, 16-byte stores between an unaligned head and tail.
constexpr int kZeroWarps = 8;
__global__ void __launch_bounds__(kZeroWarps * 32) zero_masks_kernel(uint8_t* out, uint64_t stride, uint64_t plane_stride,
                                                                     uint32_t n_planes, uint32_t y0, uint32_t n_rows, uint64_t x0,
                                                                     uint64_t row_bytes) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t total = (uint64_t)n_planes * n_rows;
    for (uint64_t r = (uint64_t)blockIdx.x * kZeroWarps + (threadIdx.x >> 5); r < total; r += (uint64_t)gridDim.x * kZeroWarps) {
        const uint64_t plane = r / n_rows, y = y0 + r % n_rows;
        uint8_t* p = out + plane * plane_stride + y * stride + x0;
        const uint64_t head = min(row_bytes, (uint64_t)((16u - (reinterpret_cast<uintptr_t>(p) & 15u)) & 15u));
        const uint64_t n_vec = (row_bytes - head) / 16u, tail = head + 16u * n_vec;
        if (lane < head) p[lane] = 0;
        uint4* q = reinterpret_cast<uint4*>(p + head);
        for (uint64_t i = lane; i < n_vec; i += 32u) q[i] = make_uint4(0u, 0u, 0u, 0u);
        if (tail + lane < row_bytes) p[tail + lane] = 0;
    }
}

uint32_t launch_paint_masks(const PaintScene& S, const uint64_t* segs, const EntryRec* recs, const uint2* tile_range,
                            const uint32_t* heavy, const uint32_t* heavy_count, uint8_t* id_flags, const MaskFrame& m,
                            uint32_t* tile_counter, cudaStream_t st, uint32_t rows, const BatchFrame* frames) {
    if (S.tx_hi <= S.tx_lo || S.ty_hi <= S.ty_lo) return 0;
    const uint32_t bpp = m.format == FORMA_MASK_U8 ? 1u : 4u;
    // The written rectangle: a stack's frames whole, a single frame's tile rectangle clipped to it.
    const uint32_t y0 = rows ? 0u : S.ty_lo * 16u, y1 = rows ? m.height : min(S.ty_hi * 16u, S.height);
    const uint32_t x0 = rows ? 0u : S.tx_lo * 16u, x1 = rows ? S.width : min(S.tx_hi * 16u, S.width);
    const uint64_t n_rows = (uint64_t)m.n_frames * m.n_orders * (y1 - y0);
    const uint32_t zero_ctas = (uint32_t)std::min<uint64_t>((n_rows + kZeroWarps - 1) / kZeroWarps, 8u * (uint64_t)device_sm_count());
    zero_masks_kernel<<<zero_ctas, kZeroWarps * 32, 0, st>>>(m.ptr, m.stride, m.plane_stride, m.n_frames * m.n_orders, y0, y1 - y0,
                                                             (uint64_t)x0 * bpp, (uint64_t)(x1 - x0) * bpp);
    const uint32_t n_tiles = (S.tx_hi - S.tx_lo) * (S.ty_hi - S.ty_lo);
    cudaMemsetAsync(tile_counter, 0, sizeof(uint32_t), st);
    MaskInputs in{IdInputs{segs, recs, tile_range, heavy, heavy_count, S.tiles_x * S.tiles_y, id_flags, nullptr, 0, 0.0f, tile_counter},
                  m.ptr, m.stride, m.plane_stride, m.first_order, m.n_orders, m.height, rows, m.format == FORMA_MASK_U8};
    static int blocks_per_sm[2][kMaxDevices] = {{0}};
    const uint32_t need = (n_tiles + kIdWarpsPerBlock - 1) / kIdWarpsPerBlock;
    if (frames) {
        const uint32_t want = id_grid_limit(paint_masks_stacked_kernel, blocks_per_sm[1]);
        paint_masks_stacked_kernel<<<min(want, need), kIdWarpsPerBlock * 32, 0, st>>>(S, in, n_tiles, frames);
    } else {
        const uint32_t want = id_grid_limit(paint_masks_kernel, blocks_per_sm[0]);
        paint_masks_kernel<<<min(want, need), kIdWarpsPerBlock * 32, 0, st>>>(S, in, n_tiles);
    }
    return 2;
}

// The statistics kernels (see add_amodal / add_visible above): the amodal walk of the mask kernel
// and the visible walk of the ID kernel, each single-frame / views and batch.
__global__ void __launch_bounds__(kIdWarpsPerBlock * 32) stats_amodal_kernel(PaintScene S, MaskInputs in, uint32_t n_tiles,
                                                                             StatsOut so) {
    paint_masks_body<false, true>(S, in, n_tiles, nullptr, so);
}
__global__ void __launch_bounds__(kIdWarpsPerBlock * 32) stats_amodal_stacked_kernel(PaintScene S, MaskInputs in, uint32_t n_tiles,
                                                                                     StatsOut so,
                                                                                     const BatchFrame* __restrict__ frames) {
    paint_masks_body<true, true>(S, in, n_tiles, frames, so);
}
__global__ void __launch_bounds__(kIdWarpsPerBlock * 32) stats_visible_kernel(PaintScene S, IdInputs in, uint32_t n_tiles,
                                                                              StatsOut so) {
#define FORMA_IDS_SINK(out, ty, tx, row, hx) add_visible(S, so, out, ty, tx, row, hx, lane, nullptr)
#include "paint_ids_body.cuh"
#undef FORMA_IDS_SINK
}
__global__ void __launch_bounds__(kIdWarpsPerBlock * 32) stats_visible_stacked_kernel(PaintScene S, IdInputs in, uint32_t n_tiles,
                                                                                      StatsOut so,
                                                                                      const BatchFrame* __restrict__ frames) {
#define FORMA_IDS_SINK(out, ty, tx, row, hx) add_visible(S, so, out, ty, tx, row, hx, lane, frames)
#include "paint_ids_body.cuh"
#undef FORMA_IDS_SINK
}

// Every record to 0 with the boxes' min / max sentinels {~0, ~0, 0, 0}.
__global__ void init_stats_kernel(forma_layer_stats* rec, uint64_t n) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        uint2* r = reinterpret_cast<uint2*>(rec + i);  // 8-byte aligned (check_stats)
        r[0] = make_uint2(0u, 0u);             // area
        r[1] = make_uint2(0u, 0u);             // pixels, visible
        r[2] = make_uint2(~0u, ~0u);           // box x0, y0
        r[3] = make_uint2(0u, 0u);             // box x1, y1
        r[4] = make_uint2(~0u, ~0u);           // visible_box x0, y0
        r[5] = make_uint2(0u, 0u);             // visible_box x1, y1
    }
}
// The box of an empty set to {0, 0, 0, 0}.
__global__ void fix_stats_kernel(forma_layer_stats* rec, uint64_t n) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        forma_layer_stats& r = rec[i];
        if (r.pixels == 0u) r.box[0] = r.box[1] = 0u;
        if (r.visible == 0u) r.visible_box[0] = r.visible_box[1] = 0u;
    }
}

uint32_t launch_paint_stats(const PaintScene& S, const uint64_t* segs, const EntryRec* recs, const uint2* tile_range,
                            const uint32_t* heavy, const uint32_t* heavy_count, uint8_t* id_flags, const StatsFrame& f,
                            uint32_t* tile_counter, cudaStream_t st, uint32_t rows, const BatchFrame* frames) {
    const uint64_t n_rec = (uint64_t)f.n_frames * f.n_orders;
    const uint32_t rec_ctas = (uint32_t)std::min<uint64_t>((n_rec + 255u) / 256u, 8u * (uint64_t)device_sm_count());
    init_stats_kernel<<<rec_ctas, 256, 0, st>>>(f.ptr, n_rec);
    uint32_t launches = 2;
    if (S.tx_hi > S.tx_lo && S.ty_hi > S.ty_lo) {
        const uint32_t n_tiles = (S.tx_hi - S.tx_lo) * (S.ty_hi - S.ty_lo);
        const IdInputs t{segs, recs, tile_range, heavy, heavy_count, S.tiles_x * S.tiles_y, id_flags, nullptr, 0, f.min_coverage,
                         tile_counter};
        const MaskInputs in{t, nullptr, 0, 0, f.first_order, f.n_orders, f.height, rows, false};
        const StatsOut so{f.ptr, f.first_order, f.n_orders, f.height, rows, f.min_coverage};
        static int blocks_per_sm[4][kMaxDevices] = {{0}};
        const uint32_t need = (n_tiles + kIdWarpsPerBlock - 1) / kIdWarpsPerBlock;
        cudaMemsetAsync(tile_counter, 0, sizeof(uint32_t), st);
        if (frames) {
            const uint32_t want = id_grid_limit(stats_amodal_stacked_kernel, blocks_per_sm[1]);
            stats_amodal_stacked_kernel<<<min(want, need), kIdWarpsPerBlock * 32, 0, st>>>(S, in, n_tiles, so, frames);
        } else {
            const uint32_t want = id_grid_limit(stats_amodal_kernel, blocks_per_sm[0]);
            stats_amodal_kernel<<<min(want, need), kIdWarpsPerBlock * 32, 0, st>>>(S, in, n_tiles, so);
        }
        cudaMemsetAsync(tile_counter, 0, sizeof(uint32_t), st);
        if (frames) {
            const uint32_t want = id_grid_limit(stats_visible_stacked_kernel, blocks_per_sm[3]);
            stats_visible_stacked_kernel<<<min(want, need), kIdWarpsPerBlock * 32, 0, st>>>(S, t, n_tiles, so, frames);
        } else {
            const uint32_t want = id_grid_limit(stats_visible_kernel, blocks_per_sm[2]);
            stats_visible_kernel<<<min(want, need), kIdWarpsPerBlock * 32, 0, st>>>(S, t, n_tiles, so);
        }
        launches += 2;
    }
    fix_stats_kernel<<<rec_ctas, 256, 0, st>>>(f.ptr, n_rec);
    return launches;
}

}  // namespace forma
