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

__global__ void __launch_bounds__(kIdWarpsPerBlock * 32) paint_ids_kernel(PaintScene S, IdInputs in, uint32_t n_tiles) {
    __shared__ __align__(16) IdWarpSmem s_warp[kIdWarpsPerBlock];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    IdWarpSmem& W = s_warp[warp];
    const uint32_t ntx = S.tx_hi - S.tx_lo;
    const uint32_t row = lane >> 1, hx = lane & 1u;
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(in.ids) | (uintptr_t)in.ids_stride) & 15u) == 0u;
    const float min_cov = in.min_coverage;
#pragma unroll
    for (int k = 0; k < 8; ++k) W.cells[k * 32 + lane] = 0u;
    __syncwarp();

    uint32_t hcount[kHeavyClasses], H = 0;
#pragma unroll
    for (int c = 0; c < kHeavyClasses; ++c) {
        hcount[c] = in.heavy ? in.heavy_count[c] : 0u;
        H += hcount[c];
    }
    const uint32_t n_tickets = H + n_tiles;
    for (;;) {
        // Ticket -> tile, as in paint_kernel: tickets [0, H) walk the heavy lists (largest class
        // first), the rest the tile rectangle row-major, skipping the listed tiles.
        uint32_t ticket = 0;
        if (lane == 0) ticket = atomicAdd(in.tile_counter, 1u);
        ticket = __shfl_sync(kFullMask, ticket, 0);
        if (ticket >= n_tickets) break;
        uint32_t tid;
        if (ticket < H) {
            uint32_t t = ticket;
            int c = kHeavyClasses - 1;
#pragma unroll
            for (int q = kHeavyClasses - 1; q > 0; --q)
                if (c == q && t >= hcount[q]) {
                    t -= hcount[q];
                    c = q - 1;
                }
            tid = in.heavy[(size_t)c * in.n_tiles_total + t];
            const uint32_t ty = tid / S.tiles_x, tx = tid - ty * S.tiles_x;
            if (ty < S.ty_lo || ty >= S.ty_hi || tx < S.tx_lo || tx >= S.tx_hi) continue;
        } else {
            const uint32_t lin = ticket - H;
            tid = (S.ty_lo + lin / ntx) * S.tiles_x + S.tx_lo + lin % ntx;
        }
        const uint2 range = in.tile_range[tid];
        const uint32_t b = range.x, e = range.y;
        if (ticket >= H && in.heavy && e - b >= kHeavyMin) continue;  // done from its list
        const uint32_t ty = tid / S.tiles_x, tx = tid - ty * S.tiles_x;

        bool clip_tile = false;
        for (uint32_t p0 = b; p0 < e && !clip_tile; p0 += 32u) {
            const uint32_t p = p0 + lane;
            clip_tile = __any_sync(kFullMask, p < e && (in.recs[p].flags0 & kFlagClipish) != 0u);
        }

        uint32_t* out = W.ids + 8u * lane;  // this lane's eight pixels
#pragma unroll
        for (int j = 0; j < 8; ++j) out[j] = FORMA_ID_NONE;
        float cov[8];
        if (!clip_tile) {
            uint32_t open = 0xFFu;  // this lane's pixels without a hit yet
            bool done = e == b;
            for (uint32_t hi = e; hi > b && !done;) {
                const uint32_t lo = hi - b >= 32u ? hi - 32u : b;
                stage_group(W, in, lo, hi - lo, false, lane);
                for (uint32_t k = hi - lo; k-- > 0u;) {
                    const EntryRec& h = W.hdr[k];
                    const uint32_t flags = h.pad;
                    if (flags & kFlagMaskedOut) continue;
                    if (flags & kFlagFull) {  // an unclipped Draw entry of coverage 1 everywhere
#pragma unroll
                        for (int j = 0; j < 8; ++j)
                            if ((open >> j) & 1u) out[j] = h.layer;
                        done = true;
                        break;
                    }
                    entry_coverage(W, h, in.segs, lane, cov);
#pragma unroll
                    for (int j = 0; j < 8; ++j)
                        if (((open >> j) & 1u) && cov[j] > min_cov) {
                            out[j] = h.layer;
                            open &= ~(1u << j);
                        }
                    if (__all_sync(kFullMask, open == 0u)) {
                        done = true;
                        break;
                    }
                }
                hi = lo;
            }
        } else {
            if (lane == 0) skip_trivial_clips_ids(in.recs, in.id_flags, b, e);
            __syncwarp();
            // The painter's first layer (skip_fully_covered_layers): the top-most visible full,
            // unclipped, opaque entry.
            uint32_t first = b;
            for (uint32_t hi = e; hi > b;) {
                const uint32_t lo = hi - b >= 32u ? hi - 32u : b;
                bool cand = false;
                if (lo + lane < hi) {
                    const uint32_t f = in.id_flags[lo + lane];
                    const bool clipped = (f & kFlagClippedDraw) && !(f & kFlagSkipClip);
                    cand = !(f & kFlagMaskedOut) && !clipped && (f & kFlagFull) && (f & kFlagOpaque);
                }
                const uint32_t m = __ballot_sync(kFullMask, cand);
                if (m) {
                    first = lo + 31u - (uint32_t)__clz((int)m);
                    break;
                }
                hi = lo;
            }
            bool clip_active = false;
            uint32_t clip_last = 0;
            for (uint32_t p0 = first; p0 < e; p0 += 32u) {
                const uint32_t cnt = min(32u, e - p0);
                stage_group(W, in, p0, cnt, true, lane);
                for (uint32_t k = 0; k < cnt; ++k) {
                    const EntryRec& h = W.hdr[k];
                    const uint32_t flags = h.pad;
                    if (flags & kFlagMaskedOut) continue;
                    const uint32_t layer = h.layer, meta = h.meta;
                    if (clip_active && clip_last < layer) clip_active = false;  // mod.rs:302-306
                    const bool is_clip = ((meta >> 1) & 1u) != 0u;
                    const bool apply_clip = !is_clip && ((meta >> 2) & 1u) && !(flags & kFlagSkipClip);
                    if (!is_clip && !apply_clip && (flags & kFlagFull)) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) out[j] = layer;
                        continue;
                    }
                    if (apply_clip && !clip_active) continue;  // mod.rs:317-323
                    entry_coverage(W, h, in.segs, lane, cov);
                    if (is_clip) {  // clip_at, mod.rs:449-464
                        if (!clip_active) {
                            clip_active = true;
                            clip_last = layer + h.clip_layers;
                        }
                        float4* m4 = reinterpret_cast<float4*>(W.clip);
                        m4[2u * lane] = make_float4(cov[0], cov[1], cov[2], cov[3]);
                        m4[2u * lane + 1u] = make_float4(cov[4], cov[5], cov[6], cov[7]);
                        __syncwarp();
                        continue;
                    }
                    if (apply_clip) {
                        const float4* m4 = reinterpret_cast<const float4*>(W.clip);
                        const float4 m0 = m4[2u * lane], m1 = m4[2u * lane + 1u];
                        const float m[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
#pragma unroll
                        for (int j = 0; j < 8; ++j) cov[j] = __fmul_rn(cov[j], m[j]);
                    }
#pragma unroll
                    for (int j = 0; j < 8; ++j)
                        if (cov[j] > min_cov) out[j] = layer;
                }
            }
        }

        const uint32_t py = ty * 16u + row, x0 = tx * 16u + hx * 8u;
        if (py < S.height && x0 < S.width) {
            uint32_t* rowp = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(in.ids) + (size_t)py * in.ids_stride) + x0;
            if (vec_ok && x0 + 8u <= S.width) {
                reinterpret_cast<uint4*>(rowp)[0] = reinterpret_cast<const uint4*>(out)[0];
                reinterpret_cast<uint4*>(rowp)[1] = reinterpret_cast<const uint4*>(out)[1];
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    if (x0 + (uint32_t)j < S.width) rowp[j] = out[j];
            }
        }
    }
}

void launch_paint_ids(const PaintScene& S, const uint64_t* segs, const EntryRec* recs, const uint2* tile_range,
                      const uint32_t* heavy, const uint32_t* heavy_count, uint8_t* id_flags, uint32_t* ids, size_t ids_stride,
                      float min_coverage, uint32_t* tile_counter, cudaStream_t st) {
    if (S.tx_hi <= S.tx_lo || S.ty_hi <= S.ty_lo) return;
    const uint32_t n_tiles = (S.tx_hi - S.tx_lo) * (S.ty_hi - S.ty_lo);
    cudaMemsetAsync(tile_counter, 0, sizeof(uint32_t), st);
    IdInputs in{segs, recs, tile_range, heavy, heavy_count, S.tiles_x * S.tiles_y, id_flags, ids, ids_stride, min_coverage,
                tile_counter};
    static int blocks_per_sm[kMaxDevices] = {0};
    static std::mutex config_mu;
    int per_sm = 0;
    {
        std::lock_guard<std::mutex> lk(config_mu);
        int& slot = blocks_per_sm[current_device_index()];
        if (!slot) {
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&slot, paint_ids_kernel, kIdWarpsPerBlock * 32, 0);
            if (slot < 1) slot = 1;
        }
        per_sm = slot;
    }
    const uint32_t want = (uint32_t)(per_sm * device_sm_count());
    const uint32_t need = (n_tiles + kIdWarpsPerBlock - 1) / kIdWarpsPerBlock;
    paint_ids_kernel<<<min(want, need), kIdWarpsPerBlock * 32, 0, st>>>(S, in, n_tiles);
}

}  // namespace forma
