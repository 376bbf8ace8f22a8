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
// shifted space; paint_ids_stacked_kernel, the same walk, takes the frame's base off every ID it
// stores (one look-up per tile).
//
// The ID walk (ids_walk) and the amodal walk of the mask and statistics kernels (amodal_walk) hand
// each tile's result to a sink: the ID frame's store or add_visible, store_mask or add_amodal.
#include <algorithm>

#include "../../include/forma_b200.h"
#include "paint_common.cuh"

namespace forma {

// The tables every walk reads (TileTables, with the scratch and the ticket counter of the call).
struct IdTables {
    const uint64_t* segs;
    const EntryRec* recs;
    const uint2* tile_range;
    const uint32_t* heavy;        // kHeavyClasses lists of heavy tiles (linear ids), n_tiles_total each; may be null
    const uint32_t* heavy_count;
    uint32_t n_tiles_total;
    uint8_t* id_flags;            // per sorted entry: the flags after skip_trivial_clips (clip tiles only)
    uint32_t* tile_counter;
};
// The orders [first_order, first_order + n_orders) of the mask and statistics kernels, and the
// frames of a stack.
struct OrderWindow {
    uint32_t first_order, n_orders;
    uint32_t height;  // rows of one frame
    uint32_t rows;    // stacks: tile rows per frame; 0: a single frame
};
struct IdsOut {
    uint32_t* ids;  // the ID frame
    size_t stride;  // bytes
    float min_coverage;
};
struct MaskOut {
    uint8_t* ptr;
    uint64_t stride, plane_stride;
    bool u8;
};
struct StatsOut {
    forma_layer_stats* rec;  // n_frames x n_orders records
    float min_coverage;
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
__device__ __forceinline__ void stage_group(IdWarpSmem& W, const IdTables& T, uint32_t lo, uint32_t cnt, bool clip_tile,
                                            uint32_t lane) {
    __syncwarp();  // the previous group's records are no longer read
    if (lane < cnt) {
        const uint4* src = reinterpret_cast<const uint4*>(T.recs + lo + lane);
        uint4* dst = reinterpret_cast<uint4*>(&W.hdr[lane]);
        uint4 q3 = src[3];
        q3.w = clip_tile ? (uint32_t)T.id_flags[lo + lane] : q3.z;  // pad <- flags (q3.z = flags0)
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

// The warp's tiles, as paint_kernel takes them: tickets [0, H) walk the heavy lists (largest class
// first), the rest the tile rectangle row-major. Listed tiles outside the rectangle are skipped,
// and so are the rectangle's tiles that a list holds. Only H and the ticket count live in registers
// (a heavy ticket reads the list lengths again), and a skipped ticket returns to the walk's loop
// instead of looping here: with the lengths in registers or a loop here, the walk kernels spill
// more or keep fewer CTAs resident (-Xptxas -v).
struct TileTickets {
    const PaintScene& S;
    const IdTables& T;
    uint32_t lane, H = 0, n_tickets;

    __device__ __forceinline__ TileTickets(const PaintScene& S_, const IdTables& T_, uint32_t n_tiles, uint32_t lane_)
        : S(S_), T(T_), lane(lane_) {
#pragma unroll
        for (int c = 0; c < kHeavyClasses; ++c) H += T.heavy ? T.heavy_count[c] : 0u;
        n_tickets = H + n_tiles;
    }
    // Takes the next ticket: false once they have run out. Otherwise `tile` says whether it names a
    // tile to walk, with its linear id and entry range [b, e).
    __device__ __forceinline__ bool next(bool& tile, uint32_t& tid, uint32_t& b, uint32_t& e) {
        uint32_t ticket = 0;
        if (lane == 0) ticket = atomicAdd(T.tile_counter, 1u);
        ticket = __shfl_sync(kFullMask, ticket, 0);
        if (ticket >= n_tickets) return false;
        tile = false;
        if (ticket < H) {
            uint32_t t = ticket;
            int c = kHeavyClasses - 1;
#pragma unroll
            for (int q = kHeavyClasses - 1; q > 0; --q)
                if (c == q && t >= T.heavy_count[q]) {
                    t -= T.heavy_count[q];
                    c = q - 1;
                }
            tid = T.heavy[(size_t)c * T.n_tiles_total + t];
            const uint32_t ty = tid / S.tiles_x, tx = tid - ty * S.tiles_x;
            if (ty < S.ty_lo || ty >= S.ty_hi || tx < S.tx_lo || tx >= S.tx_hi) return true;
        } else {
            const uint32_t lin = ticket - H, ntx = S.tx_hi - S.tx_lo;
            tid = (S.ty_lo + lin / ntx) * S.tiles_x + S.tx_lo + lin % ntx;
        }
        const uint2 range = T.tile_range[tid];
        b = range.x;
        e = range.y;
        tile = !(ticket >= H && T.heavy && e - b >= kHeavyMin);  // done from its list
        return true;
    }
};

// Tile row ty of a stack of `rows` tile rows per frame (rows 0: a single frame): its frame, its
// row in the frame and the order base of the frame's entries (frames: a batch; otherwise 0).
struct FrameRow {
    uint32_t frame, fty, base;
};
__device__ __forceinline__ FrameRow frame_row(uint32_t ty, uint32_t rows, const BatchFrame* __restrict__ frames) {
    const uint32_t frame = rows ? ty / rows : 0u;
    return FrameRow{frame, ty - frame * rows, frames ? frames[frame].order_base : 0u};
}

// Whether entries [b, e) hold a clip-ish one (Func::Clip, or a clipped Draw). Called by the whole warp.
__device__ __forceinline__ bool clip_tile_of(const IdTables& T, uint32_t b, uint32_t e, uint32_t lane) {
    bool clip_tile = false;
    for (uint32_t p0 = b; p0 < e && !clip_tile; p0 += 32u) {
        const uint32_t p = p0 + lane;
        clip_tile = __any_sync(kFullMask, p < e && (T.recs[p].flags0 & kFlagClipish) != 0u);
    }
    return clip_tile;
}

// The ID walk of every tile: sink(ids, ty, tx, lane) gets the lane's eight IDs (shared memory) of
// the tile in row ty, column tx. IDs are the entries' layers, FORMA_ID_NONE where no layer hits.
template <class Sink>
__device__ __forceinline__ void ids_walk(const PaintScene& S, const IdTables& T, uint32_t n_tiles, float min_cov, Sink sink) {
    __shared__ __align__(16) IdWarpSmem s_warp[kIdWarpsPerBlock];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    IdWarpSmem& W = s_warp[warp];
#pragma unroll
    for (int k = 0; k < 8; ++k) W.cells[k * 32 + lane] = 0u;
    __syncwarp();

    TileTickets tickets(S, T, n_tiles, lane);
    uint32_t tid, b, e;
    for (bool tile; tickets.next(tile, tid, b, e);) {
        if (!tile) continue;
        const uint32_t ty = tid / S.tiles_x, tx = tid - ty * S.tiles_x;
        const bool clip_tile = clip_tile_of(T, b, e, lane);

        uint32_t* out = W.ids + 8u * lane;  // this lane's eight pixels
#pragma unroll
        for (int j = 0; j < 8; ++j) out[j] = FORMA_ID_NONE;
        float cov[8];
        if (!clip_tile) {
            uint32_t open = 0xFFu;  // this lane's pixels without a hit yet
            bool done = e == b;
            for (uint32_t hi = e; hi > b && !done;) {
                const uint32_t lo = hi - b >= 32u ? hi - 32u : b;
                stage_group(W, T, lo, hi - lo, false, lane);
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
                    entry_coverage(W, h, T.segs, lane, cov);
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
            if (lane == 0) skip_trivial_clips_ids(T.recs, T.id_flags, b, e);
            __syncwarp();
            // The painter's first layer (skip_fully_covered_layers): the top-most visible full,
            // unclipped, opaque entry.
            uint32_t first = b;
            for (uint32_t hi = e; hi > b;) {
                const uint32_t lo = hi - b >= 32u ? hi - 32u : b;
                bool cand = false;
                if (lo + lane < hi) {
                    const uint32_t f = T.id_flags[lo + lane];
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
                stage_group(W, T, p0, cnt, true, lane);
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
                    entry_coverage(W, h, T.segs, lane, cov);
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
        sink(out, ty, tx, lane);
    }
}

// The ID frame's sink: the lane's eight IDs of tile (tx, ty), less `base` (a batch frame's order
// base), into the frame.
__device__ __forceinline__ void store_ids(const PaintScene& S, const IdsOut& f, const uint32_t* out, uint32_t ty, uint32_t tx,
                                          uint32_t lane, uint32_t base) {
    const uint32_t py = ty * 16u + (lane >> 1), x0 = tx * 16u + (lane & 1u) * 8u;
    if (py >= S.height || x0 >= S.width) return;
    const uint4 a = reinterpret_cast<const uint4*>(out)[0], c = reinterpret_cast<const uint4*>(out)[1];
    uint32_t v[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
#pragma unroll
    for (int j = 0; j < 8; ++j)
        if (v[j] != FORMA_ID_NONE) v[j] -= base;
    uint32_t* rowp = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(f.ids) + (size_t)py * f.stride) + x0;
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(f.ids) | (uintptr_t)f.stride) & 15u) == 0u;
    if (vec_ok && x0 + 8u <= S.width) {
        reinterpret_cast<uint4*>(rowp)[0] = make_uint4(v[0], v[1], v[2], v[3]);
        reinterpret_cast<uint4*>(rowp)[1] = make_uint4(v[4], v[5], v[6], v[7]);
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (x0 + (uint32_t)j < S.width) rowp[j] = v[j];
    }
}

__global__ void __launch_bounds__(kIdWarpsPerBlock * 32) paint_ids_kernel(PaintScene S, IdTables T, IdsOut f, uint32_t n_tiles) {
    chain_begin();
    ids_walk(S, T, n_tiles, f.min_coverage,
             [&](const uint32_t* ids, uint32_t ty, uint32_t tx, uint32_t lane) { store_ids(S, f, ids, ty, tx, lane, 0u); });
}
// S stacks the frames of a batch, `rows` tile rows each; frame c's entries carry
// frames[c].order_base + order, and the IDs stored are the frame's own orders.
__global__ void __launch_bounds__(kIdWarpsPerBlock * 32) paint_ids_stacked_kernel(PaintScene S, IdTables T, IdsOut f, uint32_t n_tiles,
                                                                                  uint32_t rows, const BatchFrame* __restrict__ frames) {
    chain_begin();
    ids_walk(S, T, n_tiles, f.min_coverage, [&](const uint32_t* ids, uint32_t ty, uint32_t tx, uint32_t lane) {
        store_ids(S, f, ids, ty, tx, lane, frame_row(ty, rows, frames).base);
    });
}

static IdTables id_tables(const PaintScene& S, const TileTables& t, uint8_t* id_flags, uint32_t* tile_counter) {
    return IdTables{t.segs, t.recs, t.tile_range, t.heavy, t.heavy_count, S.tiles_x * S.tiles_y, id_flags, tile_counter};
}

void launch_paint_ids(const PaintScene& S, const TileTables& t, uint8_t* id_flags, uint32_t* ids, size_t ids_stride,
                      float min_coverage, uint32_t* tile_counter, cudaStream_t st, uint32_t rows, const BatchFrame* frames) {
    const void* kernel = frames ? (const void*)paint_ids_stacked_kernel : (const void*)paint_ids_kernel;
    const TileGrid g = tile_grid(S, kernel, kIdWarpsPerBlock, tile_counter, st);
    if (!g.n_tiles) return;
    const IdTables T = id_tables(S, t, id_flags, tile_counter);
    const IdsOut f{ids, ids_stride, min_coverage};
    if (frames) launch_chained(paint_ids_stacked_kernel, g.ctas, kIdWarpsPerBlock * 32, 0, st, S, T, f, g.n_tiles, rows, frames);
    else launch_chained(paint_ids_kernel, g.ctas, kIdWarpsPerBlock * 32, 0, st, S, T, f, g.n_tiles);
}

// ---------------------------------------------------------------------------
// Layer coverage masks (forma_renderer_render_masks): plane k of a frame holds, per pixel, the
// coverage of order o = first_order + k as paint_layer computes it, times the clip mask where a
// clip applies to o. Amodal: every layer of the tile is walked, none is skipped below an opaque
// one. The same warp scheme as the ID kernel (TileTickets, lane = the painter's eight pixels), with
// entry_coverage, stage_group and skip_trivial_clips_ids reused as they are.
//
// Tiles without clip-ish entries: the entries are sorted by layer, so the walk bisects to the
// window's first entry and stops at its end; nothing outside the window is read. Tiles with
// clips walk bottom-up from their first entry with the painter's clip state after
// skip_trivial_clips (as in the ID kernel's clip tiles, without the skip below the first opaque
// layer); the clip state restarts at every entry the ID kernel could take as its first (full,
// opaque, unclipped), so that each layer's mask is its walk in the painter's render of the
// composition cut off above it. A clip below the window is only accumulated when its mask can still apply to a window
// entry (the clip state's last layer reaches the window); other entries below the window are
// skipped without reading their segments.
//
// Only tiles with window entries are stored, and each such entry stores its own plane: the zero
// fill before the kernel (zero_masks_kernel) gives every other pixel its 0.
// ---------------------------------------------------------------------------

// A lane's part of a tile of the amodal walk: the tile's frame, its row fty in the frame and its
// column tx; the lane's frame row py, first column x0 and its n_px pixels inside the frame.
struct LaneTile {
    uint32_t frame, fty, tx, py, x0, n_px, lane;
};

// compute_srgb's alpha encode (paint_math.cuh: to_byte) of a coverage in [0, 1].
__device__ __forceinline__ uint32_t mask_byte(float v) {
    const float scaled = fminf(fmaxf(v * 255.0f, 0.0f), 255.0f);
    return __float_as_uint(scaled + __uint_as_float(0x4B000000u)) & 0xFFu;
}

// The mask planes' sink: the lane's eight values of window order k into plane k of the tile's frame.
__device__ __forceinline__ void store_mask(const OrderWindow& w, const MaskOut& m, const LaneTile& t, uint32_t k, const float cov[8]) {
    const uint32_t n = t.n_px;
    if (!n) return;
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(m.ptr) | (uintptr_t)m.stride | (uintptr_t)m.plane_stride) & (m.u8 ? 7u : 15u)) == 0u;
    uint8_t* p = m.ptr + ((size_t)t.frame * w.n_orders + k) * m.plane_stride + (size_t)t.py * m.stride + (size_t)t.x0 * (m.u8 ? 1u : 4u);
    if (m.u8) {
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

// Widens `box` (x0, y0, x1, y1) to hold [x0, x1) x [y0, y1). Bounds only move outwards, so a
// relaxed read that finds one already as wide skips its atomic (a stale read only costs an atomic).
__device__ __forceinline__ void widen_box(uint32_t* box, uint32_t x0, uint32_t y0, uint32_t x1, uint32_t y1) {
    const uint2 lo = __ldcg(reinterpret_cast<const uint2*>(box)), hi = __ldcg(reinterpret_cast<const uint2*>(box + 2));
    if (x0 < lo.x) atomicMin(box, x0);
    if (y0 < lo.y) atomicMin(box + 1, y0);
    if (x1 > hi.x) atomicMax(box + 2, x1);
    if (y1 > hi.y) atomicMax(box + 3, y1);
}

// The amodal statistics' sink: the lane's eight values cov of window order k into the record of
// (frame, k). `full`: a kFlagFull entry that no clip mask scales, 1 on the tile's whole in-frame
// rectangle, taken without a reduction. Called by the whole warp.
__device__ __forceinline__ void add_amodal(const PaintScene& S, const OrderWindow& w, const StatsOut& so, const LaneTile& t,
                                           uint32_t k, const float cov[8], bool full) {
    const uint32_t lane = t.lane;
    forma_layer_stats* r = so.rec + (size_t)t.frame * w.n_orders + k;
    if (full) {
        const uint32_t tx0 = t.tx * 16u, ty0 = t.fty * 16u;
        const uint32_t tw = tx0 < S.width ? min(16u, S.width - tx0) : 0u, th = ty0 < w.height ? min(16u, w.height - ty0) : 0u;
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
        if (j >= t.n_px) continue;
        units += (uint32_t)(cov[j] * 262144.0f);  // exact: v x 2^18 is an integer <= 2^18
        if (cov[j] > so.min_coverage) {
            ++cnt;
            xl = min(xl, t.x0 + j);
            xh = t.x0 + j + 1u;
        }
    }
    units = __reduce_add_sync(kFullMask, units);  // <= 256 x 2^18
    const uint32_t n = __reduce_add_sync(kFullMask, cnt);
    if (n) {
        xl = __reduce_min_sync(kFullMask, xl);
        xh = __reduce_max_sync(kFullMask, xh);
    }
    const uint32_t yl = n ? __reduce_min_sync(kFullMask, cnt ? t.py : ~0u) : 0u;
    const uint32_t yh = n ? __reduce_max_sync(kFullMask, cnt ? t.py + 1u : 0u) : 0u;
    if (lane == 0) {
        if (units) atomicAdd(reinterpret_cast<unsigned long long*>(&r->area), (unsigned long long)units);
        if (n) {
            atomicAdd(&r->pixels, n);
            widen_box(r->box, xl, yl, xh, yh);
        }
    }
}

// The visible statistics' sink: the tile's (row ty, column tx) IDs `out`, eight of each lane, one
// reduction per distinct window ID of the tile. `frames`: a batch, whose IDs carry the frame's
// order base. Called by the whole warp.
__device__ __forceinline__ void add_visible(const PaintScene& S, const OrderWindow& w, const StatsOut& so, const uint32_t* out,
                                            uint32_t ty, uint32_t tx, uint32_t lane, const BatchFrame* __restrict__ frames) {
    const FrameRow fr = frame_row(ty, w.rows, frames);
    const uint32_t lo_w = fr.base + w.first_order;
    const uint32_t py = fr.fty * 16u + (lane >> 1), x0 = tx * 16u + (lane & 1u) * 8u;
    const uint32_t n_px = py < w.height && x0 < S.width ? min(8u, S.width - x0) : 0u;
    uint32_t k[8], pend = 0;  // window indices; the lane's pixels not reduced yet
#pragma unroll
    for (uint32_t j = 0; j < 8u; ++j) {
        k[j] = out[j] - lo_w;  // (FORMA_ID_NONE and orders outside the window land at >= n_orders)
        if (j < n_px && k[j] < w.n_orders) pend |= 1u << j;
    }
    forma_layer_stats* rec = so.rec + (size_t)fr.frame * w.n_orders;
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

// The amodal walk of every tile with entries: sink(t, k, cov, full) gets the lane's eight values of
// each window entry of order first_order + k; `full`: cov is a kFlagFull entry's 1 everywhere.
// `frames`: a batch, whose entries carry the frame's order base.
template <class Sink>
__device__ __forceinline__ void amodal_walk(const PaintScene& S, const IdTables& T, const OrderWindow& w, uint32_t n_tiles,
                                            const BatchFrame* __restrict__ frames, Sink sink) {
    __shared__ __align__(16) IdWarpSmem s_warp[kIdWarpsPerBlock];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    IdWarpSmem& W = s_warp[warp];
    const uint32_t row = lane >> 1, hx = lane & 1u;
#pragma unroll
    for (int k = 0; k < 8; ++k) W.cells[k * 32 + lane] = 0u;
    __syncwarp();

    TileTickets tickets(S, T, n_tiles, lane);
    uint32_t tid, b, e;
    for (bool tile; tickets.next(tile, tid, b, e);) {
        if (!tile) continue;
        if (e == b) continue;
        const uint32_t ty = tid / S.tiles_x, tx = tid - ty * S.tiles_x;
        const FrameRow fr = frame_row(ty, w.rows, frames);
        const uint32_t lo_w = fr.base + w.first_order, hi_w = lo_w + w.n_orders;  // the window in the entries' layer space
        const uint32_t py = fr.fty * 16u + row, x0 = tx * 16u + hx * 8u;
        const LaneTile t{fr.frame, fr.fty, tx, py, x0, py < w.height && x0 < S.width ? min(8u, S.width - x0) : 0u, lane};
        float cov[8];
        bool full = false;
        auto put = [&](uint32_t layer) { sink(t, layer - lo_w, cov, full); };
        auto coverage = [&](const EntryRec& h) {
            full = (h.pad & kFlagFull) != 0u;
            if (h.pad & kFlagFull) {  // no segments, a full carried cover: coverage 1 without reading anything
#pragma unroll
                for (int j = 0; j < 8; ++j) cov[j] = 1.0f;
            } else {
                entry_coverage(W, h, T.segs, lane, cov);
            }
        };

        if (!clip_tile_of(T, b, e, lane)) {
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
                    // A layer the painter could start from (the ID kernel's `cand`): the walk of
                    // every layer from here up starts with no clip, as the painter's would.
                    const bool clipped = (flags & kFlagClippedDraw) && !(flags & kFlagSkipClip);
                    if (!clipped && (flags & kFlagFull) && (flags & kFlagOpaque)) clip_active = false;
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

__global__ void __launch_bounds__(kIdWarpsPerBlock * 32) paint_masks_kernel(PaintScene S, IdTables T, OrderWindow w, MaskOut m,
                                                                            uint32_t n_tiles) {
    chain_begin();
    amodal_walk(S, T, w, n_tiles, nullptr, [&](const LaneTile& t, uint32_t k, const float* cov, bool) { store_mask(w, m, t, k, cov); });
}
// S stacks the frames of a batch; frame c's entries carry frames[c].order_base + order, and its
// planes hold the frame's own orders.
__global__ void __launch_bounds__(kIdWarpsPerBlock * 32) paint_masks_stacked_kernel(PaintScene S, IdTables T, OrderWindow w, MaskOut m,
                                                                                    uint32_t n_tiles, const BatchFrame* __restrict__ frames) {
    chain_begin();
    amodal_walk(S, T, w, n_tiles, frames, [&](const LaneTile& t, uint32_t k, const float* cov, bool) { store_mask(w, m, t, k, cov); });
}

// Zeroes `row_bytes` bytes from byte x0 of rows [y0, y0 + n_rows) of n_planes planes: one warp per
// row, 16-byte stores between an unaligned head and tail.
constexpr int kZeroWarps = 8;
__global__ void __launch_bounds__(kZeroWarps * 32) zero_masks_kernel(uint8_t* out, uint64_t stride, uint64_t plane_stride,
                                                                     uint32_t n_planes, uint32_t y0, uint32_t n_rows, uint64_t x0,
                                                                     uint64_t row_bytes) {
    chain_begin();
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

uint32_t launch_paint_masks(const PaintScene& S, const TileTables& t, uint8_t* id_flags, const MaskFrame& m, uint32_t* tile_counter,
                            cudaStream_t st, uint32_t rows, const BatchFrame* frames) {
    const void* kernel = frames ? (const void*)paint_masks_stacked_kernel : (const void*)paint_masks_kernel;
    const TileGrid g = tile_grid(S, kernel, kIdWarpsPerBlock, tile_counter, st);
    if (!g.n_tiles) return 0;
    const uint32_t bpp = m.format == FORMA_MASK_U8 ? 1u : 4u;
    // The written rectangle: a stack's frames whole, a single frame's tile rectangle clipped to it.
    const uint32_t y0 = rows ? 0u : S.ty_lo * 16u, y1 = rows ? m.height : min(S.ty_hi * 16u, S.height);
    const uint32_t x0 = rows ? 0u : S.tx_lo * 16u, x1 = rows ? S.width : min(S.tx_hi * 16u, S.width);
    const uint64_t n_rows = (uint64_t)m.n_frames * m.n_orders * (y1 - y0);
    const uint32_t zero_ctas = (uint32_t)std::min<uint64_t>((n_rows + kZeroWarps - 1) / kZeroWarps, 8u * (uint64_t)device_sm_count());
    launch_chained(zero_masks_kernel, zero_ctas, kZeroWarps * 32, 0, st, m.ptr, m.stride, m.plane_stride, m.n_frames * m.n_orders, y0, y1 - y0,
                                                             (uint64_t)x0 * bpp, (uint64_t)(x1 - x0) * bpp);
    const IdTables T = id_tables(S, t, id_flags, tile_counter);
    const OrderWindow w{m.first_order, m.n_orders, m.height, rows};
    const MaskOut out{m.ptr, m.stride, m.plane_stride, m.format == FORMA_MASK_U8};
    if (frames) launch_chained(paint_masks_stacked_kernel, g.ctas, kIdWarpsPerBlock * 32, 0, st, S, T, w, out, g.n_tiles, frames);
    else launch_chained(paint_masks_kernel, g.ctas, kIdWarpsPerBlock * 32, 0, st, S, T, w, out, g.n_tiles);
    return 2;
}

// The statistics kernels (see add_amodal / add_visible above): the amodal walk of the mask kernel
// and the ID walk of the ID kernel, each single-frame / views and batch.
__global__ void __launch_bounds__(kIdWarpsPerBlock * 32) stats_amodal_kernel(PaintScene S, IdTables T, OrderWindow w, StatsOut so,
                                                                             uint32_t n_tiles) {
    chain_begin();
    amodal_walk(S, T, w, n_tiles, nullptr,
                [&](const LaneTile& t, uint32_t k, const float* cov, bool full) { add_amodal(S, w, so, t, k, cov, full); });
}
__global__ void __launch_bounds__(kIdWarpsPerBlock * 32) stats_amodal_stacked_kernel(PaintScene S, IdTables T, OrderWindow w,
                                                                                     StatsOut so, uint32_t n_tiles,
                                                                                     const BatchFrame* __restrict__ frames) {
    chain_begin();
    amodal_walk(S, T, w, n_tiles, frames,
                [&](const LaneTile& t, uint32_t k, const float* cov, bool full) { add_amodal(S, w, so, t, k, cov, full); });
}
__global__ void __launch_bounds__(kIdWarpsPerBlock * 32) stats_visible_kernel(PaintScene S, IdTables T, OrderWindow w, StatsOut so,
                                                                              uint32_t n_tiles) {
    chain_begin();
    ids_walk(S, T, n_tiles, so.min_coverage, [&](const uint32_t* ids, uint32_t ty, uint32_t tx, uint32_t lane) {
        add_visible(S, w, so, ids, ty, tx, lane, nullptr);
    });
}
__global__ void __launch_bounds__(kIdWarpsPerBlock * 32) stats_visible_stacked_kernel(PaintScene S, IdTables T, OrderWindow w,
                                                                                      StatsOut so, uint32_t n_tiles,
                                                                                      const BatchFrame* __restrict__ frames) {
    chain_begin();
    ids_walk(S, T, n_tiles, so.min_coverage, [&](const uint32_t* ids, uint32_t ty, uint32_t tx, uint32_t lane) {
        add_visible(S, w, so, ids, ty, tx, lane, frames);
    });
}

// Every record to 0 with the boxes' min / max sentinels {~0, ~0, 0, 0}.
__global__ void init_stats_kernel(forma_layer_stats* rec, uint64_t n) {
    chain_begin();
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
    chain_begin();
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        forma_layer_stats& r = rec[i];
        if (r.pixels == 0u) r.box[0] = r.box[1] = 0u;
        if (r.visible == 0u) r.visible_box[0] = r.visible_box[1] = 0u;
    }
}

uint32_t launch_paint_stats(const PaintScene& S, const TileTables& t, uint8_t* id_flags, const StatsFrame& f, uint32_t* tile_counter,
                            cudaStream_t st, uint32_t rows, const BatchFrame* frames) {
    const uint64_t n_rec = (uint64_t)f.n_frames * f.n_orders;
    const uint32_t rec_ctas = (uint32_t)std::min<uint64_t>((n_rec + 255u) / 256u, 8u * (uint64_t)device_sm_count());
    launch_chained(init_stats_kernel, rec_ctas, 256, 0, st, f.ptr, n_rec);
    uint32_t launches = 2;
    const IdTables T = id_tables(S, t, id_flags, tile_counter);
    const OrderWindow w{f.first_order, f.n_orders, f.height, rows};
    const StatsOut so{f.ptr, f.min_coverage};
    const uint32_t block = kIdWarpsPerBlock * 32;
    const void* amodal = frames ? (const void*)stats_amodal_stacked_kernel : (const void*)stats_amodal_kernel;
    const TileGrid g = tile_grid(S, amodal, kIdWarpsPerBlock, tile_counter, st);
    if (g.n_tiles) {
        if (frames) launch_chained(stats_amodal_stacked_kernel, g.ctas, block, 0, st, S, T, w, so, g.n_tiles, frames);
        else launch_chained(stats_amodal_kernel, g.ctas, block, 0, st, S, T, w, so, g.n_tiles);
        const void* visible = frames ? (const void*)stats_visible_stacked_kernel : (const void*)stats_visible_kernel;
        const TileGrid v = tile_grid(S, visible, kIdWarpsPerBlock, tile_counter, st);
        if (frames) launch_chained(stats_visible_stacked_kernel, v.ctas, block, 0, st, S, T, w, so, v.n_tiles, frames);
        else launch_chained(stats_visible_kernel, v.ctas, block, 0, st, S, T, w, so, v.n_tiles);
        launches += 2;
    }
    launch_chained(fix_stats_kernel, rec_ctas, 256, 0, st, f.ptr, n_rec);
    return launches;
}

}  // namespace forma
