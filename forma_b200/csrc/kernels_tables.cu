// Stage 4: per-tile coverage accumulation and compositing to RGBA8 — replaces
// forma/src/cpu/painter/{mod.rs, layer_workbench/, styling.rs}.
//
// The reference walks each tile row left to right, carrying every layer's
// winding "cover" (16 x i8, one per pixel row) from tile to tile in a queue
// (cpu/painter/mod.rs:486-568, layer_workbench/mod.rs:196-342). To paint tiles
// independently the carries are materialised first:
//
//   cells     runs of sorted segments with equal (tile_y, tile_x, layer)
//             (cells_scan: one pass, head bits -> cell_start by decoupled look-back)
//   covers    per cell: sum of segment covers by local_y (wrapping i8), its key (same pass)
//   re-sort   cell ids stably by the layer bits only -> (layer, tile_y, tile_x)
//             (digit counts from the cells pass)
//   carries   per (tile_y, layer) group a running sum -> carry-in of every cell
//             and "carry-only" entries for the tiles a layer spans without
//             segments (layer_workbench/mod.rs:213-234,328-336), generated in
//             that order (carry_pass: segmented scan, decoupled look-back) and
//             stably sorted by the tile digits only (digit counts from the carry pass)
//   entries   cells merged with the carry-only entries by rank into 64-byte
//             records ordered by (tile_y, tile_x, layer), + per-tile ranges (same pass)
//   paint     kernels_painter.cu: one warp per tile
//
// Integer semantics: areas wrap at i16 and covers at i8 in the reference;
// sums are formed in i32 / packed bytes and truncated where the reference
// widens them (truncation commutes with wrapping addition).
#include "paint_common.cuh"

namespace forma {

// ---------------------------------------------------------------------------
// Cells
// ---------------------------------------------------------------------------
constexpr int kCellThreads = 256;

__device__ __forceinline__ bool is_cell_head(const uint64_t* __restrict__ segs, uint32_t i) {
    return i == 0 || (segs[i] >> kSortShift) != (segs[i - 1] >> kSortShift);
}

// A CTA scans kCellItems x 256 consecutive segments (warp-striped so that every
// load is coalesced and the element order inside a warp is item-major).
constexpr int kCellItems = 8;
constexpr int kCellTile = kCellThreads * kCellItems;

// Cells in one pass over the sorted segments. A CTA takes a tile of 2048 segments (by
// ticket), keeps them in registers and
//   1. marks the heads (a segment starts a cell when its key differs from its predecessor's),
//   2. gets the number of cells before its tile by decoupled look-back (state[t] = flag |
//      running count; state[tiles] = ticket counter; 32 predecessors per round),
//   3. writes cell_start for its heads,
//   4. sums the covers of every cell that lies entirely inside the tile, by local_y, in shared
//      memory (acc_segment's cover part + cover_carry, cpu/painter/mod.rs:257-271,
//      layer_workbench/mod.rs:218-224) and writes the cell's records: its cover (16 x i8),
//      its key and the (tile_y, layer, tile_x) key of the carry pass.
// Cells that cross a tile boundary (at most two per tile) are left to cells_boundary_kernel.
// Positions >= cap are not written: the kernel may run before the host knows the cell count
// (Renderer::render repeats both kernels after growing the buffers if it was too small).
constexpr unsigned long long kCellAggregate = 1ull << 62, kCellInclusive = 2ull << 62, kCellFlags = 3ull << 62;
constexpr uint32_t kCellSlots = 512;  // cells accumulated per round (a tile with more takes several rounds)

// Returns the carry-pass key written.
__device__ __forceinline__ uint64_t write_cell_records(const PaintScene& S, uint32_t c, uint64_t first_seg, const int32_t* acc16,
                                                       uint64_t* __restrict__ cell_key, uint4* __restrict__ cell_cover,
                                                       uint64_t* __restrict__ key2, uint32_t* __restrict__ perm) {
    uint32_t w[4];
#pragma unroll
    for (int q = 0; q < 4; ++q)
        w[q] = ((uint32_t)acc16[4 * q] & 0xFFu) | (((uint32_t)acc16[4 * q + 1] & 0xFFu) << 8) |
               (((uint32_t)acc16[4 * q + 2] & 0xFFu) << 16) | (((uint32_t)acc16[4 * q + 3] & 0xFFu) << 24);
    const uint64_t ck = (first_seg >> kSortShift) << kSortShift;  // the cell's key = its first segment's
    cell_key[c] = ck;
    const int32_t ty = (int32_t)key_ty(ck) - 1, tx = (int32_t)key_tx(ck) - 1;
    const bool relevant = !(ty < (int32_t)S.ty_lo || ty >= (int32_t)S.ty_hi || tx >= (int32_t)S.tx_hi);
    perm[c] = c;
    cell_cover[c] = make_uint4(w[0], w[1], w[2], w[3]);
    const uint64_t k2 = relevant ? make_key2(ck) : sentinel_key(S.tiles_y);
    key2[c] = k2;
    return k2;
}

// Digit counts of a pair sort, gathered by the kernel that writes its keys: per CTA in shared
// memory, added to the global histogram once at the end.
__device__ __forceinline__ void hist_clear(uint32_t (*s_hist)[256], uint32_t passes) {
    for (uint32_t i = threadIdx.x; i < passes * 256u; i += blockDim.x) (&s_hist[0][0])[i] = 0;
}
__device__ __forceinline__ void hist_count(uint32_t* hist /* [passes][256], shared or global */, const SortPlan& plan,
                                           uint64_t key) {
#pragma unroll
    for (uint32_t p = 0; p < (uint32_t)kMaxSortPasses; ++p)  // unrolled: the plan stays in registers
        if (p < plan.n_passes) atomicAdd(&hist[p * 256u + digit_of(key, plan.pass[p])], 1u);
}
__device__ __forceinline__ void hist_flush(const uint32_t (*s_hist)[256], uint32_t passes, uint32_t* __restrict__ hist) {
    for (uint32_t i = threadIdx.x; i < passes * 256u; i += blockDim.x) {
        const uint32_t v = (&s_hist[0][0])[i];
        if (v) atomicAdd(&hist[i], v);
    }
}

__global__ void __launch_bounds__(kCellThreads)
    cells_kernel(PaintScene S, const uint64_t* __restrict__ segs, uint32_t n, unsigned long long* __restrict__ state,
                 uint32_t tiles, uint32_t* __restrict__ cell_start, uint32_t cap, uint32_t* __restrict__ n_cells_out,
                 uint64_t* __restrict__ cell_key, uint4* __restrict__ cell_cover, uint64_t* __restrict__ key2,
                 uint32_t* __restrict__ perm, SortPlan plan, uint32_t* __restrict__ hist, const uint32_t* __restrict__ n_dev) {
    chain_begin();
    if (n_dev) n = *n_dev;
    __shared__ uint32_t warp_cnt[kCellThreads / 32];
    __shared__ uint32_t s_tile;
    __shared__ unsigned long long s_prefix;
    __shared__ int32_t s_acc[kCellSlots][16];
    __shared__ uint64_t s_first[kCellSlots];  // first segment of the cell in each slot
    __shared__ uint32_t s_hist[kMaxSortPasses][256];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    if (threadIdx.x == 0) s_tile = (uint32_t)atomicAdd(&state[tiles], 1ull);
    hist_clear(s_hist, plan.n_passes);
    __syncthreads();
    const uint32_t tile = s_tile;
    // The tiles past the segment count (a device count, n_dev) hold no segment: they return, and the
    // last tile that holds one (tile 0 without any) writes the total. Tiles are taken in order.
    const uint32_t live = max((n + (uint32_t)kCellTile - 1u) / (uint32_t)kCellTile, 1u);
    if (tile >= live) return;
    const uint32_t tile_base = tile * kCellTile;
    const uint32_t base = tile_base + warp * (32u * kCellItems);
    // 1. segments -> registers, heads
    uint64_t seg[kCellItems];
    uint32_t masks[kCellItems];
    uint32_t cnt = 0;
    uint64_t carry_key = ~0ull;  // key of the element before the warp's first (none: every key differs from it)
    if (base > 0 && base < n) carry_key = segs[base - 1] >> kSortShift;
#pragma unroll
    for (int k = 0; k < kCellItems; ++k) {
        const uint32_t i = base + k * 32u + lane;
        seg[k] = i < n ? segs[i] : 0ull;
        const uint64_t key = seg[k] >> kSortShift;
        uint64_t prev = __shfl_up_sync(kFullMask, key, 1);
        if (lane == 0) prev = carry_key;
        const bool head = i < n && (i == 0 || key != prev);
        masks[k] = __ballot_sync(kFullMask, head);
        cnt += __popc(masks[k]);
        carry_key = __shfl_sync(kFullMask, key, 31);
    }
    if (lane == 0) warp_cnt[warp] = cnt;
    __syncthreads();
    uint32_t warp_off = 0, tile_sum = 0;
#pragma unroll
    for (int w = 0; w < kCellThreads / 32; ++w) {
        if ((uint32_t)w < warp) warp_off += warp_cnt[w];
        tile_sum += warp_cnt[w];
    }
    // 2. publish this tile's count at once: successors can start summing while we accumulate
    if (threadIdx.x == 0) {
        volatile unsigned long long* st = state;
        st[tile] = (tile == 0 ? kCellInclusive : kCellAggregate) | tile_sum;
    }
    // rank of every element's cell inside the tile (-1: the cell that continues from the previous tile)
    int32_t local[kCellItems];
    {
        uint32_t pos = warp_off;
#pragma unroll
        for (int k = 0; k < kCellItems; ++k) {
            local[k] = (int32_t)(pos + __popc(masks[k] & (0xFFFFFFFFu >> (31u - lane)))) - 1;  // heads at or before this lane
            pos += __popc(masks[k]);
        }
    }
    // The tile's last cell is complete iff the next tile starts with a head (or there is no next element).
    const uint32_t tile_end = min(tile_base + (uint32_t)kCellTile, n);
    bool last_complete = true;
    if (tile_end < n) last_complete = (segs[tile_end] >> kSortShift) != (segs[tile_end - 1u] >> kSortShift);
    const uint32_t n_complete = tile_sum - ((tile_sum > 0u && !last_complete) ? 1u : 0u);  // cells [0, n_complete) of the tile

    // 3. covers of the first kCellSlots complete cells — before the look-back: its latency hides behind this
    auto accumulate = [&](uint32_t r0, uint32_t nr) {
        for (uint32_t i = threadIdx.x; i < nr * 16u; i += kCellThreads) (&s_acc[0][0])[i] = 0;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < kCellItems; ++k) {
            const uint32_t i = base + k * 32u + lane;
            const int32_t slot = local[k] - (int32_t)r0;
            if (i < n && slot >= 0 && slot < (int32_t)nr) {
                const uint64_t sg = seg[k];
                const uint32_t ly = (uint32_t)(sg >> 12) & 15u;
                const int32_t cv = (int32_t)(((uint32_t)sg & 0x3Fu) ^ 0x20u) - 0x20;
                atomicAdd(&s_acc[slot][ly], cv);
                if ((masks[k] >> lane) & 1u) s_first[slot] = sg;
            }
        }
        __syncthreads();
    };
    const uint32_t nr0 = min(kCellSlots, n_complete);
    accumulate(0u, nr0);

    // 4. look-back (first warp): 32 predecessors per round, until one holds an inclusive prefix
    if (warp == 0) {
        volatile unsigned long long* st = state;
        unsigned long long prefix = 0;
        if (tile != 0) {
            int32_t p = (int32_t)tile - 1;
            while (true) {
                const int32_t idx = p - (int32_t)lane;
                unsigned long long v = kCellInclusive;  // before the first tile: an inclusive prefix of 0
                if (idx >= 0) {
                    do {
                        v = st[idx];
                    } while ((v & kCellFlags) == 0);
                }
                const uint32_t incl = __ballot_sync(kFullMask, (v & kCellFlags) == kCellInclusive);
                const uint32_t upto = incl ? (uint32_t)__ffs((int)incl) : 32u;  // lanes [0, upto) count
                unsigned long long part = lane < upto ? (v & ~kCellFlags) : 0ull;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(kFullMask, part, o);
                prefix += part;
                if (incl) break;
                p -= 32;
            }
            if (lane == 0) st[tile] = kCellInclusive | (prefix + tile_sum);
        }
        if (lane == 0) {
            s_prefix = prefix;
            if (tile + 1 == live) {
                const uint32_t total = (uint32_t)(prefix + tile_sum);
                n_cells_out[0] = total;
                if (total < cap) cell_start[total] = n;  // one-past-the-end sentinel
            }
        }
    }
    __syncthreads();
    const uint32_t cells_before = (uint32_t)s_prefix;

    // 5. cell_start of the heads, records of the complete cells
#pragma unroll
    for (int k = 0; k < kCellItems; ++k) {
        if ((masks[k] >> lane) & 1u) {
            const uint32_t q = cells_before + (uint32_t)local[k];
            if (q < cap) cell_start[q] = base + k * 32u + lane;
        }
    }
    for (uint32_t r0 = 0; r0 < n_complete; r0 += kCellSlots) {
        const uint32_t nr = min(kCellSlots, n_complete - r0);
        if (r0) accumulate(r0, nr);  // a tile with more than kCellSlots cells: further rounds
        for (uint32_t sl = threadIdx.x; sl < nr; sl += kCellThreads) {
            const uint32_t c = cells_before + r0 + sl;
            if (c < cap) hist_count(&s_hist[0][0], plan, write_cell_records(S, c, s_first[sl], s_acc[sl], cell_key, cell_cover, key2, perm));
        }
        __syncthreads();
    }
    hist_flush(s_hist, plan.n_passes, hist);
}

// The cells that cross a tile boundary of cells_kernel: one warp per boundary b (between
// tiles b - 1 and b). The warp acts when the element after the boundary continues a cell whose
// head lies in tile b - 1 (a cell that spans whole tiles is taken at its first boundary only)
// and sums the covers over the cell's whole segment range.
__global__ void __launch_bounds__(kCellThreads)
    cells_boundary_kernel(PaintScene S, const uint64_t* __restrict__ segs, uint32_t n, const unsigned long long* __restrict__ state,
                          uint32_t tiles, const uint32_t* __restrict__ cell_start, uint32_t cap,
                          const uint32_t* __restrict__ n_cells_ptr, uint64_t* __restrict__ cell_key, uint4* __restrict__ cell_cover,
                          uint64_t* __restrict__ key2, uint32_t* __restrict__ perm, SortPlan plan, uint32_t* __restrict__ hist,
                          const uint32_t* __restrict__ n_dev) {
    chain_begin();
    if (n_dev) n = *n_dev;
    const uint32_t b = blockIdx.x * (kCellThreads / 32) + (threadIdx.x >> 5) + 1u, lane = threadIdx.x & 31u;
    if (b >= tiles) return;
    const uint32_t n_cells = *n_cells_ptr;
    if (n_cells >= cap) return;  // cell_start is incomplete: the host repeats both kernels
    const uint32_t first = b * kCellTile;  // first element after the boundary
    if (first >= n || (segs[first] >> kSortShift) != (segs[first - 1u] >> kSortShift)) return;  // a head: nothing crosses
    const uint32_t incl_prev = (uint32_t)(state[b - 1u] & ~kCellFlags);                       // cells through tile b - 1
    const uint32_t incl_prev2 = b >= 2u ? (uint32_t)(state[b - 2u] & ~kCellFlags) : 0u;
    if (incl_prev == incl_prev2) return;  // tile b - 1 holds no head: an earlier boundary owns this cell
    const uint32_t c = incl_prev - 1u;
    const uint32_t s0 = cell_start[c], s1 = cell_start[c + 1u];
    int32_t acc[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) acc[r] = 0;
    for (uint32_t i = s0 + lane; i < s1; i += 32u) {
        const uint64_t sg = segs[i];
        const uint32_t ly = (uint32_t)(sg >> 12) & 15u;
        const int32_t cv = (int32_t)(((uint32_t)sg & 0x3Fu) ^ 0x20u) - 0x20;
#pragma unroll
        for (int r = 0; r < 16; ++r) acc[r] += (ly == (uint32_t)r) ? cv : 0;
    }
#pragma unroll
    for (int r = 0; r < 16; ++r) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[r] += __shfl_xor_sync(kFullMask, acc[r], o);
    }
    if (lane == 0)  // at most one cell per boundary: straight into the global histogram
        hist_count(hist, plan, write_cell_records(S, c, segs[s0], acc, cell_key, cell_cover, key2, perm));
}

// ---------------------------------------------------------------------------
// Carries
// ---------------------------------------------------------------------------
// Counts kept on the device (DevCounts, kernels.h): a frame whose tables are built without a
// host read-back launches the kernels below over upper bounds and lets them pick up the real
// counts here. A count above its bound (the buffers are too small) turns every later kernel of
// the frame into a no-op; the host sees it at the end of the frame and builds the tables again.
__device__ __forceinline__ void resolve_cells(const DevCounts& dc, uint32_t& n_cells) {
    if (!dc.cells) return;
    const uint32_t c = *dc.cells;
    n_cells = c > dc.cell_bound ? 0u : c;
}
__device__ __forceinline__ void resolve_counts(const DevCounts& dc, uint32_t& n_cells, uint32_t& n_gaps) {
    if (!dc.cells) return;
    const uint32_t c = *dc.cells, g = *dc.gaps;
    const bool ok = c <= dc.cell_bound && g <= dc.gap_bound;
    n_cells = ok ? c : 0u;
    n_gaps = ok ? g : 0u;
}

// The carry pass: one thread per cell in carry order ((layer, tile_y, tile_x) after the carry
// sort; a (tile_y, layer) group is a run of equal key2 >> 32), CTA tiles of kCarryThreads cells
// taken by ticket. Per cell:
//   1. its carry-in: the wrapping 16 x i8 sum of the covers of the cells before it in its group
//      (a segmented scan: inside the CTA by shuffles, across CTAs by decoupled look-back),
//   2. the number of carry-only entries between it and the next cell of the group: the tiles
//      a layer spans without segments while its running cover is not empty
//      (layer_workbench/mod.rs:213-234,328-336),
//   3. their exclusive offset (a second look-back over the counts), and the entries themselves,
//      written by the cell's warp together: key, payload n_cells + entry id and carried cover.
// The entries come out in (layer, tile_y, tile_x) order: a stable sort on the tile digits alone
// then orders them by (tile_y, tile_x, layer).
// 1024-cell tiles: the CTAs of a frame's carry pass look back at about the same time, so the
// last tile's look-back walks up to tiles / 32 windows of predecessors; a quarter as many tiles
// as with 256-cell tiles (paris@4K: 225).
constexpr int kCarryThreads = 1024;
constexpr int kCarryWarps = kCarryThreads / 32;
constexpr uint32_t kCarryAggregate = 1u, kCarryInclusive = 2u;  // carry flag words (0: not published yet)
constexpr unsigned long long kGapAggregate = 1ull << 62, kGapInclusive = 2ull << 62, kGapFlags = 3ull << 62;

// State per CTA tile: the published cover and its flag word (a 128-bit cover cannot be published
// with the flag in one atomic store: payload first, then the flag with release semantics) and the
// gap-count word (flag | running count, one 64-bit word); then the ticket counter.
struct CarryPassState {
    uint4* aggregate;   // segmented sum of the tile: its cells after its last group head (all of them without a head)
    uint4* inclusive;   // running cover after the tile's last cell
    uint32_t* flag;     // kCarryAggregate / kCarryInclusive
    unsigned long long* gaps;
    uint32_t* ticket;
};
__host__ __device__ inline size_t carry_pass_state_bytes(uint32_t tiles) { return (size_t)tiles * (16 + 16 + 8 + 4) + 16; }
__host__ __device__ inline CarryPassState carry_pass_state(uint8_t* base, uint32_t tiles) {
    CarryPassState s;
    s.aggregate = reinterpret_cast<uint4*>(base);
    s.inclusive = s.aggregate + tiles;
    s.gaps = reinterpret_cast<unsigned long long*>(s.inclusive + tiles);
    s.flag = reinterpret_cast<uint32_t*>(s.gaps + tiles);
    s.ticket = s.flag + tiles;
    return s;
}
inline uint32_t carry_pass_tiles(uint32_t n_cells) { return (n_cells + kCarryThreads - 1) / kCarryThreads; }

__device__ __forceinline__ uint32_t ld_acquire(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(uint32_t* p, uint32_t v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint4 ld_relaxed_v4(const uint4* p) {
    uint4 v;
    asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p)
                 : "memory");
    return v;
}
__device__ __forceinline__ uint4 shfl_cover(uint4 v, int src) {
    return make_uint4(__shfl_sync(kFullMask, v.x, src), __shfl_sync(kFullMask, v.y, src), __shfl_sync(kFullMask, v.z, src),
                      __shfl_sync(kFullMask, v.w, src));
}
__device__ __forceinline__ uint4 shfl_up_cover(uint4 v, unsigned d) {
    return make_uint4(__shfl_up_sync(kFullMask, v.x, d), __shfl_up_sync(kFullMask, v.y, d), __shfl_up_sync(kFullMask, v.z, d),
                      __shfl_up_sync(kFullMask, v.w, d));
}
__device__ __forceinline__ uint4 shfl_xor_cover(uint4 v, int m) {
    return make_uint4(__shfl_xor_sync(kFullMask, v.x, m), __shfl_xor_sync(kFullMask, v.y, m), __shfl_xor_sync(kFullMask, v.z, m),
                      __shfl_xor_sync(kFullMask, v.w, m));
}

__global__ void __launch_bounds__(kCarryThreads)
    carry_pass_kernel(PaintScene S, const uint64_t* __restrict__ key2, const uint32_t* __restrict__ perm,
                      const uint4* __restrict__ cell_cover, uint32_t n_cells, uint8_t* __restrict__ state_base, uint32_t tiles,
                      uint4* __restrict__ carry_in, uint64_t* __restrict__ gkey, uint32_t* __restrict__ gid,
                      uint4* __restrict__ gap_carry, uint32_t cap, uint32_t* __restrict__ n_gaps_out, SortPlan plan,
                      uint32_t* __restrict__ hist, DevCounts dc) {
    chain_begin();
    __shared__ uint32_t s_tile;
    __shared__ uint4 s_warp_cover[kCarryWarps];
    __shared__ uint32_t s_warp_head[kCarryWarps];
    __shared__ uint32_t s_warp_gaps[kCarryWarps];
    __shared__ uint4 s_carry;  // running cover into the tile's first cell
    __shared__ unsigned long long s_gap_prefix;
    __shared__ uint32_t s_hist[kMaxSortPasses][256];
    const CarryPassState st = carry_pass_state(state_base, tiles);
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    resolve_cells(dc, n_cells);
    if (threadIdx.x == 0) s_tile = atomicAdd(st.ticket, 1u);
    hist_clear(s_hist, plan.n_passes);
    __syncthreads();
    const uint32_t tile = s_tile;
    const uint32_t base = tile * (uint32_t)kCarryThreads;
    if (base >= n_cells) {  // tiles are taken in order: nobody looks back at this one
        if (tile == 0 && threadIdx.x == 0) n_gaps_out[0] = 0;
        return;
    }
    const uint32_t last_tile = (n_cells - 1u) / kCarryThreads;
    const uint64_t sentinel = sentinel_key(S.tiles_y);
    const uint4 zero = make_uint4(0u, 0u, 0u, 0u);

    // 1. the cell, its group head bit and its cover (zero for cells that reach no painted tile)
    const uint32_t j = base + threadIdx.x;
    const bool valid = j < n_cells;
    const uint64_t k = valid ? key2[j] : sentinel;
    const bool relevant = valid && k != sentinel;
    const uint32_t c = valid ? perm[j] : 0u;
    const uint4 cover = relevant ? cell_cover[c] : zero;
    const bool head = !valid || j == 0 || (key2[j - 1] >> 32) != (k >> 32);

    // 2. segmented inclusive scan inside the warp: (head seen, sum since the last head)
    uint4 incl = cover;
    bool seen = head;
#pragma unroll
    for (unsigned o = 1; o < 32; o <<= 1) {
        const uint4 pv = shfl_up_cover(incl, o);
        const bool ps = __shfl_up_sync(kFullMask, seen, o);
        if (lane >= o) {
            if (!seen) incl = cover_add(pv, incl);
            seen = seen || ps;
        }
    }
    if (lane == 31) {
        s_warp_cover[warp] = incl;
        s_warp_head[warp] = seen;
    }
    __syncthreads();
    uint4 warp_prefix = zero;  // segmented sum of the warps before this one
    bool warp_prefix_seen = false;
    for (int w = (int)warp - 1; w >= 0 && !warp_prefix_seen; --w) {
        warp_prefix = cover_add(warp_prefix, s_warp_cover[w]);
        warp_prefix_seen = s_warp_head[w] != 0u;
    }

    // 3. carry look-back (first warp). A tile that holds a group head knows the running cover
    //    after its last cell by itself and publishes it at once; a tile without one publishes its
    //    sum and, after the look-back, the running cover.
    if (warp == 0) {
        uint4 agg = zero;
        bool agg_seen = false;
        for (int w = kCarryWarps - 1; w >= 0 && !agg_seen; --w) {
            agg = cover_add(agg, s_warp_cover[w]);
            agg_seen = s_warp_head[w] != 0u;
        }
        if (lane == 0) {
            if (agg_seen || tile == 0) {
                st.inclusive[tile] = agg;
                st_release(&st.flag[tile], kCarryInclusive);
            } else {
                st.aggregate[tile] = agg;
                st_release(&st.flag[tile], kCarryAggregate);
            }
        }
        uint4 prefix = zero;
        if (tile != 0 && !__shfl_sync(kFullMask, head, 0)) {  // the first cell continues a group
            int32_t p = (int32_t)tile - 1;
            while (true) {
                const int32_t idx = p - (int32_t)lane;
                uint32_t f = kCarryInclusive;  // before the first tile: a running cover of 0
                uint4 v = zero;
                if (idx >= 0) {
                    do {
                        f = ld_acquire(&st.flag[idx]);
                    } while (f == 0u);
                    v = ld_relaxed_v4(f == kCarryInclusive ? &st.inclusive[idx] : &st.aggregate[idx]);
                }
                const uint32_t done = __ballot_sync(kFullMask, f == kCarryInclusive);
                const uint32_t upto = done ? (uint32_t)__ffs((int)done) : 32u;  // lanes [0, upto) count
                uint4 part = lane < upto ? v : zero;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) part = cover_add(part, shfl_xor_cover(part, o));
                prefix = cover_add(prefix, part);
                if (done) break;
                p -= 32;
            }
            if (lane == 0 && !agg_seen) {
                st.inclusive[tile] = cover_add(prefix, agg);
                st_release(&st.flag[tile], kCarryInclusive);
            }
        }
        if (lane == 0) s_carry = prefix;
    }
    __syncthreads();

    // 4. carry-in and running cover after the cell
    uint4 before = shfl_up_cover(incl, 1);
    bool before_seen = __shfl_up_sync(kFullMask, seen, 1);
    if (lane == 0) {
        before = zero;
        before_seen = false;
    }
    if (!before_seen) {
        before = cover_add(warp_prefix, before);
        if (!warp_prefix_seen) before = cover_add(s_carry, before);
    }
    const uint4 cin = head ? zero : before;
    const uint4 run = cover_add(cin, cover);
    if (valid) carry_in[c] = cin;

    // 5. carry-only entries after the cell: tiles [first, first + gaps) of its row
    uint32_t gaps = 0;
    int32_t first = 0;
    if (relevant) {
        const int32_t ty = (int32_t)key_ty(k) - 1;
        if (ty >= (int32_t)S.ty_lo && ty < (int32_t)S.ty_hi) {
            const int32_t t = (int32_t)key2_tx(k) - 1;
            const bool has_next = j + 1u < n_cells && (key2[j + 1u] >> 32) == (k >> 32);
            const int32_t next_t = has_next ? (int32_t)key2_tx(key2[j + 1u]) - 1 : (int32_t)S.tx_hi;
            first = max(t + 1, (int32_t)S.tx_lo);
            const int32_t hi = min(next_t, (int32_t)S.tx_hi);
            if (!cover_is_empty(run, fill_rule_of(S, key2_layer(k)))) {
                gaps = hi > first ? (uint32_t)(hi - first) : 0u;
            } else if (t < (int32_t)S.tx_lo && next_t > (int32_t)S.tx_lo && S.tx_lo < S.tx_hi) {
                // covers_left_of_row: a layer with segments left of the first
                // painted tile is queued for it even when its cover sums to zero
                // (cpu/painter/mod.rs:501-522).
                gaps = 1;
            }
        }
    }

    // 6. exclusive offset of the cell's entries: inside the tile, then by look-back
    const uint32_t gaps_incl = warp_inclusive_scan(gaps);
    if (lane == 31) s_warp_gaps[warp] = gaps_incl;
    __syncthreads();
    uint32_t warp_off = 0, tile_gaps = 0;
#pragma unroll
    for (int w = 0; w < kCarryWarps; ++w) {
        if ((uint32_t)w < warp) warp_off += s_warp_gaps[w];
        tile_gaps += s_warp_gaps[w];
    }
    if (warp == 0) {
        volatile unsigned long long* gs = st.gaps;
        unsigned long long prefix = 0;
        if (tile == 0) {
            if (lane == 0) gs[0] = kGapInclusive | tile_gaps;
        } else {
            if (lane == 0) gs[tile] = kGapAggregate | tile_gaps;
            int32_t p = (int32_t)tile - 1;
            while (true) {
                const int32_t idx = p - (int32_t)lane;
                unsigned long long v = kGapInclusive;
                if (idx >= 0) {
                    do {
                        v = gs[idx];
                    } while ((v & kGapFlags) == 0);
                }
                const uint32_t done = __ballot_sync(kFullMask, (v & kGapFlags) == kGapInclusive);
                const uint32_t upto = done ? (uint32_t)__ffs((int)done) : 32u;
                unsigned long long part = lane < upto ? (v & ~kGapFlags) : 0ull;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(kFullMask, part, o);
                prefix += part;
                if (done) break;
                p -= 32;
            }
            if (lane == 0) gs[tile] = kGapInclusive | (prefix + tile_gaps);
        }
        if (lane == 0) {
            s_gap_prefix = prefix;
            if (tile == last_tile) n_gaps_out[0] = (uint32_t)(prefix + tile_gaps);
        }
    }
    __syncthreads();

    // 7. the entries, written by the warp together (entry i of the warp by lane i % 32): lane l's
    //    cell owns entries [off_l, off_l + gaps_l) of the warp, found by bisection over the lanes
    const uint32_t warp_gaps = __shfl_sync(kFullMask, gaps_incl, 31);
    const uint32_t off = gaps_incl - gaps;                                     // inside the warp
    const uint64_t q0 = s_gap_prefix + warp_off;                               // the warp's first entry
    const uint64_t bk = ((uint64_t)key_ty(k) << 53) | ((uint64_t)key2_layer(k) << 20);  // key without its tile_x
    for (uint32_t i0 = 0; i0 < warp_gaps; i0 += 32u) {
        const uint32_t i = i0 + lane;
        int src = 0;
#pragma unroll
        for (int step = 16; step > 0; step >>= 1)
            if (__shfl_sync(kFullMask, off, src + step) <= i) src += step;
        const uint32_t r = i - __shfl_sync(kFullMask, off, src);
        const int32_t f = __shfl_sync(kFullMask, first, src);
        const uint64_t kb = ((uint64_t)__shfl_sync(kFullMask, (uint32_t)(bk >> 32), src) << 32) |
                            (uint64_t)__shfl_sync(kFullMask, (uint32_t)bk, src);
        const uint4 cv = shfl_cover(run, src);
        const uint64_t q = q0 + i;
        if (i < warp_gaps && q < cap) {
            const uint64_t gk = kb | ((uint64_t)(uint32_t)(f + (int32_t)r + 1) << 41);
            gkey[q] = gk;
            gid[q] = n_cells + (uint32_t)q;
            gap_carry[q] = cv;
            hist_count(&s_hist[0][0], plan, gk);
        }
    }
    __syncthreads();
    hist_flush(s_hist, plan.n_passes, hist);
}

// Entries = cells (sorted by construction) merged with the sorted carry-only
// entries; both lists are strictly increasing and share no key, so an element's
// position is its own index plus its rank in the other list.
__device__ __forceinline__ uint32_t lower_bound_key(const uint64_t* __restrict__ a, uint32_t n, uint64_t k) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        uint32_t mid = (lo + hi) >> 1;
        if (a[mid] < k) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}
// lower_bound_key over the whole list by one warp: 32 pivots per round cut the range 33-fold,
// so a list of a million keys takes 4 dependent loads instead of 20.
__device__ __forceinline__ uint32_t warp_lower_bound_key(const uint64_t* __restrict__ a, uint32_t n, uint64_t k) {
    const uint32_t lane = threadIdx.x & 31u;
    uint32_t lo = 0, hi = n;  // the answer lies in [lo, hi]
    while (hi - lo > 32u) {
        const uint64_t len = hi - lo;
        const uint32_t below = __popc(__ballot_sync(kFullMask, a[lo + (uint32_t)(len * (lane + 1u) / 33u)] < k));
        const uint32_t nlo = below ? lo + (uint32_t)(len * below / 33u) + 1u : lo;  // past the last pivot < k
        hi = below < 32u ? lo + (uint32_t)(len * (below + 1u) / 33u) : hi;        // at the first pivot >= k
        lo = nlo;
    }
    return lo + __popc(__ballot_sync(kFullMask, lo + lane < hi && a[lo + lane] < k));
}
// lower_bound_key in a[0, i] when every key from a[i] on is >= k (a[i] itself is not read):
// galloping back from i, then bisection — a tile's entries are few and close together.
__device__ __forceinline__ uint32_t lower_bound_back(const uint64_t* __restrict__ a, uint32_t i, uint64_t k) {
    uint32_t hi = i, lo = 0;  // the answer lies in [lo, hi]
    for (uint32_t step = 1; step <= hi; step <<= 1) {
        if (a[hi - step] < k) {
            lo = hi - step + 1u;
            break;
        }
        hi -= step;
    }
    return lo + lower_bound_key(a + lo, hi - lo, k);
}
// Besides the sorted key, every entry gets a self-contained 64-byte record (its
// segment range, carry, style bits and colour) and its initial optimizer flags,
// so that the painter reaches everything it needs with one round of loads per
// 32 entries instead of chasing key -> id -> cell -> style pointers per tile.
// kPoseFills: S.styles is a pose style table (PoseFillArgs), and an in-frame entry of a Draw layer
// in the pose window takes its frame's slot; everything after reads the StyleRec at that slot.
template <bool kPoseFills>
__device__ __forceinline__ void merge_entries_body(PaintScene S, const uint64_t* __restrict__ cell_key, uint32_t n_cells,
                                                   const uint64_t* __restrict__ gkey, const uint32_t* __restrict__ gid,
                                                   uint32_t n_gaps, const uint32_t* __restrict__ cell_start,
                                                   const uint4* __restrict__ carry_in, const uint4* __restrict__ gap_carry,
                                                   uint64_t* __restrict__ ekey, EntryRec* __restrict__ recs,
                                                   uint8_t* __restrict__ eflags, uint2* __restrict__ tile_range,
                                                   uint32_t* __restrict__ heavy, uint32_t* __restrict__ heavy_count,
                                                   DevCounts dc, const BatchFrame* __restrict__ frames, uint32_t rows,
                                                   PoseFillArgs F = PoseFillArgs{}) {
    if (dc.words_out && blockIdx.x == 0 && threadIdx.x < dc.n_words) dc.words_out[threadIdx.x] = dc.words[threadIdx.x];
    resolve_counts(dc, n_cells, n_gaps);
    // Merge-path style partition: the keys of a CTA's 256 consecutive elements of
    // one list bracket a short range of the other list, found once per CTA (two
    // whole-list searches by warps 0 and 1); every thread then bisects that range only.
    __shared__ uint32_t s_bound[2];
    const uint32_t i0 = blockIdx.x * blockDim.x, i = i0 + threadIdx.x;
    const uint32_t n_all = n_cells + n_gaps;
    if (i0 >= n_all) return;  // (whole CTA; only with device-side counts)
    const bool cell_block = i0 + blockDim.x <= n_cells, gap_block = i0 >= n_cells;  // else: the one mixed CTA
    if (threadIdx.x < 64u) {
        const uint32_t w = threadIdx.x >> 5;
        const uint32_t last = min(i0 + blockDim.x, n_all) - 1u;
        uint32_t b = w == 0u ? 0u : (cell_block ? n_gaps : n_cells);
        if (cell_block) b = warp_lower_bound_key(gkey, n_gaps, cell_key[w == 0u ? i0 : last]);
        else if (gap_block) b = warp_lower_bound_key(cell_key, n_cells, gkey[(w == 0u ? i0 : last) - n_cells]);
        if ((threadIdx.x & 31u) == 0u) s_bound[w] = b;
    }
    __syncthreads();
    if (i >= n_all) return;
    uint64_t k;
    uint32_t pos;
    EntryRec r;
    // The entry's own list (a) from index ia on, the other list (b) from rank rb on: the next
    // entry in tile order is the smaller of a[ia + 1] and b[rb].
    const uint64_t *a, *b;
    uint32_t na, nb, ia, rb;
    if (i < n_cells) {
        k = cell_key[i];
        const uint32_t lo = cell_block ? s_bound[0] : 0u, hi = cell_block ? s_bound[1] : n_gaps;
        rb = lo + lower_bound_key(gkey + lo, hi - lo, k);
        a = cell_key, na = n_cells, ia = i, b = gkey, nb = n_gaps;
        r.seg0 = cell_start[i];
        r.seg1 = cell_start[i + 1];
        r.carry = carry_in[i];
    } else {
        uint32_t g = i - n_cells;
        k = gkey[g];
        const uint32_t lo = gap_block ? s_bound[0] : 0u, hi = gap_block ? s_bound[1] : n_cells;
        rb = lo + lower_bound_key(cell_key + lo, hi - lo, k);
        a = gkey, na = n_gaps, ia = g, b = cell_key, nb = n_cells;
        r.seg0 = r.seg1 = 0;
        r.carry = gap_carry[gid[g] - n_cells];
    }
    pos = ia + rb;
    // Per painted tile: [begin, end) of its entries, written by the thread of the tile's last
    // entry (it finds the first one in both lists, searching back from its own place in them:
    // every key from a[ia] and from b[rb] on is >= the tile's first key); the same thread files a tile
    // with many entries in its class list (see paint_common.cuh: kHeavyMin). Entries outside the
    // render target (biased tile coordinate 0 = tile -1, or beyond the last tile) belong to no
    // painted tile.
    const uint64_t tile_bits = k >> 41;
    const bool in_frame = key_ty(k) != 0u && key_ty(k) <= S.tiles_y && key_tx(k) != 0u && key_tx(k) <= S.tiles_x;
    if (in_frame && (ia + 1u >= na || (a[ia + 1u] >> 41) != tile_bits) && (rb >= nb || (b[rb] >> 41) != tile_bits)) {
        const uint64_t tile_key = tile_bits << 41;
        const uint32_t begin = lower_bound_back(a, ia, tile_key) + lower_bound_back(b, rb, tile_key);
        const uint32_t tid = (key_ty(k) - 1u) * S.tiles_x + (key_tx(k) - 1u);
        tile_range[tid] = make_uint2(begin, pos + 1u);
        const uint32_t count = pos + 1u - begin;
        if (heavy && count >= kHeavyMin) {
            const int hc = heavy_class(count);
            heavy[(size_t)hc * S.tiles_x * S.tiles_y + atomicAdd(&heavy_count[hc], 1u)] = tid;
        }
    }
    r.layer = key_layer(k);
    r.slot = r.layer < S.n_orders ? S.order_to_style[r.layer] : -1;
    if constexpr (kPoseFills) {
        const uint32_t o = r.layer - F.first_order;  // (wraps for orders below the window)
        if (r.slot >= 0 && in_frame && o < F.n_orders && S.styles[r.slot].func == 0u)
            r.slot = (int32_t)(F.n_styles + ((key_ty(k) - 1u) / F.rows) * F.n_orders + o);
    }
    uint32_t flags = 0;
    if (r.slot >= 0) {
        const StyleRec& st = S.styles[r.slot];
        const bool unchanged = S.unchanged && S.unchanged[r.layer];
        r.meta = pack_style_meta(st, unchanged);
        // The clip's range in the frame's own orders o (a batch's layers are order_base + o, see
        // BatchFrame): o + clip_layers wraps below o in 32 bits (the clip then ends at itself), or
        // ends at the last order there can be. Every walk adds it to the layer as it stands, and
        // then finds the range a single frame of the composition finds.
        const uint32_t o = frames && in_frame ? r.layer - frames[(key_ty(k) - 1u) / rows].order_base : r.layer;
        r.clip_layers = o + st.clip_layers < o ? 0u : min(st.clip_layers, kLayerLimit - o);
        r.color[0] = st.color[0];
        r.color[1] = st.color[1];
        r.color[2] = st.color[2];
        r.color[3] = st.color[3];
        if (r.seg1 > r.seg0) flags |= kFlagHasSegs;
        else if (cover_is_full(r.carry, st.fill_rule & 1u)) flags |= kFlagFull;  // layer_is_full, mod.rs:171-182
        if (unchanged) flags |= kFlagUnchanged;
        if (st.func == 1u || st.is_clipped) flags |= kFlagClipish;
        if (st.func == 0u && st.is_clipped) flags |= kFlagClippedDraw;
        if (st.func == 0u && st.fill_type == 0u && st.blend_mode == 0u && st.color[3] == 1.0f) flags |= kFlagOpaque;
    } else {
        r.meta = 0;
        r.clip_layers = 0;
        r.color[0] = r.color[1] = r.color[2] = r.color[3] = 0.0f;
        flags = kFlagMaskedOut;
    }
    r.flags0 = flags;
    r.pad = 0;
    ekey[pos] = k;
    recs[pos] = r;
    eflags[pos] = (uint8_t)flags;
}
__global__ void merge_entries_kernel(PaintScene S, const uint64_t* __restrict__ cell_key, uint32_t n_cells,
                                     const uint64_t* __restrict__ gkey, const uint32_t* __restrict__ gid, uint32_t n_gaps,
                                     const uint32_t* __restrict__ cell_start, const uint4* __restrict__ carry_in,
                                     const uint4* __restrict__ gap_carry, uint64_t* __restrict__ ekey,
                                     EntryRec* __restrict__ recs, uint8_t* __restrict__ eflags, uint2* __restrict__ tile_range,
                                     uint32_t* __restrict__ heavy, uint32_t* __restrict__ heavy_count, DevCounts dc,
                                     const BatchFrame* __restrict__ frames, uint32_t rows) {
    chain_begin();
    merge_entries_body<false>(S, cell_key, n_cells, gkey, gid, n_gaps, cell_start, carry_in, gap_carry, ekey, recs, eflags, tile_range,
                              heavy, heavy_count, dc, frames, rows);
}
__global__ void merge_entries_pose_fills_kernel(PaintScene S, const uint64_t* __restrict__ cell_key, uint32_t n_cells,
                                                const uint64_t* __restrict__ gkey, const uint32_t* __restrict__ gid, uint32_t n_gaps,
                                                const uint32_t* __restrict__ cell_start, const uint4* __restrict__ carry_in,
                                                const uint4* __restrict__ gap_carry, uint64_t* __restrict__ ekey,
                                                EntryRec* __restrict__ recs, uint8_t* __restrict__ eflags,
                                                uint2* __restrict__ tile_range, uint32_t* __restrict__ heavy,
                                                uint32_t* __restrict__ heavy_count, DevCounts dc, PoseFillArgs F) {
    chain_begin();
    merge_entries_body<true>(S, cell_key, n_cells, gkey, gid, n_gaps, cell_start, carry_in, gap_carry, ekey, recs, eflags, tile_range,
                             heavy, heavy_count, dc, nullptr, 0u, F);
}

// A Draw layer's StyleRec with its fill made Fill::Solid(c): no gradient or texture left.
__device__ __forceinline__ void make_solid(StyleRec& r, float4 c) {
    r.fill_type = 0u;
    r.color[0] = c.x;
    r.color[1] = c.y;
    r.color[2] = c.z;
    r.color[3] = c.w;
    r.gradient_type = 0u;
    r.start[0] = r.start[1] = r.end[0] = r.end[1] = 0.0f;
    r.stop_count = 0u;
    for (int j = 0; j < 6; ++j) r.tex_xf[j] = 0.0f;
    r.tex_max_x = r.tex_max_y = 0.0f;
    r.tex_width = r.tex_first = 0u;
}

// The tail of a pose style table, one thread per (frame b, order first_order + k) record i = b K + k:
// the StyleRec of the layer at that order with its fill made Fill::Solid(colors[i]) when the layer
// draws; a Clip layer's record is its own (merge_entries never points at it). Orders without a
// layer have no record.
__global__ void __launch_bounds__(256) pose_styles_kernel(const int32_t* __restrict__ order_to_style, uint32_t n_orders,
                                                          StyleRec* __restrict__ styles, uint32_t n_styles,
                                                          const float4* __restrict__ colors, uint32_t first_order, uint32_t K,
                                                          uint64_t n_recs) {
    chain_begin();
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_recs) return;
    const uint32_t o = first_order + (uint32_t)(i % K);
    const int32_t s = o < n_orders ? order_to_style[o] : -1;
    if (s < 0) return;
    StyleRec r = styles[s];
    if (r.func == 0u) make_solid(r, colors[i]);
    styles[n_styles + i] = r;
}

// The order -> style table of an instance call, one thread per slot r (see launch_instance_styles).
__global__ void __launch_bounds__(256) instance_styles_kernel(const int32_t* __restrict__ order_to_style, uint32_t n_orders,
                                                              const uint32_t* __restrict__ prototypes, StyleRec* __restrict__ styles,
                                                              uint32_t n_styles, const float4* __restrict__ colors, uint32_t n_recs,
                                                              int32_t* __restrict__ inst_order_to_style) {
    chain_begin();
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_recs) return;
    const uint32_t p = prototypes[r];  // (FORMA_NO_INSTANCE is no order)
    int32_t s = p < n_orders ? order_to_style[p] : -1;
    if (s >= 0 && colors && styles[s].func == 0u) {
        StyleRec rec = styles[s];
        make_solid(rec, colors[r]);
        styles[n_styles + r] = rec;
        s = (int32_t)(n_styles + r);
    }
    inst_order_to_style[r] = s;
}

// Cost of every tile row of the frame just rendered: 32 x its (tile, layer) entries + its
// pixel segments (paint time follows the entries, sort / table time the segments). The
// multi-GPU band split of the next frame is balanced on these (SURVEY.md 8e). One warp per row.
__global__ void row_cost_kernel(const uint2* __restrict__ tile_range, uint32_t tiles_x, uint32_t tiles_y,
                                const uint64_t* __restrict__ segs, uint32_t n, unsigned long long* __restrict__ out,
                                unsigned long long* __restrict__ seg_out, const uint32_t* __restrict__ n_dev) {
    chain_begin();
    if (n_dev) n = *n_dev;
    const uint32_t row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
    if (row >= tiles_y) return;
    uint32_t entries = 0;
    for (uint32_t tx = lane; tx < tiles_x; tx += 32u) {
        const uint2 r = tile_range[(size_t)row * tiles_x + tx];
        entries += r.y - r.x;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) entries += __shfl_xor_sync(kFullMask, entries, o);
    if (lane == 0) {
        auto lower = [&](uint64_t key) {  // first segment with key >= `key`
            uint32_t lo = 0, hi = n;
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (segs[mid] < key) lo = mid + 1u;
                else hi = mid;
            }
            return lo;
        };
        const uint32_t s0 = lower((uint64_t)(row + 1u) << 53), s1 = lower((uint64_t)(row + 2u) << 53);
        out[row] = 32ull * entries + (unsigned long long)(s1 - s0);
        // Pixel segments and entries of the row. The first row also takes the segments above the
        // frame (tile_y clamped to -1), the last row those below it (they sort behind every
        // painted tile), so that the rows of a frame add up to its segment count.
        if (seg_out) {
            seg_out[row] = (row + 1u == tiles_y ? n : s1) - (row == 0u ? 0u : s0);
            seg_out[tiles_y + row] = entries;
        }
    }
}

void launch_row_costs(const uint2* tile_range, uint32_t tiles_x, uint32_t tiles_y, const uint64_t* segs, uint32_t n,
                      unsigned long long* out, cudaStream_t st, unsigned long long* seg_out, const uint32_t* n_dev) {
    if (tiles_y) launch_chained(row_cost_kernel, (tiles_y + 7) / 8, 256, 0, st, tile_range, tiles_x, tiles_y, segs, n, out, seg_out, n_dev);
}

// ---------------------------------------------------------------------------
// Host launchers
// ---------------------------------------------------------------------------
uint32_t cell_num_blocks(uint32_t n) { return (n + kCellTile - 1) / kCellTile; }

static size_t align256(size_t b) { return (b + 255u) & ~(size_t)255u; }

TableScratch table_scratch_layout(uint32_t n, uint32_t n_cells, uint32_t n_gaps, const SortPlan& carry_plan,
                                  const SortPlan& gap_plan) {
    TableScratch L;
    const size_t hist_bytes = align256((size_t)kMaxSortPasses * 256u * sizeof(uint32_t));
    L.heavy_count = 0;
    L.carry_hist = align256(kHeavyListClasses * sizeof(uint32_t));
    L.gap_hist = L.carry_hist + hist_bytes;
    L.cells_state = L.gap_hist + hist_bytes;
    L.carry_sort = L.cells_state + align256(((size_t)cell_num_blocks(n) + 1u) * sizeof(unsigned long long));
    L.carry_pass = L.carry_sort + align256(sort_lookback_bytes(n_cells, carry_plan));
    L.gap_sort = L.carry_pass + align256(carry_pass_state_bytes(carry_pass_tiles(n_cells)));
    L.end = L.gap_sort + align256(sort_lookback_bytes(n_gaps, gap_plan));
    return L;
}

// Zeroes the bytes [0, a_bytes) of `a` and [0, b_bytes) of `b` (two device allocations, so 16-byte
// aligned) and the word `word` (when not null): the tile ranges, the table scratch and the paint
// kernel's tile counter of a sync-free frame, in one chained launch in place of three memsets, which
// would end the overlap of the kernels around them. Not counted in Renderer::launches, like the
// memsets it replaces.
__global__ void __launch_bounds__(256) zero_tables_kernel(uint8_t* __restrict__ a, size_t a_bytes, uint8_t* __restrict__ b, size_t b_bytes,
                                                          uint32_t* __restrict__ word) {
    chain_begin();
    const size_t stride = (size_t)gridDim.x * blockDim.x, i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (word && i0 == 0) *word = 0u;
    for (int k = 0; k < 2; ++k) {
        uint8_t* p = k ? b : a;
        const size_t bytes = k ? b_bytes : a_bytes, words = bytes / 16u;
        for (size_t i = i0; i < words; i += stride) reinterpret_cast<uint4*>(p)[i] = make_uint4(0u, 0u, 0u, 0u);
        for (size_t i = words * 16u + i0; i < bytes; i += stride) p[i] = 0u;
    }
}
void launch_zero_tables(uint8_t* a, size_t a_bytes, uint8_t* b, size_t b_bytes, uint32_t* word, cudaStream_t st) {
    const size_t words = std::max<size_t>((std::max(a_bytes, b_bytes) + 15u) / 16u, 1u);
    const uint32_t ctas = (uint32_t)std::min<size_t>((words + 255u) / 256u, (size_t)device_sm_count() * 4u);
    launch_chained(zero_tables_kernel, ctas, 256, 0, st, a, a_bytes, b, b_bytes, word);
}

void launch_cells(const PaintScene& S, const uint64_t* segs, uint32_t n, uint8_t* scratch, const TableScratch& L,
                  const SortPlan& carry_plan, uint32_t* cell_start, uint32_t cap, uint32_t* n_cells_out, uint64_t* cell_key,
                  uint4* cell_cover, uint64_t* key2, uint32_t* perm, cudaStream_t st, const uint32_t* n_dev) {
    const uint32_t tiles = cell_num_blocks(n);
    auto* state = reinterpret_cast<unsigned long long*>(scratch + L.cells_state);  // [tiles] look-back | ticket
    auto* hist = reinterpret_cast<uint32_t*>(scratch + L.carry_hist);
    launch_chained(cells_kernel, tiles, kCellThreads, 0, st, S, segs, n, state, tiles, cell_start, cap, n_cells_out, cell_key, cell_cover, key2,
                                                 perm, carry_plan, hist, n_dev);
    if (tiles > 1)
        launch_chained(cells_boundary_kernel, (tiles - 1 + kCellThreads / 32 - 1) / (kCellThreads / 32), kCellThreads, 0, st,
            S, segs, n, state, tiles, cell_start, cap, n_cells_out, cell_key, cell_cover, key2, perm, carry_plan, hist, n_dev);
}

// Largest values the three key fields can take in the pair sorts (sentinel
// included); the sort plan only spends passes on bits below these bounds.
// The cells arrive sorted by (tile_y, tile_x, layer); a stable sort on the layer
// bits alone leaves them ordered by (layer, tile_y, tile_x), which is all the
// carry pass needs: every (tile_y, layer) group contiguous, tile_x ascending.
SortPlan carry_sort_plan(const PaintScene& S) {  // fields, least significant first: tile_x, layer, tile_y
    const uint64_t bound[3] = {0u, S.n_orders ? S.n_orders - 1u : 0u, 0u};
    return make_sort_plan(carry_key_layout(), bound);
}
// Carry-only entries: tile digits only (see carry_pass_kernel).
SortPlan gap_sort_plan(const PaintScene& S) {  // layer, tile_x, tile_y
    const uint64_t bound[3] = {0u, S.tx_hi, S.ty_hi};
    return make_sort_plan(segment_key_layout(), bound);
}

void launch_carry_pass(const PaintScene& S, const uint64_t* key2, const uint32_t* perm, const uint4* cell_cover,
                       uint32_t n_cells, uint8_t* scratch, const TableScratch& L, const SortPlan& gap_plan, uint4* carry_in,
                       uint64_t* gkey, uint32_t* gid, uint4* gap_carry, uint32_t cap, uint32_t* n_gaps_out, cudaStream_t st,
                       const DevCounts& dc) {
    const uint32_t tiles = carry_pass_tiles(n_cells);
    if (!tiles) return;
    launch_chained(carry_pass_kernel, tiles, kCarryThreads, 0, st, S, key2, perm, cell_cover, n_cells, scratch + L.carry_pass, tiles, carry_in,
                                                       gkey, gid, gap_carry, cap, n_gaps_out, gap_plan,
                                                       reinterpret_cast<uint32_t*>(scratch + L.gap_hist), dc);
}

void launch_merge_entries(const PaintScene& S, const uint64_t* cell_key, uint32_t n_cells, const uint64_t* gkey,
                          const uint32_t* gid, uint32_t n_gaps, const uint32_t* cell_start, const uint4* carry_in,
                          const uint4* gap_carry, uint64_t* ekey, EntryRec* recs, uint8_t* eflags, uint2* tile_range,
                          uint32_t* heavy, uint32_t* heavy_count, cudaStream_t st, const DevCounts& dc, const BatchFrame* frames,
                          uint32_t rows, const PoseFillArgs* fills) {
    uint32_t n = n_cells + n_gaps;
    if (!n) return;
    if (fills)
        launch_chained(merge_entries_pose_fills_kernel, (n + 255) / 256, 256, 0, st, S, cell_key, n_cells, gkey, gid, n_gaps, cell_start, carry_in,
                                                                          gap_carry, ekey, recs, eflags, tile_range, heavy, heavy_count,
                                                                          dc, *fills);
    else
        launch_chained(merge_entries_kernel, (n + 255) / 256, 256, 0, st, S, cell_key, n_cells, gkey, gid, n_gaps, cell_start, carry_in,
                                                               gap_carry, ekey, recs, eflags, tile_range, heavy, heavy_count, dc,
                                                               frames, rows);
}

void launch_pose_styles(const int32_t* order_to_style, uint32_t n_orders, StyleRec* styles, uint32_t n_styles, const float4* colors,
                        uint32_t first_order, uint32_t n_window, uint64_t n_recs, cudaStream_t st) {
    if (n_recs)
        launch_chained(pose_styles_kernel, (unsigned)((n_recs + 255u) / 256u), 256, 0, st, order_to_style, n_orders, styles, n_styles, colors,
                                                                               first_order, n_window, n_recs);
}
void launch_instance_styles(const int32_t* order_to_style, uint32_t n_orders, const uint32_t* prototypes, StyleRec* styles,
                            uint32_t n_styles, const float4* colors, uint32_t n_recs, int32_t* inst_order_to_style, cudaStream_t st) {
    if (n_recs)
        launch_chained(instance_styles_kernel, (n_recs + 255u) / 256u, 256, 0, st, order_to_style, n_orders, prototypes, styles, n_styles,
                       colors, n_recs, inst_order_to_style);
}

// ---------------------------------------------------------------------------
// Batch tables
// ---------------------------------------------------------------------------
// CTA (x, k) copies every gridDim.x-th run of 256 records of composition k's tables into the
// batch's, moving the indices into the shared arrays by the composition's bases.
__global__ void __launch_bounds__(256) batch_tables_kernel(const BatchTableSrc* __restrict__ src, int32_t* __restrict__ order_to_style,
                                                           StyleRec* __restrict__ styles, GradRec* __restrict__ grads,
                                                           StopRec* __restrict__ stops, uint2* __restrict__ texels) {
    const BatchTableSrc s = src[blockIdx.y];
    const uint32_t step = gridDim.x * blockDim.x;
    const uint32_t first = blockIdx.x * blockDim.x + threadIdx.x;
    for (uint32_t i = first; i < s.n_orders; i += step) {
        const int32_t slot = s.order_to_style[i];
        order_to_style[s.order_base + i] = slot < 0 ? -1 : slot + (int32_t)s.style_base;
    }
    for (uint32_t i = first; i < s.n_styles; i += step) {
        StyleRec r = s.styles[i];
        r.stop_first += s.stop_base;
        r.tex_first += s.texel_base;
        styles[s.style_base + i] = r;
        grads[s.style_base + i] = s.grads[i];
    }
    for (uint32_t i = first; i < s.n_stops; i += step) stops[s.stop_base + i] = s.stops[i];
    const uint2* tex = reinterpret_cast<const uint2*>(s.texels);  // one texel = 4 x u16 = 8 B
    for (uint32_t i = first; i < s.n_texels; i += step) texels[s.texel_base + i] = tex[i];
}

void launch_batch_tables(const BatchTableSrc* src, uint32_t n_src, uint32_t max_items, int32_t* order_to_style, StyleRec* styles,
                         GradRec* grads, StopRec* stops, uint16_t* texels, cudaStream_t st) {
    if (!n_src || !max_items) return;
    const uint32_t per_comp = std::min<uint32_t>((max_items + 255u) / 256u, 256u);
    batch_tables_kernel<<<dim3(per_comp, n_src), 256, 0, st>>>(src, order_to_style, styles, grads, stops,
                                                               reinterpret_cast<uint2*>(texels));
}


}  // namespace forma
