// Stage 3: on-device LSD radix sort of the packed u64 pixel segments on key
// bits [20, 64) — replaces crumsort::ParCrumSort (cpu/rasterizer.rs:162-164)
// and the WGSL block-merge sort (gpu/conveyor_sort/sort.wgsl).
//
// * Plan (host): the 44 key bits are three fields (tile_y | tile_x | layer, or
//   tile_y | layer | tile_x for the painter's carry pass). The caller knows an
//   upper bound of every field (largest tile coordinates seen by the line-setup
//   pass, number of layer orders), so only the low bits of each field that can
//   be set take part: digits of <= 8 bits over the concatenation of those bits
//   (paris@4K: 16 + 8 + 8 = 32 bits = 4 passes instead of 6). Exactly the
//   planned passes are launched; after an odd number the caller swaps buffers.
// * Large key-only sorts (the pixel segments): every pass is reduce-then-scan —
//   `radix_upsweep_kernel` (per-tile digit counts), `radix_tile_scan_kernel`
//   (global offset of every (tile, digit) run) and the persistent, TMA-staged
//   `radix_downsweep_wide_kernel` (stable warp match/popc ranking, digit-order
//   staging in shared memory, coalesced scatter): 24 B/key per pass, and no CTA
//   ever waits for another one (see the comment above those kernels). For the segment sort the
//   kernels that write the keys count the tiles' digits instead (TileCounts, option sort_counts):
//   `radix_chunk_totals_kernel` replaces the upsweep, 16 B/key per pass.
// * Small sorts and (key, u32 payload) pairs (the painter's cell / gap tables):
//   one upfront histogram kernel for all passes, or none when the kernel that wrote the keys
//   counted their digits (every pass CTA scans its 256 counts itself), then one single-sweep
//   ("onesweep") kernel per pass with decoupled look-back (16 B/key per pass;
//   latency-bound at these sizes). A persistent single-sweep kernel for the large sorts
//   was measured look-back-bound and removed in favour of the reduce-then-scan passes.
#include <mutex>
#include "cuda_common.cuh"
#include "kernels.h"

namespace forma {

static std::mutex g_sort_config_mu;  // guards the per-device kernel attributes set at first use


constexpr int kRadixBits = 8;
constexpr int kRadix = 1 << kRadixBits;
constexpr int kSortThreads = 256;
constexpr int kSortWarps = kSortThreads / 32;

constexpr uint32_t kFlagAggregate = 1u << 30;
constexpr uint32_t kFlagInclusive = 2u << 30;
constexpr uint32_t kFlagMask = 3u << 30;
constexpr uint32_t kValueMask = ~kFlagMask;

__device__ __forceinline__ uint32_t ld_relaxed(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

static uint32_t bit_length(uint64_t v) {
    uint32_t n = 0;
    while (v) {
        ++n;
        v >>= 1;
    }
    return n;
}

// Field f occupies key bits [pos[f], pos[f] + maxw[f]); f = 0 is least
// significant. bound[f] = largest value field f can take.
SortPlan make_sort_plan(const KeyLayout& layout, const uint64_t bound[3]) {
    SortPlan plan{};
    uint32_t w[3], total = 0;
    for (int f = 0; f < 3; ++f) {
        w[f] = bit_length(bound[f]);
        if (w[f] > layout.maxw[f]) w[f] = layout.maxw[f];
        total += w[f];
    }
    plan.total_bits = total;
    plan.n_passes = (total + kRadixBits - 1) / kRadixBits;
    uint32_t lo = 0;  // position in the virtual (compacted) key
    for (uint32_t k = 0; k < plan.n_passes; ++k) {
        DigitSpec& d = plan.pass[k];
        uint32_t remaining = total - lo, left = plan.n_passes - k;
        uint32_t bits = (remaining + left - 1) / left;  // spread evenly, e.g. 38 bits -> 8,8,8,7,7
        d.bits = (uint8_t)bits;
        uint32_t hi = lo + bits, base = 0, got = 0;
        int r = 0;
        for (int f = 0; f < 3; ++f) {  // intersect [lo, hi) with field f's slice [base, base + w[f])
            uint32_t a = lo > base ? lo : base, b = hi < base + w[f] ? hi : base + w[f];
            if (b > a) {
                d.shift[r] = (uint8_t)(layout.pos[f] + (a - base));
                d.width[r] = (uint8_t)(b - a);
                d.lsh[r] = (uint8_t)got;
                got += b - a;
                ++r;
            }
            base += w[f];
        }
        lo = hi;
    }
    return plan;
}

// `n_dev` (optional): the key count in device memory; `n` is then only its upper bound (the
// count may not be known on the host when the sort is launched, see Renderer::build_tables). A
// count above the bound means that the producer overflowed its buffers: nothing is sorted.
__device__ __forceinline__ uint32_t resolve_key_count(uint32_t n, const uint32_t* __restrict__ n_dev) {
    if (!n_dev) return n;
    const uint32_t c = *n_dev;
    return c > n ? 0u : c;
}

// Counts every digit of every planned pass in one read of the keys.
__global__ void __launch_bounds__(kSortThreads) radix_hist_kernel(const uint64_t* __restrict__ keys, uint32_t n, SortPlan plan,
                                                                uint32_t* __restrict__ hist /*[passes][256]*/,
                                                                const uint32_t* __restrict__ n_dev) {
    chain_begin();
    n = resolve_key_count(n, n_dev);
    __shared__ uint32_t s_hist[kMaxSortPasses][kRadix];
    for (int i = threadIdx.x; i < kMaxSortPasses * kRadix; i += kSortThreads) (&s_hist[0][0])[i] = 0;
    __syncthreads();
    const uint32_t np = plan.n_passes;
    uint32_t stride = gridDim.x * kSortThreads;
    for (uint32_t i = blockIdx.x * kSortThreads + threadIdx.x; i < n; i += stride) {
        uint64_t k = keys[i];
#pragma unroll
        for (uint32_t p = 0; p < (uint32_t)kMaxSortPasses; ++p)
            if (p < np) atomicAdd(&s_hist[p][digit_of(k, plan.pass[p])], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kMaxSortPasses * kRadix; i += kSortThreads) {
        uint32_t v = (&s_hist[0][0])[i];
        if (v) atomicAdd(&hist[i], v);
    }
}

template <bool kPairs, int kItems>
__global__ void __launch_bounds__(kSortThreads, kItems == 16 ? 3 : 6)
    onesweep_pass_kernel(const uint64_t* __restrict__ keys_in, uint64_t* __restrict__ keys_out,
                         const uint32_t* __restrict__ vals_in, uint32_t* __restrict__ vals_out, uint32_t n, DigitSpec spec,
                         const uint32_t* __restrict__ digit_counts /*[256]: keys per digit (radix_hist_kernel)*/,
                         uint32_t* __restrict__ lb /*[tiles][256], zeroed*/, uint32_t* __restrict__ tile_counter,
                         const uint32_t* __restrict__ n_dev) {
    chain_begin();
    n = resolve_key_count(n, n_dev);
    constexpr int kTileKeys = kSortThreads * kItems;
    __shared__ uint64_t s_keys[kTileKeys];
    __shared__ uint32_t s_warp_hist[kSortWarps][kRadix];
    __shared__ uint32_t s_digit_start[kRadix];
    __shared__ uint32_t s_global_base[kRadix];
    __shared__ uint32_t s_warp_tot[kSortWarps];
    __shared__ uint32_t s_hist_tot[kSortWarps];
    __shared__ uint32_t s_tile;

    const uint32_t t = threadIdx.x, warp = t >> 5, lane = t & 31u;
    if (t == 0) s_tile = atomicAdd(tile_counter, 1u);
    for (int i = t; i < kSortWarps * kRadix; i += kSortThreads) (&s_warp_hist[0][0])[i] = 0;
    // Every CTA turns the pass's digit counts into exclusive offsets itself (256 values).
    const uint32_t hist_count = digit_counts[t];
    const uint32_t hist_incl = warp_inclusive_scan(hist_count);
    if (lane == 31) s_hist_tot[warp] = hist_incl;
    __syncthreads();
    uint32_t digit_offset = hist_incl - hist_count;  // first output position of digit t
    for (uint32_t w = 0; w < warp; ++w) digit_offset += s_hist_tot[w];
    const uint32_t tile = s_tile;
    const uint32_t base = tile * (uint32_t)kTileKeys;
    if (base >= n) return;  // a tile beyond the (device-side) key count: tiles are taken in order, nobody waits for it
    const uint32_t valid = min((uint32_t)kTileKeys, n - base);

    // Warp-striped load: warp w owns keys [w*32*kItems, (w+1)*32*kItems) of the tile.
    uint64_t key[kItems];
    const uint32_t warp_base = base + warp * (32u * kItems);
#pragma unroll
    for (int i = 0; i < kItems; ++i) {
        uint32_t idx = warp_base + i * 32u + lane;
        key[i] = idx < n ? keys_in[idx] : ~0ull;
    }

    // Stable rank of every key among the keys of its warp with the same digit.
    // Out-of-range slots of the last tile get the largest digit so that they
    // rank after every real key.
    uint32_t rank[kItems];
    const uint32_t lt_mask = (1u << lane) - 1u;
    const uint32_t max_digit = (1u << spec.bits) - 1u;
#pragma unroll
    for (int i = 0; i < kItems; ++i) {
        uint32_t idx = warp_base + i * 32u + lane;
        uint32_t d = idx < n ? digit_of(key[i], spec) : max_digit;
        uint32_t peers = __match_any_sync(kFullMask, d);
        uint32_t leader = __ffs(peers) - 1;
        uint32_t old = 0;
        if (lane == leader) {
            old = s_warp_hist[warp][d];
            s_warp_hist[warp][d] = old + __popc(peers);
        }
        old = __shfl_sync(kFullMask, old, leader);
        rank[i] = (old + __popc(peers & lt_mask)) | (d << 16);  // rank < 4096, digit < 256
        __syncwarp();
    }
    __syncthreads();

    // Thread t owns digit t: exclusive offsets of each warp, tile count.
    uint32_t count = 0;
#pragma unroll
    for (int w = 0; w < kSortWarps; ++w) {
        uint32_t c = s_warp_hist[w][t];
        s_warp_hist[w][t] = count;
        count += c;
    }
    // Publish this tile's digit count as early as possible.
    uint32_t* my_slot = lb + (size_t)tile * kRadix + t;
    if (tile != 0) st_relaxed(my_slot, kFlagAggregate | count);

    // Exclusive scan of the tile's digit counts (local layout in shared memory).
    uint32_t incl = warp_inclusive_scan(count);
    if (lane == 31) s_warp_tot[warp] = incl;
    __syncthreads();
    uint32_t dstart = incl - count;
    for (uint32_t w = 0; w < warp; ++w) dstart += s_warp_tot[w];
    s_digit_start[t] = dstart;

    // Decoupled look-back: exclusive count of digit t over all previous tiles,
    // four predecessors in flight at a time. The padding slots of the last tile
    // are counted under max_digit; no tile follows it, so nobody consumes that.
    {
        uint32_t prefix = 0;
        int32_t p = (int32_t)tile - 1;
        bool done = p < 0;
        while (!done) {
            uint32_t v[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] = (p - j >= 0) ? ld_relaxed(lb + (size_t)(p - j) * kRadix + t) : kFlagInclusive;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (done) break;
                uint32_t flag = v[j] & kFlagMask;
                if (flag == 0) {  // not published yet: retry from here
                    p -= j;
                    goto retry;
                }
                prefix += v[j] & kValueMask;
                if (flag == kFlagInclusive) done = true;
            }
            p -= 4;
        retry:;
        }
        st_relaxed(my_slot, kFlagInclusive | (prefix + count));
        s_global_base[t] = digit_offset + prefix - dstart;
    }
    __syncthreads();

    // Stage the tile in shared memory in digit order.
#pragma unroll
    for (int i = 0; i < kItems; ++i) {
        uint32_t d = rank[i] >> 16;
        uint32_t pos = s_digit_start[d] + s_warp_hist[warp][d] + (rank[i] & 0xFFFFu);
        s_keys[pos] = key[i];
        rank[i] = pos;
    }
    __syncthreads();

    uint32_t out_idx[kItems];
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
        uint32_t p = t + k * kSortThreads;
        out_idx[k] = 0xFFFFFFFFu;
        if (p < valid) {
            uint64_t kk = s_keys[p];
            uint32_t o = s_global_base[digit_of(kk, spec)] + p;
            keys_out[o] = kk;
            out_idx[k] = o;
        }
    }
    if (kPairs) {
        __syncthreads();
        uint32_t* s_vals = reinterpret_cast<uint32_t*>(s_keys);
#pragma unroll
        for (int i = 0; i < kItems; ++i) {
            uint32_t idx = warp_base + i * 32u + lane;
            if (idx < n) s_vals[rank[i]] = vals_in[idx];
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < kItems; ++k) {
            uint32_t p = t + k * kSortThreads;
            if (out_idx[k] != 0xFFFFFFFFu) vals_out[out_idx[k]] = s_vals[p];
        }
    }
}

// ---------------------------------------------------------------------------
// 1-D TMA (cp.async.bulk) + mbarrier helpers used by the downsweep's tile staging.
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok = 0;
    while (!ok) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    }
}

// ---------------------------------------------------------------------------
// Reduce-then-scan passes for large key-only sorts (the main pixel-segment
// sort). The look-back of the single-sweep kernels above serialises the tiles
// of a pass whatever the bandwidth; here no CTA ever waits for another one:
//   1. upsweep   — one CTA per tile counts the tile's digits     (reads  8 B/key)
//   2. tile scan — counts -> exclusive global offsets per (tile, digit)
//   3. downsweep — one CTA per tile ranks, stages in shared memory in digit
//                  order and writes coalesced runs        (reads + writes 8 B/key)
// i.e. 24 B/key per pass instead of 16, but every kernel streams.
// ---------------------------------------------------------------------------
constexpr int kDsItems = 16;
constexpr int kDsTile = kSortThreads * kDsItems;  // 4096 keys = 32 KB
static_assert(kDsTile == (int)kSortTileKeys, "the tiles of TileCounts");
// The tile scan works on chunks of consecutive tiles (one CTA each) grouped into super-chunks
// (kChunksPerSuper, kMaxSupers, kTotalsRows: kernels.h): a CTA needs 32 + 16 loads per digit to
// know what precedes it.

__global__ void __launch_bounds__(kSortThreads) radix_upsweep_kernel(const uint64_t* __restrict__ keys, uint32_t n, DigitSpec spec,
                                                                   uint32_t* __restrict__ tile_hist /*[tiles][256]*/,
                                                                   uint32_t* __restrict__ totals /*[kTotalsRows][256], zeroed*/,
                                                                   uint32_t tiles_per_chunk) {
    chain_begin();
    __shared__ uint32_t s_hist[kRadix];
    const uint32_t t = threadIdx.x, tile = blockIdx.x;
    s_hist[t] = 0;
    const uint32_t base = tile * (uint32_t)kDsTile;
    uint64_t key[kDsItems];
#pragma unroll
    for (int i = 0; i < kDsItems; ++i) {
        uint32_t idx = base + (uint32_t)i * kSortThreads + t;
        key[i] = idx < n ? keys[idx] : 0ull;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < kDsItems; ++i) {
        uint32_t idx = base + (uint32_t)i * kSortThreads + t;
        if (idx < n) atomicAdd(&s_hist[digit_of(key[i], spec)], 1u);
    }
    __syncthreads();
    const uint32_t c = s_hist[t];
    tile_hist[(size_t)tile * kRadix + t] = c;
    if (c) {
        const uint32_t chunk = tile / tiles_per_chunk;
        atomicAdd(&totals[(size_t)chunk * kRadix + t], c);
        atomicAdd(&totals[(size_t)(kMaxChunks + chunk / kChunksPerSuper) * kRadix + t], c);
    }
}

// Tile counts from the keys' producers (TileCounts): CTA c sums the counts of tiles
// [c * tiles_per_chunk, ...) into chunk row c (stores) and its super-chunk row (atomics, on rows the
// previous downsweep over this block left zero). Thread d owns digit d.
// n_dev (optional): the key count in device memory; `tiles` is then a bound, and the tiles past the
// count (all zero) are not read.
__global__ void __launch_bounds__(kRadix) radix_chunk_totals_kernel(const uint32_t* __restrict__ tile_hist,
                                                                  uint32_t* __restrict__ totals, uint32_t tiles,
                                                                  uint32_t tiles_per_chunk, const uint32_t* __restrict__ n_dev) {
    chain_begin();
    if (n_dev) tiles = min(tiles, (*n_dev + kSortTileKeys - 1u) / kSortTileKeys);
    const uint32_t d = threadIdx.x, c = blockIdx.x;
    const uint32_t t0 = c * tiles_per_chunk, t1 = min(tiles, t0 + tiles_per_chunk);
    uint32_t sum = 0;
    for (uint32_t tb = t0; tb < t1; tb += 8u) {
        uint32_t v[8];
#pragma unroll
        for (uint32_t k = 0; k < 8u; ++k) v[k] = (tb + k < t1) ? tile_hist[(size_t)(tb + k) * kRadix + d] : 0u;
#pragma unroll
        for (uint32_t k = 0; k < 8u; ++k) sum += v[k];
    }
    totals[(size_t)c * kRadix + d] = sum;
    if (sum) atomicAdd(&totals[(size_t)(kMaxChunks + c / kChunksPerSuper) * kRadix + d], sum);
}

// CTA c turns the digit counts of tiles [c * tiles_per_chunk, ...) into the
// global offset of each tile's first key of each digit. Thread d owns digit d.
// n_dev: as for radix_chunk_totals_kernel (the tiles past the count keep their zero counts).
__global__ void __launch_bounds__(kRadix) radix_tile_scan_kernel(uint32_t* __restrict__ tile_hist,
                                                               const uint32_t* __restrict__ totals, uint32_t tiles,
                                                               uint32_t tiles_per_chunk, const uint32_t* __restrict__ n_dev) {
    chain_begin();
    if (n_dev) tiles = min(tiles, (*n_dev + kSortTileKeys - 1u) / kSortTileKeys);
    __shared__ uint32_t s_warp_tot[kRadix / 32];
    const uint32_t d = threadIdx.x, c = blockIdx.x, sc = c / kChunksPerSuper;
    uint32_t before = 0, total = 0;  // keys of digit d in earlier chunks / in all chunks
    {
        uint32_t v[kMaxSupers], w[kChunksPerSuper];
#pragma unroll
        for (uint32_t k = 0; k < kMaxSupers; ++k) v[k] = totals[(size_t)(kMaxChunks + k) * kRadix + d];
#pragma unroll
        for (uint32_t k = 0; k < kChunksPerSuper; ++k) w[k] = totals[(size_t)(sc * kChunksPerSuper + k) * kRadix + d];
#pragma unroll
        for (uint32_t k = 0; k < kMaxSupers; ++k) {
            total += v[k];
            if (k < sc) before += v[k];
        }
#pragma unroll
        for (uint32_t k = 0; k < kChunksPerSuper; ++k)
            if (sc * kChunksPerSuper + k < c) before += w[k];
    }
    uint32_t incl = warp_inclusive_scan(total);
    if ((d & 31u) == 31u) s_warp_tot[d >> 5] = incl;
    __syncthreads();
    uint32_t running = incl - total + before;
    for (uint32_t w = 0; w < (d >> 5); ++w) running += s_warp_tot[w];
    const uint32_t t0 = c * tiles_per_chunk, t1 = min(tiles, t0 + tiles_per_chunk);
    for (uint32_t tb = t0; tb < t1; tb += 8u) {
        uint32_t v[8];
#pragma unroll
        for (uint32_t k = 0; k < 8u; ++k) v[k] = (tb + k < t1) ? tile_hist[(size_t)(tb + k) * kRadix + d] : 0u;
#pragma unroll
        for (uint32_t k = 0; k < 8u; ++k) {
            if (tb + k < t1) tile_hist[(size_t)(tb + k) * kRadix + d] = running;
            running += v[k];
        }
    }
}

// Persistent downsweep: CTA c owns tiles c, c + G, ...; the keys of the next
// kDsStages - 1 tiles of the CTA are always in flight as 32 KB `cp.async.bulk`
// (1-D TMA) copies into a shared-memory ring, so the HBM reads never wait for
// the ranking or the stores of the current tile. The stage that delivered a
// tile is reused as its digit-order staging buffer before the write-out.
constexpr int kDsStages = 3;
// 512 threads x 8 keys per 4096-key tile: the ranking chain per warp is short and an SM
// holds 32 warps (2 CTAs, <= 64 registers) — a 256-thread x 16-key version measured
// short-scoreboard / fixed-latency bound at low occupancy.
// Per-warp digit counters are u16 (a tile has 4096 keys) so that the shared memory still
// fits twice per SM.
constexpr int kWideThreads = 512;
constexpr int kWideItems = 8;
constexpr int kWideWarps = kWideThreads / 32;
static_assert(kWideThreads * kWideItems == kDsTile, "same tile as the upsweep");
struct DownsweepWideSmem {
    uint64_t stage[kDsStages][kDsTile];      // 3 x 32 KB
    uint16_t warp_hist[kWideWarps][kRadix];  // 8 KB
    uint32_t digit_start[kRadix];
    uint32_t global_base[kRadix];
    uint32_t warp_tot[kRadix / 32];
    uint64_t bar[kDsStages];
};

// kCount: every key written also counts for the next pass: digit next.spec, at the tile of its
// destination (TileCounts), one atomic per group of lanes with the same (tile, digit).
// kZero: what the pass consumed is left zero for the next producer (TileCounts): every tile's
// offsets once read, and the pass's super-chunk rows `supers` (CTA 0; the tile scan read them).
// n_dev (kZero only): the key count in device memory, `n` and `tiles` being bounds (resolve_key_count).
// The tiles past the count hold no key and zero counts, which the tile scan left alone.
template <bool kCount, bool kZero>
__global__ void __launch_bounds__(kWideThreads, 2)
    radix_downsweep_wide_kernel(const uint64_t* __restrict__ keys_in, uint64_t* __restrict__ keys_out, uint32_t n, DigitSpec spec,
                                uint32_t* __restrict__ tile_base, uint32_t tiles, CountArgs next, uint32_t* __restrict__ supers,
                                const uint32_t* __restrict__ n_dev) {
    chain_begin();
    extern __shared__ __align__(128) unsigned char smem_raw[];
    DownsweepWideSmem& S = *reinterpret_cast<DownsweepWideSmem*>(smem_raw);
    const uint32_t t = threadIdx.x, warp = t >> 5, lane = t & 31u;
    const uint32_t G = gridDim.x;
    if (t == 0) {
#pragma unroll
        for (int s = 0; s < kDsStages; ++s) mbar_init(&S.bar[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    auto issue = [&](uint32_t tile, uint32_t st) {  // thread 0 only
        uint32_t base = tile * (uint32_t)kDsTile;
        uint32_t valid = min((uint32_t)kDsTile, n - base);
        uint32_t bytes = ((valid + 1u) & ~1u) * 8u;  // multiple of 16 B (the buffers have one key of slack)
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_expect_tx(&S.bar[st], bytes);
        tma_load_1d(&S.stage[st][0], keys_in + base, bytes, &S.bar[st]);
    };

    uint32_t tile = blockIdx.x;
    if constexpr (kZero) {
        if (tile == 0)
            for (uint32_t i = t; i < kMaxSupers * (uint32_t)kRadix; i += kWideThreads) supers[i] = 0;
        if (n_dev) {
            n = resolve_key_count(n, n_dev);
            tiles = (n + (uint32_t)kDsTile - 1u) / (uint32_t)kDsTile;
        }
    }
    if (tile >= tiles) return;
    if (t == 0) {
#pragma unroll
        for (int s = 0; s < kDsStages - 1; ++s)
            if (tile + (uint32_t)s * G < tiles) issue(tile + (uint32_t)s * G, (uint32_t)s);
    }
    uint32_t st = 0, phases = 0;
    const uint32_t lt_mask = (1u << lane) - 1u;
    const uint32_t max_digit = (1u << spec.bits) - 1u;

    for (; tile < tiles; tile += G) {
        if (t == 0 && tile + (uint32_t)(kDsStages - 1) * G < tiles)
            issue(tile + (uint32_t)(kDsStages - 1) * G, (st + kDsStages - 1u) % kDsStages);
        uint32_t gbase = 0;
        if (t < (uint32_t)kRadix) gbase = tile_base[(size_t)tile * kRadix + t];
        {
            uint32_t* z = reinterpret_cast<uint32_t*>(&S.warp_hist[0][0]);
            for (int i = t; i < kWideWarps * kRadix / 2; i += kWideThreads) z[i] = 0;
        }
        const uint32_t base = tile * (uint32_t)kDsTile;
        const uint32_t valid = min((uint32_t)kDsTile, n - base);
        mbar_wait(&S.bar[st], (phases >> st) & 1u);
        phases ^= 1u << st;
        uint64_t* stage = S.stage[st];

        uint64_t key[kWideItems];
        const uint32_t wofs = warp * (32u * kWideItems);
#pragma unroll
        for (int i = 0; i < kWideItems; ++i) key[i] = stage[wofs + i * 32u + lane];
        __syncthreads();  // everybody has its keys (and the zeroed histograms are visible)

        uint32_t rank[kWideItems];
#pragma unroll
        for (int i = 0; i < kWideItems; ++i) {
            uint32_t slot = wofs + i * 32u + lane;
            uint32_t d = slot < valid ? digit_of(key[i], spec) : max_digit;
            uint32_t peers = __match_any_sync(kFullMask, d);
            uint32_t leader = __ffs(peers) - 1;
            uint32_t old = 0;
            if (lane == leader) {
                old = S.warp_hist[warp][d];
                S.warp_hist[warp][d] = (uint16_t)(old + __popc(peers));
            }
            old = __shfl_sync(kFullMask, old, leader);
            rank[i] = (old + __popc(peers & lt_mask)) | (d << 16);
            __syncwarp();
        }
        __syncthreads();

        if (t < (uint32_t)kRadix) {
            uint32_t count = 0;
#pragma unroll
            for (int w = 0; w < kWideWarps; ++w) {
                uint32_t c = S.warp_hist[w][t];
                S.warp_hist[w][t] = (uint16_t)count;
                count += c;
            }
            uint32_t incl = warp_inclusive_scan(count);
            if (lane == 31) S.warp_tot[warp] = incl;
            S.digit_start[t] = incl - count;  // completed below with the totals of the lower warps
            S.global_base[t] = gbase;
        }
        __syncthreads();
        if (t < (uint32_t)kRadix) {
            uint32_t add = 0;
            for (uint32_t w = 0; w < warp; ++w) add += S.warp_tot[w];
            uint32_t dstart = S.digit_start[t] + add;
            S.digit_start[t] = dstart;
            S.global_base[t] -= dstart;
        }
        __syncthreads();

#pragma unroll
        for (int i = 0; i < kWideItems; ++i) {
            uint32_t d = rank[i] >> 16;
            stage[S.digit_start[d] + S.warp_hist[warp][d] + (rank[i] & 0xFFFFu)] = key[i];
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < kWideItems; ++k) {
            uint32_t p = t + k * kWideThreads;
            if (p < valid) {
                uint64_t kk = stage[p];
                const uint32_t dst = S.global_base[digit_of(kk, spec)] + p;
                keys_out[dst] = kk;
                if constexpr (kCount) {
                    const uint32_t dt = dst / kSortTileKeys, d = digit_of(kk, next.spec);
                    const uint32_t peers = __match_any_sync(__activemask(), (dt << 8) | d);
                    if (lane == __ffs(peers) - 1u) add_tile_count(next, dt, d, (uint32_t)__popc(peers));
                }
            }
        }
        // (Zeroed here, long after the load: a store right behind it would wait for the load.)
        if (kZero && t < (uint32_t)kRadix) tile_base[(size_t)tile * kRadix + t] = 0;
        __syncthreads();  // the stage is free again: the next iteration refills it by TMA
        st = (st + 1u) % kDsStages;
    }
}

static uint32_t tiles_for(uint32_t n, int items) { return (n + kSortThreads * items - 1) / (kSortThreads * items); }
// Keys per thread: 4096-key tiles from 2^19 keys on (fewer tiles = a shorter look-back chain for
// the single-sweep pair sorts, and the reduce-then-scan path for key-only sorts), 1024-key tiles
// below that so that small sorts still spread over the SMs (option sort_big_log2, default 19).
static int items_for(uint32_t n) { return n >= (1u << options().sort_big_log2) ? 16 : 4; }

// scratch layout (u32 words): hist[6][256] | tile_counter[8] | lookback[6][tiles][256]
// or, for the reduce-then-scan passes: totals[6][kTotalsRows][256] | tile_hist[tiles][256]
size_t radix_scratch_bytes(uint32_t n) {
    size_t words = (size_t)kMaxSortPasses * kRadix + 8 + (size_t)kMaxSortPasses * tiles_for(n, items_for(n)) * kRadix;
    size_t scan_words = (size_t)kMaxSortPasses * kTotalsRows * kRadix + (size_t)tiles_for(n, kDsItems) * kRadix;
    return (words > scan_words ? words : scan_words) * sizeof(uint32_t) + 256;
}
// With the histogram counted elsewhere: tile_counter[8] | lookback[passes][tiles][256].
size_t sort_lookback_bytes(uint32_t n, const SortPlan& plan) {
    return (8 + (size_t)plan.n_passes * tiles_for(n, items_for(n)) * kRadix) * sizeof(uint32_t);
}

void launch_radix_hist(const uint64_t* keys, uint32_t n, const SortPlan& plan, uint32_t* hist, const uint32_t* n_dev,
                       cudaStream_t stream) {
    uint32_t hist_blocks = min(tiles_for(n, 16) * 4u, (uint32_t)device_sm_count() * 8u);
    launch_chained(radix_hist_kernel, hist_blocks, kSortThreads, 0, stream, keys, n, plan, hist, n_dev);
}

template <bool kPairs, int kItems>
static void launch_passes(uint64_t* keys, uint64_t* keys_tmp, uint32_t* vals, uint32_t* vals_tmp, uint32_t n,
                          const SortPlan& plan, const uint32_t* hist, uint32_t* lookback, uint32_t* counters, uint32_t tiles,
                          cudaStream_t stream, const uint32_t* n_dev) {
    static bool configured[kMaxDevices] = {false};
    const int dev = current_device_index();
    {
        std::lock_guard<std::mutex> lk(g_sort_config_mu);  // several host threads may render on one device
        if (!configured[dev]) {  // let several CTAs of 18-43 KB share one SM's shared memory
            cudaFuncSetAttribute(onesweep_pass_kernel<kPairs, kItems>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
            configured[dev] = true;
        }
    }
    for (uint32_t p = 0; p < plan.n_passes; ++p) {
        const uint64_t* kin = (p & 1u) ? keys_tmp : keys;
        uint64_t* kout = (p & 1u) ? keys : keys_tmp;
        const uint32_t* vin = (p & 1u) ? vals_tmp : vals;
        uint32_t* vout = (p & 1u) ? vals : vals_tmp;
        launch_chained(onesweep_pass_kernel<kPairs, kItems>, tiles, kSortThreads, 0, stream,
            kin, kout, vin, vout, n, plan.pass[p], hist + p * kRadix, lookback + (size_t)p * tiles * kRadix, counters + p, n_dev);
    }
}

// The persistent downsweep's grid on the current device: 2 CTAs per SM (0: the occupancy query
// failed, and the reduce-then-scan passes are not used). The attribute is set at first use.
static int downsweep_grid() {
    static int wide_grids[kMaxDevices];
    static bool ds_configured[kMaxDevices] = {false};
    const int cur_dev = current_device_index();
    // Under a lock: a second host thread rendering on the same device (a slice of a host-frame
    // pipeline) must not see the flag before the attributes are set and the grid is known.
    std::lock_guard<std::mutex> lk(g_sort_config_mu);
    if (!ds_configured[cur_dev]) {
        // The plain build, and the builds that leave the tile counts zero (+ count the next pass).
        int per_sm_all = 1 << 30;
        for (auto* k : {radix_downsweep_wide_kernel<false, false>, radix_downsweep_wide_kernel<false, true>,
                        radix_downsweep_wide_kernel<true, true>}) {
            cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DownsweepWideSmem));
            int per_sm = 0;
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, kWideThreads, sizeof(DownsweepWideSmem));
            per_sm_all = min(per_sm_all, per_sm);  // one grid for all: a persistent CTA must never wait for a slot
        }
        wide_grids[cur_dev] = per_sm_all > 0 ? per_sm_all * device_sm_count() : 0;
        ds_configured[cur_dev] = true;
    }
    return wide_grids[cur_dev];
}

bool radix_sort_scans(uint32_t n) {
    return n >= 2 && items_for(n) == 16 && n >= (1u << options().sort_scan_log2) && downsweep_grid() > 0;
}

SortResult launch_radix_sort(uint64_t* keys, uint64_t* keys_tmp, uint32_t* vals, uint32_t* vals_tmp, uint32_t n,
                             const SortPlan& plan, void* scratch, cudaStream_t stream, cudaEvent_t* pass_events,
                             const uint32_t* n_dev, const uint32_t* hist_ready, const TileCounts* counts, uint32_t* keep_counts) {
    SortResult res{0, false};
    if (n < 2 || plan.n_passes == 0) return res;
    const int items = items_for(n);
    const uint32_t tiles = tiles_for(n, items);
    // A device count (n_dev) takes the reduce-then-scan passes only with the emit's pass-0 counts.
    const bool counted = counts && tiles <= counts->tile_cap;
    if (!vals && items == 16 && n >= (1u << options().sort_scan_log2) && (!n_dev || (counted && counts->pass0)) && !hist_ready) {
        const int wide_grid = downsweep_grid();
        if (wide_grid > 0) {
            const uint32_t grid = min(tiles, (uint32_t)wide_grid);
            if (counted) {
                // Pass p's tile counts are in block p & 1: counted by the emit pass (pass 0, when
                // counts->pass0) or the upsweep (pass 0 otherwise), then by the downsweep of pass p - 1.
                const uint32_t tpc = counts->tiles_per_chunk;
                const uint32_t chunks = (tiles + tpc - 1) / tpc;
                for (uint32_t p = 0; p < plan.n_passes; ++p) {
                    const uint64_t* kin = (p & 1u) ? keys_tmp : keys;
                    uint64_t* kout = (p & 1u) ? keys : keys_tmp;
                    if (p == 0 && !counts->pass0) {  // the upsweep stores the tile counts and adds to zeroed totals
                        cudaMemsetAsync(counts->totals(0), 0, (size_t)kTotalsRows * kRadix * sizeof(uint32_t), stream);
                        launch_chained(radix_upsweep_kernel, tiles, kSortThreads, 0, stream, kin, n, plan.pass[0], counts->hist(0), counts->totals(0), tpc);
                    } else {
                        launch_chained(radix_chunk_totals_kernel, chunks, kRadix, 0, stream, counts->hist(p), counts->totals(p), tiles, tpc,
                                       n_dev);
                    }
                    if (keep_counts)
                        cudaMemcpyAsync(keep_counts + (size_t)p * tiles * kRadix, counts->hist(p), (size_t)tiles * kRadix * sizeof(uint32_t),
                                        cudaMemcpyDeviceToDevice, stream);
                    launch_chained(radix_tile_scan_kernel, chunks, kRadix, 0, stream, counts->hist(p), counts->totals(p), tiles, tpc, n_dev);
                    if (pass_events) cudaEventRecord(pass_events[3 * p + 1], stream);
                    uint32_t* supers = counts->totals(p) + (size_t)kMaxChunks * kRadix;
                    if (p + 1 < plan.n_passes) {
                        const CountArgs next{counts->hist(p + 1), plan.pass[p + 1]};
                        launch_chained(radix_downsweep_wide_kernel<true, true>, grid, kWideThreads, sizeof(DownsweepWideSmem), stream,
                            kin, kout, n, plan.pass[p], counts->hist(p), tiles, next, supers, n_dev);
                    } else {
                        launch_chained(radix_downsweep_wide_kernel<false, true>, grid, kWideThreads, sizeof(DownsweepWideSmem), stream,
                            kin, kout, n, plan.pass[p], counts->hist(p), tiles, CountArgs{}, supers, n_dev);
                    }
                    if (pass_events && p + 1 < plan.n_passes) cudaEventRecord(pass_events[3 * p + 2], stream);
                }
                res.timed_passes = pass_events ? (int)plan.n_passes : 0;
                res.launches = 3 * (int)plan.n_passes;
                res.in_tmp = (plan.n_passes & 1u) != 0u;
                return res;
            }
            const uint32_t tiles_per_chunk = (tiles + kMaxChunks - 1) / kMaxChunks;
            const uint32_t chunks = (tiles + tiles_per_chunk - 1) / tiles_per_chunk;
            uint32_t* chunk_totals = static_cast<uint32_t*>(scratch);
            uint32_t* tile_hist = chunk_totals + (size_t)kMaxSortPasses * kTotalsRows * kRadix;
            cudaMemsetAsync(chunk_totals, 0, (size_t)plan.n_passes * kTotalsRows * kRadix * sizeof(uint32_t), stream);
            for (uint32_t p = 0; p < plan.n_passes; ++p) {
                const uint64_t* kin = (p & 1u) ? keys_tmp : keys;
                uint64_t* kout = (p & 1u) ? keys : keys_tmp;
                uint32_t* totals = chunk_totals + (size_t)p * kTotalsRows * kRadix;
                launch_chained(radix_upsweep_kernel, tiles, kSortThreads, 0, stream, kin, n, plan.pass[p], tile_hist, totals, tiles_per_chunk);
                launch_chained(radix_tile_scan_kernel, chunks, kRadix, 0, stream, tile_hist, totals, tiles, tiles_per_chunk,
                               (const uint32_t*)nullptr);
                if (pass_events) cudaEventRecord(pass_events[3 * p + 1], stream);
                launch_chained(radix_downsweep_wide_kernel<false, false>, grid, kWideThreads, sizeof(DownsweepWideSmem), stream,
                    kin, kout, n, plan.pass[p], tile_hist, tiles, CountArgs{}, nullptr, (const uint32_t*)nullptr);
                if (pass_events && p + 1 < plan.n_passes) cudaEventRecord(pass_events[3 * p + 2], stream);
            }
            res.timed_passes = pass_events ? (int)plan.n_passes : 0;
            res.launches = 3 * (int)plan.n_passes;
            res.in_tmp = (plan.n_passes & 1u) != 0u;
            return res;
        }
        // (occupancy query failed: fall through to the single-sweep passes)
    }
    const uint32_t* hist = hist_ready;
    uint32_t* counters = static_cast<uint32_t*>(scratch);
    if (!hist_ready) {
        uint32_t* h = static_cast<uint32_t*>(scratch);
        counters = h + kMaxSortPasses * kRadix;
        size_t total_words = (size_t)kMaxSortPasses * kRadix + 8 + (size_t)plan.n_passes * tiles * kRadix;
        cudaMemsetAsync(scratch, 0, total_words * sizeof(uint32_t), stream);
        launch_radix_hist(keys, n, plan, h, n_dev, stream);
        res.launches = 1;
        hist = h;
    }
    uint32_t* lookback = counters + 8;
    if (vals) {
        if (items == 16) launch_passes<true, 16>(keys, keys_tmp, vals, vals_tmp, n, plan, hist, lookback, counters, tiles, stream, n_dev);
        else launch_passes<true, 4>(keys, keys_tmp, vals, vals_tmp, n, plan, hist, lookback, counters, tiles, stream, n_dev);
    } else {
        if (items == 16) launch_passes<false, 16>(keys, keys_tmp, nullptr, nullptr, n, plan, hist, lookback, counters, tiles, stream, n_dev);
        else launch_passes<false, 4>(keys, keys_tmp, nullptr, nullptr, n, plan, hist, lookback, counters, tiles, stream, n_dev);
    }
    res.launches += (int)plan.n_passes;
    res.in_tmp = (plan.n_passes & 1u) != 0u;
    return res;
}

}  // namespace forma
