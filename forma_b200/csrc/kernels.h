// Host-callable launchers of the CUDA kernels (implemented in kernels_*.cu).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>

#include "device_types.h"

struct forma_layer_stats;  // include/forma_b200.h

namespace forma {

// Schedule switches (none of them changes results). Initialised from the environment
// (FORMA_<NAME>) on first use and settable at run time through forma_set_option(), which is
// how the parity tests cover every value (tests/test_gpu_options.py).
struct Options {
    int speculate = 1;       // launch kernels ahead of their count read-backs (0: strictly after)
    int band_copy = 1;       // host frames: paint / copy back in bands of tile rows
    int copy_bands = 4;      //   ... how many (1..16)
    int sort_full_key = 0;   // 1: sort the layer digits even when the inserts are in layer order
    int sort_big_log2 = 19;  // key count from which the 4096-key tiles / reduce-then-scan passes are used
    int sort_scan_log2 = 22; // key-only sorts: key count from which the reduce-then-scan passes replace the single-sweep ones
    int sort_counts = 1;     // reduce-then-scan segment sorts: per-tile digit counts from the kernels that write the keys (0: an upsweep pass per digit)
    int test_gap_cap = 0;    // test hook: cap of the speculative carry-only-entry launch (0 = none)
    int paint_lpt = 1;       // heavy tiles first (longest-processing-time order) in the paint kernel
    int paint_wide = 0;      // 1: the general paint kernel built for 6 CTAs / SM (up to 168 registers) instead of 8 (128); sRGB8 frames only (float frames always use the 8-CTA build)
    int paint_solid = 1;     // sRGB8 frames whose layers are all solid `Over` fills without clips are painted by the paint kernel's lean build (0: by the general one)
    int band_filter = 1;     // a render cropped to a band of rows only makes the band's geometry resident
    int sync_free = 1;       // painter tables without count read-backs when the previous frame's counts bound this one's (redone the slow way if they do not)
    int test_fast_shrink = 0;  // test hook: halve the bounds of the sync-free tables (forces the redo)
    int host_slices = 1;     // host frames: > 1 = that many tile-row slices rendered as independent upload -> render -> copy-back pipelines on their own streams.
                             //   Off by default: the slices' kernel chains do not overlap on the device (latency-bound kernels that fill the SMs), see DESIGN.md section 3
    int slice_bands = 2;     //   ... copy bands inside a slice
    int slice_min_points = 65536;  //   ... only for compositions of at least this many points
    int slice_chain = 1;     //   ... uploads issued slice after slice, each waiting for the one before (0: all at once from the slices' threads)
    int pdl = 1;             // chained launches: the frame's kernels launched with programmatic dependent launch (0: plain launches)
    int sync_free_sort = 1;  // single device frames: segment sort, tables and paint launched over the previous frame's segment count and sort plan, without the mid-frame count read-back (redone the slow way if they do not hold)
    int test_sort_bound = 0; // test hook: the segment-count bound of such a frame (0 = the previous count + 25 % + 4096)
};
Options& options();

// Arguments of the fused line-setup + pixel-grid-intersection kernels.
struct RasterArgs {
    const float* x;            // segment buffer (segment.rs:530-534)
    const float* y;
    const uint32_t* gid;       // geometry id per point, 0 = None
    uint32_t n_points;
    const int32_t* geom_slot;  // geom id -> layer slot, -1 = not in the composition
    uint32_t n_geoms;
    const LayerRec* layers;    // nullptr when no layer has a transform: then ...
    const uint32_t* layer_bits;// ... order | enabled << 21 per layer slot
    float width, height;       // render target in pixels
    float band_lo, band_hi;    // pixel rows painted by this GPU ([0, height) on one GPU)
};

// ---- kernels_raster.cu ------------------------------------------------------
void launch_flatten_eval(const SplineRec* splines, const PointRec* points, const uint8_t* kinds, const QuadRec* quads,
                         const FlattenJob* jobs, const JobXf* xfs, uint32_t n_jobs, uint32_t n_points,
                         uint32_t dst_base /* first point of the batch in the segment buffer */, float* x, float* y, uint32_t* gid,
                         cudaStream_t stream);
// Rebuilds the device-resident QuadRecs from the uploaded control points (quad_math.h).
void launch_quad_expand(const QuadUp* in, QuadRec* out, uint32_t n, cudaStream_t stream);
void launch_quad_expand_poly(const QuadUpPoly* in, QuadRec* out, uint32_t n, cudaStream_t stream);  // all weights 1
uint32_t raster_num_blocks(uint32_t n_points);
// block_sums: raster_num_blocks(n) entries, turned into exclusive offsets; total[0] = #segments.
// max_tile[0..1] = largest biased tile_x / tile_y any emitted segment can carry.
// A frame launched before its segment count is known on the host (Renderer::rasterize with a
// bound): the scan that produces the count also decides whether the frame's launches hold. They
// hold when n_lo <= count <= n_hi, count < 2^30 and the bit lengths of max_tile[0..1] are tx_bits
// and ty_bits (the sort plan they were made with is then the frame's own). Then *live_n = count
// and *paint_counter = 0; otherwise *live_n = 0 (every kernel that reads it does nothing) and
// *paint_counter = kPaintAbort (every paint ticket is past the frame's tiles: nothing is written).
struct CountCheck {
    uint32_t n_lo, n_hi, tx_bits, ty_bits;
    uint32_t* live_n;
    uint32_t* paint_counter;
};
constexpr uint32_t kPaintAbort = 0x80000000u;
void launch_line_count(const RasterArgs& args, uint32_t* block_sums, uint32_t* total, uint32_t* max_tile,
                       cudaStream_t stream, const CountCheck* check = nullptr);
// Segments at positions >= cap are dropped (speculative launches, see Renderer::rasterize).
// `counts` (optional): the digit of every stored segment is added to the counts of its 4096-key
// sort tile (TileCounts); dropped segments are not counted.
struct CountArgs;
void launch_raster_emit(const RasterArgs& args, const uint32_t* block_offsets, uint64_t* out, uint32_t cap, cudaStream_t stream,
                        const CountArgs* counts = nullptr);
// Views (see forma_renderer_render_views_device): the same line setup for n_views transforms of
// the composition, stacked top to bottom in one frame of n_views * rows tile rows. View b's line
// of layer transform T is transformed by C = V_b ∘ T in f32, `*` rounded on its own:
//   C.ux = fmaf(V.ux, T.ux, V.vx * T.uy)   C.vx = fmaf(V.ux, T.vx, V.vx * T.vy)
//   C.uy = fmaf(V.uy, T.ux, V.vy * T.uy)   C.vy = fmaf(V.uy, T.vx, V.vy * T.vy)
//   C.tx = fmaf(V.ux, T.tx, fmaf(V.vx, T.ty, V.tx))   C.ty = fmaf(V.uy, T.tx, fmaf(V.vy, T.ty, V.ty))
// (by V alone without T), and rasterized in its own frame's coordinates; only the tile row of
// the sort key moves: row t of view b becomes biased b * rows + t + 1, rows outside the view 0.
struct ViewArgs {
    const float* xf;  // n_views x 6 floats, [ux, vx, uy, vy, tx, ty] (forma_layer_set_transform order)
    uint32_t rows;    // tile rows per view: ceil(height / 16)
};
// As launch_line_count / launch_raster_emit: raster_num_blocks(n_points) * n_views block sums,
// view-major; max_tile[1] is the stacked bound.
void launch_line_count_views(const RasterArgs& args, const ViewArgs& views, uint32_t n_views, uint32_t* block_sums, uint32_t* total,
                             uint32_t* max_tile, cudaStream_t stream);
void launch_raster_emit_views(const RasterArgs& args, const ViewArgs& views, uint32_t n_views, const uint32_t* block_offsets,
                              uint64_t* out, uint32_t cap, cudaStream_t stream, const CountArgs* counts = nullptr);
// Poses (see forma_renderer_render_poses_device): the views' stacked frame of n_frames frames, but
// instead of a view transform, frame b gives the layer at an order o of the window
// [first_order, first_order + n_orders) the transform and enabled bit of its record
// recs[b * n_orders + o - first_order]. Layers outside the window keep their own.
struct PoseRec {                    // 32 B
    float ux, uy, vx, vy, tx, ty;   // LayerRec order
    uint32_t bits;                  // has_xf | enabled << 1 (an identity transform is no transform)
    uint32_t pad;
};
struct PoseArgs {
    const PoseRec* recs;            // n_frames x n_orders, frame-major
    uint32_t first_order, n_orders;
    uint32_t rows;                  // tile rows per frame: ceil(height / 16)
};
// As the views launchers: raster_num_blocks(n_points) * n_frames block sums, frame-major.
void launch_line_count_poses(const RasterArgs& args, const PoseArgs& poses, uint32_t n_frames, uint32_t* block_sums, uint32_t* total,
                             uint32_t* max_tile, cudaStream_t stream);
void launch_raster_emit_poses(const RasterArgs& args, const PoseArgs& poses, uint32_t n_frames, const uint32_t* block_offsets,
                              uint64_t* out, uint32_t cap, cudaStream_t stream, const CountArgs* counts = nullptr);
// The fold of a poses call's tables into its records (pose_fold_kernel): record r = b * n_orders + k
// of frame b, order first_order + k, starts from window[k], the layer's own transform and bits with
// kPoseLayer set (or all zero: the order has no layer, and its record stays zero). transforms[r]
// replaces the transform ([ux, vx, uy, vy, tx, ty], reordered; an identity is no transform) and
// visible[r] != 0 the enabled bit. The tables are read where they are passed: in device memory of
// the caller or as the renderer's copy of host tables.
constexpr uint32_t kPoseLayer = 4u;  // PoseRec::bits of a window record: a layer is attached at this order
struct PoseFoldArgs {
    const PoseRec* window;     // n_orders records
    const float* transforms;   // nullable: 6 floats per record, 4-byte aligned
    const uint8_t* visible;    // nullable: 1 byte per record
    uint32_t n_orders;
    uint32_t* first_bad;       // nullable: atomicMin of every r whose transform forma_layer_set_transform refuses
};
void launch_pose_fold(const PoseFoldArgs& args, PoseRec* recs, uint32_t n_recs, cudaStream_t stream);
// Batches (see forma_renderer_render_batch_device): frame c of a stack of n_frames frames is a
// composition of its own. Each frame's line setup reads its composition's segment buffer and
// tables (as RasterArgs, over the whole frame), and only two key fields move: row t of frame c
// becomes biased c * rows + t + 1 (rows outside the frame 0, as for views), and the layer field
// gets the frame's order base.
struct BatchFrame {  // 64 B
    const float* x;
    const float* y;
    const uint32_t* gid;
    const int32_t* geom_slot;
    const LayerRec* layers;      // nullptr: layer_bits
    const uint32_t* layer_bits;
    uint32_t n_points, n_geoms;
    uint32_t order_base;         // first order of the composition's slice of the layer field
    uint32_t pad;
};
struct BatchArgs {
    const BatchFrame* frames;
    const uint32_t* cta_first;   // n_frames + 1: the frame's first CTA (its CTA count is the next entry minus this)
    uint32_t n_frames;
    uint32_t rows;               // tile rows per frame: ceil(height / 16)
    float width, height;
};
// One CTA of raster_num_blocks(n_points) per frame, frame-major: cta_first[n_frames] block sums.
// max_tile[1] is the stacked bound.
void launch_line_count_batch(const BatchArgs& batch, uint32_t n_ctas, uint32_t* block_sums, uint32_t* total, uint32_t* max_tile,
                             cudaStream_t stream);
void launch_raster_emit_batch(const BatchArgs& batch, uint32_t n_ctas, const uint32_t* block_offsets, uint64_t* out, uint32_t cap,
                              cudaStream_t stream, const CountArgs* counts = nullptr);
// Instance scenes (see forma_renderer_render_instances_device): a stack of n_frames frames of one
// composition (RasterArgs), frame b drawing its slots' prototypes as the layers b * n_slots + m.
// Frame b's line records lines[frame_first[b], frame_first[b + 1]) are in (slot, insert) order;
// record r covers the point pairs [first_pair, first_pair + n_pairs) of its frame, which are the
// pairs (first_point + j, first_point + j + 1) of the segment buffer, and draws them with the
// transform of recs[slot] (slot = b * n_slots + m), enabled, at layer order slot. A frame's pairs
// are padded to whole CTAs: CTA x belongs to the last frame with cta_first[b] <= x.
struct InstanceLine {  // 16 B
    uint32_t first_pair;   // frame-local: the pairs of the frame's records before this one
    uint32_t n_pairs;
    uint32_t first_point;  // in the composition's segment buffer
    uint32_t slot;         // b * n_slots + m: the layer order and the PoseRec of the instance
};
struct InstanceArgs {
    const InstanceLine* lines;
    const uint32_t* frame_first;  // n_frames + 1: each frame's first line record
    const uint32_t* cta_first;    // n_frames + 1: each frame's first CTA
    const PoseRec* recs;          // n_frames x n_slots
    uint32_t n_frames, n_slots;
    uint32_t rows;                // tile rows per frame: ceil(height / 16)
};
// cta_first[n_frames] block sums, frame-major; max_tile[1] is the stacked bound.
void launch_line_count_instances(const RasterArgs& args, const InstanceArgs& inst, uint32_t n_ctas, uint32_t* block_sums, uint32_t* total,
                                 uint32_t* max_tile, cudaStream_t stream);
void launch_raster_emit_instances(const RasterArgs& args, const InstanceArgs& inst, uint32_t n_ctas, const uint32_t* block_offsets,
                                  uint64_t* out, uint32_t cap, cudaStream_t stream, const CountArgs* counts = nullptr);
// The instance records (instance_fold_kernel): record r of slot r starts from the record of its
// prototype p = prototypes[r], base[p] (the layer's own transform and bits), or stays zero for an
// empty slot (FORMA_NO_INSTANCE). transforms[r] replaces the transform as in pose_fold_kernel, with
// the same refusal word; every instance is enabled.
struct InstanceFoldArgs {
    const uint32_t* prototypes;  // n_recs layer orders (device)
    const PoseRec* base;         // per order up to the largest prototype
    const float* transforms;     // nullable: 6 floats per record, 4-byte aligned
    uint32_t* first_bad;         // nullable: atomicMin of every r whose transform forma_layer_set_transform refuses
};
void launch_instance_fold(const InstanceFoldArgs& args, PoseRec* recs, uint32_t n_recs, cudaStream_t stream);
// Line records of the n = n_points - 1 point pairs (inspection only): orders, then
// f = {x0, y0, dx, dy, a, b, c, d}, then the per-line segment counts.
void launch_line_records(const RasterArgs& args, uint32_t n, uint32_t* orders, float* const f[8], uint32_t* lengths,
                         cudaStream_t stream);

// ---- kernels_sort.cu --------------------------------------------------------
// LSD radix sort of u64 keys on bits [kSortShift, 64) (+ optional u32 payload).
// Sorted data ends up in keys / vals; *_tmp are same-sized scratch buffers.
// `scratch` needs radix_scratch_bytes(n) bytes. Launch count is returned.
// The 44 ordering bits are three fields; pos/maxw list them from least to most
// significant. Only the low bits of each field that are set in some key (OR of
// all keys | extra_or) take part in the sort passes.
struct KeyLayout {
    uint32_t pos[3];
    uint32_t maxw[3];
};
inline KeyLayout segment_key_layout() { return KeyLayout{{20, 41, 53}, {21, 12, 11}}; }   // ty | tx | layer
inline KeyLayout carry_key_layout() { return KeyLayout{{20, 32, 53}, {12, 21, 11}}; }     // ty | layer | tx

constexpr int kMaxSortPasses = 6;  // ceil(44 / 8)
// One digit = up to three bit runs of the key, concatenated.
struct DigitSpec {
    uint8_t shift[3];
    uint8_t width[3];
    uint8_t lsh[3];
    uint8_t bits;
};
struct SortPlan {
    uint32_t n_passes;
    uint32_t total_bits;
    DigitSpec pass[kMaxSortPasses];
};
// bound[f] = largest value field f (least significant first) takes in any key.
SortPlan make_sort_plan(const KeyLayout& layout, const uint64_t bound[3]);
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t digit_of(uint64_t key, const DigitSpec& d) {
    uint32_t v = (uint32_t)(key >> d.shift[0]) & ((1u << d.width[0]) - 1u);  // lsh[0] == 0
    if (d.width[1] != 0u) {  // uniform: most digits are a single bit run
        v |= ((uint32_t)(key >> d.shift[1]) & ((1u << d.width[1]) - 1u)) << d.lsh[1];
        v |= ((uint32_t)(key >> d.shift[2]) & ((1u << d.width[2]) - 1u)) << d.lsh[2];
    }
    return v;
}
#endif
inline bool same_digit(const DigitSpec& a, const DigitSpec& b) {
    for (int r = 0; r < 3; ++r)
        if (a.shift[r] != b.shift[r] || a.width[r] != b.width[r] || a.lsh[r] != b.lsh[r]) return false;
    return a.bits == b.bits;
}
struct SortResult {
    int launches;
    bool in_tmp;  // the sorted data is in keys_tmp / vals_tmp (odd number of passes)
    int timed_passes = 0;  // passes whose kernels were bracketed by pass_events
};

// Per-tile digit counts of the reduce-then-scan passes of a key-only sort, counted by the kernels
// that write the keys instead of by an upsweep pass that reads them again (option sort_counts): the
// emit pass counts pass 0 (Renderer::rasterize), the downsweep of pass p counts pass p + 1 by the
// keys' destinations. Two blocks of u32, pass p using block p & 1:
//   block = totals[kTotalsRows][256] | hist[tile_cap][256]
// hist: per 4096-key tile, the only counts the producers add to (one atomic per warp group of equal
// (tile, digit)). totals: per chunk of tiles_per_chunk consecutive tiles, then per super-chunk of
// kChunksPerSuper chunks (what the tile scan reads), summed from hist by radix_chunk_totals_kernel.
// The downsweep of pass p zeroes what it consumed (hist of pass p, its super-chunk rows): after a
// sort both blocks are zero again, and the next frame's producers count into them without a memset.
constexpr uint32_t kSortTileKeys = 4096;
constexpr uint32_t kChunksPerSuper = 16;
constexpr uint32_t kMaxSupers = 32;
constexpr uint32_t kMaxChunks = kChunksPerSuper * kMaxSupers;  // 512
constexpr uint32_t kTotalsRows = kMaxChunks + kMaxSupers;      // chunk rows, then super-chunk rows
inline uint32_t sort_tiles(uint32_t n) { return (n + kSortTileKeys - 1u) / kSortTileKeys; }
struct TileCounts {
    uint32_t* base = nullptr;
    uint32_t tile_cap = 0;         // tiles each block is laid out for
    uint32_t tiles_per_chunk = 1;  // ceil(tile_cap / kMaxChunks)
    bool pass0 = false;            // block 0 holds pass 0's counts; otherwise the sort counts them itself (upsweep)
    size_t block_words() const { return (size_t)(kTotalsRows + tile_cap) * 256u; }
    uint32_t* totals(uint32_t p) const { return base + (p & 1u) * block_words(); }
    uint32_t* hist(uint32_t p) const { return totals(p) + (size_t)kTotalsRows * 256u; }
};
// Where a producer adds its keys' digit counts: the pass's per-tile counts and digit.
struct CountArgs {
    uint32_t* hist;
    DigitSpec spec;
};
#ifdef __CUDACC__
__device__ __forceinline__ void add_tile_count(const CountArgs& C, uint32_t tile, uint32_t digit, uint32_t count) {
    atomicAdd(&C.hist[(size_t)tile * 256u + digit], count);
}
#endif
// Whether a key-only sort of n keys runs the reduce-then-scan passes (the only ones that take TileCounts).
bool radix_sort_scans(uint32_t n);
size_t radix_scratch_bytes(uint32_t n);
// Scratch of a sort whose digit histogram comes from the kernel that wrote its keys (see
// launch_radix_sort's `hist`): tile counters and look-back tables of the single-sweep passes.
size_t sort_lookback_bytes(uint32_t n, const SortPlan& plan);
// Adds the digit counts of every planned pass of keys[0, n) (n_dev: as below) to hist[kMaxSortPasses][256].
void launch_radix_hist(const uint64_t* keys, uint32_t n, const SortPlan& plan, uint32_t* hist, const uint32_t* n_dev,
                       cudaStream_t stream);
SortResult launch_radix_sort(uint64_t* keys, uint64_t* keys_tmp, uint32_t* vals, uint32_t* vals_tmp, uint32_t n,
                             const SortPlan& plan, void* scratch, cudaStream_t stream,
                             cudaEvent_t* pass_events = nullptr /* 3 per pass, of which the sort records [3p + 1] (before the downsweep) and [3p + 2] (after it) but
                                                                  not the last pass's [3p + 2]: pass p starts at the event recorded before it (the caller's before the sort, pass p - 1's
                                                                  end) and the last pass ends at the caller's after the sort. Fewer event records between the kernels */,
                             const uint32_t* n_dev = nullptr /* the key count in device memory; `n` is then its upper bound
                                                                and a larger count sorts nothing. With `counts` (reduce-then-scan
                                                                passes) the counts of the tiles past it must be zero */,
                             const uint32_t* hist = nullptr /* [kMaxSortPasses][256] digit counts of every planned pass,
                                                               counted by the keys' producer: the sort then launches its
                                                               passes only, and `scratch` holds sort_lookback_bytes(n, plan)
                                                               bytes zeroed by the caller */,
                             const TileCounts* counts = nullptr /* reduce-then-scan passes: the tile counts, both blocks zero
                                                                   except for what the emit counted into block 0 (counts->pass0;
                                                                   without it, block 0 must be zero: pass 0 is counted by an
                                                                   upsweep); no upsweep from pass 1 on, and both blocks are zero
                                                                   again when the sort is done */,
                             uint32_t* keep_counts = nullptr /* with `counts`: pass p's tile counts are copied to
                                                                keep_counts + p * tiles * 256 before its tile scan */);

// ---- kernels_paint.cu -------------------------------------------------------
struct PaintScene {
    const StyleRec* styles;       // indexed by style slot
    const int32_t* order_to_style;// layer id (order) -> style slot
    uint32_t n_orders;
    const StopRec* stops;
    const GradRec* grads;         // per style slot (valid where the style is a gradient of <= 4 stops)
    const uint16_t* texels;       // RGBA f16 (styling.rs:224-249), 4 per texel
    float clear[4];
    uint32_t channels[4];         // already upgraded Alpha -> One when clear.a == 1
    uint32_t width, height;       // pixels
    uint32_t stride;              // bytes
    uint32_t tiles_x, tiles_y;    // ceil(width / 16), ceil(height / 16)
    uint32_t tx_lo, tx_hi;        // tile columns painted (crop), [lo, hi)
    uint32_t ty_lo, ty_hi;        // tile rows painted (crop ∩ band), [lo, hi)
    // Layer cache (damage reuse, cpu/buffer/mod.rs:114-197); all null/0 without a cache.
    const uint8_t* unchanged;     // per layer order: Layer::is_unchanged(cache_id)
    uint2* cache_tiles;           // per tile: x = has_count<<31 | has_solid<<30 | layer_count(24), y = solid colour
    uint32_t* written_list;       // optional: linear ids of the tiles this frame wrote (unordered)
    uint32_t* written_count;      //           ... and how many
    uint32_t clear_unchanged;     // previous clear colour == this frame's
};

uint32_t cell_num_blocks(uint32_t n);
// Plans of the painter's two pair sorts (their key bounds are host-known).
SortPlan carry_sort_plan(const PaintScene& S);
SortPlan gap_sort_plan(const PaintScene& S);
// The painter tables' scratch: one block that is zeroed before the tables of a frame are built
// (byte offsets; every region starts 256-byte aligned). n = segments; n_cells / n_gaps: the
// counts (or bounds) that size the carry sort / carry pass and the gap sort.
struct TableScratch {
    size_t heavy_count;  // kHeavyListClasses u32: lengths of the heavy-tile lists (read by the painter)
    size_t carry_hist;   // [kMaxSortPasses][256] u32: digit counts of the carry sort (cells pass)
    size_t gap_hist;     // [kMaxSortPasses][256] u32: digit counts of the gap sort (carry pass)
    size_t cells_state;  // cells pass look-back
    size_t carry_sort;   // carry sort tile counters + look-back tables
    size_t carry_pass;   // carry pass look-back (carries, gap offsets) + ticket
    size_t gap_sort;     // gap sort tile counters + look-back tables
    size_t end;
};
TableScratch table_scratch_layout(uint32_t n, uint32_t n_cells, uint32_t n_gaps, const SortPlan& carry_plan,
                                  const SortPlan& gap_plan);
// Bytes [0, a_bytes) of a and [0, b_bytes) of b, and *word when not null, set to zero by one chained
// kernel (not counted as a launch).
void launch_zero_tables(uint8_t* a, size_t a_bytes, uint8_t* b, size_t b_bytes, uint32_t* word, cudaStream_t st);
// dst[0, n) = src[0, n), n <= 256, by one chained kernel (not counted as a launch); dst may be the
// device address of pinned host memory.
// Cells in one pass over the sorted segments (+ a small kernel for the cells that cross a
// CTA tile): cell_start[c] = first segment of cell c (cell_start[#cells] = n), the cell's
// cover (16 x i8 by local_y), its key, the (tile_y, layer, tile_x) key of the carry pass and
// perm[c] = c, for every c < cap - 1; n_cells_out[0] = #cells. All five arrays need `cap`
// entries. The digits of every written carry-pass key are added to `carry_hist` ([passes][256]
// of `carry_plan`). `scratch`: the zeroed table scratch (cells_state). May be launched before the
// host knows the count; the caller repeats it if #cells >= cap. n_dev (optional): the segment count
// in device memory, `n` then being its upper bound (the grid).
void launch_cells(const PaintScene& S, const uint64_t* segs, uint32_t n, uint8_t* scratch, const TableScratch& L,
                  const SortPlan& carry_plan, uint32_t* cell_start, uint32_t cap, uint32_t* n_cells_out, uint64_t* cell_key,
                  uint4* cell_cover, uint64_t* key2, uint32_t* perm, cudaStream_t st, const uint32_t* n_dev = nullptr);
// Cell / carry-only-entry counts that stay on the device (frames whose tables are built without a
// host read-back, Options::sync_free): with `cells` set, the n_cells / n_gaps arguments of the
// launchers below are upper bounds (grid sizes) and the kernels read the counts here; a count
// above its bound makes them no-ops (the host then rebuilds the tables with known counts).
// words / words_out / n_words (merge only): the merge kernel, the last kernel of the tables, also
// copies n_words (<= 256) count words to the host's pinned words (words_out: their device
// address), which the host reads after the frame's final synchronisation; no kernel of its own
// behind the paint carries them.
struct DevCounts {
    const uint32_t* cells = nullptr;
    const uint32_t* gaps = nullptr;
    uint32_t cell_bound = 0, gap_bound = 0;
    const uint32_t* words = nullptr;
    uint32_t* words_out = nullptr;
    uint32_t n_words = 0;
};
// One pass over the carry-sorted cells: the carry-in of every cell (carry_in, by cell id) and the
// carry-only entries in (layer, tile_y, tile_x) order: key, payload n_cells + entry id, carried
// cover. Entries at positions >= cap are not written; n_gaps_out[0] = their exact count. The
// digits of every written key are added to `gap_hist` ([passes][256] of `gap_plan`). `scratch`:
// the zeroed table scratch (carry_pass).
void launch_carry_pass(const PaintScene& S, const uint64_t* key2, const uint32_t* perm, const uint4* cell_cover,
                       uint32_t n_cells, uint8_t* scratch, const TableScratch& L, const SortPlan& gap_plan, uint4* carry_in,
                       uint64_t* gkey, uint32_t* gid, uint4* gap_carry, uint32_t cap, uint32_t* n_gaps_out, cudaStream_t st,
                       const DevCounts& dc = DevCounts());
// One painter entry = one (tile, layer) pair with segments and / or a carried cover.
struct EntryRec {  // 64 B
    uint32_t layer, seg0, seg1;  // layer order; [seg0, seg1) in the sorted segments (empty for carry-only entries)
    uint32_t meta;               // packed style bits, see pack_style_meta (paint_common.cuh)
    uint4 carry;                 // 16 x i8 cover carried in from the tiles on the left
    float color[4];              // solid fill colour
    int32_t slot;                // style slot
    uint32_t clip_layers;
    uint32_t flags0;             // initial optimizer flags (kFlag*)
    uint32_t pad;
};
// Merges the cells with the sorted carry-only entries: ekey, entry records and
// initial flags of the n_cells + n_gaps entries, ordered by (tile_y, tile_x, layer), and
// the per-tile entry ranges (tile_range: zeroed by the caller, left zero for tiles without
// entries) and, when `heavy` is not null, the lists of tiles with many entries:
// kHeavyListClasses arrays of tiles_x * tiles_y ids each, their lengths in
// heavy_count[kHeavyListClasses] (zeroed by the caller). frames != nullptr: S stacks the frames of
// a batch, `rows` tile rows each (their order bases bound each entry's clip_layers to the range a
// single frame of its composition has). fills != nullptr: S.styles is a pose style table (see
// PoseFillArgs), and the entries of a pose stack's Draw layers in the window take their frame's
// slot (merge_entries_pose_fills_kernel; frames is then null).
constexpr int kHeavyListClasses = 4;
// Pose fills (see forma_poses::colors): a pose style table holds the composition's n_styles style
// records at their own slots, then per frame b and order first_order + k of the window the record of
// slot n_styles + b * n_orders + k: the layer's StyleRec with the frame's solid fill
// (launch_pose_styles). n_styles + n * n_orders < 2^31 (EntryRec::slot).
struct PoseFillArgs {
    uint32_t n_styles;
    uint32_t first_order, n_orders;  // the pose window
    uint32_t rows;                   // tile rows per frame
};
void launch_merge_entries(const PaintScene& S, const uint64_t* cell_key, uint32_t n_cells, const uint64_t* gkey,
                          const uint32_t* gid, uint32_t n_gaps, const uint32_t* cell_start, const uint4* carry_in,
                          const uint4* gap_carry, uint64_t* ekey, EntryRec* recs, uint8_t* eflags, uint2* tile_range,
                          uint32_t* heavy, uint32_t* heavy_count, cudaStream_t st, const DevCounts& dc = DevCounts(),
                          const BatchFrame* frames = nullptr, uint32_t rows = 0, const PoseFillArgs* fills = nullptr);
// The tail of a pose style table `styles` (its slots [0, n_styles) already hold the composition's
// records): record i = b * n_window + k of the n_recs records is the StyleRec of the layer at order
// first_order + k (order_to_style, n_orders orders), with a Draw layer's fill replaced by the solid
// colour colors[i] (linear RGBA) and no gradient or texture left; orders without a layer get none.
void launch_pose_styles(const int32_t* order_to_style, uint32_t n_orders, StyleRec* styles, uint32_t n_styles, const float4* colors,
                        uint32_t first_order, uint32_t n_window, uint64_t n_recs, cudaStream_t st);
// The order -> style table of an instance call, one thread per slot r: -1 for an empty slot
// (FORMA_NO_INSTANCE) or a prototype without a style, the prototype's own slot when colors is null
// or the prototype does not draw, else n_styles + r, where `styles` (whose slots [0, n_styles) hold
// the composition's records) receives the prototype's StyleRec made solid with colors[r], as
// launch_pose_styles makes it.
void launch_instance_styles(const int32_t* order_to_style, uint32_t n_orders, const uint32_t* prototypes, StyleRec* styles,
                            uint32_t n_styles, const float4* colors, uint32_t n_recs, int32_t* inst_order_to_style, cudaStream_t st);
// The painter tables of a frame as every tile kernel (paint, ID, mask, statistics) reads them: the
// sorted segments, the entry records, the per-tile entry ranges and, when `heavy` is not null, the
// heavy-tile lists with their lengths (launch_merge_entries).
struct TileTables {
    const uint64_t* segs;
    const EntryRec* recs;
    const uint2* tile_range;
    const uint32_t* heavy;
    const uint32_t* heavy_count;
};
// The tile kernels below are persistent: their warps take the tiles of S's tile rectangle by ticket
// from `tile_counter`, which the launcher resets on `st` (launch_paint: unless counter_zeroed, when a
// kernel earlier on `st` has cleared it). Nothing is launched for an empty rectangle.
// view_rows != 0: S stacks views of view_rows tile rows each (ViewArgs); gradients and textures are
// then sampled in each view's own coordinates. solid_over: every layer of the frame is a solid `Over`
// fill without clips (Composition::solid_over_only); the lean build of the kernel paints it.
void launch_paint(const PaintScene& S, const TileTables& t, uint8_t* eflags, uint8_t* framebuffer, uint32_t* tile_counter,
                  cudaStream_t st, uint32_t view_rows = 0, bool solid_over = false, bool counter_zeroed = false);
// launch_paint for a linear float frame of `bpp` bytes per pixel: 8 (RGBA16F) or 16 (RGBA32F), the
// painter's planes in channel order where launch_paint stores their sRGB bytes (see
// forma_renderer_render_linear). `framebuffer` and S.stride: multiples of 4 bytes.
void launch_paint_linear(const PaintScene& S, const TileTables& t, uint8_t* eflags, uint8_t* framebuffer, uint32_t* tile_counter,
                         cudaStream_t st, uint32_t view_rows, uint32_t bpp, bool counter_zeroed = false);
// launch_paint over the pixels already in `framebuffer` (see forma_renderer_render_over_device):
// each pixel's own value, decoded, is its clear colour; tiles without entries are not written.
// bpp 4 (sRGB8, channels a permutation with A last), 8 (RGBA16F) or 16 (RGBA32F, both: any
// permutation); S.channels are not upgraded (the kernels upgrade Alpha -> One per pixel).
// `framebuffer` and S.stride: multiples of 4 bytes.
void launch_paint_over(const PaintScene& S, const TileTables& t, uint8_t* eflags, uint8_t* framebuffer, uint32_t* tile_counter,
                       cudaStream_t st, uint32_t view_rows, uint32_t bpp, bool counter_zeroed = false);
// The inverse of launch_repack_views: rows [0, height) of the n_views frames at src + b * view_stride
// (row r at + r * stride) to the stacked frame at dst, frame b's first row at
// dst + b * view_rows_px * dst_stride. `width` in 4-byte words; every pointer and stride a multiple of 4.
void launch_unpack_views(const uint8_t* src, uint64_t stride, uint64_t view_stride, uint8_t* dst, uint64_t dst_stride,
                         uint32_t view_rows_px, uint32_t width, uint32_t height, uint32_t n_views, cudaStream_t st);
// Copies rows [0, height) of the n_views views of a stacked frame (view b's first row at
// src + b * view_rows_px * src_stride) to dst + b * view_stride, row r at + r * stride.
void launch_repack_views(const uint8_t* src, uint64_t src_stride, uint32_t view_rows_px, uint8_t* dst, uint64_t stride,
                         uint64_t view_stride, uint32_t width, uint32_t height, uint32_t n_views, cudaStream_t st);
// ID frame (kernels_ids.cu): per pixel of the tile rectangle of S (clipped to the frame), the
// order of the top-most Draw layer whose coverage x clip mask exceeds min_coverage, or
// FORMA_ID_NONE. Reads the tables like launch_paint (never `eflags`); id_flags: one byte per
// entry of scratch. ids_stride in bytes.
// frames != nullptr: S stacks the frames of a batch, `rows` tile rows each, whose entries carry
// frames[c].order_base + order (BatchArgs); every ID stored is the frame's own order
// (paint_ids_stacked_kernel). The stacked views of one composition need neither.
void launch_paint_ids(const PaintScene& S, const TileTables& t, uint8_t* id_flags, uint32_t* ids, size_t ids_stride,
                      float min_coverage, uint32_t* tile_counter, cudaStream_t st, uint32_t rows = 0,
                      const BatchFrame* frames = nullptr);
// Layer coverage masks (kernels_ids.cu, see forma_renderer_render_masks): n_orders planes per frame
// of n_frames, plane (b, k) at ptr + (b * n_orders + k) * plane_stride with rows `stride` bytes
// apart, holding order first_order + k: f32 (format 0) or the u8 encode of alpha (format 1).
struct MaskFrame {
    uint8_t* ptr;
    uint64_t stride, plane_stride;
    uint32_t first_order, n_orders, format;
    uint32_t height;    // rows of one frame
    uint32_t n_frames;  // 1 for a single frame
};
// Zeroes the written rectangle of every plane (the crop's tile rectangle of a single frame, each
// frame's width x height pixels of a stack), then paints the masks from the tables like
// launch_paint_ids (id_flags: the same scratch). rows != 0: S stacks frames of `rows` tile rows;
// frames != nullptr: a batch, whose entries carry frames[c].order_base + order. Returns the launches.
uint32_t launch_paint_masks(const PaintScene& S, const TileTables& t, uint8_t* id_flags, const MaskFrame& m, uint32_t* tile_counter,
                            cudaStream_t st, uint32_t rows = 0, const BatchFrame* frames = nullptr);
// Layer statistics (kernels_ids.cu, see forma_renderer_render_stats): n_orders records of order
// first_order + k per frame of n_frames, frame b's at ptr + b * n_orders.
struct StatsFrame {
    forma_layer_stats* ptr;
    uint32_t first_order, n_orders;
    float min_coverage;
    uint32_t height;    // rows of one frame
    uint32_t n_frames;  // 1 for a single frame
};
// Initialises the records, reduces the amodal walk (the mask kernel's) and the visible walk (the
// ID kernel's) into them, then writes the empty sets' boxes: the whole of the records, so that the
// sync-free redo can repeat it. rows / frames as for launch_paint_masks. Returns the launches.
uint32_t launch_paint_stats(const PaintScene& S, const TileTables& t, uint8_t* id_flags, const StatsFrame& f, uint32_t* tile_counter,
                            cudaStream_t st, uint32_t rows = 0, const BatchFrame* frames = nullptr);
// The painter tables of a batch: the device tables of its distinct compositions, concatenated.
// Composition k's orders land at order_base + order (the slots they name shifted by style_base,
// -1 kept), its StyleRecs at style_base with stop_first + stop_base and tex_first + texel_base;
// stops, texels (in texels of 4 x u16) and GradRecs are copied as they are.
struct BatchTableSrc {
    const int32_t* order_to_style;
    const StyleRec* styles;
    const GradRec* grads;
    const StopRec* stops;
    const uint16_t* texels;
    uint32_t n_orders, n_styles, n_stops, n_texels;  // n_texels: texels (4 x u16 each)
    uint32_t order_base, style_base, stop_base, texel_base;
};
void launch_batch_tables(const BatchTableSrc* src, uint32_t n_src, uint32_t max_items, int32_t* order_to_style, StyleRec* styles,
                         GradRec* grads, StopRec* stops, uint16_t* texels, cudaStream_t st);
// GradRec of every style slot (see device_types.h).
void launch_grad_setup(const StyleRec* styles, const StopRec* stops, uint32_t n_styles, GradRec* grads, cudaStream_t st);
// Pixel-pair fp32 arithmetic of the painter against scalar IEEE operations; mismatches are added to out[0].
void launch_f32x2_selftest(const float* a, const float* b, const float* c, uint32_t n, uint32_t* out, cudaStream_t st);
// out[row] = 32 x entries + pixel segments of tile row `row` (see row_cost_kernel). n_dev: as for launch_cells.
void launch_row_costs(const uint2* tile_range, uint32_t tiles_x, uint32_t tiles_y, const uint64_t* segs, uint32_t n,
                      unsigned long long* out, cudaStream_t st, unsigned long long* seg_out = nullptr, const uint32_t* n_dev = nullptr);
// Packs the tiles in S.written_list into `packed` (256 u32 per tile, row-major).
void launch_gather_tiles(const PaintScene& S, const uint8_t* framebuffer, uint32_t* packed, cudaStream_t st);

}  // namespace forma
