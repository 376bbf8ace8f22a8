// forma_b200 — the per-device Renderer (renderer.cu) and the C ABI objects that c_abi.cu and
// multi_renderer.cu share.
#pragma once

#include <algorithm>
#include <exception>

#include "../../include/forma_b200.h"
#include "host_scene.hpp"
#include "kernels.h"

namespace forma {

// ---------------------------------------------------------------------------
// Renderer
// ---------------------------------------------------------------------------
// BufferLayerCache (cpu/buffer/mod.rs:114-197). The per-tile records live on the
// device (the painter reads and updates them); the host only keeps the size and
// clear colour of the last frame.
struct LayerCache {
    uint8_t id = 0;
    DeviceBuffer<uint2> tiles;  // CachedTile per tile, see PaintScene::cache_tiles
    bool has_size = false;
    uint64_t width = 0, height = 0;
    bool has_clear = false;
    float clear_color[4] = {0, 0, 0, 0};
    bool needs_reset = true;  // the tile records must be zeroed before their next use
    void clear() {            // BufferLayerCache::clear, mod.rs:189-196
        has_clear = false;
        needs_reset = true;
    }
};

struct Timer {
    cudaEvent_t ev[8];
    cudaEvent_t sort_ev[3 * kMaxSortPasses];  // main sort, per pass: before upsweep, before / after downsweep
    bool ok = false;
};

// A target of a FrameRequest: pixels of `bpp` bytes, RGBA8 (4), RGBA16F (8) or RGBA32F (16) for the
// RGBA target (see forma_renderer_render_linear), the 4-byte layer IDs of ID frames (see
// forma_renderer_render_ids). Row r of frame b at ptr + b * frame_stride + r * stride
// (frame_stride: stacks only).
struct FrameTarget {
    uint8_t* ptr = nullptr;  // null: the request has no such target
    bool on_device = false;
    uint64_t stride = 0, frame_stride = 0;
    float min_coverage = 0.0f;  // the ID target
    uint32_t bpp = 4;
    bool over = false;  // the RGBA target: painted over its own pixels, each its clear colour (see forma_renderer_render_over_device)
};

// The masks target of a FrameRequest (see forma_renderer_render_masks): n_orders planes of order
// first_order + k per frame, plane (b, k) at ptr + (b * n_orders + k) * plane_stride, rows `stride`
// bytes apart, f32 or u8 values (format).
struct MaskTarget {
    uint8_t* ptr = nullptr;  // null: the request has no masks
    bool on_device = false;
    uint32_t first_order = 0, n_orders = 0, format = 0;
    uint64_t stride = 0, plane_stride = 0;
    uint32_t bpp() const { return format == FORMA_MASK_U8 ? 1u : 4u; }
};

// The statistics target of a FrameRequest (see forma_renderer_render_stats): n_orders records of
// order first_order + k per frame, frame b's at ptr + b * n_orders.
struct StatsTarget {
    forma_layer_stats* ptr = nullptr;  // null: the request has no statistics
    bool on_device = false;
    uint32_t first_order = 0, n_orders = 0;
    float min_coverage = 0.0f;
};

// What a FrameRequest renders. single: one frame of a composition. views: n views of one
// composition in one pass, stacked top to bottom as one frame of n * ceil(height / 16) tile rows;
// line setup rasterizes every view in its own coordinates and moves its segments' tile rows to the
// view's place in the stack (ViewArgs), and the tables, the sort and the painter see one frame.
// batch: n compositions, one frame each, stacked as views are; frame c's line setup reads
// comps[c]'s segment buffer and moves its segments' layers to the composition's slice of the
// layer field (bind_batch), so that the batch tables serve every frame, and frame c's IDs are
// comps[c]'s own orders. poses: n frames of one composition stacked as views are, frame b giving
// each layer of a window of orders its own transform and enabled state (PoseArgs); line setup
// reads frame b's pose records in place of a view transform, and from there on a pose stack is a
// views stack. instances: n frames of one composition stacked as views are, frame b drawing its M
// slots' prototype layers as the layers b M + m (Renderer::upload_instances); from line setup on an
// instance stack is a batch of n compositions of M orders each, whose tables are built per call.
// A stack takes no layer cache and no band filter: every composition is resident whole.
enum class FrameKind { single, views, batch, poses, instances };

// One call of Renderer::render: what is rendered, the size of one frame, and its targets: an
// RGBA target, an ID target (channels {0, 1, 2, 3}, clear colour 0 when it is alone) or both, or
// masks or statistics, alone or with an sRGB8 RGBA target.
struct FrameRequest {
    FrameKind kind = FrameKind::single;
    uint32_t n = 0;  // stacks: the frames
    uint64_t width = 0, height = 0;
    const uint32_t* channels = nullptr;  // of the RGBA target
    const float* clear = nullptr;
    forma_timings* timings = nullptr;
    const forma_rect* crop = nullptr;  // single frames only
    LayerCache* cache = nullptr;       // single RGBA frames only
    FrameTarget rgba, ids;
    MaskTarget masks;
    StatsTarget stats;
    Composition* comp = nullptr;          // single, views
    const float* views = nullptr;         // views: n transforms [ux, vx, uy, vy, tx, ty]
    Composition* const* batch = nullptr;  // batch: n compositions (null entries are refused)
    const forma_poses* poses = nullptr;   // poses: the window and its tables (null is refused)
    const forma_instances* instances = nullptr;  // instances: the slots and their tables (null is refused)
    // Views, poses and instances: a stack of frames of one composition (q.comp).
    bool one_comp_stack() const {
        return kind == FrameKind::views || kind == FrameKind::poses || kind == FrameKind::instances;
    }
    // Poses with colours: the painter tables are built over a pose style table (PoseFillArgs).
    bool pose_fills() const { return kind == FrameKind::poses && poses && poses->colors; }
};

// Where Renderer::render paints a request's targets: per target the frame on the device (the
// caller's buffer when `direct`, the renderer's scratch otherwise) and its row stride.
struct DeviceFrame {
    uint8_t* ptr;
    uint64_t stride;
    bool direct;
};
struct FramePlan {
    DeviceFrame rgba, ids;
    uint32_t rows;      // stacks: tile rows of each frame; 0: a single frame
    bool in_bands;      // a single host sRGB8 frame painted and copied back band by band (see paint)
    bool pack_written;  // a cached host frame: only the tiles it writes travel back (scatter_written_tiles)
    DeviceFrame masks;  // the caller's planes on the device, or (host masks) the renderer's scratch ...
    uint64_t mask_plane_stride;  // ... with this plane stride
    forma_layer_stats* stats;    // the caller's records on the device, or (host statistics) the renderer's scratch
};

// The line setup of an instance call (see Renderer::upload_instances).
struct InstanceLines {
    InstanceArgs args;
    BatchArgs frames;      // only frames (order_base = b M) and rows: the tables' and tile kernels' view of the stack
    uint32_t n_ctas;
    uint64_t layer_bound;  // the sort plan's bound of the layer field
    uint64_t n_lines;      // point pairs of all frames (forma_timings)
};

// The line setup of a batch (see Renderer::bind_batch).
struct BatchLines {
    BatchArgs args;
    uint32_t n_ctas;
    uint64_t layer_bound;  // the sort plan's bound of the layer field
    uint64_t n_lines;      // point pairs of all frames (forma_timings)
};

class Renderer {
   public:
    int device = 0;
    int res_key = 0;  // key of this renderer's residency record in a Composition: the device ordinal, or
                      // device + 4096 * (k + 1) for the k-th slice renderer of a host-frame pipeline
    int copy_bands_override = 0;  // slice renderers: copy bands inside the slice (0 = option copy_bands)
    cudaStream_t stream = 0;
    bool owns_stream = false;
    uint64_t launches = 0;
    uint32_t caches_in_use = 0;
    Timer timer;

    // Per-frame device scratch (high-water-mark allocations).
    DeviceBuffer<uint32_t> block_sums, totals;
    SortPlan segment_plan{};  // digits of the main sort, from the bounds seen by the line-setup pass
    uint64_t segment_bound[3] = {0, 0, 0};  // ... those bounds: layer, tile_x, tile_y (forma_renderer_sort_bounds)

    template <class T>
    static void swap_buffers(DeviceBuffer<T>& a, DeviceBuffer<T>& b) {
        std::swap(a.ptr, b.ptr);
        std::swap(a.capacity, b.capacity);
    }
    // launch_radix_sort of keys (+ vals, may be null) with sort_scratch, or with `scratch` and the
    // digit histogram `hist` counted by the keys' producer; the sorted data ends up in keys /
    // vals: the buffers trade places with their twins when it landed there.
    SortResult sort(DeviceBuffer<uint64_t>& keys, DeviceBuffer<uint64_t>& keys_tmp, DeviceBuffer<uint32_t>* vals,
                    DeviceBuffer<uint32_t>* vals_tmp, uint32_t n, const SortPlan& plan, cudaEvent_t* pass_events = nullptr,
                    const uint32_t* n_dev = nullptr, const uint32_t* hist = nullptr, void* scratch = nullptr,
                    const TileCounts* counts = nullptr, uint32_t* keep_counts = nullptr);
    DeviceBuffer<uint64_t> segs, segs_tmp;
    DeviceBuffer<uint8_t> sort_scratch;
    // The segment sort's per-tile digit counts (TileCounts, option sort_counts), counted by the emit
    // pass and the downsweeps. Laid out for tile_counts.tile_cap tiles: reserved before the emit pass
    // that counts into it (prepare_tile_counts), never moved between that pass and the sort.
    DeviceBuffer<uint32_t> sort_counts;
    TileCounts tile_counts;
    // Pass 0 of the last frame whose sort used the tile counts: the speculative emit pass of the next
    // frame counts that digit (the frame's own plan is only known after the count read-back).
    DigitSpec count_spec{};
    bool count_spec_valid = false;
    // Where the last frame's pass-0 counts came from (see forma_renderer_sort_counts): 0 none,
    // 1 the speculative emit, 2 the emit after the read-back, 3 an upsweep.
    int last_count_source = 0;
    bool keep_sort_counts = false;  // forma_renderer_sort_counts: keep every pass's counts of the next frames
    DeviceBuffer<uint32_t> kept_counts;
    uint32_t kept_passes = 0, kept_tiles = 0;
    bool counts_clean = false;  // both blocks of tile_counts are zero (TileCounts)
    // Reserves the tile counts for max_keys keys and zeroes them unless they are clean.
    cudaError_t prepare_tile_counts(uint32_t max_keys);
    DeviceBuffer<uint8_t> table_scratch;  // see TableScratch (kernels.h); zeroed per frame by build_tables
    uint32_t* heavy_count() const { return reinterpret_cast<uint32_t*>(table_scratch.ptr); }  // TableScratch::heavy_count == 0
    DeviceBuffer<uint32_t> cell_start, perm, perm_tmp, eid, eid_tmp, gid_tmp, heavy_tiles;
    DeviceBuffer<uint2> tile_range;
    DeviceBuffer<uint64_t> cell_key, key2, key2_tmp, ekey, ekey_tmp, gkey_tmp;
    DeviceBuffer<uint4> cell_cover, carry_in, gap_carry;
    DeviceBuffer<uint8_t> eflags, framebuffer;
    DeviceBuffer<EntryRec> recs;
    // The painter-table scratch by the count that sizes it (see build_tables): per cell, per
    // carry-only entry, per entry. n + 1 per cell and per carry-only entry: the cells pass writes
    // its outputs below cap - 1, and the pair sorts need a slack slot.
    template <class... B>
    static cudaError_t reserve_all(size_t n, B&... bufs) {
        cudaError_t e = cudaSuccess;
        ((e = e != cudaSuccess ? e : bufs.reserve(n)), ...);
        return e;
    }
    cudaError_t reserve_cell_tables(size_t n_cells) {
        return reserve_all(n_cells + 1, cell_start, cell_key, cell_cover, carry_in, key2, key2_tmp, perm, perm_tmp);
    }
    cudaError_t reserve_gap_tables(size_t n_gaps) { return reserve_all(n_gaps + 1, ekey_tmp, eid_tmp, gkey_tmp, gid_tmp, gap_carry); }
    cudaError_t reserve_entry_tables(size_t n_entries) { return reserve_all(n_entries, ekey, eid, eflags, recs); }
    // Band-wise copy-back of host frames (see render()).
    static constexpr uint32_t kMaxCopyBands = 16;
    uint32_t copy_bands() const {
        return (uint32_t)std::min(std::max(copy_bands_override ? copy_bands_override : options().copy_bands, 1), (int)kMaxCopyBands);
    }
    cudaStream_t aux_stream = nullptr;  // side stream of the geometry upload (see flush_geometry)
    cudaEvent_t aux_ev[2];
    cudaStream_t band_stream[kMaxCopyBands];
    uint32_t band_streams_made = 0;  // created as needed: streams beyond the device's hardware queues alias onto them
    bool band_streams_ok = false;    // the band events exist
    cudaEvent_t band_ev[kMaxCopyBands + 1];
    cudaEvent_t count_ev = nullptr;  // completion of a count read-back (waited on instead of the whole stream)
    cudaError_t ensure_count_event() {
        return count_ev ? cudaSuccess : cudaEventCreateWithFlags(&count_ev, cudaEventDisableTiming);
    }
    static bool speculation_enabled() { return options().speculate != 0; }
    static size_t test_gap_cap_override() { return (size_t)std::max(options().test_gap_cap, 0); }
    static bool band_copies_enabled() { return options().band_copy != 0; }
    // Layer-cache frames: per-slot `is_unchanged` flags, the list of written
    // tiles and their packed pixels (only these travel back to a host buffer).
    DeviceBuffer<uint8_t> d_unchanged;
    PinnedBuffer<uint8_t> h_unchanged;
    DeviceBuffer<uint32_t> written_list, packed_tiles;
    PinnedBuffer<uint32_t> h_written_list, h_packed_tiles;
    uint32_t last_written_tiles = 0;
    // Upload staging.
    DeviceBuffer<QuadUp> up_quads_raw;  // as uploaded; expanded into up_quads on the device
    DeviceBuffer<SplineRec> up_splines;
    DeviceBuffer<PointRec> up_points;
    DeviceBuffer<uint8_t> up_kinds;
    DeviceBuffer<QuadRec> up_quads;
    DeviceBuffer<FlattenJob> up_jobs;
    DeviceBuffer<JobXf> up_xfs;

    uint32_t last_segments = 0, last_cells = 0, last_entries = 0, last_gaps = 0;
    bool last_tables_sync_free = false, last_tables_redone = false;  // how the last frame's painter tables were built
    uint32_t last_tiles_x = 0, last_tiles_y = 0;  // tile grid of the last render (forma_renderer_row_costs)
    RasterArgs last_raster{};        // line-setup arguments of the last render (device pointers owned by its composition)
    bool last_raster_valid = false;
    uint64_t h2d_bytes = 0, d2h_bytes = 0;  // bytes copied over PCIe since creation
    double stage_ms[8] = {0};               // see forma_renderer_stage_times (valid after resolve_times)
    double kernel_ms[4] = {0};              // see forma_renderer_kernel_times
    uint32_t kernel_launches[4] = {0};
    bool times_pending = false;             // the last render's events have not been turned into stage_ms / kernel_ms yet
    int pending_sort_passes = 0;
    uint32_t pending_paint_launches = 0;
    void resolve_times() {
        if (!times_pending || !timer.ok) return;
        times_pending = false;
        cudaSetDevice(device);
        auto el = [&](int a, int b) {
            float ms = 0;
            cudaEventElapsedTime(&ms, timer.ev[a], timer.ev[b]);
            return (double)ms;
        };
        stage_ms[0] = el(0, 7);  // uploads (geometry programs + flatten eval + tables)
        stage_ms[1] = el(7, 1);  // line setup: count pass + scan (+ count read-back)
        stage_ms[2] = el(1, 2);  // pixel-grid intersection (emit)
        stage_ms[3] = el(2, 3);  // sort (upsweep / tile scan / downsweep per digit), no host sync inside
        stage_ms[4] = el(3, 4);  // painter tables: cells, carries, entries (2 pair sorts)
        stage_ms[5] = el(4, 5);  // paint kernel alone (host frames: its band launches)
        stage_ms[6] = el(5, 6);  // device -> host copy of the framebuffer
        stage_ms[7] = el(0, 6);  // whole call on the device timeline
        kernel_ms[0] = kernel_ms[1] = 0;
        // (the sort records no event of its own where a pass starts or the sort ends: launch_radix_sort)
        for (int p = 0; p < pending_sort_passes; ++p) {
            float a = 0, b = 0;
            cudaEventElapsedTime(&a, p ? timer.sort_ev[3 * p - 1] : timer.ev[2], timer.sort_ev[3 * p + 1]);
            cudaEventElapsedTime(&b, timer.sort_ev[3 * p + 1], p + 1 < pending_sort_passes ? timer.sort_ev[3 * p + 2] : timer.ev[3]);
            kernel_ms[1] += a;  // upsweep + tile scan
            kernel_ms[0] += b;  // downsweep
        }
        kernel_launches[0] = kernel_launches[1] = (uint32_t)pending_sort_passes;
        kernel_ms[2] = stage_ms[5];
        kernel_launches[2] = pending_paint_launches;
    }
    uint32_t* pinned_totals = nullptr;  // 16 x u32 pinned host words for count read-backs
    uint32_t* pinned_totals_dev = nullptr;  // their device address (set at first use)
    bool paint_counter_zeroed = false;  // sync-free tables cleared the paint kernel's tile counter (totals[3])
    // Renderers of a multi-device / sliced frame: the per-row costs of the frame (see
    // row_cost_kernel) travel back behind the frame itself, without a synchronisation of their own.
    bool track_row_costs = false;
    DeviceBuffer<unsigned long long> d_row_costs;
    PinnedBuffer<unsigned long long> h_row_costs;
    uint32_t row_costs_rows = 0;  // rows of h_row_costs that belong to the last render (0 = none)
    uint32_t last_slices = 0;     // slices of the last host frame (0 = rendered as one piece)
    // Slice renderers of a host-frame pipeline: the uploads of the slices are issued by one thread,
    // slice after slice, and chained (a slice's copies wait for the previous slice's), so that slice k
    // has its geometry - and starts computing - while slices k + 1 ... are still crossing PCIe.
    cudaEvent_t upload_done_ev = nullptr;  // recorded behind this renderer's last host -> device copy
    cudaEvent_t upload_after = nullptr;    // this renderer's copies wait for it (the previous slice's upload_done_ev)
    bool prefetched = false;               // prefetch() ran for the coming render: timer.ev[0] is already recorded
    int prefetch(Composition& comp, uint64_t width, uint64_t height, const forma_rect* crop);
    int ensure_timer() {
        if (!timer.ok) {
            for (auto& e : timer.ev) FORMA_CUDA_TRY(cudaEventCreate(&e));
            for (auto& e : timer.sort_ev) FORMA_CUDA_TRY(cudaEventCreate(&e));
            timer.ok = true;
        }
        return FORMA_STATUS_OK;
    }

    ~Renderer() {
        if (pinned_totals) cudaFreeHost(pinned_totals);
        if (count_ev) cudaEventDestroy(count_ev);
        if (upload_done_ev) cudaEventDestroy(upload_done_ev);
        if (band_streams_ok)
            for (auto& e : band_ev) cudaEventDestroy(e);
        for (uint32_t k = 0; k < band_streams_made; ++k) cudaStreamDestroy(band_stream[k]);
        if (timer.ok) {
            for (auto& e : timer.ev) cudaEventDestroy(e);
            for (auto& e : timer.sort_ev) cudaEventDestroy(e);
        }
        if (aux_stream) {
            cudaEventDestroy(aux_ev[0]);
            cudaEventDestroy(aux_ev[1]);
            cudaStreamDestroy(aux_stream);
        }
        if (owns_stream && stream) cudaStreamDestroy(stream);
    }

    int flush_geometry(Composition& comp, float band_lo = 0.0f, float band_hi = 0.0f, bool band_is_partial = false);
    int upload_tables(Composition& comp, int64_t cache_id);
    int upload_tables_device(Composition& comp, CompDevice& cd);
    // views / n_views: the line setup of a views request (a stacked frame of n_views views); batch:
    // that of a batch request (comp is then null).
    // poses: that of a poses request (n_views frames).
    // inst: that of an instance request.
    // n_bound (a single frame, see sort_bound): launch the emit over that many segments and the
    // previous frame's sort plan without reading the count back; *n_out = n_bound, and the real
    // count follows in totals[0] (its live copy for the kernels in totals[7], CountCheck).
    int rasterize(Composition* comp, uint32_t width, uint32_t height, float band_lo, float band_hi, uint32_t* n_out,
                  const ViewArgs* views = nullptr, uint32_t n_views = 0, const BatchLines* batch = nullptr,
                  const PoseArgs* poses = nullptr, const InstanceLines* inst = nullptr, uint32_t n_bound = 0);
    // The segment-count bound of a frame that takes the sync_free_sort path, or 0 when it reads its
    // count back (see run_frame).
    uint32_t sort_bound(const FrameRequest& q, const FramePlan& p);
    static uint32_t sort_count_floor();
    // Refuses a frame of n >= 2^30 segments (the limit of the sort's look-back counters).
    int refuse_segments(uint32_t n);
    bool last_sort_sync_free = false, last_sort_redone = false;  // how the last frame's segment count reached the sort
    // Every frame, whatever its kind and targets: check_request, the PaintScene (begin_frame), each
    // target's device frame, run_frame and, for a layer cache, its bookkeeping.
    int render(const FrameRequest& q);
    int check_request(const FrameRequest& q);
    int check_masks(const FrameRequest& q);
    int check_stats(const FrameRequest& q);
    int check_poses(const FrameRequest& q);
    int check_instances(const FrameRequest& q);
    // One frame of S: uploads, line setup, sort, then the painter tables, paint_step and
    // output_step once or, when the sync-free bounds were too small, twice.
    int run_frame(const FrameRequest& q, PaintScene& S, const FramePlan& p);
    int paint_step(const FrameRequest& q, const PaintScene& S, const FramePlan& p, const TileTables& t, uint32_t* paint_launches);
    int output_step(const FrameRequest& q, const PaintScene& S, const FramePlan& p);
    DeviceBuffer<uint8_t> id_flags;   // per entry: the ID kernel's optimizer flags (clip tiles)
    DeviceBuffer<uint32_t> id_frame;  // the ID target's scratch frame
    DeviceBuffer<uint8_t> mask_frame; // the planes of host masks
    DeviceBuffer<forma_layer_stats> stats_scratch;  // the records of host statistics
    PinnedBuffer<float> h_views;
    DeviceBuffer<float> d_views;
    // Poses: where the current request's transforms, visible and colors tables are (check_poses:
    // true = device memory of this device, read there), the window's K records as the host builds
    // them, the copies of host tables, the n x K pose records and the fold's first failing record.
    bool pose_tables_on_device[3] = {false, false, false};
    PinnedBuffer<PoseRec> h_pose_window;
    DeviceBuffer<PoseRec> d_pose_window;
    PinnedBuffer<float> h_pose_xf;
    DeviceBuffer<float> d_pose_xf;
    PinnedBuffer<uint8_t> h_pose_vis;
    DeviceBuffer<uint8_t> d_pose_vis;
    DeviceBuffer<PoseRec> d_poses;
    PinnedBuffer<uint32_t> h_pose_first_bad;
    DeviceBuffer<uint32_t> d_pose_first_bad;
    // Queues the window records, the host tables' bytes and pose_fold_kernel, which writes the
    // n x K pose records; with device transforms, reads back whether the fold refused one.
    int upload_poses(const FrameRequest& q);
    // Pose fills (forma_poses::colors): the colours as uploaded, 16 bytes per record, and the pose
    // style table the call's PaintScene reads (PoseFillArgs).
    PinnedBuffer<float4> h_pose_colors;
    DeviceBuffer<float4> d_pose_colors;
    DeviceBuffer<StyleRec> pose_styles;
    // Queues the upload of a poses request's colours and the build of its pose style table, and
    // points S at the table; `fills` receives the merge's arguments.
    int upload_pose_fills(const FrameRequest& q, PaintScene& S, PoseFillArgs& fills);
    // Instances: where the current request's prototypes, transforms and colors tables are
    // (check_instances: true = device memory of this device), the host's copy of the prototypes
    // (a device table's is read back there), the line records with the frame records ahead of them,
    // the prototypes' own transforms by order, the device copies of host tables, the n M instance
    // records and the fold's first failing record, and the call's order -> style table.
    bool inst_tables_on_device[3] = {false, false, false};
    std::vector<const Layer*> inst_layers;               // the distinct prototypes, in order of first appearance
    std::unordered_map<uint32_t, uint32_t> inst_index;   // prototype order -> its index in inst_layers
    PinnedBuffer<uint32_t> h_inst_protos;
    DeviceBuffer<uint32_t> d_inst_protos;
    PinnedBuffer<uint8_t> h_inst_lines;  // BatchFrame per frame, cta_first, frame_first, then the InstanceLines
    DeviceBuffer<uint8_t> d_inst_lines;
    PinnedBuffer<PoseRec> h_inst_base;
    DeviceBuffer<PoseRec> d_inst_base;
    PinnedBuffer<float> h_inst_xf;
    DeviceBuffer<float> d_inst_xf;
    DeviceBuffer<PoseRec> d_inst_recs;
    PinnedBuffer<float4> h_inst_colors;
    DeviceBuffer<float4> d_inst_colors;
    DeviceBuffer<StyleRec> inst_styles;
    DeviceBuffer<int32_t> inst_order_to_style;
    // Queues the records and tables of an instance request and points S at its tables; with
    // device transforms, reads back whether the fold refused one.
    int upload_instances(const FrameRequest& q, PaintScene& S, InstanceLines& lines);
    // A batch's distinct compositions' tables are gathered into the batch tables below, which are
    // kept until a batch of other compositions or other table versions comes (batch_key).
    std::vector<std::pair<uint64_t, uint64_t>> batch_key;  // (Composition::serial, tables_version) of the distinct compositions
    std::vector<std::pair<uint64_t, uint64_t>> batch_key_next;
    std::vector<Composition*> batch_distinct;  // of the current call, in order of first appearance (check_request)
    std::vector<uint32_t> batch_slot;          // per frame: its composition's index in batch_distinct
    PinnedBuffer<uint8_t> h_batch_lines;  // BatchFrame per frame, then cta_first
    DeviceBuffer<uint8_t> d_batch_lines;
    PinnedBuffer<BatchTableSrc> h_batch_src;
    DeviceBuffer<BatchTableSrc> d_batch_src;
    DeviceBuffer<int32_t> batch_order_to_style;
    DeviceBuffer<StyleRec> batch_styles;
    DeviceBuffer<GradRec> batch_grads;
    DeviceBuffer<StopRec> batch_stops;
    DeviceBuffer<uint16_t> batch_texels;
    int bind_batch(Composition* const* comps, uint32_t n, PaintScene& S, uint32_t height, BatchLines& lines);
    // The stages of a frame, in the order they run: begin_frame in render, the rest in run_frame.
    int begin_frame(PaintScene& S, uint64_t width, uint64_t stride, uint64_t height, const uint32_t channels[4],
                    const float clear[4], const forma_rect* crop);
    int bind_frame(Composition& comp, PaintScene& S, LayerCache* cache, const float clear[4], bool pack_written);
    // n_dev (sync_free only): the segment count in device memory, n being its bound.
    int build_tables(const PaintScene& S, uint32_t n, bool sync_free, uint32_t prev_cells, uint32_t prev_gaps, uint32_t* heavy_lists,
                     DevCounts& dc, const BatchArgs* batch, const PoseFillArgs* fills = nullptr, const uint32_t* n_dev = nullptr);
    int queue_row_costs(const PaintScene& S, uint32_t n, const uint32_t* n_dev = nullptr);
    int paint(const PaintScene& S, const TileTables& t, uint8_t* fb, uint8_t* buffer, uint64_t stride, bool in_bands,
              uint32_t* paint_launches, uint32_t view_rows = 0, uint32_t bpp = 4, bool solid_over = false, bool over = false);
    int copy_to_host(const PaintScene& S, uint8_t* buffer, const uint8_t* fb, uint64_t stride, cudaStream_t s, uint32_t bpp = 4);
    int scatter_written_tiles(const PaintScene& S, const uint8_t* fb, uint8_t* buffer, uint64_t stride);
};

// Rect::new (renderer.rs:43-52): the tile columns and rows [lo, hi) a crop covers (the whole
// frame without one).
struct TileRect {
    uint32_t tx_lo, tx_hi, ty_lo, ty_hi;
};
// The most views of `height` rows one views request takes: the stacked frame's tile rows
// are the biased rows 1 ... n * rows of the 11-bit tile_y field, and the painter tables' sentinel
// row (tiles_y + 1, see sentinel_key) must fit in it too: n * rows <= 2046.
inline uint32_t max_views(uint64_t height) {
    if (height == 0 || height > FORMA_MAX_HEIGHT) return 0;
    return (uint32_t)(2046u / ((height + 15u) / 16u));
}

inline TileRect tile_rect(uint64_t width, uint64_t height, const forma_rect* crop) {
    const uint32_t tiles_x = (uint32_t)((width + 15u) / 16u), tiles_y = (uint32_t)((height + 15u) / 16u);
    TileRect t{0, tiles_x, 0, tiles_y};
    if (crop) {
        t.tx_lo = (uint32_t)std::min<uint64_t>(crop->hor_start / 16u, tiles_x);
        t.tx_hi = (uint32_t)std::min<uint64_t>((crop->hor_end + 15u) / 16u, tiles_x);
        t.ty_lo = (uint32_t)std::min<uint64_t>(crop->vert_start / 16u, tiles_y);
        t.ty_hi = (uint32_t)std::min<uint64_t>((crop->vert_end + 15u) / 16u, tiles_y);
        if (t.tx_hi < t.tx_lo) t.tx_hi = t.tx_lo;
        if (t.ty_hi < t.ty_lo) t.ty_hi = t.ty_lo;
    }
    return t;
}

QuadUp quad_upload(const QuadRec& q);


// No C++ exception crosses the C ABI: a failed host allocation (std::bad_alloc
// from the containers behind these calls) is reported through the call's error
// value and forma_last_error() like any other failure.
template <class R, class F>
static R guarded(R on_error, F&& f) noexcept {
    try {
        return f();
    } catch (const std::exception& e) {
        set_error("host error: %s", e.what());
    } catch (...) {
        set_error("host error: unknown exception");
    }
    return on_error;
}
template <class F>
static void guarded_void(F&& f) noexcept {
    guarded(0, [&] { f(); return 0; });
}

}  // namespace forma

struct forma_composition { forma::Composition c; };
struct forma_renderer {
    forma::Renderer r;
    // Host-frame pipeline (forma_renderer_render): slice renderers on this renderer's device,
    // created at the first frame that is sliced.
    forma_renderer_multi* slicer = nullptr;
    ~forma_renderer() { forma_renderer_multi_free(slicer); }
};

// Host-frame pipeline (multi_renderer.cu) of a single host RGBA frame without a layer cache:
// returns -1 when the frame is not sliced and the plain path has to render it.
int sliced_host_render(forma_renderer* r, const forma::FrameRequest& q);
