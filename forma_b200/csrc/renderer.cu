// forma_b200 — Renderer: the uploads and the frames.
//
// A frame (Renderer::run_frame, and render's layer-cache steps) follows forma/src/cpu/renderer.rs:75-224 stage by stage;
// every stage is a CUDA kernel sequence on one stream, and there is no CPU
// fallback: without a usable sm_90 device forma_renderer_new() fails.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "renderer.hpp"

namespace forma {

QuadUp quad_upload(const QuadRec& q) {
    QuadUp u;
    for (int k = 0; k < 3; ++k) {
        u.px[k] = q.px[k];
        u.py[k] = q.py[k];
        u.pw[k] = q.pw[k];
    }
    u.prev_curv = q.prev_curv;
    u.total = q.total;
    u.step = q.step;
    return u;
}

// Evaluates the Layer::insert jobs that are not resident on this device yet into its
// segment buffer: one batched upload from pinned staging + one kernel. With a band
// ([band_lo, band_hi) in pixel rows, narrower than the frame) and no layer transform in
// the composition, inserts that cannot reach the band are left out: a GPU that paints a
// band of tile rows then uploads, evaluates and scans only the geometry of its band.
int Renderer::flush_geometry(Composition& comp, float band_lo, float band_hi, bool band_is_partial) {
    comp.compact_geom();
    CompDevice& cd = comp.on(res_key);
    if (cd.geom_epoch != comp.geom_epoch) {  // compacted since: the resident points are stale
        cd.reset_residency();
        cd.geom_epoch = comp.geom_epoch;
    }
    // The filter only holds while no layer moves its geometry (a layer transform would have to be
    // applied to the bounds, and changes from frame to frame): fall back to everything otherwise.
    // (comp.layers_have_xf is maintained by rebuild_tables, which every caller runs first.)
    const bool want_filter = band_is_partial && !comp.layers_have_xf && options().band_filter != 0;
    if (cd.jobs_resident > 0) {
        // What is resident must cover what this render needs.
        const bool covers = !cd.filtered || (want_filter && band_lo >= cd.band_lo && band_hi <= cd.band_hi);
        if (!covers) cd.reset_residency();
    }
    if (cd.jobs_resident == 0) {
        cd.filtered = want_filter;
        cd.band_lo = band_lo;
        cd.band_hi = band_hi;
    }
    const size_t from = cd.jobs_resident, to = comp.jobs.size();
    if (from == to) return FORMA_STATUS_OK;
    if (to - from >= (1u << 30)) {
        set_error("too many inserts in one batch");
        return FORMA_STATUS_CAPACITY;
    }
    auto wanted = [&](const PendingInsert& p) { return !cd.filtered || !(p.y_min >= cd.band_hi || p.y_max <= cd.band_lo); };

    if (!cd.staged_valid || cd.staged_from != from || cd.staged_to != to || cd.staged_filtered != cd.filtered ||
        (cd.filtered && (cd.staged_lo != cd.band_lo || cd.staged_hi != cd.band_hi))) {
        // (Re)build the pinned staging copy of the flatten programs of the wanted jobs in [from, to).
        size_t n_jobs = 0, n_splines = 0, n_quads = 0, n_pts = 0, n_recs = 0, n_xfs = 0;
        bool rational = false;  // any weight != 1 in the batch: 48-byte QuadUp, else 36-byte QuadUpPoly
        for (size_t j = from; j < to; ++j) {
            if (!wanted(comp.jobs[j])) continue;
            const FlattenProgram& prog = comp.jobs[j].data->program();
            rational = rational || prog.rational;
            ++n_jobs;
            n_xfs += comp.jobs[j].has_xf ? 1u : 0u;
            n_splines += prog.splines.size();
            n_recs += prog.points.size();
            n_quads += prog.quads.size();
            n_pts += prog.n_points;
        }
        if ((uint64_t)cd.n_resident + n_pts >= (1ull << 32)) {
            set_error("too many points in the segment buffer");
            return FORMA_STATUS_CAPACITY;
        }
        FORMA_CUDA_TRY(cudaStreamSynchronize(stream));  // staging may still be in flight
        FORMA_CUDA_TRY(cd.h_splines.reserve(n_splines + 1));
        FORMA_CUDA_TRY(cd.h_points.reserve(n_recs + 1));
        FORMA_CUDA_TRY(cd.h_kinds.reserve(n_recs + 1));
        FORMA_CUDA_TRY(cd.h_quads.reserve(n_quads + 1));
        FORMA_CUDA_TRY(cd.h_jobs.reserve(n_jobs + 1));
        FORMA_CUDA_TRY(cd.h_xfs.reserve(n_xfs + 1));
        size_t ji = 0, si = 0, qi = 0, pi = 0, ri = 0, xi = 0;
        for (size_t j = from; j < to; ++j) {
            const PendingInsert& p = comp.jobs[j];
            if (!wanted(p)) continue;
            const FlattenProgram& prog = p.data->program();
            FlattenJob& job = cd.h_jobs.ptr[ji++];
            job.first_point = (uint32_t)pi;  // relative to the batch; the batch lands at the device's resident point count
            job.quad_base = (uint32_t)qi;
            job.spline_base = (uint32_t)(prog.splines.empty() ? ri : si);
            job.n_splines = (uint32_t)prog.splines.size();
            job.geom_id = p.geom_id;
            job.xf_index = 0;
            if (p.has_xf) {
                std::memcpy(cd.h_xfs.ptr[xi].xf, p.xf, sizeof(p.xf));
                job.xf_index = (uint32_t)++xi;
            }
            if (!prog.splines.empty())
                std::memcpy(cd.h_splines.ptr + si, prog.splines.data(), prog.splines.size() * sizeof(SplineRec));
            if (!prog.points.empty()) {
                std::memcpy(cd.h_points.ptr + ri, prog.points.data(), prog.points.size() * sizeof(PointRec));
                std::memcpy(cd.h_kinds.ptr + ri, prog.kinds.data(), prog.kinds.size());
                ri += prog.points.size();
            }
            if (rational) {
                for (size_t q = 0; q < prog.quads.size(); ++q) cd.h_quads.ptr[qi + q] = quad_upload(prog.quads[q]);
            } else {  // the pinned buffer is sized for QuadUp; the smaller records share it
                QuadUpPoly* poly = reinterpret_cast<QuadUpPoly*>(cd.h_quads.ptr);
                for (size_t q = 0; q < prog.quads.size(); ++q) {
                    const QuadRec& s = prog.quads[q];
                    QuadUpPoly& u = poly[qi + q];
                    for (int k = 0; k < 3; ++k) {
                        u.px[k] = s.px[k];
                        u.py[k] = s.py[k];
                    }
                    u.prev_curv = s.prev_curv;
                    u.total = s.total;
                    u.step = s.step;
                }
            }
            si += prog.splines.size();
            qi += prog.quads.size();
            pi += prog.n_points;
        }
        cd.staged_valid = true;
        cd.staged_from = from;
        cd.staged_to = to;
        cd.staged_filtered = cd.filtered;
        cd.staged_lo = cd.band_lo;
        cd.staged_hi = cd.band_hi;
        cd.staged_jobs = n_jobs;
        cd.staged_splines = n_splines;
        cd.staged_recs = n_recs;
        cd.staged_quads = n_quads;
        cd.staged_points = n_pts;
        cd.staged_xfs = n_xfs;
        cd.staged_rational = rational;
    }  // else: the same batch as last time (an evicted composition) is uploaded again from the same staging
    cd.jobs_resident = to;
    if (!cd.staged_jobs) return FORMA_STATUS_OK;
    const uint32_t n_after = cd.n_resident + (uint32_t)cd.staged_points;
    FORMA_CUDA_TRY(cd.d_x.reserve(n_after, true, stream));
    FORMA_CUDA_TRY(cd.d_y.reserve(n_after, true, stream));
    FORMA_CUDA_TRY(cd.d_gid.reserve(n_after, true, stream));
    const size_t quad_bytes = cd.staged_rational ? sizeof(QuadUp) : sizeof(QuadUpPoly);
    FORMA_CUDA_TRY(up_splines.reserve(cd.staged_splines + 1));
    FORMA_CUDA_TRY(up_points.reserve(cd.staged_recs + 1));
    FORMA_CUDA_TRY(up_kinds.reserve(cd.staged_recs + 1));
    FORMA_CUDA_TRY(up_quads.reserve(cd.staged_quads + 1));
    FORMA_CUDA_TRY(up_jobs.reserve(cd.staged_jobs));
    FORMA_CUDA_TRY(up_xfs.reserve(cd.staged_xfs + 1));
    // The quadratics go first: their expansion kernel runs on a side stream while the copy
    // engine keeps sending the other records.
    bool expanding = false;
    if (upload_after) FORMA_CUDA_TRY(cudaStreamWaitEvent(stream, upload_after, 0));
    if (cd.staged_quads) {
        FORMA_CUDA_TRY(up_quads_raw.reserve(cd.staged_quads + 1));
        FORMA_CUDA_TRY(cudaMemcpyAsync(up_quads_raw.ptr, cd.h_quads.ptr, cd.staged_quads * quad_bytes, cudaMemcpyHostToDevice,
                                       stream));
        if (!aux_stream) {
            FORMA_CUDA_TRY(cudaStreamCreateWithFlags(&aux_stream, cudaStreamNonBlocking));
            FORMA_CUDA_TRY(cudaEventCreateWithFlags(&aux_ev[0], cudaEventDisableTiming));
            FORMA_CUDA_TRY(cudaEventCreateWithFlags(&aux_ev[1], cudaEventDisableTiming));
        }
        FORMA_CUDA_TRY(cudaEventRecord(aux_ev[0], stream));
        FORMA_CUDA_TRY(cudaStreamWaitEvent(aux_stream, aux_ev[0], 0));
        if (cd.staged_rational)
            launch_quad_expand(up_quads_raw.ptr, up_quads.ptr, (uint32_t)cd.staged_quads, aux_stream);
        else
            launch_quad_expand_poly(reinterpret_cast<const QuadUpPoly*>(up_quads_raw.ptr), up_quads.ptr,
                                    (uint32_t)cd.staged_quads, aux_stream);
        FORMA_CUDA_TRY(cudaEventRecord(aux_ev[1], aux_stream));
        expanding = true;
        ++launches;
    }
    if (cd.staged_splines)
        FORMA_CUDA_TRY(cudaMemcpyAsync(up_splines.ptr, cd.h_splines.ptr, cd.staged_splines * sizeof(SplineRec),
                                       cudaMemcpyHostToDevice, stream));
    if (cd.staged_recs) {
        FORMA_CUDA_TRY(cudaMemcpyAsync(up_points.ptr, cd.h_points.ptr, cd.staged_recs * sizeof(PointRec), cudaMemcpyHostToDevice,
                                       stream));
        FORMA_CUDA_TRY(cudaMemcpyAsync(up_kinds.ptr, cd.h_kinds.ptr, cd.staged_recs, cudaMemcpyHostToDevice, stream));
    }
    FORMA_CUDA_TRY(cudaMemcpyAsync(up_jobs.ptr, cd.h_jobs.ptr, cd.staged_jobs * sizeof(FlattenJob), cudaMemcpyHostToDevice, stream));
    if (cd.staged_xfs)
        FORMA_CUDA_TRY(cudaMemcpyAsync(up_xfs.ptr, cd.h_xfs.ptr, cd.staged_xfs * sizeof(JobXf), cudaMemcpyHostToDevice, stream));
    if (upload_done_ev) FORMA_CUDA_TRY(cudaEventRecord(upload_done_ev, stream));
    h2d_bytes += cd.staged_splines * sizeof(SplineRec) + cd.staged_recs * (sizeof(PointRec) + 1) +
                 cd.staged_quads * quad_bytes + cd.staged_jobs * sizeof(FlattenJob) + cd.staged_xfs * sizeof(JobXf);
    if (expanding) FORMA_CUDA_TRY(cudaStreamWaitEvent(stream, aux_ev[1], 0));
    launch_flatten_eval(up_splines.ptr, up_points.ptr, up_kinds.ptr, up_quads.ptr, up_jobs.ptr, up_xfs.ptr, (uint32_t)cd.staged_jobs,
                        (uint32_t)cd.staged_points, cd.n_resident, cd.d_x.ptr, cd.d_y.ptr, cd.d_gid.ptr, stream);
    ++launches;
    FORMA_CUDA_TRY(cudaGetLastError());
    cd.n_resident = n_after;
    return FORMA_STATUS_OK;
}

// geom id -> layer slot, layer records, style table (segment.rs:141-149 does
// these look-ups per point). The pinned host copies are rebuilt when the
// composition changed and re-uploaded when they are not resident.
int Renderer::upload_tables(Composition& comp, int64_t cache_id) {
    comp.compact_geom();  // renumbers the geometry ids the tables are built from (no-op unless half of the points are dead)
    CompDevice& cd = comp.on(res_key);
    if (comp.tables_dirty || comp.tables_cache_id != cache_id) {
        FORMA_CUDA_TRY(cudaStreamSynchronize(stream));  // an upload from the pinned tables may still be in flight
        int st = comp.rebuild_tables(cache_id);
        if (st) return st;
    }
    if (cd.tables_version == comp.tables_version) return FORMA_STATUS_OK;
    return upload_tables_device(comp, cd);
}

int Renderer::upload_tables_device(Composition& comp, CompDevice& cd) {
    auto up = [&](auto& dbuf, const auto& hbuf, size_t n) -> cudaError_t {
        cudaError_t e = dbuf.reserve(n + 1);
        if (e != cudaSuccess || n == 0) return e;
        h2d_bytes += n * sizeof(*hbuf.ptr);
        return cudaMemcpyAsync(dbuf.ptr, hbuf.ptr, n * sizeof(*hbuf.ptr), cudaMemcpyHostToDevice, stream);
    };
    // Layers without transforms (the common case) travel as 4 bytes each instead of 36.
    if (comp.layers_have_xf) FORMA_CUDA_TRY(up(cd.d_layers, comp.h_layers, comp.n_layer_recs));
    else FORMA_CUDA_TRY(up(cd.d_layer_bits, comp.h_layer_bits, comp.n_layer_recs));
    FORMA_CUDA_TRY(up(cd.d_styles, comp.h_styles, comp.n_style_recs));
    FORMA_CUDA_TRY(up(cd.d_stops, comp.h_stops, comp.n_stops));
    FORMA_CUDA_TRY(up(cd.d_texels, comp.h_texels, comp.n_texels));
    FORMA_CUDA_TRY(up(cd.d_order_to_style, comp.h_order_to_style, comp.n_orders));
    FORMA_CUDA_TRY(up(cd.d_geom_slot, comp.h_geom_slot, comp.n_geoms));
    // Gradient records of the styles (only when some style is a gradient: n_stops > 0).
    FORMA_CUDA_TRY(cd.d_grads.reserve(comp.n_style_recs + 1));
    if (comp.n_stops) {
        launch_grad_setup(cd.d_styles.ptr, cd.d_stops.ptr, (uint32_t)comp.n_style_recs, cd.d_grads.ptr, stream);
        ++launches;
    }
    cd.tables_version = comp.tables_version;
    return FORMA_STATUS_OK;
}

// Stages 1½ + 2: fills `segs` with the unsorted pixel segments.
int Renderer::rasterize(Composition* comp, uint32_t width, uint32_t height, float band_lo, float band_hi,
                        uint32_t* n_out, const ViewArgs* views, uint32_t n_views, const BatchLines* batch) {
    RasterArgs& ra = last_raster;  // kept for forma_renderer_lines (a stacked frame has no line records)
    last_raster_valid = !views && !batch;
    if (comp) {
        CompDevice& cd = comp->on(res_key);
        ra.x = cd.d_x.ptr;
        ra.y = cd.d_y.ptr;
        ra.gid = cd.d_gid.ptr;
        ra.n_points = cd.n_resident;
        ra.geom_slot = cd.d_geom_slot.ptr;
        ra.n_geoms = comp->n_geoms;
        ra.layers = comp->layers_have_xf ? cd.d_layers.ptr : nullptr;
        ra.layer_bits = cd.d_layer_bits.ptr;
        ra.width = (float)width;
        ra.height = (float)height;
        ra.band_lo = band_lo;
        ra.band_hi = band_hi;
    }
    uint32_t nb = batch ? batch->n_ctas : raster_num_blocks(ra.n_points);
    if (views) {
        if ((uint64_t)nb * n_views >= (1ull << 32)) {
            set_error("%u views of %u points exceed the line-setup grid", n_views, ra.n_points);
            return FORMA_STATUS_CAPACITY;
        }
        nb *= n_views;  // one CTA sum per (view, CTA of points)
    }
    FORMA_CUDA_TRY(block_sums.reserve(nb + 1));
    if (batch) launch_line_count_batch(batch->args, nb, block_sums.ptr, totals.ptr + 0, totals.ptr + 4, stream);
    else if (views) launch_line_count_views(ra, *views, n_views, block_sums.ptr, totals.ptr + 0, totals.ptr + 4, stream);
    else launch_line_count(ra, block_sums.ptr, totals.ptr + 0, totals.ptr + 4, stream);
    launches += nb ? 2 : 0;
    auto emit = [&](uint32_t cap, const CountArgs* counts) {
        if (batch) launch_raster_emit_batch(batch->args, nb, block_sums.ptr, segs.ptr, cap, stream, counts);
        else if (views) launch_raster_emit_views(ra, *views, n_views, block_sums.ptr, segs.ptr, cap, stream, counts);
        else launch_raster_emit(ra, block_sums.ptr, segs.ptr, cap, stream, counts);
    };
    // The emit pass counts the sort's pass-0 digits (TileCounts) when the sort will take them: with
    // the digit of the previous frame when it runs ahead of the read-back (used when this frame's
    // plan has the same pass 0), with the plan's own when it runs after it.
    const bool counting = options().sort_counts != 0;
    auto pass0_counts = [&](const DigitSpec& spec) {
        counts_clean = false;  // what the emit counts is zero again only once a sort has consumed it
        return CountArgs{tile_counts.hist(0), spec};
    };
    last_count_source = 0;
    tile_counts.pass0 = false;
    uint32_t n = 0;
    // One read-back: segment count + the largest tile coordinates (totals[4..5]).
    FORMA_CUDA_TRY(cudaMemcpyAsync(pinned_totals, totals.ptr, 6 * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
    // The emit pass does not need the count, only room for its output: launch it
    // into the buffer of the previous frames before waiting for the read-back, so
    // that the GPU keeps working while the host wakes up. Segments beyond the
    // capacity are dropped and the pass is repeated below in that (rare) case.
    const size_t spec_cap = speculation_enabled() ? std::min<size_t>(segs.capacity, 0xFFFFFFFFu) : 0;
    const bool speculated = spec_cap > 1 && nb;
    FORMA_CUDA_TRY(ensure_count_event());
    FORMA_CUDA_TRY(cudaEventRecord(count_ev, stream));
    const bool spec_counted = speculated && counting && count_spec_valid;
    if (spec_counted) {
        FORMA_CUDA_TRY(prepare_tile_counts((uint32_t)(spec_cap - 1)));
    }
    if (speculated) {
        if (timer.ok) FORMA_CUDA_TRY(cudaEventRecord(timer.ev[1], stream));  // end of line setup (count pass)
        const CountArgs c = spec_counted ? pass0_counts(count_spec) : CountArgs{};
        emit((uint32_t)(spec_cap - 1), spec_counted ? &c : nullptr);
        ++launches;
    }
    FORMA_CUDA_TRY(cudaEventSynchronize(count_ev));  // the read-back only, not the speculative launch
    n = pinned_totals[0];
    {
        // Already ordered by layer: no layer digits (see Composition::layers_in_order).
        const bool skip_layer_digits = options().sort_full_key == 0;
        const uint64_t layer_bound = batch ? batch->layer_bound
                                     : (comp->layers_in_order && skip_layer_digits) ? 0u
                                                                                    : (comp->n_orders ? comp->n_orders - 1u : 0u);
        const uint64_t bound[3] = {layer_bound, pinned_totals[4], pinned_totals[5]};
        segment_plan = make_sort_plan(segment_key_layout(), bound);  // layer, tile_x, tile_y
        std::copy(bound, bound + 3, segment_bound);
    }
    *n_out = 0;
    last_segments = 0;  // (forma_renderer_segments / _row_costs read segs[0, last_segments))
    // n saturates at 0xFFFFFFFF (line_count_kernel, scan_block_sums_kernel): a frame at or above
    // the limit is refused, never rendered from a wrapped count. Nothing of it stays behind: the
    // speculative emit wrote only inside `segs`, and the layer cache, its unchanged bits and the
    // sync-free bounds (last_cells / last_gaps) are updated only by a frame that gets past here,
    // and the segment count and tile rows of the last frame read 0.
    if (n >= (1u << 30)) {
        count_spec_valid = false;
        if (n == 0xFFFFFFFFu)
            set_error("at least 2^32 - 1 pixel segments exceed the 2^30 limit of the sort's look-back counters");
        else
            set_error("%u pixel segments exceed the 2^30 limit of the sort's look-back counters", n);
        last_tiles_x = last_tiles_y = 0;  // no row costs either
        return FORMA_STATUS_CAPACITY;
    }
    *n_out = n;
    last_segments = n;
    FORMA_CUDA_TRY(reserve_all(n + 1, segs, segs_tmp));
    const bool sort_counted = counting && radix_sort_scans(n);
    int source = 0;
    if (!speculated || (size_t)n + 1 > spec_cap) {
        if (!speculated && timer.ok) FORMA_CUDA_TRY(cudaEventRecord(timer.ev[1], stream));  // end of line setup (count pass)
        if (sort_counted) {  // (re)counted from zero with the plan's own digit
            FORMA_CUDA_TRY(prepare_tile_counts(n));
            source = 2;
        }
        const CountArgs c = sort_counted ? pass0_counts(segment_plan.pass[0]) : CountArgs{};
        emit(n, sort_counted ? &c : nullptr);
        launches += nb ? 1 : 0;
    } else if (sort_counted) {
        if (spec_counted && same_digit(segment_plan.pass[0], count_spec)) {
            source = 1;
        } else {  // the sort counts pass 0 itself (upsweep)
            FORMA_CUDA_TRY(prepare_tile_counts(n));
            source = 3;
        }
    }
    last_count_source = source;
    tile_counts.pass0 = source == 1 || source == 2;
    count_spec_valid = sort_counted;
    count_spec = segment_plan.pass[0];
    FORMA_CUDA_TRY(cudaGetLastError());
    return FORMA_STATUS_OK;
}

cudaError_t Renderer::prepare_tile_counts(uint32_t max_keys) {
    const uint32_t tiles = std::max(sort_tiles(max_keys), 1u);
    if (tiles > tile_counts.tile_cap) {
        TileCounts t;
        counts_clean = false;
        t.tile_cap = tiles;
        cudaError_t e = sort_counts.reserve(2 * t.block_words());
        if (e != cudaSuccess) return e;
        t.tile_cap = (uint32_t)(sort_counts.capacity / 2u / 256u) - kTotalsRows;  // all that was reserved
        t.base = sort_counts.ptr;
        t.tiles_per_chunk = (t.tile_cap + kMaxChunks - 1u) / kMaxChunks;
        tile_counts = t;
    }
    tile_counts.pass0 = false;
    // A sort that took the counts leaves both blocks zero (its downsweeps clear what they read): only
    // a new buffer, or counts that no sort consumed (a fallback, rasterize_only), need the memset.
    if (counts_clean) return cudaSuccess;
    counts_clean = true;
    return cudaMemsetAsync(tile_counts.base, 0, 2 * tile_counts.block_words() * sizeof(uint32_t), stream);
}

// The pixel rows [lo, hi) a frame paints; partial: not all of its rows (flush_geometry's band filter).
struct FrameBand {
    float lo, hi;
    bool partial;
};
// The band of the tile rows [ty_lo, ty_hi) of a frame `height` rows high.
static FrameBand tile_band(uint32_t ty_lo, uint32_t ty_hi, uint64_t height) {
    return {(float)(ty_lo * 16u), (float)std::min<uint64_t>((uint64_t)ty_hi * 16u, height),
            ty_lo > 0u || ty_hi < (height + 15u) / 16u};
}

// The upload half of run_frame() on its own: tables + the geometry that the rows of `crop` need and
// that is not resident yet. The next frame then finds everything in place.
int Renderer::prefetch(Composition& comp, uint64_t width, uint64_t height, const forma_rect* crop) {
    FORMA_CUDA_TRY(cudaSetDevice(device));
    const int ts = ensure_timer();
    if (ts) return ts;
    const TileRect t = tile_rect(width, height, crop);
    FORMA_CUDA_TRY(cudaEventRecord(timer.ev[0], stream));
    prefetched = true;
    if (upload_after) FORMA_CUDA_TRY(cudaStreamWaitEvent(stream, upload_after, 0));
    const FrameBand band = tile_band(t.ty_lo, t.ty_hi, height);
    int st = upload_tables(comp, -1);
    if (st) return st;
    return flush_geometry(comp, band.lo, band.hi, band.partial);
}

// One frame of S, whatever its kind: uploads, line setup, sort, then the painter tables,
// paint_step (the frame's kernels) and output_step (the copy to where the caller wants the frame)
// once or, when the sync-free bounds were too small, twice.
int Renderer::run_frame(const FrameRequest& q, PaintScene& S, const FramePlan& p) {
    if (!prefetched) FORMA_CUDA_TRY(cudaEventRecord(timer.ev[0], stream));
    prefetched = false;
    // Lines entirely above / below the painted tile rows cannot reach a painted tile: they are
    // culled per line (rasterize), and whole inserts are left out of the device's segment
    // buffer when the band is narrower than the frame (flush_geometry). Line setup sees every
    // frame of a stack as a frame of its own: all its rows are painted.
    const uint32_t height = (uint32_t)q.height;
    const FrameBand band = p.rows ? FrameBand{0.0f, (float)height, false} : tile_band(S.ty_lo, S.ty_hi, height);
    const bool views = q.kind == FrameKind::views, batched = q.kind == FrameKind::batch;
    int st = FORMA_STATUS_OK;
    BatchLines batch{};
    if (batched) {  // every composition's uploads, then the batch tables
        st = bind_batch(q.batch, q.n, S, height, batch);
        if (st) return st;
    } else {
        st = upload_tables(*q.comp, -1);
        if (st) return st;
        st = flush_geometry(*q.comp, band.lo, band.hi, band.partial);
        if (st) return st;
        st = bind_frame(*q.comp, S, q.cache, S.clear, p.pack_written);
        if (st) return st;
    }
    if (views) {
        const uint32_t nv = q.n;
        FORMA_CUDA_TRY(h_views.reserve(6u * nv));
        FORMA_CUDA_TRY(d_views.reserve(6u * nv));
        std::memcpy(h_views.ptr, q.views, 6u * nv * sizeof(float));  // (the previous call's copy is complete: rasterize waited for it)
        FORMA_CUDA_TRY(cudaMemcpyAsync(d_views.ptr, h_views.ptr, 6u * nv * sizeof(float), cudaMemcpyHostToDevice, stream));
        h2d_bytes += 6u * nv * sizeof(float);
    }
    const ViewArgs va{d_views.ptr, (height + 15u) / 16u};

    FORMA_CUDA_TRY(cudaEventRecord(timer.ev[7], stream));
    uint32_t n = 0;
    st = rasterize(q.comp, S.width, height, band.lo, band.hi, &n, views ? &va : nullptr, q.n, batched ? &batch : nullptr);
    if (st) return st;

    // Stage 3: sort.
    FORMA_CUDA_TRY(cudaEventRecord(timer.ev[2], stream));
    int timed_sort_passes = 0;
    if (n > 1) {
        FORMA_CUDA_TRY(sort_scratch.reserve(radix_scratch_bytes(n)));
        uint32_t* keep = nullptr;
        kept_passes = kept_tiles = 0;
        if (keep_sort_counts && last_count_source) {
            FORMA_CUDA_TRY(kept_counts.reserve((size_t)segment_plan.n_passes * sort_tiles(n) * 256u));
            keep = kept_counts.ptr;
            kept_passes = segment_plan.n_passes;
            kept_tiles = sort_tiles(n);
        }
        timed_sort_passes = sort(segs, segs_tmp, nullptr, nullptr, n, segment_plan, timer.sort_ev, nullptr, nullptr, nullptr,
                                 last_count_source ? &tile_counts : nullptr, keep)
                                .timed_passes;
        if (last_count_source) counts_clean = true;  // (rasterize reserved the counts for n keys: the sort took them)
        FORMA_CUDA_TRY(cudaGetLastError());
    }
    FORMA_CUDA_TRY(cudaEventRecord(timer.ev[3], stream));

    // Stage 4: cells -> carries -> entries -> paint.
    const size_t n_tiles_total = (size_t)S.tiles_x * S.tiles_y;
    last_tiles_x = S.tiles_x;
    last_tiles_y = S.tiles_y;
    FORMA_CUDA_TRY(tile_range.reserve(n_tiles_total));
    FORMA_CUDA_TRY(heavy_tiles.reserve(n_tiles_total * kHeavyListClasses));
    // Heavy tiles first (longest-processing-time order): their lists + counts (heavy_count()). The
    // tile kernels read them with the rest of the tables (TileTables), taken after build_tables,
    // which may move any of them.
    uint32_t* const heavy_lists = options().paint_lpt ? heavy_tiles.ptr : nullptr;
    // Tables + paint + output, once or (rarely) twice. sync_free = without count read-backs: the
    // tables of a frame are normally about as large as those of the frame before, so every
    // kernel is launched over bounds derived from the previous counts and reads the real counts
    // from device memory (DevCounts); the host looks at them only after the frame's final
    // synchronisation. A count above its bound (the kernels then did nothing, the frame holds
    // the clear colour) sends the frame through again with counted tables.
    // A frame with a layer cache is never sync-free: its first attempt would write the clear colour
    // into the caller's buffer and record it in the cache's tiles, and the redo would then skip the
    // tiles it finds unchanged (and the host scatter of the written tiles must not see a redone frame).
    const uint32_t prev_cells = last_cells, prev_gaps = last_gaps;  // of this renderer's previous frame
    const bool fast = options().sync_free && n > 0 && prev_cells > 0 && !q.cache;
    last_cells = last_entries = 0;
    last_written_tiles = 0;
    last_tables_redone = false;
    uint32_t paint_launches = 1;
    for (bool sync_free = fast;; sync_free = false) {
        DevCounts dc;
        st = build_tables(S, n, sync_free, prev_cells, prev_gaps, heavy_lists, dc, batched ? &batch.args : nullptr);
        if (st) return st;
        st = queue_row_costs(S, n);
        if (st) return st;
        FORMA_CUDA_TRY(cudaEventRecord(timer.ev[4], stream));
        st = paint_step(q, S, p, TileTables{segs.ptr, recs.ptr, tile_range.ptr, heavy_lists, heavy_count()}, &paint_launches);
        if (st) return st;
        FORMA_CUDA_TRY(cudaEventRecord(timer.ev[5], stream));
        st = output_step(q, S, p);
        if (st) return st;
        FORMA_CUDA_TRY(cudaEventRecord(timer.ev[6], stream));
        FORMA_CUDA_TRY(cudaStreamSynchronize(stream));
        if (!sync_free) break;
        last_cells = pinned_totals[1];
        last_gaps = pinned_totals[2];
        last_entries = last_cells + last_gaps;
        if (last_cells <= dc.cell_bound && last_gaps <= dc.gap_bound) break;
        last_tables_redone = true;
    }
    last_tables_sync_free = fast && !last_tables_redone;
    // The stage times are read from the events when somebody asks for them (resolve_times): a dozen
    // event queries are not part of rendering a frame.
    times_pending = true;
    pending_sort_passes = timed_sort_passes;
    pending_paint_launches = paint_launches;
    if (forma_timings* timings = q.timings) {
        resolve_times();
        timings->line_setup_ms = stage_ms[1];
        timings->rasterize_ms = stage_ms[2];
        timings->sort_ms = stage_ms[3];
        timings->paint_ms = stage_ms[4] + stage_ms[5];
        if (q.comp) {
            const CompDevice& cd = q.comp->on(res_key);
            timings->n_lines = cd.n_resident ? cd.n_resident - 1 : 0;
        } else {
            timings->n_lines = batch.n_lines;
        }
        timings->n_segments = n;
    }
    return FORMA_STATUS_OK;
}

int Renderer::render(const FrameRequest& q) {
    int st = check_request(q);
    if (st) return st;
    const bool stack = q.kind != FrameKind::single, rgba = q.rgba.ptr != nullptr;
    // Each target's frame on the device. A single frame keeps the caller's stride and is painted in
    // place when it is on the device. A stack is painted in place when its frames are whole tile
    // rows laid out as the stacked frame's rows; each target decides for itself.
    auto device_frame = [&](const FrameTarget& t) {
        const bool direct = t.on_device && (!stack || (q.height % 16u == 0u && t.frame_stride == q.height * t.stride));
        return DeviceFrame{t.ptr, direct || !stack ? t.stride : t.bpp * q.width, direct};
    };
    FramePlan p{device_frame(q.rgba), device_frame(q.ids), stack ? (uint32_t)((q.height + 15u) / 16u) : 0u, false, false};
    // Masks are painted straight into the caller's planes on the device (a stack's tile rows are
    // mapped to its frames by the kernel), host masks into scratch planes of 16-byte aligned rows.
    p.masks = DeviceFrame{q.masks.ptr, q.masks.stride, q.masks.on_device};
    p.mask_plane_stride = q.masks.plane_stride;
    if (q.masks.ptr && !q.masks.on_device) {
        p.masks.stride = (q.masks.bpp() * q.width + 15u) / 16u * 16u;
        p.mask_plane_stride = p.masks.stride * q.height;
    }
    p.stats = q.stats.ptr;
    // The PaintScene of the RGBA target, or of the ID target, the masks or the statistics when they
    // are alone (statistics have no frame: the stride is that of an sRGB8 frame's rows).
    // An over frame has no clear colour: its kernels read each pixel's, and upgrade Alpha -> One per
    // pixel, so the scene's channels stay as given.
    static const uint32_t kIdChannels[4] = {0, 1, 2, 3};
    static const float kIdClear[4] = {0, 0, 0, 0};
    PaintScene S{};
    st = begin_frame(S, q.width, rgba ? p.rgba.stride : q.ids.ptr ? p.ids.stride : q.masks.ptr ? p.masks.stride : 4u * q.width,
                     stack ? (uint64_t)q.n * p.rows * 16u : q.height,
                     rgba ? q.channels : kIdChannels, rgba && !q.rgba.over ? q.clear : kIdClear, q.crop);
    if (st) return st;
    if (rgba && !p.rgba.direct) {
        FORMA_CUDA_TRY(framebuffer.reserve((size_t)p.rgba.stride * S.height));
        p.rgba.ptr = framebuffer.ptr;
    }
    if (q.ids.ptr && !p.ids.direct) {
        FORMA_CUDA_TRY(id_frame.reserve((size_t)(p.ids.stride / 4u) * S.height));
        p.ids.ptr = reinterpret_cast<uint8_t*>(id_frame.ptr);
    }
    if (q.masks.ptr && !p.masks.direct) {
        FORMA_CUDA_TRY(mask_frame.reserve((size_t)p.mask_plane_stride * q.masks.n_orders));
        p.masks.ptr = mask_frame.ptr;
    }
    if (q.stats.ptr && !q.stats.on_device) {
        FORMA_CUDA_TRY(stats_scratch.reserve((size_t)q.stats.n_orders));
        p.stats = stats_scratch.ptr;
    }
    // (A host float frame is painted whole and copied back once.)
    p.in_bands = rgba && q.rgba.bpp == 4u && !stack && !q.rgba.on_device && !q.cache && S.ty_hi - S.ty_lo >= (copy_bands_override ? 8u : 32u) &&
                 S.tx_hi > S.tx_lo && band_copies_enabled();
    p.pack_written = q.cache && !q.rgba.on_device;
    st = run_frame(q, S, p);
    if (st) return st;
    if (q.cache) {  // renderer.rs:217-223
        q.cache->has_clear = true;
        std::memcpy(q.cache->clear_color, q.clear, sizeof(q.cache->clear_color));
        for (auto& kv : q.comp->layers) {
            if (kv.second->enabled) kv.second->unchanged_bits |= 1u << q.cache->id;
            else kv.second->unchanged_bits &= ~(1u << q.cache->id);
        }
    }
    return FORMA_STATUS_OK;
}

// The checks of a request, before anything is written: each target (LinearLayout::new asserts,
// layout/mod.rs:188-193, consts.rs limits, and for a stack the frame count and frame stride), the
// ID target's own, then the views or the compositions of a batch. An ID-only request has no RGBA
// target to check.
int Renderer::check_request(const FrameRequest& q) {
    const bool stack = q.kind != FrameKind::single;
    const char* what = q.kind == FrameKind::views ? "view" : "frame";
    const uint64_t width = q.width, height = q.height;
    auto check_target = [&](const FrameTarget& t) {
        if (!t.ptr || width == 0 || height == 0 || width * t.bpp > t.stride || width > FORMA_MAX_WIDTH || height > FORMA_MAX_HEIGHT) {
            set_error("invalid render target %llux%llu stride %llu", (unsigned long long)width, (unsigned long long)height,
                      (unsigned long long)t.stride);
            return (int)FORMA_STATUS_INVALID;
        }
        if (!stack) return (int)FORMA_STATUS_OK;
        if (q.n == 0 || q.n > max_views(height)) {
            set_error("%u %ss of height %llu: between 1 and %u %ss of this height fit in one call", q.n, what,
                      (unsigned long long)height, max_views(height), what);
            return (int)FORMA_STATUS_INVALID;
        }
        if (t.frame_stride < (height - 1u) * t.stride + t.bpp * width) {
            set_error("%s stride %llu is smaller than one %s (%llu bytes)", what, (unsigned long long)t.frame_stride, what,
                      (unsigned long long)((height - 1u) * t.stride + t.bpp * width));
            return (int)FORMA_STATUS_INVALID;
        }
        return (int)FORMA_STATUS_OK;
    };
    int st = q.rgba.ptr || (!q.ids.ptr && !q.masks.ptr && !q.stats.ptr) ? check_target(q.rgba) : FORMA_STATUS_OK;
    if (st) return st;
    if (q.rgba.bpp != 4u && (((uintptr_t)q.rgba.ptr | q.rgba.stride | q.rgba.frame_stride) & 3u) != 0u) {
        set_error("invalid float frame: buffer, stride %llu and %s stride %llu must be multiples of 4 bytes",
                  (unsigned long long)q.rgba.stride, what, (unsigned long long)q.rgba.frame_stride);
        return FORMA_STATUS_INVALID;
    }
    if (q.rgba.over) {
        // Over frames: device memory, 4-byte aligned in every format, no ID target or layer cache, and
        // a channel order that can be decoded: a permutation of R, G, B, A, for sRGB8 with A last (a
        // solid tile's bytes encode by position, so only then do they decode to its colour).
        bool seen[4] = {false, false, false, false}, perm = q.channels != nullptr;
        for (int k = 0; perm && k < 4; ++k) {
            const uint32_t c = q.channels[k];
            perm = perm && c < 4u && !seen[c];
            if (c < 4u) seen[c] = true;
        }
        if (!q.rgba.on_device || q.ids.ptr || q.cache || !perm || (q.rgba.bpp == 4u && q.channels[3] != FORMA_CHANNEL_ALPHA) ||
            (((uintptr_t)q.rgba.ptr | q.rgba.stride | q.rgba.frame_stride) & 3u) != 0u) {
            set_error("invalid over frame: a device buffer without IDs or layer cache, channels a permutation of R, G, B, A%s, "
                      "and buffer, stride %llu and %s stride %llu multiples of 4 bytes",
                      q.rgba.bpp == 4u ? " with A last" : "", (unsigned long long)q.rgba.stride, what,
                      (unsigned long long)q.rgba.frame_stride);
            return FORMA_STATUS_INVALID;
        }
    }
    if (q.ids.ptr) {
        const FrameTarget& t = q.ids;
        if (t.stride % 4u != 0u || t.frame_stride % 4u != 0u || !std::isfinite(t.min_coverage) || t.min_coverage < 0.0f ||
            t.min_coverage >= 1.0f) {
            set_error("invalid ID frame: stride %llu, %s stride %llu (multiples of 4 bytes), min_coverage %g (finite, in [0, 1))",
                      (unsigned long long)t.stride, what, (unsigned long long)t.frame_stride, (double)t.min_coverage);
            return FORMA_STATUS_INVALID;
        }
        st = check_target(t);
        if (st) return st;
    }
    if (q.masks.ptr) {
        st = check_masks(q);
        if (st) return st;
    }
    if (q.stats.ptr) {
        st = check_stats(q);
        if (st) return st;
    }
    if ((q.kind == FrameKind::views && !q.views) || (q.kind == FrameKind::batch && !q.batch)) {
        set_error("no %s", q.kind == FrameKind::views ? "views" : "compositions");
        return FORMA_STATUS_INVALID;
    }
    for (uint32_t b = 0; q.kind == FrameKind::views && b < q.n; ++b) {  // [ux, vx, uy, vy, tx, ty], as forma_layer_set_transform checks them
        const float* v = q.views + 6u * b;
        bool finite = true;
        for (int k = 0; k < 6; ++k) finite = finite && std::isfinite(v[k]);
        if (!finite || !geom_pres_ok(v[0], v[2], v[1], v[3])) {
            set_error("view %u is not a finite transform that does not scale up", b);
            return FORMA_STATUS_INVALID;
        }
    }
    if (q.kind != FrameKind::batch) return FORMA_STATUS_OK;
    // The distinct compositions in order of first appearance, and the slices of the layer field
    // they need: n_orders each, as rebuild_tables counts them.
    batch_distinct.clear();
    batch_slot.resize(q.n);
    std::unordered_map<const Composition*, uint32_t> index;
    uint64_t order_sum = 0;
    for (uint32_t c = 0; c < q.n; ++c) {
        if (!q.batch[c]) {
            set_error("batch entry %u is null", c);
            return FORMA_STATUS_INVALID;
        }
        auto it = index.emplace(q.batch[c], (uint32_t)batch_distinct.size()).first;
        batch_slot[c] = it->second;
        if (it->second < batch_distinct.size()) continue;
        batch_distinct.push_back(q.batch[c]);
        const auto& layers = q.batch[c]->layers;
        order_sum += layers.empty() ? 0u : (uint64_t)layers.rbegin()->first + 1u;
    }
    if (order_sum > (1ull << 21)) {
        set_error("the batch's compositions need %llu layer orders; the layer field holds %u",
                  (unsigned long long)order_sum, 1u << 21);
        return FORMA_STATUS_ORDER;
    }
    return FORMA_STATUS_OK;
}

// The masks target's own checks (see forma_renderer_render_masks), then those of any target for
// its size, the frame count and its planes: masks go alone or with an sRGB8 RGBA target that is
// neither painted over its pixels nor cached, never with an ID target.
int Renderer::check_masks(const FrameRequest& q) {
    const MaskTarget& m = q.masks;
    const uint64_t width = q.width, height = q.height, bpp = m.bpp(), frames = q.kind == FrameKind::single ? 1u : q.n;
    if (q.ids.ptr || (q.rgba.ptr && (q.rgba.bpp != 4u || q.rgba.over || q.cache))) {
        set_error("masks go alone or with an sRGB8 RGBA frame without a layer cache");
        return FORMA_STATUS_INVALID;
    }
    if (m.n_orders == 0u || (uint64_t)m.first_order + m.n_orders > (1ull << 21) || m.format > FORMA_MASK_U8) {
        set_error("invalid masks: orders [%u, %u + %u) (1 to 2^21 orders below 2^21), format %u", m.first_order, m.first_order,
                  m.n_orders, m.format);
        return FORMA_STATUS_INVALID;
    }
    if (width == 0 || height == 0 || width > FORMA_MAX_WIDTH || height > FORMA_MAX_HEIGHT || m.stride < bpp * width ||
        m.plane_stride < (height - 1u) * m.stride + bpp * width ||
        (bpp == 4u && (((uintptr_t)m.ptr | m.stride | m.plane_stride) & 3u) != 0u)) {
        set_error("invalid masks %llux%llu: stride %llu, plane stride %llu (f32: multiples of 4 bytes)", (unsigned long long)width,
                  (unsigned long long)height, (unsigned long long)m.stride, (unsigned long long)m.plane_stride);
        return FORMA_STATUS_INVALID;
    }
    // The whole stack of planes: (frames * K - 1) * plane_stride + one plane, within 64 bits.
    uint64_t planes = 0, span = 0, end = 0;
    if (__builtin_mul_overflow(frames, (uint64_t)m.n_orders, &planes) || __builtin_mul_overflow(planes - 1u, m.plane_stride, &span) ||
        __builtin_add_overflow(span, (height - 1u) * m.stride + bpp * width, &end)) {
        set_error("the masks' planes overflow 64 bits: %llu planes of stride %llu", (unsigned long long)planes,
                  (unsigned long long)m.plane_stride);
        return FORMA_STATUS_INVALID;
    }
    if (q.kind != FrameKind::single && (q.n == 0 || q.n > max_views(height))) {
        set_error("%u %ss of height %llu: between 1 and %u fit in one call", q.n, q.kind == FrameKind::views ? "view" : "frame",
                  (unsigned long long)height, max_views(height));
        return FORMA_STATUS_INVALID;
    }
    return FORMA_STATUS_OK;
}

// The statistics target's own checks (see forma_renderer_render_stats), then those of any target
// for its size and the frame count: statistics go alone or with an sRGB8 RGBA target that is
// neither painted over its pixels nor cached, never with IDs or masks.
int Renderer::check_stats(const FrameRequest& q) {
    const StatsTarget& t = q.stats;
    const uint64_t width = q.width, height = q.height, frames = q.kind == FrameKind::single ? 1u : q.n;
    if (q.ids.ptr || q.masks.ptr || (q.rgba.ptr && (q.rgba.bpp != 4u || q.rgba.over || q.cache))) {
        set_error("statistics go alone or with an sRGB8 RGBA frame without a layer cache");
        return FORMA_STATUS_INVALID;
    }
    if (((uintptr_t)t.ptr & 7u) != 0u || t.n_orders == 0u || (uint64_t)t.first_order + t.n_orders > (1ull << 21) ||
        !std::isfinite(t.min_coverage) || t.min_coverage < 0.0f || t.min_coverage >= 1.0f) {
        set_error("invalid statistics: records 8-byte aligned, orders [%u, %u + %u) (1 to 2^21 orders below 2^21), "
                  "min_coverage %g (finite, in [0, 1))", t.first_order, t.first_order, t.n_orders, (double)t.min_coverage);
        return FORMA_STATUS_INVALID;
    }
    if (width == 0 || height == 0 || width > FORMA_MAX_WIDTH || height > FORMA_MAX_HEIGHT) {
        set_error("invalid statistics frame %llux%llu", (unsigned long long)width, (unsigned long long)height);
        return FORMA_STATUS_INVALID;
    }
    uint64_t n_rec = 0, bytes = 0;
    if (__builtin_mul_overflow(frames, (uint64_t)t.n_orders, &n_rec) ||
        __builtin_mul_overflow(n_rec, (uint64_t)sizeof(forma_layer_stats), &bytes)) {
        set_error("the statistics' records overflow 64 bits: %llu frames of %u records", (unsigned long long)frames, t.n_orders);
        return FORMA_STATUS_INVALID;
    }
    if (q.kind != FrameKind::single && (q.n == 0 || q.n > max_views(height))) {
        set_error("%u %ss of height %llu: between 1 and %u fit in one call", q.n, q.kind == FrameKind::views ? "view" : "frame",
                  (unsigned long long)height, max_views(height));
        return FORMA_STATUS_INVALID;
    }
    return FORMA_STATUS_OK;
}

// Every distinct composition of the batch (batch_distinct, as check_request found them) is uploaded
// (tables, then all of its geometry), in the order of first appearance, and gets its slices:
// orders from order_base, style slots, stops and texels from their bases, each the sum of the
// counts of the compositions before it. The batch tables are gathered from the compositions'
// device tables when their list of (serial, version) changed; the per-frame line-setup records
// are uploaded every call (the segment buffers move as they grow).
int Renderer::bind_batch(Composition* const* comps, uint32_t n, PaintScene& S, uint32_t height, BatchLines& lines) {
    const uint32_t nd = (uint32_t)batch_distinct.size();
    FORMA_CUDA_TRY(h_batch_src.reserve(nd));
    batch_key_next.clear();
    uint64_t orders = 0, styles = 0, stops = 0, texels = 0, max_items = 0;
    bool in_order = options().sort_full_key == 0;
    for (uint32_t k = 0; k < nd; ++k) {
        Composition& comp = *batch_distinct[k];
        int st = upload_tables(comp, -1);
        if (st) return st;
        st = flush_geometry(comp, 0.0f, (float)height, false);
        if (st) return st;
        const CompDevice& cd = comp.on(res_key);
        const uint64_t n_texels = comp.n_texels / 4u;
        h_batch_src.ptr[k] = BatchTableSrc{cd.d_order_to_style.ptr, cd.d_styles.ptr, cd.d_grads.ptr, cd.d_stops.ptr, cd.d_texels.ptr,
                                           comp.n_orders, (uint32_t)comp.n_style_recs, (uint32_t)comp.n_stops, (uint32_t)n_texels,
                                           (uint32_t)orders, (uint32_t)styles, (uint32_t)stops, (uint32_t)texels};
        max_items = std::max<uint64_t>({max_items, comp.n_orders, comp.n_style_recs, comp.n_stops, n_texels});
        orders += comp.n_orders;
        styles += comp.n_style_recs;
        stops += comp.n_stops;
        texels += n_texels;
        in_order = in_order && comp.layers_in_order;
        batch_key_next.emplace_back(comp.serial, comp.tables_version);
    }
    if (stops > 0xFFFFFFFFu || texels > 0xFFFFFFFFu || styles > 0x7FFFFFFFu) {
        set_error("the batch's %llu gradient stops / %llu texels / %llu styles exceed the 32-bit indices of its tables",
                  (unsigned long long)stops, (unsigned long long)texels, (unsigned long long)styles);
        return FORMA_STATUS_CAPACITY;
    }
    if (batch_key_next != batch_key) {
        batch_key.clear();  // (until the gather below is queued)
        FORMA_CUDA_TRY(batch_order_to_style.reserve(orders + 1));
        FORMA_CUDA_TRY(batch_styles.reserve(styles + 1));
        FORMA_CUDA_TRY(batch_grads.reserve(styles + 1));
        FORMA_CUDA_TRY(batch_stops.reserve(stops + 1));
        FORMA_CUDA_TRY(batch_texels.reserve(4u * texels + 4u));
        FORMA_CUDA_TRY(d_batch_src.reserve(nd));
        FORMA_CUDA_TRY(cudaMemcpyAsync(d_batch_src.ptr, h_batch_src.ptr, nd * sizeof(BatchTableSrc), cudaMemcpyHostToDevice, stream));
        h2d_bytes += nd * sizeof(BatchTableSrc);
        launch_batch_tables(d_batch_src.ptr, nd, (uint32_t)max_items, batch_order_to_style.ptr, batch_styles.ptr, batch_grads.ptr,
                            batch_stops.ptr, batch_texels.ptr, stream);
        launches += max_items ? 1 : 0;
        FORMA_CUDA_TRY(cudaGetLastError());
        batch_key.swap(batch_key_next);
    }
    S.styles = batch_styles.ptr;
    S.order_to_style = batch_order_to_style.ptr;
    S.n_orders = (uint32_t)orders;
    S.stops = batch_stops.ptr;
    S.grads = batch_grads.ptr;
    S.texels = batch_texels.ptr;

    // Line setup: one record per frame, then the frames' first CTAs.
    const size_t frames_bytes = (size_t)n * sizeof(BatchFrame), bytes = frames_bytes + (n + 1u) * sizeof(uint32_t);
    FORMA_CUDA_TRY(h_batch_lines.reserve(bytes));
    FORMA_CUDA_TRY(d_batch_lines.reserve(bytes));
    BatchFrame* frames = reinterpret_cast<BatchFrame*>(h_batch_lines.ptr);
    uint32_t* cta_first = reinterpret_cast<uint32_t*>(h_batch_lines.ptr + frames_bytes);
    uint64_t ctas = 0, n_lines = 0;
    for (uint32_t c = 0; c < n; ++c) {
        const Composition& comp = *comps[c];
        const CompDevice& cd = *comp.devices.at(res_key);
        frames[c] = BatchFrame{cd.d_x.ptr, cd.d_y.ptr, cd.d_gid.ptr, cd.d_geom_slot.ptr, comp.layers_have_xf ? cd.d_layers.ptr : nullptr,
                               cd.d_layer_bits.ptr, cd.n_resident, comp.n_geoms, h_batch_src.ptr[batch_slot[c]].order_base, 0u};
        cta_first[c] = (uint32_t)std::min<uint64_t>(ctas, 0xFFFFFFFFu);
        ctas += raster_num_blocks(cd.n_resident);
        n_lines += cd.n_resident ? cd.n_resident - 1u : 0u;
    }
    if (ctas >= (1ull << 31)) {  // the launch's largest grid
        set_error("the batch's %llu line-setup CTAs exceed the largest grid", (unsigned long long)ctas);
        return FORMA_STATUS_CAPACITY;
    }
    cta_first[n] = (uint32_t)ctas;
    FORMA_CUDA_TRY(cudaMemcpyAsync(d_batch_lines.ptr, h_batch_lines.ptr, bytes, cudaMemcpyHostToDevice, stream));
    h2d_bytes += bytes;
    lines.args = BatchArgs{reinterpret_cast<const BatchFrame*>(d_batch_lines.ptr),
                           reinterpret_cast<const uint32_t*>(d_batch_lines.ptr + frames_bytes), n, (height + 15u) / 16u,
                           (float)S.width, (float)height};
    lines.n_ctas = (uint32_t)ctas;
    // Layer digits can be skipped when every composition emits its segments in layer order: a
    // painted tile holds one frame's segments, in emission order (stacked row 0 mixes frames, and
    // no painted tile reads it).
    lines.layer_bound = in_order ? 0u : (orders ? orders - 1u : 0u);
    lines.n_lines = n_lines;
    return FORMA_STATUS_OK;
}

// The frame's kernels: paint() for the RGBA target (in copy bands, or with the rows of a stack's
// frames), then the ID kernel for the ID target, or the mask or statistics kernels. The sync-free
// redo repeats them all.
int Renderer::paint_step(const FrameRequest& q, const PaintScene& S, const FramePlan& p, const TileTables& t,
                         uint32_t* paint_launches) {
    if (q.rgba.ptr) {
        bool solid_over = true;
        if (q.kind == FrameKind::batch)
            for (const Composition* c : batch_distinct) solid_over = solid_over && c->solid_over_only;
        else
            solid_over = solid_over && q.comp->solid_over_only;
        if (q.rgba.over && p.rows && !p.rgba.direct) {
            // A stack painted in scratch starts from its background (the redo of a sync-free frame
            // copies it again: the first attempt wrote nothing, and its repack gave the buffer back as it was).
            launch_unpack_views(q.rgba.ptr, q.rgba.stride, q.rgba.frame_stride, p.rgba.ptr, p.rgba.stride, p.rows * 16u,
                                S.width * (q.rgba.bpp / 4u), (uint32_t)q.height, q.n, stream);
            ++launches;
            FORMA_CUDA_TRY(cudaGetLastError());
        }
        const int st = paint(S, t, p.rgba.ptr, q.rgba.ptr, q.rgba.stride, p.in_bands, paint_launches, p.rows, q.rgba.bpp, solid_over,
                             q.rgba.over);
        if (st || (!q.ids.ptr && !q.masks.ptr && !q.stats.ptr)) return st;
        if (q.ids.ptr) ++*paint_launches;
    }
    FORMA_CUDA_TRY(id_flags.reserve(std::max<size_t>(recs.capacity, 1)));
    const BatchFrame* frames = q.kind == FrameKind::batch ? reinterpret_cast<const BatchFrame*>(d_batch_lines.ptr) : nullptr;
    if (q.masks.ptr) {  // the zero fill of the planes, then the masks (the redo of a sync-free frame repeats both)
        const MaskFrame m{p.masks.ptr, p.masks.stride, p.mask_plane_stride, q.masks.first_order, q.masks.n_orders, q.masks.format,
                          (uint32_t)q.height, q.kind == FrameKind::single ? 1u : q.n};
        const uint32_t n = launch_paint_masks(S, t, id_flags.ptr, m, totals.ptr + 8, stream, p.rows, frames);
        launches += n;
        *paint_launches = q.rgba.ptr ? *paint_launches + n : n;
        FORMA_CUDA_TRY(cudaGetLastError());
        return FORMA_STATUS_OK;
    }
    if (q.stats.ptr) {  // the records' initialisation, both walks, the empty boxes (the redo of a sync-free frame repeats all)
        const StatsFrame f{p.stats, q.stats.first_order, q.stats.n_orders, q.stats.min_coverage, (uint32_t)q.height,
                           q.kind == FrameKind::single ? 1u : q.n};
        const uint32_t n = launch_paint_stats(S, t, id_flags.ptr, f, totals.ptr + 8, stream, p.rows, frames);
        launches += n;
        *paint_launches = q.rgba.ptr ? *paint_launches + n : n;
        FORMA_CUDA_TRY(cudaGetLastError());
        return FORMA_STATUS_OK;
    }
    // A batch's entries carry each frame's order base (bind_batch): the kernel takes it off.
    launch_paint_ids(S, t, id_flags.ptr, reinterpret_cast<uint32_t*>(p.ids.ptr), p.ids.stride, q.ids.min_coverage, totals.ptr + 8, stream,
                     p.rows, frames);
    ++launches;
    FORMA_CUDA_TRY(cudaGetLastError());
    return FORMA_STATUS_OK;
}

// Moves every target's frames from the device frame to the caller's buffer: only the written
// tiles of a cached host frame, the crop's tile rectangle of a single host frame, and for a stack
// repack_views_kernel into another device layout or one copy per frame to a host buffer. Nothing
// for a frame painted in place or copied back band by band.
int Renderer::output_step(const FrameRequest& q, const PaintScene& S, const FramePlan& p) {
    if (p.pack_written) return scatter_written_tiles(S, p.rgba.ptr, q.rgba.ptr, q.rgba.stride);
    auto output = [&](const FrameTarget& t, const DeviceFrame& f) {
        if (!t.ptr || f.direct) return (int)FORMA_STATUS_OK;
        if (!p.rows) return copy_to_host(S, t.ptr, f.ptr, t.stride, stream, t.bpp);
        const uint32_t height = (uint32_t)q.height;
        if (t.on_device) {  // (a frame of 8- or 16-byte pixels is a frame of 4-byte words bpp / 4 times as wide)
            launch_repack_views(f.ptr, f.stride, p.rows * 16u, t.ptr, t.stride, t.frame_stride, S.width * (t.bpp / 4u), height, q.n,
                                stream);
            ++launches;
            FORMA_CUDA_TRY(cudaGetLastError());
            return (int)FORMA_STATUS_OK;
        }
        // Rows [0, height) of every frame, one copy per frame with the pitches copy_to_host uses
        // for a single frame (a copy over all frames would have a frame as its pitch, which can
        // exceed the device's largest pitch).
        for (uint32_t b = 0; b < q.n; ++b) {
            uint8_t* dst = t.ptr + (size_t)b * t.frame_stride;
            const uint8_t* src = f.ptr + (size_t)b * p.rows * 16u * f.stride;
            if (t.stride == f.stride)
                FORMA_CUDA_TRY(cudaMemcpyAsync(dst, src, (height - 1u) * t.stride + t.bpp * q.width, cudaMemcpyDeviceToHost, stream));
            else
                FORMA_CUDA_TRY(cudaMemcpy2DAsync(dst, t.stride, src, f.stride, t.bpp * q.width, height, cudaMemcpyDeviceToHost, stream));
        }
        d2h_bytes += (uint64_t)q.n * height * q.width * t.bpp;
        return (int)FORMA_STATUS_OK;
    };
    int st = p.in_bands ? FORMA_STATUS_OK : output(q.rgba, p.rgba);
    st = st ? st : output(q.ids, p.ids);
    if (st) return st;
    if (q.stats.ptr && !q.stats.on_device) {  // host statistics (single frames): the records
        const size_t bytes = (size_t)q.stats.n_orders * sizeof(forma_layer_stats);
        FORMA_CUDA_TRY(cudaMemcpyAsync(q.stats.ptr, p.stats, bytes, cudaMemcpyDeviceToHost, stream));
        d2h_bytes += bytes;
    }
    if (!q.masks.ptr || q.masks.on_device) return FORMA_STATUS_OK;
    // Host masks (single frames): the crop's tile rectangle of every plane.
    const MaskTarget& m = q.masks;
    const uint64_t bpp = m.bpp();
    const uint64_t x0 = (uint64_t)S.tx_lo * 16u, x1 = std::min<uint64_t>((uint64_t)S.tx_hi * 16u, S.width);
    const uint64_t y0 = (uint64_t)S.ty_lo * 16u, y1 = std::min<uint64_t>((uint64_t)S.ty_hi * 16u, S.height);
    if (x1 <= x0 || y1 <= y0) return FORMA_STATUS_OK;
    for (uint32_t k = 0; k < m.n_orders; ++k)
        FORMA_CUDA_TRY(cudaMemcpy2DAsync(m.ptr + k * m.plane_stride + y0 * m.stride + x0 * bpp, m.stride,
                                         p.masks.ptr + k * p.mask_plane_stride + y0 * p.masks.stride + x0 * bpp, p.masks.stride,
                                         (x1 - x0) * bpp, y1 - y0, cudaMemcpyDeviceToHost, stream));
    d2h_bytes += (uint64_t)m.n_orders * (x1 - x0) * bpp * (y1 - y0);
    return FORMA_STATUS_OK;
}

// The frame's PaintScene without its composition tables, for a target that check_request
// accepted: size, channels, clear colour and the tile rectangle of the crop.
int Renderer::begin_frame(PaintScene& S, uint64_t width, uint64_t stride, uint64_t height, const uint32_t channels_in[4],
                          const float clear[4], const forma_rect* crop) {
    FORMA_CUDA_TRY(cudaSetDevice(device));
    last_slices = 0;
    const int ts = ensure_timer();
    if (ts) return ts;
    for (int k = 0; k < 4; ++k) {
        uint32_t c = channels_in[k];
        if (c > 5u) {
            set_error("invalid channel %u", c);
            return FORMA_STATUS_INVALID;
        }
        if (clear[3] == 1.0f && c == FORMA_CHANNEL_ALPHA) c = FORMA_CHANNEL_ONE;  // renderer.rs:87-92
        S.channels[k] = c;
        S.clear[k] = clear[k];
    }
    S.width = (uint32_t)width;
    S.height = (uint32_t)height;
    S.stride = (uint32_t)stride;
    S.tiles_x = (S.width + 15u) / 16u;
    S.tiles_y = (S.height + 15u) / 16u;
    const TileRect tiles = tile_rect(width, height, crop);
    S.tx_lo = tiles.tx_lo; S.tx_hi = tiles.tx_hi; S.ty_lo = tiles.ty_lo; S.ty_hi = tiles.ty_hi;
    return FORMA_STATUS_OK;
}

// Points the scene at the composition's device tables and prepares the layer cache.
int Renderer::bind_frame(Composition& comp, PaintScene& S, LayerCache* cache, const float clear[4], bool pack_written) {
    CompDevice& cd = comp.on(res_key);
    S.styles = cd.d_styles.ptr;
    S.order_to_style = cd.d_order_to_style.ptr;
    S.n_orders = comp.n_orders;
    S.stops = cd.d_stops.ptr;
    S.grads = cd.d_grads.ptr;
    S.texels = cd.d_texels.ptr;

    if (cache) {  // renderer.rs:94-110
        const size_t cache_tiles = (size_t)S.tiles_x * S.tiles_y;
        if (!cache->has_size || cache->width != S.width || cache->height != S.height) {
            cache->has_size = true;
            cache->width = S.width;
            cache->height = S.height;
            cache->clear();
        }
        FORMA_CUDA_TRY(cache->tiles.reserve(cache_tiles));
        if (cache->needs_reset) {
            FORMA_CUDA_TRY(cudaMemsetAsync(cache->tiles.ptr, 0, cache_tiles * sizeof(uint2), stream));
            cache->needs_reset = false;
        }
        S.cache_tiles = cache->tiles.ptr;
        S.clear_unchanged = cache->has_clear && cache->clear_color[0] == clear[0] && cache->clear_color[1] == clear[1] &&
                            cache->clear_color[2] == clear[2] && cache->clear_color[3] == clear[3];
        // Layer::is_unchanged(cache_id) per style slot (renderer.rs:144-157); the slots
        // follow the iteration order of upload_tables.
        FORMA_CUDA_TRY(h_unchanged.reserve(comp.n_orders + 1));
        FORMA_CUDA_TRY(d_unchanged.reserve(comp.n_orders + 1));
        size_t slot = comp.n_orders;  // one byte per layer order
        std::memset(h_unchanged.ptr, 0, slot);
        for (auto& kv : comp.layers)
            if (kv.first < comp.n_orders) h_unchanged.ptr[kv.first] = (uint8_t)((kv.second->unchanged_bits >> cache->id) & 1u);
        if (slot) {
            FORMA_CUDA_TRY(cudaMemcpyAsync(d_unchanged.ptr, h_unchanged.ptr, slot, cudaMemcpyHostToDevice, stream));
            h2d_bytes += slot;
        }
        S.unchanged = d_unchanged.ptr;
        if (pack_written) {
            FORMA_CUDA_TRY(written_list.reserve(cache_tiles));
            FORMA_CUDA_TRY(cudaMemsetAsync(totals.ptr + 6, 0, sizeof(uint32_t), stream));
            S.written_list = written_list.ptr;
            S.written_count = totals.ptr + 6;
        }
    }
    return FORMA_STATUS_OK;
}

SortResult Renderer::sort(DeviceBuffer<uint64_t>& keys, DeviceBuffer<uint64_t>& keys_tmp, DeviceBuffer<uint32_t>* vals,
                          DeviceBuffer<uint32_t>* vals_tmp, uint32_t n, const SortPlan& plan, cudaEvent_t* pass_events,
                          const uint32_t* n_dev, const uint32_t* hist, void* scratch, const TileCounts* counts,
                          uint32_t* keep_counts) {
    SortResult sr = launch_radix_sort(keys.ptr, keys_tmp.ptr, vals ? vals->ptr : nullptr, vals ? vals_tmp->ptr : nullptr, n, plan,
                                      scratch ? scratch : sort_scratch.ptr, stream, pass_events, n_dev, hist, counts, keep_counts);
    launches += sr.launches;
    if (sr.in_tmp) {
        swap_buffers(keys, keys_tmp);
        if (vals) swap_buffers(*vals, *vals_tmp);
    }
    return sr;
}

// The painter tables of the n sorted segments: cells (+ the carry sort's digit counts) -> carry
// pair sort -> carry pass: carries, carry-only entries ("gaps") (+ the gap sort's digit counts)
// -> gap pair sort -> entries, tile ranges and heavy-tile lists. The modes differ only in how
// they get the cell and gap counts:
// - sync_free: a count is a bound (the previous frame's + 25 % + 4096), everything is reserved
//   for the bounds up front, and the kernels read the real counts from device memory (dc). Two
//   memsets (tile ranges, table scratch) and the kernels, nothing else.
// - counted: a count is read back; the kernel that produces it runs ahead of the read-back into
//   the buffers of the previous frames and is launched again when they turn out too small.
// batch: the frames of a batch (the merge bounds each entry's clip range by its frame's orders).
int Renderer::build_tables(const PaintScene& S, uint32_t n, bool sync_free, uint32_t prev_cells, uint32_t prev_gaps,
                           uint32_t* heavy_lists, DevCounts& dc, const BatchArgs* batch) {
    // Tiles without entries keep an empty range: a frame whose tables are redone paints only the
    // clear colour in its first attempt. A count above its bound leaves every range empty (the
    // merge kernel then writes none), so that attempt of an over frame writes nothing at all.
    FORMA_CUDA_TRY(cudaMemsetAsync(tile_range.ptr, 0, (size_t)S.tiles_x * S.tiles_y * sizeof(uint2), stream));
    const SortPlan carry_plan = carry_sort_plan(S), gap_plan = gap_sort_plan(S);
    auto zero_scratch = [&](size_t from, size_t to) -> cudaError_t {
        return to > from ? cudaMemsetAsync(table_scratch.ptr + from, 0, to - from, stream) : cudaSuccess;
    };
    if (n == 0) {  // nothing to index; the painter still reads the heavy-list lengths
        const TableScratch L = table_scratch_layout(0, 0, 0, carry_plan, gap_plan);
        FORMA_CUDA_TRY(table_scratch.reserve(L.carry_hist));
        FORMA_CUDA_TRY(zero_scratch(0, L.carry_hist));
        return FORMA_STATUS_OK;
    }
    uint32_t n_cells = 0, n_gaps = 0;  // sync_free: their bounds
    TableScratch L{};
    auto cells_pass = [&](uint32_t cap) {
        launch_cells(S, segs.ptr, n, table_scratch.ptr, L, carry_plan, cell_start.ptr, cap, totals.ptr + 1, cell_key.ptr,
                     cell_cover.ptr, key2.ptr, perm.ptr, stream);
        launches += cell_num_blocks(n) > 1 ? 2 : 1;
    };
    auto carry_pass = [&](uint32_t cap) {
        launch_carry_pass(S, key2.ptr, perm.ptr, cell_cover.ptr, n_cells, table_scratch.ptr, L, gap_plan, carry_in.ptr,
                          ekey_tmp.ptr, eid_tmp.ptr, gap_carry.ptr, cap, totals.ptr + 2, stream, dc);
        ++launches;
    };
    if (sync_free) {
        const uint64_t shrink = options().test_fast_shrink ? 2u : 1u;
        n_cells = (uint32_t)std::min<uint64_t>(((uint64_t)prev_cells + prev_cells / 4u + 4096u) / shrink, n);
        n_gaps = (uint32_t)std::min<uint64_t>(((uint64_t)prev_gaps + prev_gaps / 4u + 4096u) / shrink, 0x7FFFFFFFu);
        FORMA_CUDA_TRY(reserve_cell_tables(n_cells));
        FORMA_CUDA_TRY(reserve_gap_tables(n_gaps));
        FORMA_CUDA_TRY(reserve_entry_tables((size_t)n_cells + n_gaps));
        L = table_scratch_layout(n, n_cells, n_gaps, carry_plan, gap_plan);
        FORMA_CUDA_TRY(table_scratch.reserve(L.end));
        FORMA_CUDA_TRY(zero_scratch(0, L.end));
        dc = DevCounts{totals.ptr + 1, totals.ptr + 2, n_cells, n_gaps};
        // Cells beyond cell_bound + 1 are dropped by the pass; the count it leaves in totals[1] is the real one.
        cells_pass(n_cells + 1u);
    } else {
        // Cells: one pass finds the cell heads, counts them and sums their covers. The count is
        // read back, but nothing waits for it: the pass runs into the buffers of the previous
        // frames (writes beyond their capacity are dropped) and is repeated below only if
        // those turn out too small.
        L = table_scratch_layout(n, 0, 0, carry_plan, gap_plan);
        FORMA_CUDA_TRY(table_scratch.reserve(L.carry_sort));
        FORMA_CUDA_TRY(zero_scratch(0, L.carry_sort));
        if (!cell_start.capacity)  // first frame: a guess that usually holds (cells ~ segments / 20)
            FORMA_CUDA_TRY(reserve_all((size_t)n / 8u + 4096u, cell_start, cell_key, cell_cover, key2, perm));
        auto cells_capacity = [&] {
            return (uint32_t)std::min({cell_start.capacity, cell_key.capacity, cell_cover.capacity, key2.capacity, perm.capacity,
                                       (size_t)0xFFFFFFFFu});
        };
        const uint32_t cell_cap = cells_capacity();
        cells_pass(cell_cap);
        FORMA_CUDA_TRY(cudaMemcpyAsync(pinned_totals + 1, totals.ptr + 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
        FORMA_CUDA_TRY(cudaEventRecord(count_ev, stream));
        FORMA_CUDA_TRY(cudaEventSynchronize(count_ev));
        n_cells = pinned_totals[1];
        FORMA_CUDA_TRY(reserve_cell_tables(n_cells));
        L = table_scratch_layout(n, n_cells, 0, carry_plan, gap_plan);
        const uint8_t* held = table_scratch.ptr;
        FORMA_CUDA_TRY(table_scratch.reserve(L.gap_sort));
        // The buffers were too small (the pass dropped the overflow), or the scratch moved (the
        // digit counts went with it): once more.
        if ((size_t)n_cells + 1 > cell_cap || table_scratch.ptr != held) {
            FORMA_CUDA_TRY(zero_scratch(0, L.carry_sort));
            cells_pass(cells_capacity());
        }
        FORMA_CUDA_TRY(zero_scratch(L.carry_sort, L.gap_sort));
    }
    sort(key2, key2_tmp, &perm, &perm_tmp, n_cells, carry_plan, nullptr, dc.cells,
         reinterpret_cast<const uint32_t*>(table_scratch.ptr + L.carry_hist), table_scratch.ptr + L.carry_sort);
    if (sync_free) {
        carry_pass(n_gaps);
    } else {
        // Same scheme for the number of carry-only entries: the carry pass counts them and writes
        // them ahead of the read-back, into the buffers of the previous frames (at most gap_cap;
        // 0: the carries and the count only, the entries follow the read-back). The speculative
        // output survives only if the reserve(n_gaps + 1) calls below do not reallocate: one
        // element of every buffer is kept back (the sort's slack slot).
        size_t gap_cap = 0;
        if (speculation_enabled()) {
            const size_t room = std::min({ekey_tmp.capacity, eid_tmp.capacity, gap_carry.capacity});
            gap_cap = std::min<size_t>(room ? room - 1u : 0u, (size_t)last_gaps * 2u + 4096u);
            if (test_gap_cap_override() && gap_cap) gap_cap = std::min<size_t>(gap_cap, test_gap_cap_override());
        }
        carry_pass((uint32_t)gap_cap);
        FORMA_CUDA_TRY(cudaMemcpyAsync(pinned_totals + 2, totals.ptr + 2, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
        FORMA_CUDA_TRY(cudaEventRecord(count_ev, stream));
        FORMA_CUDA_TRY(cudaEventSynchronize(count_ev));
        n_gaps = pinned_totals[2];
        last_gaps = n_gaps;
        last_cells = n_cells;
        last_entries = n_cells + n_gaps;
        FORMA_CUDA_TRY(reserve_gap_tables(n_gaps));
        FORMA_CUDA_TRY(reserve_entry_tables((size_t)n_cells + n_gaps));
        L = table_scratch_layout(n, n_cells, n_gaps, carry_plan, gap_plan);
        const uint8_t* held = table_scratch.ptr;
        FORMA_CUDA_TRY(table_scratch.reserve(L.end));
        const bool moved = table_scratch.ptr != held;
        const bool again = n_gaps && (n_gaps > gap_cap || moved);  // entries dropped, or their digit counts lost
        if (again || moved) {
            FORMA_CUDA_TRY(zero_scratch(0, L.end));
        } else {
            FORMA_CUDA_TRY(zero_scratch(L.gap_sort, L.end));
        }
        if (again) carry_pass(n_gaps);
    }
    if (n_gaps)
        sort(ekey_tmp, gkey_tmp, &eid_tmp, &gid_tmp, n_gaps, gap_plan, nullptr, dc.gaps,
             reinterpret_cast<const uint32_t*>(table_scratch.ptr + L.gap_hist), table_scratch.ptr + L.gap_sort);
    launch_merge_entries(S, cell_key.ptr, n_cells, ekey_tmp.ptr, eid_tmp.ptr, n_gaps, cell_start.ptr, carry_in.ptr, gap_carry.ptr,
                         ekey.ptr, recs.ptr, eflags.ptr, tile_range.ptr, heavy_lists, heavy_count(), stream, dc,
                         batch ? batch->frames : nullptr, batch ? batch->rows : 0u);
    ++launches;
    // sync_free: the counts travel to the host behind everything else of the frame.
    if (sync_free)
        FORMA_CUDA_TRY(cudaMemcpyAsync(pinned_totals + 1, totals.ptr + 1, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
    return FORMA_STATUS_OK;
}

// Renderers of a multi-device / sliced frame queue the per-row costs of the frame and their copy
// to the host.
int Renderer::queue_row_costs(const PaintScene& S, uint32_t n) {
    row_costs_rows = 0;
    if (track_row_costs && n > 0) {
        FORMA_CUDA_TRY(d_row_costs.reserve(3u * S.tiles_y));  // per row: cost, pixel segments, entries
        FORMA_CUDA_TRY(h_row_costs.reserve(3u * S.tiles_y));
        launch_row_costs(tile_range.ptr, S.tiles_x, S.tiles_y, segs.ptr, n, d_row_costs.ptr, stream, d_row_costs.ptr + S.tiles_y);
        ++launches;
        FORMA_CUDA_TRY(cudaMemcpyAsync(h_row_costs.ptr, d_row_costs.ptr, 3u * S.tiles_y * sizeof(unsigned long long),
                                       cudaMemcpyDeviceToHost, stream));
        row_costs_rows = S.tiles_y;
    }
    return FORMA_STATUS_OK;
}

// Paints S into fb. in_bands (a host frame without a layer cache): paint in bands of tile rows,
// every band on its own stream followed by the copy of its rows to the host buffer. The band
// kernels are persistent (one CTA per resident slot), so the CTAs of band k + 1 start as the warps
// of band k run dry: the kernels overlap at their tails, and the PCIe transfer of a band overlaps
// the painting of the following ones.
// bpp: bytes per pixel of fb, 4 (sRGB8), or 8 / 16 for a linear float frame (never in bands).
// solid_over: see launch_paint (sRGB8 frames; a float frame is painted by the general build).
// over: paint over fb's own pixels (launch_paint_over), in any of the three formats.
int Renderer::paint(const PaintScene& S, const TileTables& t, uint8_t* fb, uint8_t* buffer, uint64_t stride, bool in_bands,
                    uint32_t* paint_launches, uint32_t view_rows, uint32_t bpp, bool solid_over, bool over) {
    *paint_launches = 1;
    if (over) {  // (never in bands: an over frame is on the device)
        launch_paint_over(S, t, eflags.ptr, fb, totals.ptr + 3, stream, view_rows, bpp);
        ++launches;
    } else if (in_bands) {
        if (!band_streams_ok) {
            for (auto& e : band_ev) FORMA_CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
            band_streams_ok = true;
        }
        const uint32_t paint_rows = S.ty_hi - S.ty_lo;
        const uint32_t kCopyBands = std::max(1u, std::min(copy_bands(), paint_rows / 8u));
        // One band: paint and copy on the render stream itself.
        while (kCopyBands > 1u && band_streams_made < kCopyBands) {
            FORMA_CUDA_TRY(cudaStreamCreateWithFlags(&band_stream[band_streams_made], cudaStreamNonBlocking));
            ++band_streams_made;
        }
        if (kCopyBands > 1u) FORMA_CUDA_TRY(cudaEventRecord(band_ev[kMaxCopyBands], stream));  // the tables are ready
        for (uint32_t k = 0; k < kCopyBands; ++k) {
            PaintScene Sb = S;
            Sb.ty_lo = S.ty_lo + paint_rows * k / kCopyBands;
            Sb.ty_hi = S.ty_lo + paint_rows * (k + 1u) / kCopyBands;
            cudaStream_t bs = kCopyBands > 1u ? band_stream[k] : stream;
            if (kCopyBands > 1u) FORMA_CUDA_TRY(cudaStreamWaitEvent(bs, band_ev[kMaxCopyBands], 0));
            launch_paint(Sb, t, eflags.ptr, fb, totals.ptr + 16 + k, bs, 0, solid_over);
            ++launches;
            const int st = copy_to_host(Sb, buffer, fb, stride, bs);
            if (st) return st;
            if (kCopyBands > 1u) FORMA_CUDA_TRY(cudaEventRecord(band_ev[k], bs));
        }
        for (uint32_t k = 0; kCopyBands > 1u && k < kCopyBands; ++k) FORMA_CUDA_TRY(cudaStreamWaitEvent(stream, band_ev[k], 0));
        *paint_launches = kCopyBands;
    } else if (bpp == 4u) {
        launch_paint(S, t, eflags.ptr, fb, totals.ptr + 3, stream, view_rows, solid_over);
        ++launches;
    } else {
        launch_paint_linear(S, t, eflags.ptr, fb, totals.ptr + 3, stream, view_rows, bpp);
        ++launches;
    }
    FORMA_CUDA_TRY(cudaGetLastError());
    return FORMA_STATUS_OK;
}

// Copies the painted tile rectangle of S from the frame on the device to the host buffer. Only the
// cropped tile rectangle is written by the reference (cpu/painter/mod.rs:524-529,589-593); padding
// bytes beyond width * bpp stay untouched.
int Renderer::copy_to_host(const PaintScene& S, uint8_t* buffer, const uint8_t* fb, uint64_t stride, cudaStream_t s, uint32_t bpp) {
    const uint64_t x0 = (uint64_t)S.tx_lo * 16u, x1 = std::min<uint64_t>((uint64_t)S.tx_hi * 16u, S.width);
    const uint64_t y0 = (uint64_t)S.ty_lo * 16u, y1 = std::min<uint64_t>((uint64_t)S.ty_hi * 16u, S.height);
    if (x1 > x0 && y1 > y0) {
        if (x0 == 0 && x1 * bpp == stride)  // whole rows without padding: one contiguous copy
            FORMA_CUDA_TRY(cudaMemcpyAsync(buffer + y0 * stride, fb + y0 * stride, (y1 - y0) * stride, cudaMemcpyDeviceToHost, s));
        else
            FORMA_CUDA_TRY(cudaMemcpy2DAsync(buffer + y0 * stride + x0 * bpp, stride, fb + y0 * stride + x0 * bpp, stride,
                                             (x1 - x0) * bpp, y1 - y0, cudaMemcpyDeviceToHost, s));
        d2h_bytes += (x1 - x0) * bpp * (y1 - y0);
    }
    return FORMA_STATUS_OK;
}

// With a layer cache only the tiles this frame wrote may touch the host
// buffer (TileWriteOp::None leaves its bytes alone): pack them on the
// device, copy count + ids + pixels, scatter on the host.
int Renderer::scatter_written_tiles(const PaintScene& S, const uint8_t* fb, uint8_t* buffer, uint64_t stride) {
    FORMA_CUDA_TRY(packed_tiles.reserve((size_t)S.tiles_x * S.tiles_y * 256u));
    launch_gather_tiles(S, fb, packed_tiles.ptr, stream);
    ++launches;
    FORMA_CUDA_TRY(cudaMemcpyAsync(pinned_totals + 6, totals.ptr + 6, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
    FORMA_CUDA_TRY(cudaStreamSynchronize(stream));
    const uint32_t n_written = pinned_totals[6];
    last_written_tiles = n_written;
    if (n_written) {
        FORMA_CUDA_TRY(h_written_list.reserve(n_written));
        FORMA_CUDA_TRY(h_packed_tiles.reserve((size_t)n_written * 256u));
        FORMA_CUDA_TRY(cudaMemcpyAsync(h_written_list.ptr, written_list.ptr, n_written * sizeof(uint32_t),
                                       cudaMemcpyDeviceToHost, stream));
        FORMA_CUDA_TRY(cudaMemcpyAsync(h_packed_tiles.ptr, packed_tiles.ptr, (size_t)n_written * 1024u,
                                       cudaMemcpyDeviceToHost, stream));
        FORMA_CUDA_TRY(cudaStreamSynchronize(stream));
        d2h_bytes += (uint64_t)n_written * (1024u + 4u);
        for (uint32_t i = 0; i < n_written; ++i) {  // LinearLayout::write, layout/mod.rs:265-282
            const uint32_t tile = h_written_list.ptr[i];
            const uint64_t x0 = (uint64_t)(tile % S.tiles_x) * 16u, y0 = (uint64_t)(tile / S.tiles_x) * 16u;
            const uint64_t cols = std::min<uint64_t>(16u, S.width - x0), rows = std::min<uint64_t>(16u, S.height - y0);
            const uint32_t* src = h_packed_tiles.ptr + (size_t)i * 256u;
            uint8_t* dst = buffer + y0 * stride + x0 * 4u;
            if (cols == 16u) {  // whole tile rows: fixed-size copies the compiler turns into vector moves
                for (uint64_t r = 0; r < rows; ++r) std::memcpy(dst + r * stride, src + r * 16u, 64);
            } else {
                for (uint64_t r = 0; r < rows; ++r) std::memcpy(dst + r * stride, src + r * 16u, cols * 4u);
            }
        }
    }
    return FORMA_STATUS_OK;
}

}  // namespace forma
