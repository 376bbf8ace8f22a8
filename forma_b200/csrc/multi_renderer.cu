// forma_b200 — several renderers behind one frame: the multi-GPU renderer (one tile-row band per
// device) and the sliced host-frame pipeline (tile-row slices on one device), with the worker
// pool that drives them and the balancing of their bands on the previous frame's row costs.
#include <condition_variable>
#include <cstring>
#include <functional>
#include <mutex>
#include <string>
#include <thread>

#include "renderer.hpp"

using namespace forma;

// ---------------------------------------------------------------------------
// Several GPUs behind one renderer (single process): tile-row bands, one worker thread and
// one forma_renderer per device. Every device makes the geometry of its band resident
// (flush_geometry's band filter), rasterizes, sorts and paints its band, and either copies
// the band's rows to the caller's host buffer or stores them into the frame in the first
// device's memory over NVLink (peer access). No collective: the bands are disjoint row
// ranges of one frame. The bands of the next frame are balanced on this frame's row costs.
// ---------------------------------------------------------------------------

// Persistent worker threads of a multi-device (or sliced) renderer: run(n, f) executes f(0) on
// the calling thread and f(1) ... f(n - 1) on workers that live as long as the pool, so a frame
// of a millisecond does not pay for thread creation.
class WorkerPool {
   public:
    ~WorkerPool() {
        {
            std::lock_guard<std::mutex> lk(mu);
            stop = true;
        }
        cv_work.notify_all();
        for (std::thread& t : threads) t.join();
    }
    void run(size_t n, const std::function<void(size_t)>& f) {
        if (n == 0) return;
        while (threads.size() + 1 < n) {
            const size_t index = threads.size() + 1;
            uint64_t seen;
            {
                std::lock_guard<std::mutex> lk(mu);
                seen = generation;
            }
            threads.emplace_back([this, index, seen] { worker(index, seen); });
        }
        if (n > 1) {
            std::lock_guard<std::mutex> lk(mu);
            job = &f;
            active = n;
            pending = threads.size();
            ++generation;
        }
        if (n > 1) cv_work.notify_all();
        f(0);
        if (n > 1) {
            std::unique_lock<std::mutex> lk(mu);
            cv_done.wait(lk, [&] { return pending == 0; });
            job = nullptr;
        }
    }

   private:
    void worker(size_t index, uint64_t seen) {
        for (;;) {
            std::unique_lock<std::mutex> lk(mu);
            cv_work.wait(lk, [&] { return stop || generation != seen; });
            if (stop) return;
            seen = generation;
            const std::function<void(size_t)>* f = job;
            const size_t n = active;
            lk.unlock();
            if (index < n && f) {
                try {
                    (*f)(index);
                } catch (...) {  // jobs report through their own status words
                }
            }
            lk.lock();
            if (--pending == 0) cv_done.notify_one();
        }
    }
    std::vector<std::thread> threads;
    std::mutex mu;
    std::condition_variable cv_work, cv_done;
    const std::function<void(size_t)>* job = nullptr;
    size_t active = 0, pending = 0;
    uint64_t generation = 0;
    bool stop = false;
};

struct forma_renderer_multi {
    std::vector<forma_renderer*> dev;
    std::vector<uint32_t> bounds;  // tile rows: band i = [bounds[i], bounds[i + 1])
    uint32_t bounds_lo = 0, bounds_hi = 0;
    bool peer_ok = true;           // every device may store into the first device's memory
    std::vector<double> last_ms;   // device-timeline ms of each band in the last frame
    size_t active = 0;             // bands used by the last frame (a sliced host frame may use fewer than dev.size())
    uint64_t last_own_segments = 0, last_own_entries = 0;  // pixel segments / entries of the last frame, every band counting its own rows only
    WorkerPool pool;
    ~forma_renderer_multi() {
        for (forma_renderer* r : dev) forma_renderer_free(r);
    }
};

static int multi_render_impl(forma_renderer_multi* m, forma_composition* c, uint8_t* buffer, bool on_device, uint64_t width,
                             uint64_t stride, uint64_t height, const uint32_t channels[4], const float clear[4],
                             const forma_rect* crop, forma_timings* timings, size_t n_use = 0, bool chained_uploads = false) {
    const size_t n = n_use ? std::min(n_use, m->dev.size()) : m->dev.size();
    m->active = n;
    if (!n || !width || !height || width > FORMA_MAX_WIDTH || height > FORMA_MAX_HEIGHT) {
        set_error("forma_renderer_multi_render: invalid arguments");
        return FORMA_STATUS_INVALID;
    }
    if (on_device && n > 1 && !m->peer_ok) {
        set_error("forma_renderer_multi_render_device: peer access to the first device is not available");
        return FORMA_STATUS_INVALID;
    }
    Composition& comp = c->c;
    // Tile rows to paint (crop is tile-granular like cpu/renderer.rs:43-52).
    const uint32_t tiles_y = (uint32_t)((height + 15u) / 16u);
    const TileRect tiles = tile_rect(width, height, crop);
    const uint32_t row_lo = tiles.ty_lo, row_hi = tiles.ty_hi;
    const forma_rect full = crop ? *crop : forma_rect{0, width, 0, height};
    if (m->bounds.size() != n + 1 || m->bounds_lo != row_lo || m->bounds_hi != row_hi) {  // first frame / new target: equal bands
        m->bounds.assign(n + 1, row_lo);
        for (size_t i = 0; i <= n; ++i) m->bounds[i] = row_lo + (uint32_t)(((uint64_t)(row_hi - row_lo) * i) / n);
        m->bounds_lo = row_lo;
        m->bounds_hi = row_hi;
    }
    // Host-side preparation, once: compaction, the pinned tables, the per-device records.
    comp.compact_geom();
    if (comp.tables_dirty || comp.tables_cache_id != -1) {
        for (forma_renderer* r : m->dev) {
            FORMA_CUDA_TRY(cudaSetDevice(r->r.device));
            FORMA_CUDA_TRY(cudaStreamSynchronize(r->r.stream));
        }
        int st = comp.rebuild_tables(-1);
        if (st) return st;
    }
    for (forma_renderer* r : m->dev) comp.on(r->r.res_key);  // the workers only look their records up

    std::vector<int> status(n, FORMA_STATUS_OK);
    std::vector<std::string> errors(n);
    std::vector<forma_timings> tms(n);
    std::vector<std::vector<uint64_t>> costs(n);
    std::vector<uint64_t> own_segments(n, 0), own_entries(n, 0);
    m->last_ms.assign(n, 0.0);
    auto band_of = [&](size_t i, forma_rect* band) {
        const uint32_t r0 = m->bounds[i], r1 = m->bounds[i + 1];
        if (r1 <= r0) return false;
        *band = full;
        band->vert_start = std::max<uint64_t>(full.vert_start, (uint64_t)r0 * 16u);
        band->vert_end = std::min<uint64_t>(std::min<uint64_t>(full.vert_end, height), (uint64_t)r1 * 16u);
        return band->vert_end > band->vert_start;
    };
    if (chained_uploads) {
        // Slices of one device share its PCIe link: their uploads are issued here, in slice order,
        // each waiting for the one before (Renderer::upload_after), instead of all at once.
        for (size_t i = 0; i < n; ++i) {
            forma_rect band;
            if (!band_of(i, &band)) continue;
            const int st = m->dev[i]->r.prefetch(comp, width, height, &band);
            if (st) {
                for (size_t k = 0; k < n; ++k) m->dev[k]->r.prefetched = false;
                return st;
            }
        }
    }
    auto work = [&](size_t i) {
        const uint32_t r0 = m->bounds[i], r1 = m->bounds[i + 1];
        std::memset(&tms[i], 0, sizeof(forma_timings));
        forma_rect band;
        if (!band_of(i, &band)) return;
        Renderer& R = m->dev[i]->r;
        status[i] = guarded((int)FORMA_ERR_CAPACITY, [&] {
            return R.render(comp, buffer, on_device, width, stride, height, channels, clear, &band, nullptr, &tms[i]);
        });
        if (status[i]) {
            errors[i] = forma_last_error();
            return;
        }
        m->last_ms[i] = R.stage_ms[7];
        costs[i].assign(tiles_y, 0);  // the frame's row costs came back behind the frame (track_row_costs)
        for (uint32_t r = 0; r < std::min(R.row_costs_rows, tiles_y); ++r) costs[i][r] = R.h_row_costs.ptr[r];
        // A line that crosses a band boundary is rasterized by both neighbours: the frame's
        // segment count is the sum of the segments every band has in its own rows.
        if (R.row_costs_rows == tiles_y) {
            uint64_t own = 0, own_e = 0;
            for (uint32_t r = r0; r < std::min(r1, tiles_y); ++r) {
                own += R.h_row_costs.ptr[tiles_y + r];
                own_e += R.h_row_costs.ptr[2u * tiles_y + r];
            }
            own_segments[i] = own;
            own_entries[i] = own_e;
        } else {
            own_segments[i] = R.last_segments;
            own_entries[i] = R.last_entries;
        }
    };
    m->pool.run(n, [&](size_t i) {
        try {
            work(i);
        } catch (const std::exception& e) {
            status[i] = FORMA_STATUS_CAPACITY;
            errors[i] = e.what();
        }
    });
    for (size_t i = 0; i < n; ++i)
        if (status[i]) {
            set_error("device %d: %s", m->dev[i]->r.device, errors[i].c_str());
            return status[i];
        }
    if (timings) {
        std::memset(timings, 0, sizeof(*timings));
        for (size_t i = 0; i < n; ++i) {  // stages: the slowest band; sizes: the whole frame
            timings->line_setup_ms = std::max(timings->line_setup_ms, tms[i].line_setup_ms);
            timings->rasterize_ms = std::max(timings->rasterize_ms, tms[i].rasterize_ms);
            timings->sort_ms = std::max(timings->sort_ms, tms[i].sort_ms);
            timings->paint_ms = std::max(timings->paint_ms, tms[i].paint_ms);
            timings->n_lines += tms[i].n_lines;
            timings->n_segments += own_segments[i];
        }
    }
    m->last_own_segments = m->last_own_entries = 0;
    for (size_t i = 0; i < n; ++i) {
        m->last_own_segments += own_segments[i];
        m->last_own_entries += own_entries[i];
    }
    // Next frame's bands: equal shares of this frame's row costs (+ a floor per row: every
    // tile is at least cleared and stored).
    if (n > 1 && row_hi > row_lo) {
        std::vector<double> cost(tiles_y, 0.0);
        const double floor_cost = 2.0 * (double)((width + 15u) / 16u);
        for (size_t i = 0; i < n; ++i)
            for (uint32_t r = m->bounds[i]; r < m->bounds[i + 1] && r < (uint32_t)costs[i].size(); ++r)
                cost[r] = (double)costs[i][r];
        double total = 0.0;
        for (uint32_t r = row_lo; r < row_hi; ++r) total += (cost[r] += floor_cost);
        // Bands that are still within 8 % of an equal share stay as they are: moving a boundary
        // makes the devices on both sides re-stage and re-upload their geometry.
        double worst = 0.0;
        for (size_t i = 0; i < n; ++i) {
            double band = 0.0;
            for (uint32_t r = m->bounds[i]; r < m->bounds[i + 1]; ++r) band += cost[r];
            worst = std::max(worst, band);
        }
        if (worst * (double)n <= 1.08 * total) return FORMA_STATUS_OK;
        std::vector<uint32_t> nb(1, row_lo);
        double run = 0.0;
        size_t k = 1;
        for (uint32_t r = row_lo; r < row_hi; ++r) {
            while (k < n && run + 0.5 * cost[r] >= total * (double)k / (double)n) {
                nb.push_back(r);
                ++k;
            }
            run += cost[r];
        }
        while (nb.size() < n) nb.push_back(row_hi);
        nb.push_back(row_hi);
        m->bounds = nb;
    }
    return FORMA_STATUS_OK;
}

// Host frames as a pipeline of tile-row slices. A host frame is upload (the geometry that is not
// resident) -> line setup / rasterize / sort / tables -> paint -> copy-back; on one stream the
// copy engines idle while the SMs work and the other way round, and PCIe carries one direction
// at a time. Here the frame is cut into `host_slices` bands of tile rows; every slice is a
// renderer of its own on this device (own stream, own scratch, own residency record with the
// band filter of the multi-GPU path, so it uploads and evaluates only the geometry that can
// reach its rows) driven by its own host thread: slice k + 1 uploads while slice k computes
// and slice k - 1 copies back, and the two PCIe directions run at the same time. The slices are
// balanced on the previous frame's row costs like the bands of a multi-GPU frame. Results are
// those of a band render (tests/test_gpu_bench_scale.py: bands == whole frame).
// Not sliced: frames with a layer cache (the cache records belong to one renderer), layers with
// transforms (no band filter: every slice would upload everything), small compositions, short frames.
int sliced_host_render(forma_renderer* r, forma_composition* c, uint8_t* buffer, uint64_t width, uint64_t stride,
                       uint64_t height, const uint32_t channels[4], const float clear[4], const forma_rect* crop,
                       forma_timings* timings) {
    Renderer& P = r->r;
    const int want = options().host_slices;
    if (want < 2 || !buffer || !width || !height || width > FORMA_MAX_WIDTH || height > FORMA_MAX_HEIGHT || width * 4 > stride)
        return -1;  // (invalid targets are reported by the plain path)
    for (int k = 0; k < 4; ++k)
        if (channels[k] > 5u) return -1;
    Composition& comp = c->c;
    if ((uint64_t)comp.n_points < (uint64_t)std::max(options().slice_min_points, 0)) return -1;
    if (crop && crop->hor_end <= crop->hor_start) return -1;
    const TileRect tiles = tile_rect(width, height, crop);
    const uint32_t row_lo = tiles.ty_lo, row_hi = tiles.ty_hi;
    if (row_hi <= row_lo) return -1;
    const size_t n = std::min<size_t>((size_t)want, (row_hi - row_lo) / 16u);  // at least 16 tile rows per slice
    if (n < 2) return -1;
    if (cudaSetDevice(P.device) != cudaSuccess) return -1;
    // The tables are rebuilt here (the slices find them clean) so that layers_have_xf is known.
    comp.compact_geom();
    if (comp.tables_dirty || comp.tables_cache_id != -1) {
        FORMA_CUDA_TRY(cudaStreamSynchronize(P.stream));
        if (r->slicer)
            for (forma_renderer* q : r->slicer->dev) FORMA_CUDA_TRY(cudaStreamSynchronize(q->r.stream));
        const int st = comp.rebuild_tables(-1);
        if (st) return st;
    }
    if (comp.layers_have_xf) return -1;
    if (!r->slicer || r->slicer->dev.size() < n) {
        if (r->slicer) forma_renderer_multi_free(r->slicer);
        r->slicer = nullptr;
        std::unique_ptr<forma_renderer_multi> m(new forma_renderer_multi());
        for (size_t i = 0; i < (size_t)want; ++i) {
            forma_renderer* q = forma_renderer_new(P.device);
            if (!q) return FORMA_STATUS_CUDA;
            cudaStream_t st = nullptr;
            if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) {
                forma_renderer_free(q);
                set_error("sliced host frame: cannot create a stream");
                return FORMA_STATUS_CUDA;
            }
            q->r.stream = st;
            q->r.owns_stream = true;
            q->r.res_key = P.device + 4096 * (int)(i + 1);
            q->r.track_row_costs = true;
            if (cudaEventCreateWithFlags(&q->r.upload_done_ev, cudaEventDisableTiming) != cudaSuccess) q->r.upload_done_ev = nullptr;
            if (i > 0) q->r.upload_after = m->dev[i - 1]->r.upload_done_ev;
            m->dev.push_back(q);
        }
        r->slicer = m.release();
    }
    forma_renderer_multi* m = r->slicer;
    // The slices start behind whatever the caller has queued on this renderer's stream.
    if (!P.count_ev) FORMA_CUDA_TRY(P.ensure_count_event());
    FORMA_CUDA_TRY(cudaEventRecord(P.count_ev, P.stream));
    struct Before { uint64_t launches, h2d, d2h; };
    std::vector<Before> before(n);
    for (size_t i = 0; i < n; ++i) {
        Renderer& Q = m->dev[i]->r;
        Q.copy_bands_override = std::max(options().slice_bands, 1);
        FORMA_CUDA_TRY(cudaStreamWaitEvent(Q.stream, P.count_ev, 0));
        before[i] = {Q.launches, Q.h2d_bytes, Q.d2h_bytes};
    }
    const int st = multi_render_impl(m, c, buffer, false, width, stride, height, channels, clear, crop, timings, n,
                                     options().slice_chain != 0);
    if (st) {  // a failed frame describes nothing: no segments, cells, row costs or slices to inspect
        P.last_segments = P.last_cells = P.last_entries = 0;
        P.last_tiles_x = P.last_tiles_y = 0;
        P.last_slices = 0;
        P.last_raster_valid = false;
        return st;
    }
    // What the caller reads from this renderer after a frame: sums over the slices; stage times:
    // the slowest slice (the slices overlap, so their sum means nothing).
    P.last_segments = P.last_cells = P.last_entries = 0;
    for (double& v : P.stage_ms) v = 0.0;
    bool redone = false, all_fast = true;
    for (size_t i = 0; i < n; ++i) {
        const Renderer& Q = m->dev[i]->r;
        P.launches += Q.launches - before[i].launches;
        P.h2d_bytes += Q.h2d_bytes - before[i].h2d;
        P.d2h_bytes += Q.d2h_bytes - before[i].d2h;
        P.last_cells += Q.last_cells;
        for (int k = 0; k < 8; ++k) P.stage_ms[k] = std::max(P.stage_ms[k], Q.stage_ms[k]);
        redone = redone || Q.last_tables_redone;
        all_fast = all_fast && Q.last_tables_sync_free;
    }
    for (int k = 0; k < 4; ++k) {
        P.kernel_ms[k] = 0.0;
        P.kernel_launches[k] = 0;
    }
    P.last_tables_redone = redone;
    P.last_tables_sync_free = all_fast && !redone;
    P.times_pending = false;      // stage_ms was just set from the slices
    P.last_raster_valid = false;  // forma_renderer_lines describes the last unsliced render only
    P.last_written_tiles = 0;
    P.last_tiles_x = P.last_tiles_y = 0;
    P.last_segments = (uint32_t)std::min<uint64_t>(m->last_own_segments, 0xFFFFFFFFu);
    P.last_entries = (uint32_t)std::min<uint64_t>(m->last_own_entries, 0xFFFFFFFFu);
    // (cells: a slice also forms the cells of segments that boundary-crossing lines leave in its
    // neighbours' rows, so the sum over the slices is an upper bound of the frame's cell count)
    P.last_slices = (uint32_t)n;
    return FORMA_STATUS_OK;
}

extern "C" {

forma_renderer_multi* forma_renderer_multi_new(const int* devices, int n) {
    return guarded((forma_renderer_multi*)nullptr, [&]() -> forma_renderer_multi* {
        if (!devices || n < 1 || n > 64) {
            set_error("forma_renderer_multi_new: need 1..64 device ordinals");
            return nullptr;
        }
        std::unique_ptr<forma_renderer_multi> m(new forma_renderer_multi());
        for (int i = 0; i < n; ++i) {
            for (int j = 0; j < i; ++j)
                if (devices[j] == devices[i]) {
                    set_error("forma_renderer_multi_new: device %d listed twice", devices[i]);
                    return nullptr;
                }
            forma_renderer* r = forma_renderer_new(devices[i]);
            if (!r) return nullptr;
            // Each device renders on its own (non-blocking) stream.
            cudaStream_t st = nullptr;
            if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) == cudaSuccess) {
                r->r.stream = st;
                r->r.owns_stream = true;
            }
            r->r.track_row_costs = true;
            m->dev.push_back(r);
        }
        for (int i = 1; i < n; ++i) {  // stores into the first device's frame go over NVLink
            int can = 0;
            if (cudaDeviceCanAccessPeer(&can, devices[i], devices[0]) != cudaSuccess || !can) {
                m->peer_ok = false;
                continue;
            }
            cudaSetDevice(devices[i]);
            cudaError_t e = cudaDeviceEnablePeerAccess(devices[0], 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) m->peer_ok = false;
            cudaGetLastError();
        }
        return m.release();
    });
}
void forma_renderer_multi_free(forma_renderer_multi* m) { delete m; }
/* Slices of this renderer's last host frame (0 = rendered as one piece); out_ms (may be null,
 * room for 16) receives the device-timeline ms of every slice, out_stage_ms (may be null, room for
 * 16 x 8) every slice's stage times in the order of forma_renderer_stage_times. */
int forma_renderer_host_slices(const forma_renderer* r, double* out_ms, double* out_stage_ms) {
    if (!r || !r->r.last_slices || !r->slicer) return 0;
    const size_t n = std::min<size_t>(r->r.last_slices, 16);
    for (size_t i = 0; i < n && i < r->slicer->dev.size(); ++i) {
        if (out_ms) out_ms[i] = r->slicer->dev[i]->r.stage_ms[7];
        for (int k = 0; out_stage_ms && k < 8; ++k) out_stage_ms[8 * i + k] = r->slicer->dev[i]->r.stage_ms[k];
    }
    return (int)r->r.last_slices;
}

int forma_renderer_multi_device_count(const forma_renderer_multi* m) { return m ? (int)m->dev.size() : 0; }
int forma_renderer_multi_render(forma_renderer_multi* m, forma_composition* c, uint8_t* buffer, uint64_t width, uint64_t stride,
                                uint64_t height, const uint32_t channels[4], const float clear[4], const forma_rect* crop,
                                forma_timings* timings) {
    return guarded((int)FORMA_ERR_CAPACITY,
                   [&] { return multi_render_impl(m, c, buffer, false, width, stride, height, channels, clear, crop, timings); });
}
int forma_renderer_multi_render_device(forma_renderer_multi* m, forma_composition* c, uint8_t* buffer_on_first_device,
                                       uint64_t width, uint64_t stride, uint64_t height, const uint32_t channels[4],
                                       const float clear[4], const forma_rect* crop, forma_timings* timings) {
    return guarded((int)FORMA_ERR_CAPACITY, [&] {
        return multi_render_impl(m, c, buffer_on_first_device, true, width, stride, height, channels, clear, crop, timings);
    });
}
/* Tile-row boundaries of the bands the next frame will use (n + 1 values) and the
 * device-timeline ms every band took in the last frame (n values). */
int forma_renderer_multi_bands(const forma_renderer_multi* m, uint32_t* bounds, double* band_ms) {
    if (!m) return 0;
    for (size_t i = 0; bounds && i < m->bounds.size(); ++i) bounds[i] = m->bounds[i];
    for (size_t i = 0; band_ms && i < m->last_ms.size(); ++i) band_ms[i] = m->last_ms[i];
    return (int)m->dev.size();
}
}  // extern "C"
