// forma_b200 host side — Composition / Layer bookkeeping and the HBM-resident
// segment buffer. Mirrors forma/src/composition/{mod,layer,state}.rs and the
// storage half of forma/src/segment.rs.
//
// Unlike the reference, the flattened points never live in host memory:
// Layer::insert queues a flatten job and the points are evaluated straight into
// the device segment buffer (x, y, geometry id per point) the next time the
// composition is rendered.
#pragma once

#include <atomic>
#include <map>
#include <memory>
#include <unordered_map>
#include <vector>

#include "cuda_common.cuh"
#include "host_path.hpp"

namespace forma {

struct HostProps {
    StyleRec rec{};                 // stop_first / tex_first are assigned at upload time
    std::vector<StopRec> stops;
    std::shared_ptr<std::vector<uint16_t>> texels;  // RGBA f16
    bool equals(const HostProps& o) const;
};

struct Layer {
    bool enabled = true;
    bool has_xf = false;
    float xf[6] = {1, 0, 0, 1, 0, 0};  // ux, uy, vx, vy, tx, ty
    int64_t order = -1;               // InnerLayer.order (kept when detached, layer.rs:148-158)
    uint64_t geom_id = 0;             // GeomId (public, never reused)
    uint32_t dense_id = 0;            // this geometry's index in the device's id -> layer table (0 = None);
                                      // renumbered by Composition::compact_geom
    HostProps props;
    uint32_t unchanged_bits = 0;      // SmallBitSet over layer-cache ids
    size_t lines_count = 0;
    uint64_t points = 0;              // points this layer's current geometry id owns in the segment buffer
};

struct PendingInsert {
    std::shared_ptr<PathData> data;
    bool has_xf;
    float xf[6];
    uint32_t geom_id;  // Layer::dense_id at the time of the insert
    uint32_t dst;    // first point in the (unfiltered) segment buffer
    uint32_t count;  // number of points
    float y_min, y_max;  // rows the insert's points can take before the layer's transform (+- a safety margin)
};

// What one CUDA device holds of a composition: the evaluated points of the inserts that can
// reach the rows it renders, the lookup tables, and the pinned staging of its uploads.
struct CompDevice {
    DeviceBuffer<float> d_x, d_y;
    DeviceBuffer<uint32_t> d_gid;
    uint32_t n_resident = 0;          // points evaluated on this device
    size_t jobs_resident = 0;         // jobs [0, jobs_resident) were considered (evaluated, or left out by the band filter)
    uint64_t geom_epoch = 0;          // Composition::geom_epoch these points belong to
    // Band filter: when set, only inserts whose bounds meet the pixel rows [band_lo, band_hi) are
    // resident (a GPU that paints a band of tile rows never needs the rest, SURVEY.md 8e).
    bool filtered = false;
    float band_lo = 0.0f, band_hi = 0.0f;
    // Pinned staging of the flatten programs of jobs [staged_from, staged_to) for this device.
    PinnedBuffer<SplineRec> h_splines;
    PinnedBuffer<PointRec> h_points;
    PinnedBuffer<uint8_t> h_kinds;
    PinnedBuffer<QuadUp> h_quads;
    PinnedBuffer<FlattenJob> h_jobs;
    PinnedBuffer<JobXf> h_xfs;        // transforms of the staged jobs that carry one (FlattenJob::xf_index)
    bool staged_valid = false;
    bool staged_rational = true;      // the staged quadratics are QuadUp (else QuadUpPoly)
    bool staged_filtered = false;
    float staged_lo = 0.0f, staged_hi = 0.0f;
    size_t staged_from = 0, staged_to = 0, staged_jobs = 0, staged_splines = 0, staged_recs = 0, staged_quads = 0,
           staged_points = 0, staged_xfs = 0;
    // Tables.
    uint64_t tables_version = 0;      // Composition::tables_version of the device copies (0 = none)
    DeviceBuffer<uint32_t> d_layer_bits;
    DeviceBuffer<int32_t> d_geom_slot;
    DeviceBuffer<LayerRec> d_layers;
    DeviceBuffer<StyleRec> d_styles;
    DeviceBuffer<int32_t> d_order_to_style;
    DeviceBuffer<StopRec> d_stops;
    DeviceBuffer<GradRec> d_grads;    // built on the device from d_styles / d_stops (grad_setup_kernel)
    DeviceBuffer<uint16_t> d_texels;
    // keep_staging: the pinned copies of the last batch stay valid (an evicted composition is
    // re-uploaded from them without touching the host-side programs again).
    void reset_residency(bool keep_staging = false) {
        n_resident = 0;
        jobs_resident = 0;
        filtered = false;
        if (!keep_staging) staged_valid = false;
        tables_version = 0;
    }
};

class Composition {
   public:
    // Unique in the process and never reused (an address can be: a freed composition and a new
    // one may share it): what a renderer's batch tables are keyed on, with tables_version.
    const uint64_t serial = new_serial();
    static uint64_t new_serial() {
        static std::atomic<uint64_t> next{1};
        return next++;
    }
    std::map<uint32_t, Layer*> layers;              // attached layers by order
    std::unordered_map<Layer*, std::unique_ptr<Layer>> pool;  // every live layer (attached or not)
    std::unordered_map<uint32_t, int64_t> geom_to_order;  // dense id -> order, -1 == None
    uint64_t next_geom_id = 1;
    uint32_t next_dense_id = 1;

    Layer* create_layer();
    Layer* insert(uint32_t order, Layer* layer);    // returns the displaced layer
    Layer* remove(uint32_t order);
    Layer* get(uint32_t order);
    Layer* get_or_insert_default(uint32_t order);
    void drop(Layer* layer);

    void layer_insert(Layer* layer, const Path& path);
    void layer_clear(Layer* layer);
    // Composition::compact_geom (composition/mod.rs:184-218): drops the inserts of
    // cleared / dropped layers and re-packs the segment buffer (the survivors are
    // re-evaluated at the next render). Runs when at least half of the points are dead.
    void compact_geom();
    uint64_t garbage_points = 0;      // points whose geometry id no longer maps to a layer
    void mark_dirty() { tables_dirty = true; }

    // --- segment buffer ------------------------------------------------------------
    uint32_t n_points = 0;            // points appended so far (dead geometry included until compacted)
    uint64_t some_ids = 0;            // SegmentBuffer::len(): ids that are Some
    std::vector<PendingInsert> jobs;  // every Layer::insert so far, in order
    uint64_t geom_epoch = 1;          // bumped by compact_geom: device copies of an older epoch are stale
    // Residency per CUDA device (one process may render the composition on several GPUs).
    std::map<int, std::unique_ptr<CompDevice>> devices;
    CompDevice& on(int device) {
        auto& p = devices[device];
        if (!p) p.reset(new CompDevice());
        return *p;
    }
    // Drops device residency: the next render re-uploads everything from pinned
    // host memory (used to measure the cold, end-to-end path).
    void evict() {
        for (auto& kv : devices) kv.second->reset_residency(true);
    }

    // --- per-frame lookup tables: pinned host copies, rebuilt when dirty -------------
    bool tables_dirty = true;         // host-side pinned copies are stale
    uint64_t tables_version = 0;      // bumped at every rebuild; a device copy of an older version is stale
    PinnedBuffer<LayerRec> h_layers;
    PinnedBuffer<uint32_t> h_layer_bits;  // order | enabled << 21: uploaded instead of h_layers when no layer has a transform
    bool layers_have_xf = false;
    PinnedBuffer<StyleRec> h_styles;
    PinnedBuffer<int32_t> h_order_to_style, h_geom_slot;
    PinnedBuffer<StopRec> h_stops;
    PinnedBuffer<uint16_t> h_texels;
    size_t n_layer_recs = 0, n_style_recs = 0, n_stops = 0, n_texels = 0;
    uint32_t n_geoms = 0, n_orders = 0;
    // The inserts' layer orders never decrease along the segment buffer, so the
    // rasterizer emits the pixel segments already ordered by layer and the
    // (stable) sort only needs the tile_x / tile_y digits.
    bool layers_in_order = false;
    // Every layer is a Draw layer with a solid fill, BlendMode::Over and no clip: its frames are
    // painted by the lean build of the paint kernel (launch_paint).
    bool solid_over_only = false;
    int64_t tables_cache_id = -2;     // cache id the `unchanged` bits were uploaded for
    int rebuild_tables(int64_t cache_id);  // FORMA_STATUS_*

   private:
    void set_order(Layer* l, int64_t order);
};

}  // namespace forma
