// forma_b200 — errors, schedule options, layer props and the Composition
// bookkeeping (composition/mod.rs, composition/layer.rs), including the pinned
// lookup tables every render uploads.
#include <algorithm>
#include <cctype>
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>

#include "../../include/forma_b200.h"
#include "host_scene.hpp"
#include "kernels.h"

namespace forma {

// ---------------------------------------------------------------------------
// Errors
// ---------------------------------------------------------------------------
static thread_local std::string g_error;

void set_error(const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_error = buf;
}

// ---------------------------------------------------------------------------
// Options
// ---------------------------------------------------------------------------
struct OptionName {
    const char* name;
    int Options::*field;
    int lo, hi;
};
static const OptionName kOptionNames[] = {
    {"speculate", &Options::speculate, 0, 1},         {"band_copy", &Options::band_copy, 0, 1},
    {"copy_bands", &Options::copy_bands, 1, 16},      {"sort_full_key", &Options::sort_full_key, 0, 1},
    {"sort_big_log2", &Options::sort_big_log2, 10, 30}, {"test_gap_cap", &Options::test_gap_cap, 0, 1 << 30},
    {"paint_lpt", &Options::paint_lpt, 0, 1},         {"band_filter", &Options::band_filter, 0, 1},
    {"paint_wide", &Options::paint_wide, 0, 1},       {"sort_scan_log2", &Options::sort_scan_log2, 10, 31},
    {"paint_solid", &Options::paint_solid, 0, 1},     {"sort_counts", &Options::sort_counts, 0, 1},
    {"sync_free", &Options::sync_free, 0, 1},         {"test_fast_shrink", &Options::test_fast_shrink, 0, 1},
    {"host_slices", &Options::host_slices, 1, 16},    {"slice_bands", &Options::slice_bands, 1, 16},
    {"slice_min_points", &Options::slice_min_points, 0, 1 << 30}, {"slice_chain", &Options::slice_chain, 0, 1},
    {"pdl", &Options::pdl, 0, 1},                     {"sync_free_sort", &Options::sync_free_sort, 0, 1},
    {"test_sort_bound", &Options::test_sort_bound, 0, 1 << 30},
};
Options& options() {
    static Options o = [] {
        Options v;
        for (const OptionName& n : kOptionNames) {
            std::string env = "FORMA_";
            for (const char* c = n.name; *c; ++c) env += (char)toupper((unsigned char)*c);
            if (const char* e = getenv(env.c_str())) {
                long x = strtol(e, nullptr, 10);
                if (x >= n.lo && x <= n.hi) v.*(n.field) = (int)x;
            }
        }
        return v;
    }();
    return o;
}

bool chained_launches() { return options().pdl != 0; }

// ---------------------------------------------------------------------------
// Props
// ---------------------------------------------------------------------------
static bool same4(const float* a, const float* b, int n) {
    for (int i = 0; i < n; ++i)
        if (!(a[i] == b[i])) return false;
    return true;
}

// Props: PartialEq (styling.rs derives + Gradient/Image impls).
bool HostProps::equals(const HostProps& o) const {
    const StyleRec &a = rec, &b = o.rec;
    if (a.fill_rule != b.fill_rule || a.func != b.func) return false;
    if (a.func == 1u) return a.clip_layers == b.clip_layers;
    if (a.is_clipped != b.is_clipped || a.blend_mode != b.blend_mode || a.fill_type != b.fill_type) return false;
    if (a.fill_type == 0u) return same4(a.color, b.color, 4);
    if (a.fill_type == 1u) {
        if (a.gradient_type != b.gradient_type || !same4(a.start, b.start, 2) || !same4(a.end, b.end, 2) ||
            stops.size() != o.stops.size())
            return false;
        for (size_t i = 0; i < stops.size(); ++i)
            if (!same4(stops[i].color, o.stops[i].color, 4) || !(stops[i].stop == o.stops[i].stop)) return false;
        return true;
    }
    return texels == o.texels && a.tex_max_x == b.tex_max_x && a.tex_max_y == b.tex_max_y &&
           same4(a.tex_xf, b.tex_xf, 6);
}

// ---------------------------------------------------------------------------
// Composition (composition/mod.rs, composition/layer.rs)
// ---------------------------------------------------------------------------
Layer* Composition::create_layer() {  // mod.rs:65-83
    std::unique_ptr<Layer> owned(new Layer());
    Layer* l = owned.get();
    pool.emplace(l, std::move(owned));
    l->geom_id = next_geom_id++;
    l->dense_id = next_dense_id++;
    return l;
}

void Composition::set_order(Layer* l, int64_t order) {  // layer.rs:148-158
    if (order >= 0 && l->order != order) {
        l->order = order;
        l->unchanged_bits = 0;
    }
    geom_to_order[l->dense_id] = order;
    tables_dirty = true;
}

Layer* Composition::insert(uint32_t order, Layer* layer) {  // mod.rs:121-138
    // The reference takes the Layer by value: a layer cannot sit at two orders. Through
    // the C ABI the same handle can be inserted again, which moves it.
    if (layer->order >= 0 && (uint32_t)layer->order != order) {
        auto at = layers.find((uint32_t)layer->order);
        if (at != layers.end() && at->second == layer) layers.erase(at);
    }
    set_order(layer, order);
    Layer* old = nullptr;
    auto it = layers.find(order);
    if (it != layers.end()) {
        old = it->second;
        it->second = layer;
    } else {
        layers.emplace(order, layer);
    }
    if (old == layer) return nullptr;
    if (old) set_order(old, -1);
    return old;
}

Layer* Composition::remove(uint32_t order) {  // mod.rs:141-149
    auto it = layers.find(order);
    if (it == layers.end()) return nullptr;
    Layer* l = it->second;
    layers.erase(it);
    set_order(l, -1);
    return l;
}

Layer* Composition::get(uint32_t order) {
    auto it = layers.find(order);
    return it == layers.end() ? nullptr : it->second;
}

Layer* Composition::get_or_insert_default(uint32_t order) {  // mod.rs:175-182
    Layer* l = get(order);
    if (!l) {
        l = create_layer();
        insert(order, l);
    }
    return l;
}

void Composition::drop(Layer* l) {  // Drop for Layer, layer.rs:355-363
    if (l->order >= 0) {  // attached layers are found by their order; a detached one keeps a stale order
        auto it = layers.find((uint32_t)l->order);
        if (it != layers.end() && it->second == l) layers.erase(it);
    }
    geom_to_order.erase(l->dense_id);
    garbage_points += l->points;
    pool.erase(l);
    tables_dirty = true;
}

// Layer::insert (layer.rs:90-111) + SegmentBuffer::push_path (segment.rs:181-198).
void Composition::layer_insert(Layer* layer, const Path& path) {
    const FlattenProgram& prog = path.data->program();
    uint32_t count = prog.n_points;
    if (count) {
        if ((uint64_t)n_points + count >= (1ull << 32)) compact_geom();  // dead geometry counts until compacted
        if ((uint64_t)n_points + count >= (1ull << 32))
            throw std::length_error("segment buffer would exceed 2^32 points");
        PendingInsert job;
        job.data = path.data;
        job.has_xf = path.has_xf;
        std::memcpy(job.xf, path.xf, sizeof(job.xf));
        job.geom_id = layer->dense_id;
        job.dst = n_points;
        job.count = count;
        // Rows the insert can reach (for the band filter of multi-GPU frames): the program's
        // bounds through the path's transform, widened by half a pixel plus a relative term
        // that covers the rounding of the evaluation; infinite when the hull argument fails.
        job.y_min = -INFINITY;
        job.y_max = INFINITY;
        if (prog.bounded) {
            float lo = prog.min_y, hi = prog.max_y;
            if (path.has_xf) {  // ty = fma(uy, x, fma(vy, y, t.y)) over the four corners
                lo = INFINITY;
                hi = -INFINITY;
                for (int cx = 0; cx < 2; ++cx)
                    for (int cy = 0; cy < 2; ++cy) {
                        const float px = cx ? prog.max_x : prog.min_x, py = cy ? prog.max_y : prog.min_y;
                        const float ty = fmaf(path.xf[1], px, fmaf(path.xf[3], py, path.xf[5]));
                        lo = std::fmin(lo, ty);
                        hi = std::fmax(hi, ty);
                    }
            }
            if (lo == lo && hi == hi && std::isfinite(lo) && std::isfinite(hi)) {
                const float margin = 0.5f + 1e-4f * std::fmax(std::fabs(lo), std::fabs(hi));
                job.y_min = lo - margin;
                job.y_max = hi + margin;
            }
        }
        jobs.push_back(std::move(job));
        // ids that are Some: every point that does not end a contour, except the
        // last point of the insert (its id is the trailing None).
        uint64_t some = (uint64_t)(count - 1u) - prog.n_contour_ends;
        some_ids += some;
        layer->lines_count += some;
        layer->points += count;
        n_points += count;
    }
    geom_to_order[layer->dense_id] = layer->order;
    layer->unchanged_bits = 0;
    tables_dirty = true;
}

void Composition::compact_geom() {
    const bool dead_points = garbage_points >= 65536u && garbage_points * 2u >= n_points;
    const bool dead_ids = (uint64_t)next_dense_id > 2u * (uint64_t)pool.size() + 65536u;
    if (!dead_points && !dead_ids) return;
    // Dense ids are handed out again from 1, in the order the live layers got theirs, so
    // that the device's id -> layer table stays proportional to the live layers however
    // often layers are cleared (every Layer::clear takes a new id, layer.rs:131-146).
    std::vector<Layer*> alive;
    alive.reserve(pool.size());
    for (auto& kv : pool) alive.push_back(kv.first);
    std::sort(alive.begin(), alive.end(), [](const Layer* a, const Layer* b) { return a->dense_id < b->dense_id; });
    std::unordered_map<uint32_t, uint32_t> renumbered;
    std::unordered_map<uint32_t, int64_t> orders;
    renumbered.reserve(alive.size());
    orders.reserve(alive.size());
    uint32_t next = 1;
    for (Layer* l : alive) {
        auto it = geom_to_order.find(l->dense_id);
        if (it != geom_to_order.end()) orders.emplace(next, it->second);
        renumbered.emplace(l->dense_id, next);
        l->dense_id = next++;
    }
    std::vector<PendingInsert> live;
    live.reserve(jobs.size());
    uint64_t pts = 0;
    for (PendingInsert& j : jobs) {
        auto it = renumbered.find(j.geom_id);  // inserts of cleared / dropped geometry have no live id
        if (it == renumbered.end() || !orders.count(it->second)) continue;
        j.geom_id = it->second;
        j.dst = (uint32_t)pts;
        pts += j.count;
        live.push_back(std::move(j));
    }
    jobs.swap(live);
    geom_to_order.swap(orders);
    next_dense_id = next;
    n_points = (uint32_t)pts;
    garbage_points = 0;
    ++geom_epoch;  // everything is evaluated again into the re-packed buffers (see Renderer::flush_geometry)
    tables_dirty = true;
}

void Composition::layer_clear(Layer* layer) {  // layer.rs:131-146
    garbage_points += layer->points;
    layer->points = 0;
    geom_to_order.erase(layer->dense_id);
    layer->geom_id = next_geom_id++;
    layer->dense_id = next_dense_id++;
    geom_to_order[layer->dense_id] = layer->order;
    layer->lines_count = 0;
    layer->unchanged_bits = 0;
    tables_dirty = true;
}

// Host part: the pinned copies of the tables (no CUDA work besides pinned allocations). A
// caller that renders one composition on several devices runs it once before its workers start.
int Composition::rebuild_tables(int64_t cache_id) {
    std::vector<StopRec> stops;
    std::vector<uint16_t> texels;
    std::unordered_map<const void*, uint32_t> tex_offsets;
    uint32_t max_order = 0;
    for (auto& kv : layers) max_order = std::max(max_order, kv.first);
    uint32_t n_orders = layers.empty() ? 0u : max_order + 1u;
    uint32_t n_geoms = next_dense_id;
    FORMA_CUDA_TRY(h_layers.reserve(layers.size() + 1));
    FORMA_CUDA_TRY(h_styles.reserve(layers.size() + 1));
    FORMA_CUDA_TRY(h_order_to_style.reserve(n_orders + 1));
    FORMA_CUDA_TRY(h_geom_slot.reserve(n_geoms + 1));
    std::fill(h_order_to_style.ptr, h_order_to_style.ptr + n_orders, -1);
    std::fill(h_geom_slot.ptr, h_geom_slot.ptr + n_geoms, -1);
    uint32_t slot = 0, n_styles = 0;
    bool any_xf = false, solid_over = true;
    FORMA_CUDA_TRY(h_layer_bits.reserve(layers.size() + 1));
    std::unordered_map<std::string, uint32_t> interned;
    std::vector<int32_t> order_to_slot(n_orders, -1);
    for (auto& kv : layers) {
        const Layer& l = *kv.second;
        LayerRec& r = h_layers.ptr[slot];
        r.order = kv.first;
        r.enabled = l.enabled ? 1u : 0u;
        r.has_xf = l.has_xf ? 1u : 0u;
        r.ux = l.xf[0]; r.uy = l.xf[1]; r.vx = l.xf[2]; r.vy = l.xf[3]; r.tx = l.xf[4]; r.ty = l.xf[5];
        h_layer_bits.ptr[slot] = (kv.first & 0x1FFFFFu) | (r.enabled << 21);
        any_xf = any_xf || l.has_xf;
        StyleRec s = l.props.rec;
        solid_over = solid_over && s.func == 0u && !s.is_clipped && s.fill_type == 0u && s.blend_mode == 0u;
        s.stop_first = (uint32_t)stops.size();
        s.stop_count = (uint32_t)l.props.stops.size();
        stops.insert(stops.end(), l.props.stops.begin(), l.props.stops.end());
        if (s.fill_type == 2u && l.props.texels) {
            auto it = tex_offsets.find(l.props.texels.get());
            if (it == tex_offsets.end()) {
                uint32_t off = (uint32_t)(texels.size() / 4);
                texels.insert(texels.end(), l.props.texels->begin(), l.props.texels->end());
                it = tex_offsets.emplace(l.props.texels.get(), off).first;
            }
            s.tex_first = it->second;
        }
        s.unchanged = 0u;
        // Styles are interned like the reference's props interner (composition/interner.rs):
        // solid fills that compare equal share one record (paris-30k: 66 records for 50 620
        // layers); gradients / textures keep one record per layer.
        uint32_t style_index = n_styles;
        if (s.fill_type == 0u && s.func == 0u) {
            std::string key(reinterpret_cast<const char*>(&s), offsetof(StyleRec, gradient_type));
            auto it = interned.find(key);
            if (it == interned.end()) interned.emplace(std::move(key), n_styles);
            else style_index = it->second;
        }
        if (style_index == n_styles) h_styles.ptr[n_styles++] = s;
        h_order_to_style.ptr[kv.first] = (int32_t)style_index;
        order_to_slot[kv.first] = (int32_t)slot;
        ++slot;
    }
    for (auto& kv : geom_to_order) {
        if (kv.second < 0 || kv.first >= n_geoms || (uint64_t)kv.second >= n_orders) continue;
        h_geom_slot.ptr[kv.first] = order_to_slot[kv.second];
    }
    layers_in_order = true;
    {
        int64_t last = -1;
        for (const PendingInsert& job : jobs) {
            if (job.geom_id >= n_geoms) continue;
            int32_t s = h_geom_slot.ptr[job.geom_id];
            if (s < 0) continue;
            int64_t order = (int64_t)h_layers.ptr[s].order;
            if (order < last) {
                layers_in_order = false;
                break;
            }
            last = order;
        }
    }
    FORMA_CUDA_TRY(h_stops.reserve(stops.size() + 1));
    FORMA_CUDA_TRY(h_texels.reserve(texels.size() + 1));
    if (!stops.empty()) std::memcpy(h_stops.ptr, stops.data(), stops.size() * sizeof(StopRec));
    if (!texels.empty()) std::memcpy(h_texels.ptr, texels.data(), texels.size() * sizeof(uint16_t));
    n_layer_recs = slot;
    layers_have_xf = any_xf;
    solid_over_only = solid_over;
    n_style_recs = n_styles;
    n_stops = stops.size();
    n_texels = texels.size();
    this->n_geoms = n_geoms;
    this->n_orders = n_orders;
    tables_dirty = false;
    tables_cache_id = cache_id;
    ++tables_version;
    return FORMA_STATUS_OK;
}

}  // namespace forma

using namespace forma;

extern "C" {

const char* forma_last_error(void) { return g_error.c_str(); }

int forma_set_option(const char* name, int value) {
    if (name)
        for (const OptionName& n : kOptionNames)
            if (!strcmp(n.name, name)) {
                if (value < n.lo || value > n.hi) break;
                options().*(n.field) = value;
                return FORMA_OK;
            }
    set_error("forma_set_option: unknown option or value out of range (%s = %d)", name ? name : "(null)", value);
    return FORMA_ERR_INVALID_ARGUMENT;
}
int forma_get_option(const char* name, int* value) {
    if (name && value)
        for (const OptionName& n : kOptionNames)
            if (!strcmp(n.name, name)) {
                *value = options().*(n.field);
                return FORMA_OK;
            }
    set_error("forma_get_option: unknown option %s", name ? name : "(null)");
    return FORMA_ERR_INVALID_ARGUMENT;
}

}  // extern "C"
