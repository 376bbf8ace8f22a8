// ORACLE — TEST INFRASTRUCTURE ONLY (see fmath.hpp).
//
// Layer statistics of the oracle: fo_renderer_render_stats, the counterpart of
// forma_renderer_render_stats, in a library of its own (libforma_oracle_stats.so, built by
// stats.mk) next to libforma_oracle.so. It works on the compositions libforma_oracle.so builds
// (same headers, same flags, see forma_oracle_ids.cpp). The renderer argument is not used.
//
// Every tile is walked twice, each walk with a Workbench of its own: the mask walk
// (painter_masks.hpp: paint_layer_masks, as drive_tile_masks does it) for area, pixels and box,
// and the ID walk (painter_ids.hpp: drive_tile_ids) for visible and visible_box. Each window
// layer's plane is reduced into its record as soon as it is painted, so one 16 x 16 plane is all
// the scratch a tile needs, whatever the window's size.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "painter_ids.hpp"
#include "painter_masks.hpp"

namespace fo {

// Same layout as forma_layer_stats (include/forma_b200.h).
struct LayerStats {
    uint64_t area;
    uint32_t pixels, visible;
    uint32_t box[4], visible_box[4];
};

// An empty record with min / max sentinels in its boxes.
static LayerStats empty_stats() {
    LayerStats r{};
    r.box[0] = r.box[1] = r.visible_box[0] = r.visible_box[1] = 0xFFFFFFFFu;
    return r;
}

static void widen(uint32_t box[4], uint32_t x, uint32_t y) {
    box[0] = std::min(box[0], x);
    box[1] = std::min(box[1], y);
    box[2] = std::max(box[2], x + 1);
    box[3] = std::max(box[3], y + 1);
}

// The tile's frame pixels: column-major planes like the colour planes, pixel (x, y) of the tile
// at x * kTile + y, counted where x0 + x < width and y0 + y < height.
struct TilePixels {
    size_t x0, y0, width, height;
    bool in(int x, int y) const { return x0 + x < width && y0 + y < height; }
};

// drive_tile_masks with each window layer's plane reduced into recs[id - window.first] instead
// of kept.
static void drive_tile_stats(Workbench& wb, Painter& painter, const TileContext& ctx, const MaskWindow& window, float min_coverage,
                             const TilePixels& px, float* plane, LayerStats* recs) {
    wb.populate_layers(ctx);
    wb.skip_trivial_clips_pass(ctx);
    painter.clip_active = false;
    for (size_t k = 0; k < wb.ids.size(); ++k) {
        const uint32_t id = wb.ids[k].id;
        const Props& props = ctx.props->get(id);
        const bool is_clip = props.func != kDraw, in_window = window.holds(id);
        if (wb.ids[k].mask || (is_clip && in_window)) {
            painter.clear_cells();
            if (const Workbench::SegRange* r = wb.segments_of(id))
                for (size_t i = r->first; i <= r->last; ++i) painter.acc_segment(ctx.segs[i]);
            if (const Cover* c = wb.cover(id)) painter.acc_cover(*c);
            const bool apply_clip = !is_clip && props.is_clipped && !wb.ids[k].skip_clipping;
            if (in_window) std::fill(plane, plane + kTile * kTile, 0.0f);
            Cover cv = paint_layer_masks(painter, id, props, apply_clip, wb.ids[k].mask, in_window ? plane : nullptr);
            if (in_window) {
                LayerStats& r = recs[id - window.first];
                for (int x = 0; x < kTile; ++x)
                    for (int y = 0; y < kTile; ++y) {
                        if (!px.in(x, y)) continue;
                        const float v = plane[x * kTile + y];
                        r.area += (uint64_t)(v * 262144.0f);  // exact: v is k / 512 or a product of two such values
                        if (v > min_coverage) {
                            ++r.pixels;
                            widen(r.box, (uint32_t)(px.x0 + x), (uint32_t)(px.y0 + y));
                        }
                    }
            }
            if (wb.ids[k].mask) {
                if (!cv.is_empty(props.fill_rule)) wb.next_queue.push_back({cv, id});
                continue;
            }
        }
        CoverCarry cc;
        if (wb.cover_carry(ctx, id, &cc)) wb.next_queue.push_back(cc);
    }
    wb.next_tile();
}

// Starts a tile row on `wb` with the carries of the tiles left of the crop (as paint_tile_row
// does); returns the first segment of the crop's first tile.
static size_t begin_row(Workbench& wb, const uint64_t* segs, size_t n, const Rect* crop) {
    std::map<uint32_t, Cover> left;
    int16_t tile_x_start = crop ? (int16_t)crop->hor0 : 0;
    size_t pos = 0;
    while (pos < n && seg_tile_x(segs[pos]) < tile_x_start) {
        Cover& c = left[seg_layer(segs[pos])];
        int y = seg_local_y(segs[pos]);
        c.c[y] = (int8_t)(c.c[y] + seg_cover(segs[pos]));
        ++pos;
    }
    std::vector<CoverCarry> carries;
    for (auto& kv : left) carries.push_back({kv.second, kv.first});
    wb.init(std::move(carries));
    wb.next_queue.clear();
    wb.ids.clear();
    wb.skipped = 0;
    wb.segment_ranges.clear();
    wb.layers_were_removed = true;
    return pos;
}

static void stats_tile_row(Painter& painter, Workbench& wb_masks, Workbench& wb_ids, size_t tile_y, const uint64_t* segs, size_t n,
                           const PropsSource& props, size_t width, size_t height, const Rect* crop, const MaskWindow& window,
                           float min_coverage, float* plane, LayerStats* recs) {
    size_t pos = begin_row(wb_masks, segs, n, crop);
    begin_row(wb_ids, segs, n, crop);
    const Channel ch[4] = {kRed, kGreen, kBlue, kAlpha};
    size_t width_in_tiles = (width + kTile - 1) / kTile;
    uint32_t ids[kTile * kTile];
    for (size_t tile_x = 0; tile_x < width_in_tiles; ++tile_x) {
        if (crop && !(tile_x >= crop->hor0 && tile_x < crop->hor1)) continue;
        size_t begin = pos;
        while (pos < n && seg_tile_x(segs[pos]) == (int16_t)tile_x) ++pos;
        TileContext ctx;
        ctx.tile_x = tile_x;
        ctx.tile_y = tile_y;
        ctx.segs = segs + begin;
        ctx.n_segs = pos - begin;
        ctx.props = &props;
        ctx.has_cached_clear = false;
        ctx.cached_clear = Color();
        ctx.cached_tile = nullptr;
        ctx.channels = ch;
        ctx.clear_color = Color();
        const TilePixels px{tile_x * kTile, tile_y * kTile, width, height};
        drive_tile_stats(wb_masks, painter, ctx, window, min_coverage, px, plane, recs);
        painter.clip_active = false;
        drive_tile_ids(wb_ids, painter, ctx, min_coverage, ids);
        for (int x = 0; x < kTile; ++x)
            for (int y = 0; y < kTile; ++y) {
                const uint32_t id = ids[x * kTile + y];
                if (!px.in(x, y) || !window.holds(id)) continue;
                LayerStats& r = recs[id - window.first];
                ++r.visible;
                widen(r.visible_box, (uint32_t)(px.x0 + x), (uint32_t)(px.y0 + y));
            }
    }
}

static bool render_stats(Composition& comp, LayerStats* out, uint32_t first, uint32_t count, size_t width, size_t height,
                         const Rect* crop, float min_coverage, size_t* n_lines, size_t* n_segments) {
    size_t ht = (height + kTile - 1) / kTile;
    comp.compact_geom();
    Lines lines;
    std::vector<uint64_t> segments;
    comp.fill_cpu_view(width, height, lines);
    if (!rasterize(lines, segments)) return false;  // more pixel segments than u32 sums can index
    std::sort(segments.begin(), segments.end(), [](uint64_t a, uint64_t b) { return (a >> kSortShift) < (b >> kSortShift); });
    PropsSource props;
    props.index(comp.layers);
    const uint32_t n_orders = comp.layers.empty() ? 0u : comp.layers.rbegin()->first + 1u;
    const MaskWindow window{first, first < n_orders ? std::min(count, n_orders - first) : 0u};
    const uint64_t* segs = segments.data();
    size_t n = segments.size();
    size_t first_seg = std::partition_point(segs, segs + n, [](uint64_t s) { return seg_tile_y(s) < 0; }) - segs;
    std::vector<size_t> row_start(ht + 1);
    for (size_t j = 0; j <= ht; ++j) {
        row_start[j] =
            std::partition_point(segs + first_seg, segs + n, [j](uint64_t s) { return (size_t)seg_tile_y(s) < j; }) - segs;
    }
    for (uint32_t k = 0; k < count; ++k) out[k] = empty_stats();
    if (window.count) {
#pragma omp parallel
        {
            Painter painter;
            Workbench wb_masks, wb_ids;
            std::vector<float> plane(kTile * kTile);
            std::vector<LayerStats> recs(window.count, empty_stats());
#pragma omp for schedule(dynamic, 1)
            for (size_t j = 0; j < ht; ++j) {
                if (crop && !(j >= crop->vert0 && j < crop->vert1)) continue;
                stats_tile_row(painter, wb_masks, wb_ids, j, segs + row_start[j], row_start[j + 1] - row_start[j], props, width, height,
                               crop, window, min_coverage, plane.data(), recs.data());
            }
#pragma omp critical
            for (uint32_t k = 0; k < window.count; ++k) {
                LayerStats& o = out[k];
                const LayerStats& r = recs[k];
                o.area += r.area;
                o.pixels += r.pixels;
                o.visible += r.visible;
                for (int c = 0; c < 2; ++c) {
                    o.box[c] = std::min(o.box[c], r.box[c]);
                    o.box[2 + c] = std::max(o.box[2 + c], r.box[2 + c]);
                    o.visible_box[c] = std::min(o.visible_box[c], r.visible_box[c]);
                    o.visible_box[2 + c] = std::max(o.visible_box[2 + c], r.visible_box[2 + c]);
                }
            }
        }
    }
    for (uint32_t k = 0; k < count; ++k) {
        if (!out[k].pixels) std::memset(out[k].box, 0, sizeof(out[k].box));
        if (!out[k].visible) std::memset(out[k].visible_box, 0, sizeof(out[k].visible_box));
    }
    *n_lines = lines.size();
    *n_segments = segments.size();
    return true;
}

}  // namespace fo

using namespace fo;

// Same layouts as forma_rect / forma_timings / forma_stats (include/forma_b200.h).
struct fo_stats_rect {
    uint64_t hor_start, hor_end, vert_start, vert_end;
};
struct fo_stats_timings {
    double line_setup_ms, rasterize_ms, sort_ms, paint_ms;
    uint64_t n_lines, n_segments;
};
struct fo_stats {
    LayerStats* ptr;
    uint32_t first_order, n_orders;
    float min_coverage;
};

extern "C" {

// The refusals of forma_renderer_render_stats that apply to a host frame.
int fo_renderer_render_stats(void*, void* cv, const fo_stats* s, uint64_t width, uint64_t height, const fo_stats_rect* crop,
                             fo_stats_timings* timings) {
    if (!s || !s->ptr || ((uintptr_t)s->ptr & 7u) != 0 || s->n_orders == 0 || (uint64_t)s->first_order + s->n_orders > (1ull << 21) ||
        !std::isfinite(s->min_coverage) || s->min_coverage < 0.0f || s->min_coverage >= 1.0f || width == 0 || height == 0)
        return 1;
    Rect rect;
    if (crop) {
        rect.hor0 = crop->hor_start / kTile;
        rect.hor1 = (crop->hor_end + kTile - 1) / kTile;
        rect.vert0 = crop->vert_start / kTile;
        rect.vert1 = (crop->vert_end + kTile - 1) / kTile;
    }
    size_t n_lines = 0, n_segments = 0;
    if (!render_stats(*(Composition*)cv, s->ptr, s->first_order, s->n_orders, (size_t)width, (size_t)height, crop ? &rect : nullptr,
                      s->min_coverage, &n_lines, &n_segments))
        return 5;  // FORMA_ERR_CAPACITY
    if (timings) {
        *timings = fo_stats_timings{};
        timings->n_lines = n_lines;
        timings->n_segments = n_segments;
    }
    return 0;
}

}  // extern "C"
