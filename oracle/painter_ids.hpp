// ORACLE — TEST INFRASTRUCTURE ONLY (see fmath.hpp).
//
// ID frames: the painter walk of painter.hpp (Workbench passes, Painter cells and clip state)
// recording where blend_at would run instead of blending. Free functions over the painter's
// own types, so that painter.hpp and the RGBA path built from it stay exactly as they are.
#pragma once

#include "painter.hpp"

namespace fo {

constexpr uint32_t kIdNone = 0xFFFFFFFFu;

// Painter::paint_layer without colour arithmetic: where blend_at would run for the layer with
// coverage x clip mask > min_coverage, ids[idx] (column-major like the colour planes) becomes
// layer_id. Same clip state and returned cover as paint_layer.
inline Cover paint_layer_ids(Painter& p, uint32_t layer_id, const Props& props, bool apply_clip, float min_coverage,
                             uint32_t* ids) {
    int8_t run[kTile] = {0};
    if (p.clip_active && p.clip_last < layer_id) p.clip_active = false;
    for (int x = 0; x <= kTile; ++x) {
        if (x != 0) {
            int px = x - 1;
            int32_t da[kTile];
            for (int y = 0; y < kTile; ++y) da[y] = 32 * (int32_t)run[y] + (int32_t)p.areas[px * kTile + y];
            for (int half = 0; half < 2; ++half) {
                float cov[8];
                bool all_zero = true;
                for (int l = 0; l < 8; ++l) cov[l] = Painter::coverage_of(da[half * 8 + l], props.fill_rule);
                for (int l = 0; l < 8; ++l)
                    if (!(cov[l] == 0.0f)) all_zero = false;
                const int base = px * kTile + half * 8;
                if (props.func == kDraw) {
                    if (all_zero) continue;
                    if (apply_clip && !p.clip_active) continue;
                    for (int l = 0; l < 8; ++l) {
                        float f = cov[l];
                        if (apply_clip && p.clip_active) f *= p.clip_mask[base + l];
                        if (f > min_coverage) ids[base + l] = layer_id;
                    }
                } else {  // clip_at, cpu/painter/mod.rs:449-464
                    if (!p.clip_active) {
                        p.clip_active = true;
                        for (float& m : p.clip_mask) m = 0.0f;
                        p.clip_last = layer_id + props.clip_layers;
                    }
                    for (int l = 0; l < 8; ++l) p.clip_mask[base + l] = cov[l];
                }
            }
        }
        for (int y = 0; y < kTile; ++y) run[y] = (int8_t)(run[y] + p.covers[x * kTile + y]);
    }
    Cover out;
    std::memcpy(out.c, run, sizeof(run));
    return out;
}

// Workbench::drive_tile_painting for an ID frame (no layer cache: tile_unchanged_pass changes
// nothing). out[256], column-major: the order of the top-most Draw layer that hits each pixel,
// or kIdNone. A tile that folds into one solid colour gets the top-most layer of the fold.
inline void drive_tile_ids(Workbench& wb, Painter& painter, const TileContext& ctx, float min_coverage,
                           uint32_t out[kTile * kTile]) {
    wb.populate_layers(ctx);
    for (int i = 0; i < kTile * kTile; ++i) out[i] = kIdNone;
    wb.skip_trivial_clips_pass(ctx);
    Color solid;
    if (wb.skip_fully_covered_layers_pass(ctx, &solid) == Workbench::Flow::BreakSolid) {
        for (size_t k = wb.ids.size(); k-- > wb.skipped;)
            if (wb.ids[k].mask) {
                for (int i = 0; i < kTile * kTile; ++i) out[i] = wb.ids[k].id;
                break;
            }
        for (auto& e : wb.ids) {
            CoverCarry cc;
            if (wb.cover_carry(ctx, e.id, &cc)) wb.next_queue.push_back(cc);
        }
        wb.next_tile();
        return;
    }
    for (size_t k = 0; k < wb.ids.size(); ++k) {
        uint32_t id = wb.ids[k].id;
        if (k >= wb.skipped && wb.ids[k].mask) {
            painter.clear_cells();
            if (const Workbench::SegRange* r = wb.segments_of(id))
                for (size_t i = r->first; i <= r->last; ++i) painter.acc_segment(ctx.segs[i]);
            if (const Cover* c = wb.cover(id)) painter.acc_cover(*c);
            const Props& props = ctx.props->get(id);
            bool apply_clip = props.func == kDraw && props.is_clipped && !wb.ids[k].skip_clipping;
            Cover cv = paint_layer_ids(painter, id, props, apply_clip, min_coverage, out);
            if (!cv.is_empty(props.fill_rule)) wb.next_queue.push_back({cv, id});
        } else {
            CoverCarry cc;
            if (wb.cover_carry(ctx, id, &cc)) wb.next_queue.push_back(cc);
        }
    }
    wb.next_tile();
}

// paint_tile_row for an ID frame: `ids` has `stride` bytes per row; only the tiles of the crop
// are written.
inline void paint_tile_row_ids(Painter& painter, Workbench& wb, size_t tile_y, const uint64_t* segs, size_t n,
                               const PropsSource& props, uint32_t* ids, size_t width, size_t height, size_t stride,
                               const Rect* crop, float min_coverage) {
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

    const Channel ch[4] = {kRed, kGreen, kBlue, kAlpha};
    size_t width_in_tiles = (width + kTile - 1) / kTile;
    uint32_t out[kTile * kTile];
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
        painter.clip_active = false;
        drive_tile_ids(wb, painter, ctx, min_coverage, out);
        size_t x0 = tile_x * kTile, y0 = tile_y * kTile;
        for (size_t y = 0; y < (size_t)kTile && y0 + y < height; ++y) {
            uint32_t* row = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(ids) + (y0 + y) * stride);
            for (size_t x = 0; x < (size_t)kTile && x0 + x < width; ++x) row[x0 + x] = out[x * kTile + y];
        }
    }
}

}  // namespace fo
