// ORACLE — TEST INFRASTRUCTURE ONLY (see fmath.hpp).
//
// Layer coverage masks: the painter walk of painter.hpp (Workbench passes, Painter cells and clip
// state) recording each layer's coverage x clip mask instead of blending. Free functions over the
// painter's own types, so that painter.hpp and the RGBA path built from it stay exactly as they are.
// Every layer of a tile is painted: skip_trivial_clips decides which clips are painted and which
// clipped layers keep their clip, as in the painter, but no layer is skipped below an opaque one.
#pragma once

#include "painter.hpp"

namespace fo {

// The window of layer orders a mask frame holds, and its planes for one tile: plane k of the
// window at planes + k * 256, column-major like the colour planes.
struct MaskWindow {
    uint32_t first, count;
    bool holds(uint32_t id) const { return id >= first && id - first < count; }
};

// Painter::paint_layer without colour arithmetic: the layer's coverage (x the clip mask where a
// clip applies to it) into `plane` (may be null), with the same clip state and returned cover as
// paint_layer. A Draw layer writes only the f32x8 groups paint_layer blends (the others are 0); a
// clip layer (paint_clip = true) updates the clip state and writes its coverage everywhere.
// paint_clip = false: a clip the skip pass masks out: its coverage only, no clip state.
inline Cover paint_layer_masks(Painter& p, uint32_t layer_id, const Props& props, bool apply_clip, bool paint_clip, float* plane) {
    int8_t run[kTile] = {0};
    if (paint_clip && p.clip_active && p.clip_last < layer_id) p.clip_active = false;
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
                        if (plane) plane[base + l] = f;
                    }
                } else {
                    if (paint_clip) {  // clip_at, cpu/painter/mod.rs:449-464
                        if (!p.clip_active) {
                            p.clip_active = true;
                            for (float& m : p.clip_mask) m = 0.0f;
                            p.clip_last = layer_id + props.clip_layers;
                        }
                        for (int l = 0; l < 8; ++l) p.clip_mask[base + l] = cov[l];
                    }
                    if (plane)
                        for (int l = 0; l < 8; ++l) plane[base + l] = cov[l];
                }
            }
        }
        for (int y = 0; y < kTile; ++y) run[y] = (int8_t)(run[y] + p.covers[x * kTile + y]);
    }
    Cover out;
    std::memcpy(out.c, run, sizeof(run));
    return out;
}

// Workbench::drive_tile_painting for a mask frame (no layer cache): populate_layers and
// skip_trivial_clips, then every layer bottom-up. `planes` (window.count x 256, zeroed by the
// caller) receives the window's layers.
inline void drive_tile_masks(Workbench& wb, Painter& painter, const TileContext& ctx, const MaskWindow& window, float* planes) {
    wb.populate_layers(ctx);
    wb.skip_trivial_clips_pass(ctx);
    painter.clip_active = false;
    for (size_t k = 0; k < wb.ids.size(); ++k) {
        const uint32_t id = wb.ids[k].id;
        const Props& props = ctx.props->get(id);
        const bool is_clip = props.func != kDraw;
        float* plane = window.holds(id) ? planes + (size_t)(id - window.first) * (kTile * kTile) : nullptr;
        if (wb.ids[k].mask || (is_clip && plane)) {
            painter.clear_cells();
            if (const Workbench::SegRange* r = wb.segments_of(id))
                for (size_t i = r->first; i <= r->last; ++i) painter.acc_segment(ctx.segs[i]);
            if (const Cover* c = wb.cover(id)) painter.acc_cover(*c);
            const bool apply_clip = !is_clip && props.is_clipped && !wb.ids[k].skip_clipping;
            Cover cv = paint_layer_masks(painter, id, props, apply_clip, wb.ids[k].mask, plane);
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

// paint_tile_row for a mask frame: `out` holds window.count planes `plane_stride` bytes apart, rows
// `stride` bytes apart, of `bpp` bytes per value (4: f32, 1: compute_srgb's alpha byte); only the
// tiles of the crop are written.
inline void paint_tile_row_masks(Painter& painter, Workbench& wb, size_t tile_y, const uint64_t* segs, size_t n,
                                 const PropsSource& props, uint8_t* out, size_t width, size_t height, size_t stride,
                                 size_t plane_stride, size_t bpp, const Rect* crop, const MaskWindow& window,
                                 std::vector<float>& planes) {
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
    planes.assign((size_t)window.count * kTile * kTile, 0.0f);
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
        std::fill(planes.begin(), planes.end(), 0.0f);
        drive_tile_masks(wb, painter, ctx, window, planes.data());
        size_t x0 = tile_x * kTile, y0 = tile_y * kTile;
        for (uint32_t k = 0; k < window.count; ++k) {
            const float* src = planes.data() + (size_t)k * kTile * kTile;
            for (size_t y = 0; y < (size_t)kTile && y0 + y < height; ++y) {
                uint8_t* row = out + k * plane_stride + (y0 + y) * stride;
                for (size_t x = 0; x < (size_t)kTile && x0 + x < width; ++x) {
                    const float v = src[x * kTile + y];
                    if (bpp == 4) std::memcpy(row + (x0 + x) * 4, &v, 4);
                    else row[x0 + x] = to_byte(v);
                }
            }
        }
    }
}

}  // namespace fo
