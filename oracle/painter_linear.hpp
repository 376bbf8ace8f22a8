// ORACLE — TEST INFRASTRUCTURE ONLY (see fmath.hpp).
//
// Linear float frames: the painter walk of painter.hpp without the sRGB encode. A tile folded to
// one colour yields its Color, a painted tile leaves its planes in the Painter. Free functions
// over the painter's own types, so that painter.hpp and the RGBA path built from it stay exactly
// as they are.
#pragma once

#include "painter.hpp"

namespace fo {

// Workbench::drive_tile_painting without a layer cache (tile_unchanged_pass changes nothing and
// no tile is left alone). Returns true with the folded colour in *solid when
// skip_fully_covered_layers folds the tile; false when the tile is painted into the painter's
// planes (red, green, blue, alpha: what compute_srgb would encode).
inline bool drive_tile_linear(Workbench& wb, Painter& painter, const TileContext& ctx, Color* solid) {
    wb.populate_layers(ctx);
    wb.skip_trivial_clips_pass(ctx);
    if (wb.skip_fully_covered_layers_pass(ctx, solid) == Workbench::Flow::BreakSolid) {
        for (auto& e : wb.ids) {
            CoverCarry cc;
            if (wb.cover_carry(ctx, e.id, &cc)) wb.next_queue.push_back(cc);
        }
        wb.next_tile();
        return true;
    }
    painter.clear(ctx.clear_color);
    for (size_t k = 0; k < wb.ids.size(); ++k) {
        uint32_t id = wb.ids[k].id;
        if (k >= wb.skipped && wb.ids[k].mask) {
            painter.clear_cells();
            if (const Workbench::SegRange* r = wb.segments_of(id))
                for (size_t i = r->first; i <= r->last; ++i) painter.acc_segment(ctx.segs[i]);
            if (const Cover* c = wb.cover(id)) painter.acc_cover(*c);
            const Props& props = ctx.props->get(id);
            bool apply_clip = props.func == kDraw && props.is_clipped && !wb.ids[k].skip_clipping;
            Cover out = painter.paint_layer(ctx.tile_x, ctx.tile_y, id, props, apply_clip);
            if (!out.is_empty(props.fill_rule)) wb.next_queue.push_back({out, id});
        } else {
            CoverCarry cc;
            if (wb.cover_carry(ctx, id, &cc)) wb.next_queue.push_back(cc);
        }
    }
    wb.next_tile();
    return false;
}

// paint_tile_row for a linear frame: `out` has `stride` bytes per row and four f32 per pixel in
// the order of `ch` (kZero 0, kOne 1); only the tiles of the crop are written.
inline void paint_tile_row_linear(Painter& painter, Workbench& wb, size_t tile_y, const uint64_t* segs, size_t n,
                                  const PropsSource& props, const Channel ch[4], const Color& clear_color, float* out, size_t width,
                                  size_t height, size_t stride, const Rect* crop) {
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

    size_t width_in_tiles = (width + kTile - 1) / kTile;
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
        ctx.clear_color = clear_color;
        painter.clip_active = false;
        Color solid;
        const bool folded = drive_tile_linear(wb, painter, ctx, &solid);
        size_t x0 = tile_x * kTile, y0 = tile_y * kTile;
        for (size_t y = 0; y < (size_t)kTile && y0 + y < height; ++y) {
            float* row = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(out) + (y0 + y) * stride);
            for (size_t x = 0; x < (size_t)kTile && x0 + x < width; ++x) {
                const size_t i = x * kTile + y;
                const Color c = folded ? solid : Color{painter.red[i], painter.green[i], painter.blue[i], painter.alpha[i]};
                for (int k = 0; k < 4; ++k) row[(x0 + x) * 4 + k] = color_channel(c, ch[k]);
            }
        }
    }
}

}  // namespace fo
