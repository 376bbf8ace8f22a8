// ORACLE — TEST INFRASTRUCTURE ONLY (see fmath.hpp).
//
// Frames over a background: the painter walk of painter.hpp with a clear colour per pixel, the
// pixel's own decoded value. painter.clear per pixel; skip_fully_covered_layers' fold per pixel
// from the pixel's colour (or once from an opaque bottom layer, which does not depend on it); the
// Alpha -> One upgrade per pixel where the decoded alpha is 1. Every tile of the crop is written
// as the RGBA path writes it (a solid tile by position through to_srgb_bytes, a painted tile
// through compute_srgb), so that the device's choice not to write tiles without entries is
// checked against the bytes those tiles would get. Free functions over the painter's own types,
// so that painter.hpp and the RGBA path built from it stay exactly as they are.
#pragma once

#include "../forma_b200/csrc/srgb_decode.h"
#include "painter.hpp"

namespace fo {

static const float kSrgbDecode[256] = FORMA_SRGB_DECODE_TABLE;

// sRGB8 decode of one channel's byte: alpha as byte / 255, a colour channel through D.
inline float decode_srgb8(uint8_t b, Channel c) { return c == kAlpha ? (float)b / 255.0f : kSrgbDecode[b]; }

// skip_fully_covered_layers_pass (passes/skip_fully_covered_layers.rs:27-119) with a clear colour per
// pixel, for a tile without a layer cache. Returns true when the tile folds: every visible layer
// is full and solid; then *opaque tells whether an opaque layer is the bottom (its colour in
// *bottom) or the pixels' own colours are, and *first the first entry the fold blends.
inline bool fold_over(Workbench& wb, const TileContext& ctx, bool* opaque, Color* bottom, size_t* first, size_t* skip_n) {
    enum { kNoneYet, kOpaque, kIncomplete } state = kNoneYet;
    for (size_t k = wb.ids.size(); k-- > wb.skipped;) {
        if (!wb.ids[k].mask) continue;
        uint32_t id = wb.ids[k].id;
        const Props& props = ctx.props->get(id);
        bool is_clipped = props.func == kDraw && props.is_clipped && !wb.ids[k].skip_clipping;
        if (is_clipped || !wb.layer_is_full(id, props.fill_rule)) {
            if (state == kNoneYet) state = kIncomplete;
        } else if (props.func == kDraw && props.fill_type == kSolid && props.blend_mode == kOver) {
            if (props.color.a == 1.0f) {
                if (state == kNoneYet) {
                    state = kOpaque;
                    *bottom = props.color;
                }
                wb.skipped = k;
                break;
            }
        }
    }
    if (state == kIncomplete) return false;
    *opaque = state == kOpaque;
    *skip_n = *opaque ? 1 : 0;
    *first = wb.skipped;
    size_t seen = 0;
    for (size_t k = wb.skipped; k < wb.ids.size(); ++k) {
        if (!wb.ids[k].mask) continue;
        if (seen++ < *skip_n) continue;
        const Props& props = ctx.props->get(wb.ids[k].id);
        if (!(props.func == kDraw && props.fill_type == kSolid)) return false;
    }
    return true;
}

// The folded colour of one pixel whose clear colour is `clear`.
inline Color fold_pixel(const Workbench& wb, const TileContext& ctx, Color dst, size_t first, size_t skip_n) {
    size_t seen = 0;
    for (size_t k = first; k < wb.ids.size(); ++k) {
        if (!wb.ids[k].mask) continue;
        if (seen++ < skip_n) continue;
        const Props& props = ctx.props->get(wb.ids[k].id);
        dst = scalar_blend::blend(props.blend_mode, dst, props.color);
    }
    return dst;
}

// One tile over its background bg (256 colours, index x * 16 + y as the painter's planes). Fills
// out_color (per pixel, linear) and solid (true: the tile folded, written by position as a solid
// tile; false: painted, written per channel by compute_srgb).
inline void drive_tile_over(Workbench& wb, Painter& painter, const TileContext& ctx, const Color* bg, Color* out_color, bool* solid) {
    wb.populate_layers(ctx);
    wb.skip_trivial_clips_pass(ctx);
    bool opaque = false;
    Color bottom;
    size_t first = 0, skip_n = 0;
    if (fold_over(wb, ctx, &opaque, &bottom, &first, &skip_n)) {
        const Color once = opaque ? fold_pixel(wb, ctx, bottom, first, skip_n) : Color();
        for (int i = 0; i < kTile * kTile; ++i) out_color[i] = opaque ? once : fold_pixel(wb, ctx, bg[i], first, skip_n);
        for (auto& e : wb.ids) {
            CoverCarry cc;
            if (wb.cover_carry(ctx, e.id, &cc)) wb.next_queue.push_back(cc);
        }
        wb.next_tile();
        *solid = true;
        return;
    }
    for (int i = 0; i < kTile * kTile; ++i) {  // painter.clear, per pixel
        painter.red[i] = bg[i].r;
        painter.green[i] = bg[i].g;
        painter.blue[i] = bg[i].b;
        painter.alpha[i] = bg[i].a;
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
            Cover out = painter.paint_layer(ctx.tile_x, ctx.tile_y, id, props, apply_clip);
            if (!out.is_empty(props.fill_rule)) wb.next_queue.push_back({out, id});
        } else {
            CoverCarry cc;
            if (wb.cover_carry(ctx, id, &cc)) wb.next_queue.push_back(cc);
        }
    }
    wb.next_tile();
    for (int i = 0; i < kTile * kTile; ++i) out_color[i] = Color{painter.red[i], painter.green[i], painter.blue[i], painter.alpha[i]};
    *solid = false;
}

// paint_tile_row over a background: `frame` (bpp 4: sRGB8 bytes, 16: f32) is read for each tile's
// background and then written with its result; only the tiles of the crop.
inline void paint_tile_row_over(Painter& painter, Workbench& wb, size_t tile_y, const uint64_t* segs, size_t n, const PropsSource& props,
                                const Channel ch[4], uint8_t* frame, size_t bpp, size_t width, size_t height, size_t stride,
                                const Rect* crop) {
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

    Color bg[kTile * kTile], out[kTile * kTile];
    size_t width_in_tiles = (width + kTile - 1) / kTile;
    for (size_t tile_x = 0; tile_x < width_in_tiles; ++tile_x) {
        if (crop && !(tile_x >= crop->hor0 && tile_x < crop->hor1)) continue;
        size_t begin = pos;
        while (pos < n && seg_tile_x(segs[pos]) == (int16_t)tile_x) ++pos;
        size_t x0 = tile_x * kTile, y0 = tile_y * kTile;
        for (size_t y = 0; y < (size_t)kTile; ++y) {
            for (size_t x = 0; x < (size_t)kTile; ++x) {
                Color& c = bg[x * kTile + y];
                c = Color();
                if (x0 + x >= width || y0 + y >= height) continue;
                const uint8_t* px = frame + (y0 + y) * stride + (x0 + x) * bpp;
                float v[4];
                for (int k = 0; k < 4; ++k) {
                    if (bpp == 4) {
                        v[k] = decode_srgb8(px[k], ch[k]);
                    } else {
                        std::memcpy(&v[k], px + 4 * k, 4);
                    }
                }
                for (int k = 0; k < 4; ++k) {
                    switch (ch[k]) {
                        case kRed: c.r = v[k]; break;
                        case kGreen: c.g = v[k]; break;
                        case kBlue: c.b = v[k]; break;
                        default: c.a = v[k]; break;
                    }
                }
            }
        }
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
        bool solid = false;
        drive_tile_over(wb, painter, ctx, bg, out, &solid);
        for (size_t y = 0; y < (size_t)kTile && y0 + y < height; ++y) {
            for (size_t x = 0; x < (size_t)kTile && x0 + x < width; ++x) {
                const size_t i = x * kTile + y;
                Channel pc[4];  // renderer.rs:87-92 with this pixel's clear colour
                for (int k = 0; k < 4; ++k) pc[k] = bg[i].a == 1.0f && ch[k] == kAlpha ? kOne : ch[k];
                uint8_t* px = frame + (y0 + y) * stride + (x0 + x) * bpp;
                if (bpp == 16) {
                    for (int k = 0; k < 4; ++k) {
                        const float v = color_channel(out[i], pc[k]);
                        std::memcpy(px + 4 * k, &v, 4);
                    }
                } else if (solid) {  // to_srgb_bytes by position, as drive_tile_painting writes a solid tile
                    float sel[4];
                    for (int k = 0; k < 4; ++k) sel[k] = color_channel(out[i], pc[k]);
                    to_srgb_bytes(sel, px);
                } else {  // compute_srgb: colour channels encoded, alpha / ZERO / ONE not
                    const Color s{linear_to_srgb(out[i].r), linear_to_srgb(out[i].g), linear_to_srgb(out[i].b), out[i].a};
                    for (int k = 0; k < 4; ++k) px[k] = to_byte(color_channel(s, pc[k]));
                }
            }
        }
    }
}

}  // namespace fo
