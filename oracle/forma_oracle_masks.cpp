// ORACLE — TEST INFRASTRUCTURE ONLY (see fmath.hpp).
//
// Layer coverage masks of the oracle: fo_renderer_render_masks, the counterpart of
// forma_renderer_render_masks, in a library of its own (libforma_oracle_masks.so, built by
// masks.mk) next to libforma_oracle.so. It works on the compositions libforma_oracle.so builds
// (same headers, same flags, see forma_oracle_ids.cpp). The renderer argument is not used.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "painter_masks.hpp"

namespace fo {

// Zeroes the written rectangle of every plane, then paints the window's orders that exist (planes
// beyond the composition's last order stay 0).
static bool render_masks(Composition& comp, uint8_t* out, uint32_t first, uint32_t count, size_t bpp, size_t width, size_t height,
                         size_t stride, size_t plane_stride, const Rect* crop, size_t* n_lines, size_t* n_segments) {
    size_t wt = (width + kTile - 1) / kTile, ht = (height + kTile - 1) / kTile;
    size_t x0 = crop ? std::min(crop->hor0, wt) * kTile : 0, x1 = std::min((crop ? std::min(crop->hor1, wt) : wt) * kTile, width);
    size_t y0 = crop ? std::min(crop->vert0, ht) * kTile : 0, y1 = std::min((crop ? std::min(crop->vert1, ht) : ht) * kTile, height);
    if (x1 > x0)
        for (uint32_t k = 0; k < count; ++k)
            for (size_t y = y0; y < y1; ++y) std::memset(out + k * plane_stride + y * stride + x0 * bpp, 0, (x1 - x0) * bpp);
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
    if (window.count) {
#pragma omp parallel
        {
            Painter painter;
            Workbench wb;
            std::vector<float> planes;
#pragma omp for schedule(dynamic, 1)
            for (size_t j = 0; j < ht; ++j) {
                if (crop && !(j >= crop->vert0 && j < crop->vert1)) continue;
                paint_tile_row_masks(painter, wb, j, segs + row_start[j], row_start[j + 1] - row_start[j], props, out, width, height,
                                     stride, plane_stride, bpp, crop, window, planes);
            }
        }
    }
    *n_lines = lines.size();
    *n_segments = segments.size();
    return true;
}

}  // namespace fo

using namespace fo;

// Same layouts as forma_rect / forma_timings / forma_masks (include/forma_b200.h).
struct fo_masks_rect {
    uint64_t hor_start, hor_end, vert_start, vert_end;
};
struct fo_masks_timings {
    double line_setup_ms, rasterize_ms, sort_ms, paint_ms;
    uint64_t n_lines, n_segments;
};
struct fo_masks {
    void* ptr;
    uint32_t first_order, n_orders, format;
    uint64_t stride, plane_stride;
};

extern "C" {

// The refusals of forma_renderer_render_masks that apply to a host frame.
int fo_renderer_render_masks(void*, void* cv, const fo_masks* m, uint64_t width, uint64_t height, const fo_masks_rect* crop,
                             fo_masks_timings* timings) {
    if (!m || !m->ptr || m->n_orders == 0 || (uint64_t)m->first_order + m->n_orders > (1ull << 21) || m->format > 1 || width == 0 ||
        height == 0)
        return 1;
    const uint64_t bpp = m->format == 0 ? 4 : 1;
    if (m->stride < bpp * width || m->plane_stride < (height - 1) * m->stride + bpp * width ||
        (bpp == 4 && (((uintptr_t)m->ptr | m->stride | m->plane_stride) & 3u) != 0))
        return 1;
    Rect rect;
    if (crop) {
        rect.hor0 = crop->hor_start / kTile;
        rect.hor1 = (crop->hor_end + kTile - 1) / kTile;
        rect.vert0 = crop->vert_start / kTile;
        rect.vert1 = (crop->vert_end + kTile - 1) / kTile;
    }
    size_t n_lines = 0, n_segments = 0;
    if (!render_masks(*(Composition*)cv, (uint8_t*)m->ptr, m->first_order, m->n_orders, (size_t)bpp, (size_t)width, (size_t)height,
                      (size_t)m->stride, (size_t)m->plane_stride, crop ? &rect : nullptr, &n_lines, &n_segments))
        return 5;  // FORMA_ERR_CAPACITY
    if (timings) {
        *timings = fo_masks_timings{};
        timings->n_lines = n_lines;
        timings->n_segments = n_segments;
    }
    return 0;
}

}  // extern "C"
