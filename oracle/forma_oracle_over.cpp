// ORACLE — TEST INFRASTRUCTURE ONLY (see fmath.hpp).
//
// Frames over a background: fo_renderer_render_over, the counterpart of
// forma_renderer_render_over_device for FORMA_PIXEL_SRGB8 and FORMA_PIXEL_RGBA32F on host memory,
// and fo_srgb_decode_table, the decode table D it shares with the paint kernels. A library of its
// own (libforma_oracle_over.so, built by over.mk) next to libforma_oracle.so, working on the
// compositions that library builds, like libforma_oracle_linear.so. The renderer argument is not
// used. Built apart so that the RGBA oracle, the timed CPU baseline, stays exactly as it is.
#include <algorithm>

#include "painter_over.hpp"

namespace fo {

static bool render_over(Composition& comp, uint8_t* frame, size_t bpp, size_t width, size_t stride, size_t height, const Channel ch[4],
                        const Rect* crop, size_t* n_lines, size_t* n_segments) {
    size_t ht = (height + kTile - 1) / kTile;
    comp.compact_geom();
    Lines lines;
    std::vector<uint64_t> segments;
    comp.fill_cpu_view(width, height, lines);
    if (!rasterize(lines, segments)) return false;  // more pixel segments than u32 sums can index
    std::sort(segments.begin(), segments.end(), [](uint64_t a, uint64_t b) { return (a >> kSortShift) < (b >> kSortShift); });
    PropsSource props;
    props.index(comp.layers);
    const uint64_t* segs = segments.data();
    size_t n = segments.size();
    size_t first = std::partition_point(segs, segs + n, [](uint64_t s) { return seg_tile_y(s) < 0; }) - segs;
    std::vector<size_t> row_start(ht + 1);
    for (size_t j = 0; j <= ht; ++j) {
        row_start[j] = std::partition_point(segs + first, segs + n, [j](uint64_t s) { return (size_t)seg_tile_y(s) < j; }) - segs;
    }
#pragma omp parallel
    {
        Painter painter;
        Workbench wb;
#pragma omp for schedule(dynamic, 1)
        for (size_t j = 0; j < ht; ++j) {
            if (crop && !(j >= crop->vert0 && j < crop->vert1)) continue;
            paint_tile_row_over(painter, wb, j, segs + row_start[j], row_start[j + 1] - row_start[j], props, ch, frame, bpp, width,
                                height, stride, crop);
        }
    }
    *n_lines = lines.size();
    *n_segments = segments.size();
    return true;
}

}  // namespace fo

using namespace fo;

// Same layouts as forma_rect / forma_timings (include/forma_b200.h) and forma_oracle.cpp's.
struct fo_over_rect {
    uint64_t hor_start, hor_end, vert_start, vert_end;
};
struct fo_over_timings {
    double line_setup_ms, rasterize_ms, sort_ms, paint_ms;
    uint64_t n_lines, n_segments;
};

extern "C" {

// format 0 (FORMA_PIXEL_SRGB8) or 2 (FORMA_PIXEL_RGBA32F); channels a permutation of R, G, B, A.
int fo_renderer_render_over(void*, void* cv, void* buffer, uint64_t width, uint64_t stride, uint64_t height, const uint32_t channels[4],
                            const fo_over_rect* crop, uint32_t format, fo_over_timings* timings) {
    const size_t bpp = format == 0u ? 4 : format == 2u ? 16 : 0;
    if (!buffer || !bpp || width * bpp > stride || stride % 4 != 0) return 1;
    Channel ch[4];
    bool seen[4] = {false, false, false, false};
    for (int k = 0; k < 4; ++k) {
        if (channels[k] > kAlpha || seen[channels[k]]) return 1;
        seen[channels[k]] = true;
        ch[k] = (Channel)channels[k];
    }
    Rect rect;
    if (crop) {
        rect.hor0 = crop->hor_start / kTile;
        rect.hor1 = (crop->hor_end + kTile - 1) / kTile;
        rect.vert0 = crop->vert_start / kTile;
        rect.vert1 = (crop->vert_end + kTile - 1) / kTile;
    }
    size_t n_lines = 0, n_segments = 0;
    if (!render_over(*(Composition*)cv, (uint8_t*)buffer, bpp, (size_t)width, (size_t)stride, (size_t)height, ch, crop ? &rect : nullptr,
                     &n_lines, &n_segments))
        return 5;  // FORMA_ERR_CAPACITY
    if (timings) {
        *timings = fo_over_timings{};
        timings->n_lines = n_lines;
        timings->n_segments = n_segments;
    }
    return 0;
}

// The sRGB8 decode table D (forma_b200/csrc/srgb_decode.h) as the oracle and the kernels see it.
void fo_srgb_decode_table(float out[256]) { std::copy(kSrgbDecode, kSrgbDecode + 256, out); }

}  // extern "C"
