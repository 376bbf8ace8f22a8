// ORACLE — TEST INFRASTRUCTURE ONLY (see fmath.hpp).
//
// Linear float frames of the oracle: fo_renderer_render_linear, the counterpart of
// forma_renderer_render_linear for FORMA_PIXEL_RGBA32F, and fo_linear_to_srgb8, compute_srgb's
// encode of such a frame (which ties it to the sRGB8 frames of libforma_oracle.so). A library of
// its own (libforma_oracle_linear.so, built by linear.mk) next to libforma_oracle.so, working on
// the compositions that library builds, like libforma_oracle_ids.so. The renderer argument is not
// used. Built apart so that the RGBA oracle, the timed CPU baseline, stays exactly as it is.
#include <algorithm>

#include "painter_linear.hpp"

namespace fo {

static bool render_linear(Composition& comp, float* out, size_t width, size_t stride, size_t height, const Channel ch[4],
                          const Color& clear_color, const Rect* crop, size_t* n_lines, size_t* n_segments) {
    size_t ht = (height + kTile - 1) / kTile;
    comp.compact_geom();
    Lines lines;
    std::vector<uint64_t> segments;
    comp.fill_cpu_view(width, height, lines);
    if (!rasterize(lines, segments)) return false;  // more pixel segments than u32 sums can index
    // By key only, like the reference's sort: the order inside a key does not change the painter's
    // wrapping sums.
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
            paint_tile_row_linear(painter, wb, j, segs + row_start[j], row_start[j + 1] - row_start[j], props, ch, clear_color, out,
                                  width, height, stride, crop);
        }
    }
    *n_lines = lines.size();
    *n_segments = segments.size();
    return true;
}

}  // namespace fo

using namespace fo;

// Same layouts as forma_rect / forma_timings (include/forma_b200.h) and forma_oracle.cpp's.
struct fo_linear_rect {
    uint64_t hor_start, hor_end, vert_start, vert_end;
};
struct fo_linear_timings {
    double line_setup_ms, rasterize_ms, sort_ms, paint_ms;
    uint64_t n_lines, n_segments;
};

extern "C" {

// format must be 2 (FORMA_PIXEL_RGBA32F): the oracle's frames are f32.
int fo_renderer_render_linear(void*, void* cv, void* buffer, uint64_t width, uint64_t stride, uint64_t height,
                              const uint32_t channels[4], const float clear[4], const fo_linear_rect* crop, uint32_t format,
                              fo_linear_timings* timings) {
    if (!buffer || format != 2u || width * 16 > stride || stride % 4 != 0) return 1;
    Channel ch[4];
    for (int k = 0; k < 4; ++k) {
        if (channels[k] > kOne) return 1;
        ch[k] = (Channel)channels[k];
        if (clear[3] == 1.0f && ch[k] == kAlpha) ch[k] = kOne;  // cpu/renderer.rs:87-92
    }
    Rect rect;
    if (crop) {
        rect.hor0 = crop->hor_start / kTile;
        rect.hor1 = (crop->hor_end + kTile - 1) / kTile;
        rect.vert0 = crop->vert_start / kTile;
        rect.vert1 = (crop->vert_end + kTile - 1) / kTile;
    }
    size_t n_lines = 0, n_segments = 0;
    if (!render_linear(*(Composition*)cv, (float*)buffer, (size_t)width, (size_t)stride, (size_t)height, ch,
                       Color{clear[0], clear[1], clear[2], clear[3]}, crop ? &rect : nullptr, &n_lines, &n_segments))
        return 5;  // FORMA_ERR_CAPACITY
    if (timings) {
        *timings = fo_linear_timings{};
        timings->n_lines = n_lines;
        timings->n_segments = n_segments;
    }
    return 0;
}

// compute_srgb's encode (cpu/painter/mod.rs:466-483) of a linear f32 frame whose four values per
// pixel are in the order of `channels`: a colour channel's value goes through linear_to_srgb,
// alpha, ZERO and ONE do not, and every value is rounded to a byte by to_byte. Rows are `stride`
// bytes apart in `frame` and `out_stride` bytes apart in `out` (4 bytes per pixel).
void fo_linear_to_srgb8(const float* frame, uint64_t width, uint64_t stride, uint64_t height, const uint32_t channels[4], uint8_t* out,
                        uint64_t out_stride) {
    for (uint64_t y = 0; y < height; ++y) {
        const float* src = reinterpret_cast<const float*>(reinterpret_cast<const uint8_t*>(frame) + y * stride);
        uint8_t* dst = out + y * out_stride;
        for (uint64_t i = 0; i < 4 * width; ++i) {
            const uint32_t c = channels[i % 4];
            dst[i] = to_byte(c == kRed || c == kGreen || c == kBlue ? linear_to_srgb(src[i]) : src[i]);
        }
    }
}

}  // extern "C"
