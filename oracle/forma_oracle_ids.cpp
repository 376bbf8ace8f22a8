// ORACLE — TEST INFRASTRUCTURE ONLY (see fmath.hpp).
//
// ID frames of the oracle: fo_renderer_render_ids, the counterpart of forma_renderer_render_ids,
// in a library of its own (libforma_oracle_ids.so, built by ids.mk) next to libforma_oracle.so.
// It works on the compositions libforma_oracle.so builds: both are compiled from the same
// headers with the same flags, so a `fo::Composition*` means the same object in either. The
// renderer argument is not used (the ID frame keeps its own segments). Built apart so that the
// RGBA oracle, the timed CPU baseline, stays exactly as it is.
#include <algorithm>
#include <cmath>

#include "painter_ids.hpp"

namespace fo {

static void render_ids(Composition& comp, uint32_t* ids, size_t width, size_t stride, size_t height, const Rect* crop,
                       float min_coverage, size_t* n_lines, size_t* n_segments) {
    size_t ht = (height + kTile - 1) / kTile;
    comp.compact_geom();
    Lines lines;
    std::vector<uint64_t> segments;
    comp.fill_cpu_view(width, height, lines);
    rasterize(lines, segments);
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
            paint_tile_row_ids(painter, wb, j, segs + row_start[j], row_start[j + 1] - row_start[j], props, ids, width, height,
                               stride, crop, min_coverage);
        }
    }
    *n_lines = lines.size();
    *n_segments = segments.size();
}

}  // namespace fo

using namespace fo;

// Same layouts as forma_rect / forma_timings (include/forma_b200.h) and forma_oracle.cpp's.
struct fo_ids_rect {
    uint64_t hor_start, hor_end, vert_start, vert_end;
};
struct fo_ids_timings {
    double line_setup_ms, rasterize_ms, sort_ms, paint_ms;
    uint64_t n_lines, n_segments;
};

extern "C" {

int fo_renderer_render_ids(void*, void* cv, uint32_t* ids, uint64_t width, uint64_t stride, uint64_t height,
                           const fo_ids_rect* crop, float min_coverage, fo_ids_timings* timings) {
    if (!ids || width * 4 > stride || stride % 4 != 0 || !std::isfinite(min_coverage) || min_coverage < 0.0f ||
        min_coverage >= 1.0f)
        return 1;
    Rect rect;
    if (crop) {
        rect.hor0 = crop->hor_start / kTile;
        rect.hor1 = (crop->hor_end + kTile - 1) / kTile;
        rect.vert0 = crop->vert_start / kTile;
        rect.vert1 = (crop->vert_end + kTile - 1) / kTile;
    }
    size_t n_lines = 0, n_segments = 0;
    render_ids(*(Composition*)cv, ids, (size_t)width, (size_t)stride, (size_t)height, crop ? &rect : nullptr, min_coverage,
               &n_lines, &n_segments);
    if (timings) {
        *timings = fo_ids_timings{};
        timings->n_lines = n_lines;
        timings->n_segments = n_segments;
    }
    return 0;
}

}  // extern "C"
