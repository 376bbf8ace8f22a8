// ORACLE — TEST INFRASTRUCTURE ONLY (see fmath.hpp).
//
// Stage 2 (pixel-grid intersection) and stage 3 (sort). Restates
// forma/src/cpu/rasterizer.rs, forma/src/cpu/pixel_segment.rs and
// forma/src/utils/prefix_scan.rs.
#pragma once

#include <algorithm>
#include <vector>

#include "scene.hpp"

namespace fo {

// consts.rs:68-93 with TW = TH = 16: tile_y 11 | tile_x 12 | layer 21 |
// local_x 4 | local_y 4 | double_area_multiplier 6 | cover 6.
constexpr int kBitsTileY = 11, kBitsTileX = 12, kBitsLayer = 21, kBitsLocalX = 4, kBitsLocalY = 4,
              kBitsDam = 6, kBitsCover = 6;
constexpr int kSortShift = kBitsLocalX + kBitsLocalY + kBitsDam + kBitsCover;  // 20

// pixel_segment.rs:36-71
inline uint64_t pack_segment(uint32_t layer, int16_t tile_x, int16_t tile_y, uint8_t local_x, uint8_t local_y,
                             uint8_t dam, int8_t cover) {
    uint64_t v = 0;
    auto biased = [](int16_t t) -> uint64_t {
        int16_t s = (int16_t)(t + 1);
        return (uint64_t)(int64_t)(s < 0 ? 0 : s);
    };
    v |= ((1ull << kBitsTileY) - 1) & biased(tile_y);
    v <<= kBitsTileX;
    v |= ((1ull << kBitsTileX) - 1) & biased(tile_x);
    v <<= kBitsLayer;
    v |= ((1ull << kBitsLayer) - 1) & (uint64_t)layer;
    v <<= kBitsLocalX;
    v |= ((1ull << kBitsLocalX) - 1) & (uint64_t)local_x;
    v <<= kBitsLocalY;
    v |= ((1ull << kBitsLocalY) - 1) & (uint64_t)local_y;
    v <<= kBitsDam;
    v |= ((1ull << kBitsDam) - 1) & (uint64_t)dam;
    v <<= kBitsCover;
    v |= ((1ull << kBitsCover) - 1) & (uint64_t)(int64_t)cover;
    return v;
}

// pixel_segment.rs:100-138
inline int16_t seg_tile_y(uint64_t s) { return (int16_t)((s >> 53) & 0x7FF) - 1; }
inline int16_t seg_tile_x(uint64_t s) { return (int16_t)((s >> 41) & 0xFFF) - 1; }
inline uint32_t seg_layer(uint64_t s) { return (uint32_t)((s >> 20) & 0x1FFFFF); }
inline uint8_t seg_local_x(uint64_t s) { return (uint8_t)((s >> 16) & 0xF); }
inline uint8_t seg_local_y(uint64_t s) { return (uint8_t)((s >> 12) & 0xF); }
inline uint8_t seg_dam(uint64_t s) { return (uint8_t)((s >> 6) & 0x3F); }
inline int8_t seg_cover(uint64_t s) { return (int8_t)(((int64_t)(s << 58)) >> 58); }
inline int16_t seg_double_area(uint64_t s) { return (int16_t)((int16_t)seg_dam(s) * (int16_t)seg_cover(s)); }

// cpu/rasterizer.rs:32-61
inline float find_param(int32_t i_in, double a_over, double b_over, double cd_over, float a, float b, float c, float d) {
    float i = (float)i_in;
    float ja = std::isfinite(b) ? (float)std::ceil(std::fma(b_over, (double)i, -cd_over)) : i;
    float jb = std::isfinite(a) ? (float)std::ceil(std::fma(a_over, (double)i, cd_over)) : i;
    float guess_a = std::fmaf(a, ja, c);
    float guess_b = std::fmaf(b, jb, d);
    return rmin(guess_a, guess_b);
}

// cpu/rasterizer.rs:63-76
inline void ith_params(uint32_t i_in, float a, float b, float c, float d, float* t0, float* t1) {
    int32_t i = (int32_t)i_in - (c != 0.0f ? 1 : 0) - (d != 0.0f ? 1 : 0);
    double sum_recip = 1.0 / ((double)a + (double)b);
    double a_over = (double)a * sum_recip;
    double b_over = (double)b * sum_recip;
    double cd_over = ((double)c - (double)d) * sum_recip;
    float f0 = find_param(i, a_over, b_over, cd_over, a, b, c, d);
    float f1 = find_param(i + 1, a_over, b_over, cd_over, a, b, c, d);
    *t0 = rmax(f0, 0.0f);
    *t1 = rmin(f1, 1.0f);
}

// cpu/rasterizer.rs:78-80: `(v + 0.5).floor().to_int_unchecked()`, undefined in Rust for NaN and
// values outside i32. The reference's x86 build (cvttss2si) gives i32::MIN for them; so does this,
// explicitly rather than by the same undefined cast in C++.
inline int32_t round_sub(float v) {
    const float f = std::floor(v + 0.5f);
    return (f >= -2147483648.0f && f < 2147483648.0f) ? (int32_t)f : INT32_MIN;
}

// cpu/rasterizer.rs:100-157 — the k-th pixel segment of line `li`.
inline uint64_t pixel_segment(const Lines& L, size_t li, uint32_t k) {
    float t0, t1;
    ith_params(k, L.a[li], L.b[li], L.c[li], L.d[li], &t0, &t1);
    float x0f = std::fmaf(t0, L.dx[li], L.x0[li]);
    float y0f = std::fmaf(t0, L.dy[li], L.y0[li]);
    float x1f = std::fmaf(t1, L.dx[li], L.x0[li]);
    float y1f = std::fmaf(t1, L.dy[li], L.y0[li]);
    int32_t x0s = round_sub(x0f), x1s = round_sub(x1f), y0s = round_sub(y0f), y1s = round_sub(y1f);
    int32_t border_x = std::min(x0s, x1s) >> 4;
    int32_t border_y = std::min(y0s, y1s) >> 4;
    int16_t tile_x = (int16_t)(border_x >> 4);
    int16_t tile_y = (int16_t)(border_y >> 4);
    uint8_t local_x = (uint8_t)(border_x & 15);
    uint8_t local_y = (uint8_t)(border_y & 15);
    int32_t border = (border_x << 4) + 16;
    int32_t height = y1s - y0s;
    uint8_t dam = (uint8_t)(std::abs(x1s - x0s) + 2 * (border - std::max(x0s, x1s)));
    int8_t cover = (int8_t)height;
    return pack_segment(L.orders[li], tile_x, tile_y, local_x, local_y, dam, cover);
}

constexpr uint64_t kSegmentLimit = 0xFFFFFFFFull;  // what u32 prefix sums can index

// cpu/rasterizer.rs:93-159 with utils/prefix_scan.rs:30-63 enumerating
// (line, k) pairs from the inclusive prefix sums. Returns false, with no segments, when the
// true count exceeds kSegmentLimit: the wrapped sums would index past `out`.
inline bool rasterize(const Lines& L, std::vector<uint64_t>& out) {
    size_t n_lines = L.size();
    if (L.total > kSegmentLimit) {
        out.clear();
        return false;
    }
    size_t total = L.total;
    out.resize(total);
#pragma omp parallel for schedule(dynamic, 1024)
    for (size_t li = 0; li < n_lines; ++li) {
        uint32_t excl = li ? L.lengths[li - 1] : 0;
        uint32_t incl = L.lengths[li];
        for (uint32_t s = excl; s < incl; ++s) out[s] = pixel_segment(L, li, s - excl);
    }
    return true;
}

// cpu/rasterizer.rs:162-164 — crumsort is an unstable comparison sort on the
// top 44 bits (pixel_segment.rs:161-171); any sort with that key is a valid
// stand-in. See oracle/README.md ("parity unpinned beyond the invariant").
inline void sort_segments(std::vector<uint64_t>& segs);

}  // namespace fo
