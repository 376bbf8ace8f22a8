// POD records shared between the host side and the CUDA kernels.
#pragma once

#include <cstdint>
#include <vector>

namespace forma {

// --- pixel-segment bit layout (forma/src/consts.rs:68-93, TW = TH = 16) -----
//   63..53 tile_y(11, bias 1) | 52..41 tile_x(12, bias 1) | 40..20 layer(21) |
//   19..16 local_x | 15..12 local_y | 11..6 double_area_multiplier | 5..0 cover
constexpr int kSortShift = 20;   // ordering ignores the low 20 bits (pixel_segment.rs:161-171)
constexpr int kTile = 16;
constexpr uint32_t kLayerLimit = (1u << 21) - 1;

// One quadratic of a flatten program (path.rs:190-204: Primitives SoA, gathered).
struct QuadRec {
    float px[3], py[3], pw[3];  // control points, pre-multiplied by their weights
    float x0, dx_recip, k0, dk, curv_recip;
    float prev_curv;  // running curvature of the previous quad iff same spline, else 0 (path.rs:508-514)
    float total;      // running curvature of the spline including this quad
    float step;       // curvature / subdivisions of the spline (same for all its quads)
};

// What crosses PCIe per quadratic (48 B): the control points and the running
// curvatures of its spline; quad_expand_kernel rebuilds the full QuadRec on the
// device (the Levien parameters are recomputed there, quad_math.h).
struct QuadUp {
    float px[3], py[3], pw[3];
    float prev_curv, total, step;
};
// The same without weights (36 B), used when no quadratic of the uploaded batch is
// rational (all weights are exactly 1: SVG-like content).
struct QuadUpPoly {
    float px[3], py[3];
    float prev_curv, total, step;
};

// Point-wise encoding of a flatten program, used instead of SplineRecs when it
// is smaller (paths made of many short line splines): 8 B + 1 B per output point.
//   kind 0: literal point (a, b)                  (Start / End of a spline)
//   kind 1: literal point (a, b), ends a contour  (End with new_contour)
//   kind 2: a = quad index (u32 bits), b = pi; evaluated at quad.step * pi
//   kind 3: a = quad index (u32 bits), b = fma(step, pi, -quad.prev_curv) with the step of the
//           spline being walked, which need not be the quad's own (programs whose quad walk
//           falls behind, see host_path.cpp)
struct PointRec {
    float a, b;
};

// One spline of a flatten program: the point commands populate_buffers
// (path.rs:400-445) emits for it, in closed form. Its output points are
//   [p0 if it emits a start point] ++ [quads evaluated at step * pi, pi = 1..E] ++ [p2]
// (path.rs:138-168 PointCommand::Start / Incr / End); the quad of evaluated
// point pi is the first one whose running curvature reaches pi.
struct SplineRec {
    float p0x, p0y, p2x, p2y;
    float step;            // curvature / subdivisions
    uint32_t first_quad;   // program-relative
    uint32_t n_quads;
    uint32_t first_point;  // program-relative index of the spline's first output point
    uint32_t info;         // E (= subdivisions - 1, or 0) | emits its start point << 30 | ends a contour << 31
};
constexpr uint32_t kSplineEvalMask = (1u << 30) - 1u;

struct FlattenProgram {
    std::vector<QuadRec> quads;
    std::vector<SplineRec> splines;  // spline encoding (points / kinds empty) ...
    std::vector<PointRec> points;    // ... or point encoding (splines empty), whichever is smaller
    std::vector<uint8_t> kinds;
    bool rational = false;        // some quadratic has a weight != 1
    uint32_t n_points = 0;        // output points
    uint32_t n_contour_ends = 0;  // points that end a contour, the last point of the program excluded
    // Bounds of every point the program can emit: its literal points and the (projected)
    // control points of its quadratics, whose convex hull contains the evaluated points.
    // bounded == false when a weight is not positive (no hull property): never filter then.
    bool bounded = true;
    float min_x = 0.0f, min_y = 0.0f, max_x = 0.0f, max_y = 0.0f;
};

// A batch entry of flatten_eval_kernel: points [first, first+count) of the
// batch belong to this insert job (Layer::insert, composition/layer.rs:90-111).
struct FlattenJob {          // 24 B per Layer::insert of an uploaded batch
    uint32_t first_point;   // first output point of the job in the batch = its offset in the destination; the job's
                            // point count is the next job's first_point (the batch's point count for the last) minus this
    uint32_t quad_base;     // added to SplineRec::first_quad
    uint32_t spline_base;   // the job's splines in the batch's SplineRec array, or its first PointRec
    uint32_t n_splines;     // 0 = point encoding
    uint32_t geom_id;       // id written for non-contour-end points (0 = None)
    uint32_t xf_index;      // 1 + index of the insert's transform in the batch's JobXf array; 0 = none
};
// GeomPresTransform of an insert whose path carries one (path.rs:689-706): ux, uy, vx, vy, tx, ty.
struct JobXf {
    float xf[6];
};

// Per-layer record used by line setup (composition/layer.rs:27-31 InnerLayer).
struct LayerRec {
    uint32_t order;
    uint32_t enabled;
    uint32_t has_xf;
    float ux, uy, vx, vy, tx, ty;
};

// Per-layer style record used by the painter (styling.rs:397-442 Props, flattened).
struct StyleRec {
    uint32_t fill_rule;     // 0 NonZero, 1 EvenOdd
    uint32_t func;          // 0 Draw, 1 Clip
    uint32_t clip_layers;
    uint32_t is_clipped;
    uint32_t blend_mode;
    uint32_t fill_type;     // 0 solid, 1 gradient, 2 texture
    float color[4];
    uint32_t gradient_type; // 0 linear, 1 radial
    float start[2], end[2];
    uint32_t stop_first, stop_count;  // into the stops array
    // texture
    float tex_xf[6];        // ux, uy, vx, vy, tx, ty
    float tex_max_x, tex_max_y;
    uint32_t tex_width;
    uint32_t tex_first;     // into the texel array (4 x u16 per texel)
    uint32_t unchanged;     // Layer::is_unchanged(cache_id) for the cache in use
};

struct StopRec {
    float color[4];
    float stop;
};

// A gradient of at most four stops, ready for the painter (built on the device from the
// StyleRec and its stops whenever the tables are uploaded): the per-gradient terms of
// Gradient::get_t and color_at (cpu/painter/styling.rs:59-143) that do not depend on the pixel.
struct GradRec {  // 128 B: one float per lane of a warp
    float sx, sy, dx, dy;   // start, end - start
    float dot_recip;        // (dx * dx + dy * dy).recip()
    uint32_t type;          // 0 linear, 1 radial
    uint32_t count;         // stops (2..4); 0xFFFFFFFF = not a small gradient
    uint32_t pad;
    float color[4][4];      // stop colours; entries past the last stop repeat it
    float stop[4];
    float rcp_d[4];         // [i - 1] = (stop[i] - start_stop).recip(), start_stop = 0 for i = 1, else stop[i - 1]
};

}  // namespace forma
