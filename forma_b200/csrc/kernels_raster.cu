// Stage 1 (point evaluation), stage 1½ (per-frame line setup) and stage 2
// (pixel-grid intersection) kernels.
//
//   flatten_eval_kernel   <- path.rs:487-534 (one thread per output point)
//   line_count_kernel     <- segment.rs:298-383 (lengths only) — pass 1
//   scan_block_sums       <- segment.rs:90-98 prefix_sum (device-wide, exclusive)
//   raster_emit_kernel    <- segment.rs:298-383 + cpu/rasterizer.rs:93-159 — pass 2
//
// The reference materialises a 40 B/line SoA between line setup and
// rasterization and finds each pixel segment's line with a binary search over
// the prefix sums (utils/prefix_scan.rs). Here both stages are fused: the line
// parameters live in shared memory for the 256 lines of a CTA and the CTA's
// threads share out the block's pixel segments evenly (bisection over the block's
// prefix of line lengths), so global traffic is 12 B/point in (twice) and
// 8 B/segment out, emitted in exactly the reference's (line, k) order with
// coalesced stores.
#include "cuda_common.cuh"
#include "kernels.h"
#include "quad_math.h"

namespace forma {

// ---------------------------------------------------------------------------
// Stage 1: flatten point evaluation
// ---------------------------------------------------------------------------
__device__ __forceinline__ float inv_curvature(float k) {  // path.rs:53-56
    const float c = 0.39f;
    return k * (1.0f - c + sqrtf(fmaf(k * k, 0.25f, c * c)));
}

// QuadUp (48 B, uploaded) -> QuadRec (68 B, device only): the Levien parameters are
// recomputed with the host's own formulas (quad_math.h).
__global__ void quad_expand_kernel(const QuadUp* __restrict__ in, QuadRec* __restrict__ out, uint32_t n) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const QuadUp u = in[i];
    const QuadParams qp = quad_params(u.px, u.py, u.pw);
    QuadRec r;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        r.px[k] = u.px[k];
        r.py[k] = u.py[k];
        r.pw[k] = u.pw[k];
    }
    r.x0 = qp.x0;
    r.dx_recip = qp.dx_recip;
    r.k0 = qp.k0;
    r.dk = qp.dk;
    r.curv_recip = 1.0f / qp.cur;
    r.prev_curv = u.prev_curv;
    r.total = u.total;
    r.step = u.step;
    out[i] = r;
}

__global__ void quad_expand_poly_kernel(const QuadUpPoly* __restrict__ in, QuadRec* __restrict__ out, uint32_t n) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const QuadUpPoly u = in[i];
    const float one[3] = {1.0f, 1.0f, 1.0f};
    const QuadParams qp = quad_params(u.px, u.py, one);
    QuadRec r;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        r.px[k] = u.px[k];
        r.py[k] = u.py[k];
        r.pw[k] = 1.0f;
    }
    r.x0 = qp.x0;
    r.dx_recip = qp.dx_recip;
    r.k0 = qp.k0;
    r.dk = qp.dk;
    r.curv_recip = 1.0f / qp.cur;
    r.prev_curv = u.prev_curv;
    r.total = u.total;
    r.step = u.step;
    out[i] = r;
}

void launch_quad_expand(const QuadUp* in, QuadRec* out, uint32_t n, cudaStream_t stream) {
    if (n) quad_expand_kernel<<<(n + 255) / 256, 256, 0, stream>>>(in, out, n);
}
void launch_quad_expand_poly(const QuadUpPoly* in, QuadRec* out, uint32_t n, cudaStream_t stream) {
    if (n) quad_expand_poly_kernel<<<(n + 255) / 256, 256, 0, stream>>>(in, out, n);
}

// One thread per output point: it finds its insert job, then its spline, by
// bisection over their first-point offsets (the per-point commands of the
// reference, path.rs:138-168, are never materialised — 36 B per spline cross
// PCIe instead of 16 B per point).
__global__ void flatten_eval_kernel(const SplineRec* __restrict__ splines, const PointRec* __restrict__ points,
                                    const uint8_t* __restrict__ kinds, const QuadRec* __restrict__ quads,
                                    const FlattenJob* __restrict__ jobs, const JobXf* __restrict__ xfs, uint32_t n_jobs,
                                    uint32_t n_points, uint32_t dst_base /* first point of the batch */, float* __restrict__ out_x,
                                    float* __restrict__ out_y, uint32_t* __restrict__ out_gid) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_points) return;
    uint32_t lo = 0, hi = n_jobs - 1u;  // last job with first_point <= i
    while (lo < hi) {
        uint32_t mid = (lo + hi + 1u) >> 1;
        if (jobs[mid].first_point <= i) lo = mid;
        else hi = mid - 1u;
    }
    const FlattenJob job = jobs[lo];
    const uint32_t local = i - job.first_point;
    const uint32_t count = (lo + 1u < n_jobs ? jobs[lo + 1u].first_point : n_points) - job.first_point;
    uint32_t kind;  // 0 literal, 1 literal + contour end, 2 evaluated, 3 evaluated, pi holds fma(step, pi, -prev_curv)
    float px = 0.0f, py = 0.0f, pi = 0.0f;
    const QuadRec* qp = nullptr;
    if (job.n_splines == 0u) {  // point encoding
        const PointRec p = points[job.spline_base + local];
        kind = kinds[job.spline_base + local];
        if (kind >= 2u) {
            qp = quads + job.quad_base + __float_as_uint(p.a);
            pi = p.b;
        } else {
            px = p.a;
            py = p.b;
        }
    } else {
        lo = 0;
        hi = job.n_splines - 1u;  // last spline with first_point <= local
        const SplineRec* sp = splines + job.spline_base;
        while (lo < hi) {
            uint32_t mid = (lo + hi + 1u) >> 1;
            if (sp[mid].first_point <= local) lo = mid;
            else hi = mid - 1u;
        }
        const SplineRec s = sp[lo];
        const uint32_t has_start = (s.info >> 30) & 1u, evaluated = s.info & kSplineEvalMask;
        const uint32_t j = local - s.first_point;  // point of the spline
        if (has_start && j == 0u) {
            kind = 0u;
            px = s.p0x;
            py = s.p0y;
        } else if (j - has_start == evaluated) {
            kind = (s.info >> 31) ? 1u : 0u;
            px = s.p2x;
            py = s.p2y;
        } else {
            kind = 2u;
            pi = (float)(j - has_start + 1u);
            const QuadRec* qs = quads + job.quad_base + s.first_quad;
            uint32_t a = 0, b = s.n_quads - 1u;  // first quad whose running curvature reaches pi (path.rs:424-431)
            while (a < b) {
                uint32_t mid = (a + b) >> 1;
                if (pi > qs[mid].total) a = mid + 1u;
                else b = mid;
            }
            qp = qs + a;
        }
    }
    if (kind >= 2u) {
        const QuadRec q = *qp;
        // path.rs:515-522
        float ratio = (kind == 2u ? fmaf(q.step, pi, -q.prev_curv) : pi) * q.curv_recip;
        float xx = inv_curvature(fmaf(ratio, q.dk, q.k0));
        float t = d_clamp((xx - q.x0) * q.dx_recip, 0.0f, 1.0f);
        // eval_quad, path.rs:447-471
        float w = d_mix(t, d_mix(t, q.pw[0], q.pw[1]), d_mix(t, q.pw[1], q.pw[2]));
        float w_recip = d_rcp(w);
        px = d_mix(t, d_mix(t, q.px[0], q.px[1]), d_mix(t, q.px[1], q.px[2])) * w_recip;
        py = d_mix(t, d_mix(t, q.py[0], q.py[1]), d_mix(t, q.py[1], q.py[2])) * w_recip;
    }
    if (job.xf_index) {  // path.rs:689-706, GeomPresTransform::transform
        const JobXf m = xfs[job.xf_index - 1u];
        float tx = fmaf(m.xf[0], px, fmaf(m.xf[2], py, m.xf[4]));
        float ty = fmaf(m.xf[1], px, fmaf(m.xf[3], py, m.xf[5]));
        px = tx;
        py = ty;
    }
    uint32_t dst = dst_base + i;  // the batch's points land in job order
    // ids: None at contour ends; the id of the last point of an insert is
    // replaced by the trailing None (segment.rs:181-198).
    bool none = kind == 1u || local + 1u == count;
    out_x[dst] = px;
    out_y[dst] = py;
    out_gid[dst] = none ? 0u : job.geom_id;
}

// ---------------------------------------------------------------------------
// Stage 1½: line setup (shared by the count and the emit pass)
// ---------------------------------------------------------------------------
struct LineParams {
    float x0, y0, dx, dy;  // sub-pixel space (x16)
    float a, b, c, d;
    uint32_t order;
    uint32_t length;       // number of pixel segments; 0 = no line
};

__device__ __forceinline__ uint32_t integers_between(float u, float v) {  // segment.rs:54-59
    float mn = fminf(u, v), mx = fmaxf(u, v);
    return d_sat_u32(ceilf(mx) - floorf(mn) - 1.0f);
}

// Line lengths and their sums saturate at 0xFFFFFFFF instead of wrapping (the reference wraps
// in release builds and panics in debug builds): a frame whose true total reaches 2^30 is then
// refused by Renderer::rasterize instead of being rendered from a wrapped count. Below the
// limit nothing saturates and every count is the reference's.
__device__ __forceinline__ uint32_t sat_add(uint32_t a, uint32_t b) { return min(a, ~b) + b; }

__device__ __forceinline__ uint32_t warp_inclusive_scan_sat(uint32_t v) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t n = __shfl_up_sync(kFullMask, v, o);
        if (lane_id() >= (unsigned)o) v = sat_add(v, n);
    }
    return v;
}

// segment.rs:298-383 for the point pair (i, i+1). kViews: the line as view `V` (6 floats in
// forma_layer_set_transform order) sees it: the layer's transform T becomes V ∘ T (V alone for a
// layer without one), composed exactly as ViewArgs documents; a composed identity is no transform.
// kPoses: a layer whose order lies in Q's window takes frame blockIdx.y's record (PoseArgs) in
// place of its own transform and enabled bit.
// kInst: the pair belongs to an instance (instance_line_setup), whose layer record `inst` is
// taken in place of the geometry's layer.
template <bool kViews = false, bool kPoses = false, bool kInst = false>
__device__ __forceinline__ LineParams line_setup(const RasterArgs& A, uint32_t i, const float* V = nullptr,
                                                 const PoseArgs& Q = PoseArgs{}, const LayerRec* inst = nullptr) {
    LineParams L;
    L.length = 0;
    L.order = 0;
    L.x0 = L.y0 = L.dx = L.dy = L.a = L.b = L.c = L.d = 0.0f;
    if (i + 1u >= A.n_points) return L;
    uint32_t gid = A.gid[i];
    if (gid == 0u) return L;
    LayerRec lay;
    if constexpr (kInst) {
        lay = *inst;
    } else {
        int32_t slot = gid < A.n_geoms ? A.geom_slot[gid] : -1;
        if (slot < 0) return L;
        if (A.layers) {
            lay = A.layers[slot];
        } else {  // no layer carries a transform: 4 bytes per layer (order | enabled << 21)
            const uint32_t bits = A.layer_bits[slot];
            lay.order = bits & 0x1FFFFFu;
            lay.enabled = (bits >> 21) & 1u;
            lay.has_xf = 0u;
        }
    }
    if constexpr (kPoses) {
        const uint32_t k = lay.order - Q.first_order;  // (wraps for orders below the window)
        if (k < Q.n_orders) {
            const float4* r = reinterpret_cast<const float4*>(Q.recs + (size_t)blockIdx.y * Q.n_orders + k);
            const float4 a = __ldg(r), b = __ldg(r + 1);
            lay.ux = a.x; lay.uy = a.y; lay.vx = a.z; lay.vy = a.w; lay.tx = b.x; lay.ty = b.y;
            const uint32_t bits = __float_as_uint(b.z);
            lay.has_xf = bits & 1u;
            lay.enabled = (bits >> 1) & 1u;
        }
    }
    if (!lay.enabled) return L;
    if constexpr (kViews) {
        const float vux = V[0], vvx = V[1], vuy = V[2], vvy = V[3], vtx = V[4], vty = V[5];
        float ux = vux, vx = vvx, uy = vuy, vy = vvy, tx = vtx, ty = vty;
        if (lay.has_xf) {
            ux = fmaf(vux, lay.ux, vvx * lay.uy);
            vx = fmaf(vux, lay.vx, vvx * lay.vy);
            uy = fmaf(vuy, lay.ux, vvy * lay.uy);
            vy = fmaf(vuy, lay.vx, vvy * lay.vy);
            tx = fmaf(vux, lay.tx, fmaf(vvx, lay.ty, vtx));
            ty = fmaf(vuy, lay.tx, fmaf(vvy, lay.ty, vty));
        }
        lay.has_xf = !(ux == 1.0f && uy == 0.0f && vx == 0.0f && vy == 1.0f && tx == 0.0f && ty == 0.0f) ? 1u : 0u;
        lay.ux = ux; lay.uy = uy; lay.vx = vx; lay.vy = vy; lay.tx = tx; lay.ty = ty;
    }
    float p0x = A.x[i], p0y = A.y[i], p1x = A.x[i + 1], p1y = A.y[i + 1];
    if (lay.has_xf) {  // transform_point, segment.rs:30-39
        float ax = fmaf(lay.ux, p0x, fmaf(lay.vx, p0y, lay.tx));
        float ay = fmaf(lay.uy, p0x, fmaf(lay.vy, p0y, lay.ty));
        float bx = fmaf(lay.ux, p1x, fmaf(lay.vx, p1y, lay.tx));
        float by = fmaf(lay.uy, p1x, fmaf(lay.vy, p1y, lay.ty));
        p0x = ax; p0y = ay; p1x = bx; p1y = by;
    }
    // skip_line, segment.rs:41-52, + the cull of lines that cannot produce a pixel segment in the
    // rows [band_lo, band_hi) this render paints (a crop, or one GPU's band of a multi-GPU frame).
    // A segment's row is min(y0, y1) of its end points rounded to 1/16 pixel (rasterizer.rs:
    // 111-156): rows >= band_hi follow from both end points >= band_hi; rows < band_lo need both
    // end points below band_lo by more than the rounding (1/32) — 1/16 is used. With these two
    // rules a culled line has no segment in a painted row, so a band render equals the whole
    // frame's rows exactly (cells, optimiser decisions and pixels alike).
    bool skip = p0y == p1y || (p0y >= A.height && p1y >= A.height) || (p0x >= A.width && p1x >= A.width) ||
                (p0y <= 0.0f && p1y <= 0.0f) || (p0y >= A.band_hi && p1y >= A.band_hi) ||
                (p0y <= A.band_lo - 0.0625f && p1y <= A.band_lo - 0.0625f);
    if (skip) return L;
    float dx = p1x - p0x, dy = p1y - p0y;
    float dx_recip = d_rcp(dx), dy_recip = d_rcp(dy);
    L.c = dx != 0.0f ? fmaxf((ceilf(p0x) - p0x) * dx_recip, (floorf(p0x) - p0x) * dx_recip) : 0.0f;
    L.d = dy != 0.0f ? fmaxf((ceilf(p0y) - p0y) * dy_recip, (floorf(p0y) - p0y) * dy_recip) : 0.0f;
    L.a = fabsf(dx_recip);
    L.b = fabsf(dy_recip);
    L.order = lay.order;
    L.x0 = p0x * 16.0f;
    L.y0 = p0y * 16.0f;
    L.dx = dx * 16.0f;
    L.dy = dy * 16.0f;
    L.length = sat_add(sat_add(integers_between(p0x, p1x), integers_between(p0y, p1y)), 1u);
    return L;
}

constexpr int kRasterThreads = 256;
constexpr uint32_t kRadixDigits = 256;  // digits of a sort pass (counted by the emit pass)

// Where a CTA of a batch works: its frame, its CTA within the frame's points, the frame's order base.
struct BatchPos {
    uint32_t frame, block, order_base;
};
// The CTA's frame (the last one whose first CTA is at or before it: frames without points own no
// CTA) and that frame's line-setup arguments, over the whole frame.
__device__ __forceinline__ BatchPos batch_pos(const BatchArgs& B, RasterArgs& A) {
    uint32_t lo = 0, hi = B.n_frames - 1u;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1u) >> 1;
        if (B.cta_first[mid] <= blockIdx.x) lo = mid;
        else hi = mid - 1u;
    }
    const BatchFrame& F = B.frames[lo];
    A.x = F.x;
    A.y = F.y;
    A.gid = F.gid;
    A.n_points = F.n_points;
    A.geom_slot = F.geom_slot;
    A.n_geoms = F.n_geoms;
    A.layers = F.layers;
    A.layer_bits = F.layer_bits;
    A.width = B.width;
    A.height = B.height;
    A.band_lo = 0.0f;
    A.band_hi = B.height;
    return BatchPos{lo, blockIdx.x - B.cta_first[lo], F.order_base};
}

// Where a CTA of an instance call works (InstanceArgs): its frame (the last one whose first CTA is
// at or before it: frames without point pairs own no CTA), its CTA within the frame's padded
// pairs, and the frame's order base b * n_slots.
__device__ __forceinline__ BatchPos instance_pos(const InstanceArgs& I) {
    uint32_t lo = 0, hi = I.n_frames - 1u;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1u) >> 1;
        if (__ldg(I.cta_first + mid) <= blockIdx.x) lo = mid;
        else hi = mid - 1u;
    }
    return BatchPos{lo, blockIdx.x - __ldg(I.cta_first + lo), lo * I.n_slots};
}

// The line of pair j of frame P.frame: its record is the last of the frame's records whose first
// pair is at or before j (a library shape has tens to hundreds of points, so the threads of a
// CTA share out several records); pairs past the frame's last record are the CTA padding. The
// instance's PoseRec stands in for the layer record, enabled, at the frame-local order m (the
// emit pass adds the frame's base).
__device__ __forceinline__ LineParams instance_line_setup(const RasterArgs& A, const InstanceArgs& I, const BatchPos& P, uint32_t j) {
    uint32_t lo = __ldg(I.frame_first + P.frame), hi = __ldg(I.frame_first + P.frame + 1u) - 1u;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1u) >> 1;
        if (__ldg(&I.lines[mid].first_pair) <= j) lo = mid;
        else hi = mid - 1u;
    }
    const uint4 R = __ldg(reinterpret_cast<const uint4*>(I.lines + lo));  // first_pair, n_pairs, first_point, slot
    const uint32_t k = j - R.x;
    if (k >= R.y) {
        LineParams L;
        L.length = 0;
        L.order = 0;
        L.x0 = L.y0 = L.dx = L.dy = L.a = L.b = L.c = L.d = 0.0f;
        return L;
    }
    const float4* r = reinterpret_cast<const float4*>(I.recs + R.w);
    const float4 a = __ldg(r), b = __ldg(r + 1);
    LayerRec lay;
    lay.order = R.w - P.order_base;
    lay.enabled = 1u;
    lay.has_xf = __float_as_uint(b.z) & 1u;
    lay.ux = a.x; lay.uy = a.y; lay.vx = a.z; lay.vy = a.w; lay.tx = b.x; lay.ty = b.y;
    return line_setup<false, false, true>(A, R.z + k, nullptr, PoseArgs{}, &lay);
}

// The line of thread i of a line-setup CTA in each mode (kInst: pair i of the CTA's instance frame).
template <bool kViews, bool kPoses, bool kInst>
__device__ __forceinline__ LineParams frame_line(const RasterArgs& A, uint32_t i, const ViewArgs& V, const PoseArgs& Q, const BatchPos& P,
                                                 const InstanceArgs& I) {
    if constexpr (kInst) return instance_line_setup(A, I, P, i);
    else return line_setup<kViews, kPoses>(A, i, kViews ? V.xf + 6u * blockIdx.y : nullptr, Q);
}

// Pass 1: per-CTA sum of line lengths.
// Also tracks the largest (biased) tile coordinates any pixel segment can take,
// so that the sort only spends passes on key bits that can be set.
// kViews: CTA (x, y) = the point pairs of CTA x under view y; its sum is block y * gridDim.x + x.
// kBatch: CTA x = the point pairs of CTA P.block of frame P.frame (V.rows: the frame's tile rows);
// its sum is block x.
// kPoses: as kViews, with frame y's pose records (Q) in place of a view transform.
// kInst (with kBatch): CTA x = the point pairs of CTA P.block of instance frame P.frame (I).
template <bool kViews, bool kBatch = false, bool kPoses = false, bool kInst = false>
__device__ __forceinline__ void line_count_body(const RasterArgs& A, const ViewArgs& V, uint32_t* __restrict__ block_sums,
                                                uint32_t* __restrict__ max_tile, const BatchPos& P = BatchPos{},
                                                const PoseArgs& Q = PoseArgs{}, const InstanceArgs& I = InstanceArgs{}) {
    constexpr bool kStack = kViews || kPoses;  // the stack of one composition: frame blockIdx.y
    __shared__ uint32_t warp_sums[kRasterThreads / 32];
    __shared__ uint32_t warp_max[2][kRasterThreads / 32];
    uint32_t i = (kBatch ? P.block : blockIdx.x) * kRasterThreads + threadIdx.x;
    const LineParams L = frame_line<kViews, kPoses, kInst>(A, i, V, Q, P, I);
    uint32_t len = L.length;
    {
        uint32_t bx = 0, by = 0;
        if (len) {
            // Sub-pixel end points -> tile (>> 8) -> bias (+1) -> one tile of slack for rounding.
            float ex = fmaxf(L.x0, L.x0 + L.dx), ey = fmaxf(L.y0, L.y0 + L.dy);
            int32_t tx = ((int32_t)floorf(fminf(ex, 3.0e7f) + 0.5f) >> 8) + 2;
            int32_t ty = ((int32_t)floorf(fminf(ey, 3.0e7f) + 0.5f) >> 8) + 2;
            bx = (uint32_t)min(max(tx, 0), 4095);
            by = (uint32_t)min(max(ty, 0), 2047);
            if constexpr (kStack || kBatch) {
                // The emit pass maps view y's segments to the stacked rows [y * rows + 1, (y + 1) * rows].
                by = ((kBatch ? P.frame : blockIdx.y) + 1u) * V.rows;
                // Tile columns left of -32767 wrap (int16, as in the reference) into the frame's
                // columns: such a line can set any tile_x bit.
                if (!(fminf(L.x0, L.x0 + L.dx) >= -8388352.0f)) bx = 4095;
            } else {
                // The same for the single frame, and for its rows: the skip rules drop a line only
                // when both ends are above the frame, so a line with one end in the frame and the
                // other above tile row -32767 survives, and its rows wrap into every value of the
                // 11-bit field. (A stacked frame maps every row outside the view to 0 instead. Rows
                // below the frame need no rule: from row 2045 on the clamp already gives 2047.)
                if (!(fminf(L.x0, L.x0 + L.dx) >= -8388352.0f)) bx = 4095;
                if (!(fminf(L.y0, L.y0 + L.dy) >= -8388352.0f)) by = 2047;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            bx = max(bx, __shfl_xor_sync(kFullMask, bx, o));
            by = max(by, __shfl_xor_sync(kFullMask, by, o));
        }
        if (lane_id() == 0) {
            warp_max[0][threadIdx.x >> 5] = bx;
            warp_max[1][threadIdx.x >> 5] = by;
        }
    }
    uint32_t incl = warp_inclusive_scan_sat(len);
    if (lane_id() == 31) warp_sums[threadIdx.x >> 5] = incl;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t s = 0, bx = 0, by = 0;
        for (int w = 0; w < kRasterThreads / 32; ++w) {
            s = sat_add(s, warp_sums[w]);
            bx = max(bx, warp_max[0][w]);
            by = max(by, warp_max[1][w]);
        }
        block_sums[kStack && !kBatch ? blockIdx.y * gridDim.x + blockIdx.x : blockIdx.x] = s;
        // Same-address atomics serialise in L2: only raise the maximum when needed.
        if (bx > *(volatile uint32_t*)&max_tile[0]) atomicMax(&max_tile[0], bx);
        if (by > *(volatile uint32_t*)&max_tile[1]) atomicMax(&max_tile[1], by);
    }
}
__global__ void __launch_bounds__(kRasterThreads) line_count_kernel(RasterArgs A, uint32_t* __restrict__ block_sums,
                                                                  uint32_t* __restrict__ max_tile /*[2]: x, y*/) {
    line_count_body<false>(A, ViewArgs{}, block_sums, max_tile);
}
__global__ void __launch_bounds__(kRasterThreads) line_count_views_kernel(RasterArgs A, ViewArgs V, uint32_t* __restrict__ block_sums,
                                                                        uint32_t* __restrict__ max_tile) {
    line_count_body<true>(A, V, block_sums, max_tile);
}
__global__ void __launch_bounds__(kRasterThreads) line_count_batch_kernel(BatchArgs B, uint32_t* __restrict__ block_sums,
                                                                        uint32_t* __restrict__ max_tile) {
    RasterArgs A;
    const BatchPos P = batch_pos(B, A);
    line_count_body<false, true>(A, ViewArgs{nullptr, B.rows}, block_sums, max_tile, P);
}
__global__ void __launch_bounds__(kRasterThreads) line_count_poses_kernel(RasterArgs A, PoseArgs Q, uint32_t* __restrict__ block_sums,
                                                                        uint32_t* __restrict__ max_tile) {
    line_count_body<false, false, true>(A, ViewArgs{nullptr, Q.rows}, block_sums, max_tile, BatchPos{}, Q);
}
__global__ void __launch_bounds__(kRasterThreads) line_count_instances_kernel(RasterArgs A, InstanceArgs I, uint32_t* __restrict__ block_sums,
                                                                            uint32_t* __restrict__ max_tile) {
    const BatchPos P = instance_pos(I);
    line_count_body<false, true, false, true>(A, ViewArgs{nullptr, I.rows}, block_sums, max_tile, P, PoseArgs{}, I);
}

// Device-wide exclusive scan of `n` u32 values by ONE CTA (n = number of CTAs
// of the producing kernel, a few thousand); writes the grand total to
// total[0]. 1024 threads, each owning a contiguous chunk. Saturating: every
// offset and the total are min(true value, 0xFFFFFFFF).
// kCheck: the count of a frame launched over bounds (CountCheck), judged with the largest tile
// coordinates max_tile[0..1] of the count pass this launch is chained behind.
template <bool kCheck>
__global__ void __launch_bounds__(1024) scan_block_sums_kernel(uint32_t* __restrict__ data, uint32_t n,
                                                              uint32_t* __restrict__ total, CountCheck check,
                                                              const uint32_t* __restrict__ max_tile) {
    chain_begin();
    __shared__ uint32_t warp_tot[32];
    __shared__ uint32_t carry, round_total;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const uint32_t per_round = 1024u * 4u;
    for (uint32_t base = 0; base < n; base += per_round) {
        uint32_t idx = base + threadIdx.x * 4u;
        uint32_t v[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) v[k] = (idx + k < n) ? data[idx + k] : 0u;
        uint32_t sum = sat_add(sat_add(v[0], v[1]), sat_add(v[2], v[3]));
        uint32_t incl = warp_inclusive_scan_sat(sum);
        uint32_t lane_excl = __shfl_up_sync(kFullMask, incl, 1);  // (a saturated sum cannot be subtracted from)
        if (lane_id() == 0) lane_excl = 0;
        if (lane_id() == 31) warp_tot[threadIdx.x >> 5] = incl;
        __syncthreads();
        if (threadIdx.x < 32) {
            uint32_t w = warp_tot[threadIdx.x];
            uint32_t wi = warp_inclusive_scan_sat(w);
            uint32_t we = __shfl_up_sync(kFullMask, wi, 1);
            warp_tot[threadIdx.x] = threadIdx.x ? we : 0u;  // exclusive over warps
            if (threadIdx.x == 31) round_total = wi;
        }
        __syncthreads();
        uint32_t excl = sat_add(sat_add(carry, warp_tot[threadIdx.x >> 5]), lane_excl);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (idx + k < n) data[idx + k] = excl;
            excl = sat_add(excl, v[k]);
        }
        __syncthreads();
        if (threadIdx.x == 0) carry = sat_add(carry, round_total);
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        total[0] = carry;
        if constexpr (kCheck) {
            const uint32_t tx_bits = 32u - __clz(max_tile[0]), ty_bits = 32u - __clz(max_tile[1]);
            const bool holds = carry >= check.n_lo && carry <= check.n_hi && carry < (1u << 30) && tx_bits == check.tx_bits &&
                               ty_bits == check.ty_bits;
            *check.live_n = holds ? carry : 0u;
            *check.paint_counter = holds ? 0u : kPaintAbort;
        }
    }
}
static void launch_scan_block_sums(uint32_t* data, uint32_t n, uint32_t* total, cudaStream_t stream) {
    launch_chained(scan_block_sums_kernel<false>, 1, 1024, 0, stream, data, n, total, CountCheck{}, (const uint32_t*)nullptr);
}

// ---------------------------------------------------------------------------
// Stage 2: pixel-grid intersection
// ---------------------------------------------------------------------------

// cpu/rasterizer.rs:32-61 — the i-th term of the ordered union of a*t+c, b*t+d.
__device__ __forceinline__ float find_param(int32_t ii, double a_over, double b_over, double cd_over, float a,
                                            float b, float c, float d) {
    float i = (float)ii;
    float ja = isfinite(b) ? (float)ceil(fma(b_over, (double)i, -cd_over)) : i;
    float jb = isfinite(a) ? (float)ceil(fma(a_over, (double)i, cd_over)) : i;
    float guess_a = fmaf(a, ja, c);
    float guess_b = fmaf(b, jb, d);
    return fminf(guess_a, guess_b);  // NaN-ignoring, like f32::min (SURVEY.md A.3)
}

// rasterizer.rs:78-80: `(v + 0.5).floor().to_int_unchecked()`. Rust leaves NaN and values outside
// i32 undefined there; the reference's x86 build (cvttss2si) gives i32::MIN for them, and so does
// the CPU restatement the tests compare with. A plain cast would compile to cvt.rzi.s32.f32, which saturates
// to INT_MAX instead. Sub-pixel positions reach 2^31 at 2^27 px.
__device__ __forceinline__ int32_t round_sub(float v) {
    const float f = floorf(v + 0.5f);
    return (f >= -2147483648.0f && f < 2147483648.0f) ? (int32_t)f : INT32_MIN;
}

struct SharedLines {
    float x0[kRasterThreads], y0[kRasterThreads], dx[kRasterThreads], dy[kRasterThreads];
    float a[kRasterThreads], b[kRasterThreads], c[kRasterThreads], d[kRasterThreads];
    double a_over[kRasterThreads], b_over[kRasterThreads], cd_over[kRasterThreads];
    uint32_t order[kRasterThreads];
    uint32_t excl[kRasterThreads + 1];  // exclusive offset of the line inside its CTA (one spare slot: the bisection probes index 256 - 1 at most)
};

// Pass 2: recompute the CTA's 256 lines, then the CTA expands them together: pixel segment s
// of the block (0 <= s < block total) goes to thread s % 256, which finds its line by
// bisection over the block's exclusive prefix of the line lengths. A line of several thousand
// segments (a long diagonal) is thus spread over the whole CTA instead of keeping one warp busy
// for its whole length (measured on paris@4K: the kernel's time was one warp's tail — it did
// not shrink when seven eighths of the lines were culled).
// kViews: CTA (x, y) emits view y's segments of the CTA x lines (see line_count_body).
// kBatch: CTA x emits frame P.frame's segments, its layers moved up by the frame's order base.
// kCount: the digit C.spec of every stored segment is counted for its 4096-key sort tile (TileCounts).
// A CTA's segments are consecutive, most often within two sort tiles: their counts gather in
// shared memory, warp-aggregated, and go out once per CTA; the tiles after those two (a CTA of long
// lines) take warp-aggregated global atomics.
// kPoses: as kViews, with frame y's pose records (Q) in place of a view transform.
// kInst (with kBatch): CTA x emits instance frame P.frame's segments (I), at the orders b M + m.
template <bool kViews, bool kBatch = false, bool kCount = false, bool kPoses = false, bool kInst = false>
__device__ __forceinline__ void raster_emit_body(const RasterArgs& A, const ViewArgs& V, const uint32_t* __restrict__ block_offsets,
                                                 uint64_t* __restrict__ out, uint32_t cap, const BatchPos& P = BatchPos{},
                                                 const CountArgs& C = CountArgs{}, const PoseArgs& Q = PoseArgs{},
                                                 const InstanceArgs& I = InstanceArgs{}) {
    constexpr bool kStack = kViews || kPoses;  // the stack of one composition: frame blockIdx.y
    __shared__ SharedLines S;
    __shared__ uint32_t warp_sums[kRasterThreads / 32];
    __shared__ uint32_t s_count[kCount ? 2 * kRadixDigits : 1];  // [2 tiles][digit]
    const uint32_t t = threadIdx.x;
    const uint32_t warp = t >> 5, lane = t & 31u;
    if constexpr (kCount) {
        s_count[t] = 0;
        s_count[t + kRasterThreads] = 0;
    }
    uint32_t i = (kBatch ? P.block : blockIdx.x) * kRasterThreads + t;
    LineParams L = frame_line<kViews, kPoses, kInst>(A, i, V, Q, P, I);
    if constexpr (kBatch) L.order += P.order_base;
    uint32_t incl = warp_inclusive_scan_sat(L.length);
    if (lane == 31) warp_sums[warp] = incl;
    if (L.length) {
        S.x0[t] = L.x0; S.y0[t] = L.y0; S.dx[t] = L.dx; S.dy[t] = L.dy;
        S.a[t] = L.a; S.b[t] = L.b; S.c[t] = L.c; S.d[t] = L.d;
        S.order[t] = L.order;
        // get_ith_pixel_segment_params, rasterizer.rs:67-70 — per-line f64 constants.
        double sum_recip = 1.0 / ((double)L.a + (double)L.b);
        S.a_over[t] = (double)L.a * sum_recip;
        S.b_over[t] = (double)L.b * sum_recip;
        S.cd_over[t] = ((double)L.c - (double)L.d) * sum_recip;
    }
    __syncthreads();
    uint32_t before = 0, block_total = 0;  // segments of the warps before this one / of the whole block
#pragma unroll
    for (uint32_t w = 0; w < (uint32_t)(kRasterThreads / 32); ++w) {
        if (w < warp) before = sat_add(before, warp_sums[w]);
        block_total = sat_add(block_total, warp_sums[w]);
    }
    // Exact unless the block's total saturated (a frame Renderer::rasterize refuses; the offsets
    // then only steer the bisection, which stays inside S.excl).
    S.excl[t] = before + incl - L.length;  // exclusive prefix over the block's 256 lines
    __syncthreads();
    const uint32_t block_base = block_offsets[kStack && !kBatch ? blockIdx.y * gridDim.x + blockIdx.x : blockIdx.x];
    // `cap` bounds a speculative launch made before the segment count is known on the host: the
    // loop never runs past it, whatever the (saturated) counts of an over-limit frame. The last
    // clamp keeps `s += kRasterThreads` from wrapping.
    const uint32_t limit = min(min(block_total, block_base < cap ? cap - block_base : 0u), 0xFFFFFF00u);

    for (uint32_t s = t; s < limit; s += kRasterThreads) {
        // Largest j in [0, 256) with excl[j] <= s (zero-length lines share their
        // successor's offset and are skipped by taking the largest such j).
        uint32_t j = 0;
#pragma unroll
        for (int step = kRasterThreads / 2; step > 0; step >>= 1) {
            uint32_t cand = j + step;
            if (S.excl[cand] <= s) j = cand;
        }
        const uint32_t li = j;
        const uint32_t k = s - S.excl[j];
        const float a = S.a[li], b = S.b[li], c = S.c[li], d = S.d[li];
        // rasterizer.rs:63-76
        int32_t ii = (int32_t)k - (c != 0.0f ? 1 : 0) - (d != 0.0f ? 1 : 0);
        const double ao = S.a_over[li], bo = S.b_over[li], cdo = S.cd_over[li];
        float t0 = fmaxf(find_param(ii, ao, bo, cdo, a, b, c, d), 0.0f);
        float t1 = fminf(find_param(ii + 1, ao, bo, cdo, a, b, c, d), 1.0f);
        // rasterizer.rs:111-156
        const float ldx = S.dx[li], ldy = S.dy[li], lx0 = S.x0[li], ly0 = S.y0[li];
        int32_t x0s = round_sub(fmaf(t0, ldx, lx0));
        int32_t y0s = round_sub(fmaf(t0, ldy, ly0));
        int32_t x1s = round_sub(fmaf(t1, ldx, lx0));
        int32_t y1s = round_sub(fmaf(t1, ldy, ly0));
        int32_t border_x = min(x0s, x1s) >> 4;
        int32_t border_y = min(y0s, y1s) >> 4;
        int32_t tile_x = (int32_t)(int16_t)(border_x >> 4);
        int32_t tile_y = (int32_t)(int16_t)(border_y >> 4);
        uint32_t local_x = (uint32_t)(border_x & 15);
        uint32_t local_y = (uint32_t)(border_y & 15);
        int32_t border = (border_x << 4) + 16;
        uint32_t dam = (uint32_t)(abs(x1s - x0s) + 2 * (border - max(x0s, x1s))) & 0xFFu;
        int32_t cover = (int32_t)(int8_t)(y1s - y0s);
        // PixelSegment::new, pixel_segment.rs:36-71
        uint64_t ty = (uint64_t)max((int32_t)(int16_t)(tile_y + 1), 0) & 0x7FFull;
        // A view's painted rows (biased 1 ... rows) move to its place in the stacked frame; every
        // other row becomes tile row -1 (biased 0), which no painted tile reads, so that nothing
        // bleeds into the neighbouring views. The single frame's own wrap of the field is kept.
        if constexpr (kStack || kBatch) ty = ty - 1u < V.rows ? ty + (uint64_t)(kBatch ? P.frame : blockIdx.y) * V.rows : 0u;
        uint64_t tx = (uint64_t)max((int32_t)(int16_t)(tile_x + 1), 0) & 0xFFFull;
        uint64_t v = (ty << 53) | (tx << 41) | ((uint64_t)(S.order[li] & 0x1FFFFFu) << 20) | ((uint64_t)local_x << 16) |
                     ((uint64_t)local_y << 12) | ((uint64_t)(dam & 0x3Fu) << 6) | ((uint64_t)((uint32_t)cover & 0x3Fu));
        out[(uint64_t)block_base + s] = v;
        if constexpr (kCount) {
            // block_base + s < cap < 2^32. The lanes of one (tile, digit) add their count at once.
            const uint32_t rel = ((block_base + s) / kSortTileKeys) - block_base / kSortTileKeys, d = digit_of(v, C.spec);
            const uint32_t peers = __match_any_sync(__activemask(), (rel << 8) | d);
            if (lane == __ffs(peers) - 1u) {
                if (rel < 2u) atomicAdd(&s_count[rel * kRadixDigits + d], (uint32_t)__popc(peers));
                else add_tile_count(C, block_base / kSortTileKeys + rel, d, (uint32_t)__popc(peers));
            }
        }
    }
    if constexpr (kCount) {
        __syncthreads();
        for (uint32_t i = t; i < 2u * kRadixDigits; i += kRasterThreads) {
            const uint32_t c = s_count[i];
            if (c) add_tile_count(C, block_base / kSortTileKeys + i / kRadixDigits, i % kRadixDigits, c);
        }
    }
}
// The counting builds keep the plain builds' 32 registers: 8 CTAs per SM.
template <bool kCount>
__global__ void __launch_bounds__(kRasterThreads, kCount ? 8 : 0)
    raster_emit_kernel(RasterArgs A, const uint32_t* __restrict__ block_offsets, uint64_t* __restrict__ out, uint32_t cap, CountArgs C) {
    raster_emit_body<false, false, kCount>(A, ViewArgs{}, block_offsets, out, cap, BatchPos{}, C);
}
template <bool kCount>
__global__ void __launch_bounds__(kRasterThreads, kCount ? 8 : 0) raster_emit_views_kernel(RasterArgs A, ViewArgs V, const uint32_t* __restrict__ block_offsets,
                                                                         uint64_t* __restrict__ out, uint32_t cap, CountArgs C) {
    raster_emit_body<true, false, kCount>(A, V, block_offsets, out, cap, BatchPos{}, C);
}
template <bool kCount>
__global__ void __launch_bounds__(kRasterThreads, kCount ? 8 : 0) raster_emit_batch_kernel(BatchArgs B, const uint32_t* __restrict__ block_offsets,
                                                                         uint64_t* __restrict__ out, uint32_t cap, CountArgs C) {
    RasterArgs A;
    const BatchPos P = batch_pos(B, A);
    raster_emit_body<false, true, kCount>(A, ViewArgs{nullptr, B.rows}, block_offsets, out, cap, P, C);
}
template <bool kCount>
__global__ void __launch_bounds__(kRasterThreads, kCount ? 8 : 0) raster_emit_poses_kernel(RasterArgs A, PoseArgs Q, const uint32_t* __restrict__ block_offsets,
                                                                         uint64_t* __restrict__ out, uint32_t cap, CountArgs C) {
    raster_emit_body<false, false, kCount, true>(A, ViewArgs{nullptr, Q.rows}, block_offsets, out, cap, BatchPos{}, C, Q);
}

template <bool kCount>
__global__ void __launch_bounds__(kRasterThreads, kCount ? 8 : 0) raster_emit_instances_kernel(RasterArgs A, InstanceArgs I, const uint32_t* __restrict__ block_offsets,
                                                                             uint64_t* __restrict__ out, uint32_t cap, CountArgs C) {
    const BatchPos P = instance_pos(I);
    raster_emit_body<false, true, kCount, false, true>(A, ViewArgs{nullptr, I.rows}, block_offsets, out, cap, P, C, PoseArgs{}, I);
}

// A record's transform from a table ([ux, vx, uy, vy, tx, ty] at t): tested as geom_pres_ok
// (host_path.cpp) tests it, in the same separately rounded f32 operations (a refused record r is
// atomicMin'ed into *first_bad when that is not null), and an identity is no transform.
__device__ __forceinline__ void fold_transform(const float* t, uint32_t r, uint32_t* first_bad, float& ux, float& uy, float& vx, float& vy,
                                               float& tx, float& ty, bool& has_xf) {
    ux = __ldg(t); vx = __ldg(t + 1); uy = __ldg(t + 2); vy = __ldg(t + 3); tx = __ldg(t + 4); ty = __ldg(t + 5);
    const float max_x = 1.0f + (1.0f / 16.0f) / 65536.0f, max_y = 1.0f + (1.0f / 16.0f) / 32768.0f;
    const bool ok = !(__fadd_rn(__fmul_rn(ux, ux), __fmul_rn(uy, uy)) > max_x) && !(__fadd_rn(__fmul_rn(vx, vx), __fmul_rn(vy, vy)) > max_y);
    if (first_bad && !ok) atomicMin(first_bad, r);
    has_xf = !(ux == 1.0f && uy == 0.0f && vx == 0.0f && vy == 1.0f && tx == 0.0f && ty == 0.0f);
}

// The pose records the two kernels above read, one thread per record (see PoseFoldArgs). Every
// record's transform is tested (orders without a layer included, as check_poses walks them).
__global__ void __launch_bounds__(256) pose_fold_kernel(PoseFoldArgs F, PoseRec* __restrict__ recs, uint32_t n_recs) {
    chain_begin();
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_recs) return;
    const float4* w = reinterpret_cast<const float4*>(F.window + r % F.n_orders);
    const float4 a = __ldg(w), b = __ldg(w + 1);
    float ux = a.x, uy = a.y, vx = a.z, vy = a.w, tx = b.x, ty = b.y;
    const uint32_t bits = __float_as_uint(b.z);
    bool has_xf = bits & 1u, enabled = (bits >> 1) & 1u;
    if (F.transforms) fold_transform(F.transforms + 6ull * r, r, F.first_bad, ux, uy, vx, vy, tx, ty, has_xf);
    if (F.visible) enabled = __ldg(F.visible + r) != 0;
    float4* out = reinterpret_cast<float4*>(recs + r);
    if (!(bits & kPoseLayer)) {
        out[0] = out[1] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        return;
    }
    out[0] = make_float4(ux, uy, vx, vy);
    out[1] = make_float4(tx, ty, __uint_as_float((has_xf ? 1u : 0u) | (enabled ? 2u : 0u)), 0.0f);
}

// The instance records (see InstanceFoldArgs), one thread per slot: the prototype's own record
// with the slot's transform folded in as pose_fold_kernel folds it, enabled. Only the transforms of
// slots with a prototype are tested; an empty slot's record stays zero (no line reads it).
__global__ void __launch_bounds__(256) instance_fold_kernel(InstanceFoldArgs F, PoseRec* __restrict__ recs, uint32_t n_recs) {
    chain_begin();
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_recs) return;
    const uint32_t p = __ldg(F.prototypes + r);
    float4* out = reinterpret_cast<float4*>(recs + r);
    if (p == 0xFFFFFFFFu) {  // FORMA_NO_INSTANCE
        out[0] = out[1] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        return;
    }
    const float4* w = reinterpret_cast<const float4*>(F.base + p);
    const float4 a = __ldg(w), b = __ldg(w + 1);
    float ux = a.x, uy = a.y, vx = a.z, vy = a.w, tx = b.x, ty = b.y;
    bool has_xf = __float_as_uint(b.z) & 1u;
    if (F.transforms) fold_transform(F.transforms + 6ull * r, r, F.first_bad, ux, uy, vx, vy, tx, ty, has_xf);
    out[0] = make_float4(ux, uy, vx, vy);
    out[1] = make_float4(tx, ty, __uint_as_float((has_xf ? 1u : 0u) | 2u), 0.0f);
}

// Inspection only (forma_renderer_lines): the line records of segment.rs:298-383 as the
// reference's SegmentBufferView holds them (segment.rs:530-545), one per point pair; the
// render path itself never materialises them. `lengths` are per line (the host turns them
// into the reference's inclusive prefix sums).
__global__ void line_records_kernel(RasterArgs A, uint32_t n, uint32_t* __restrict__ orders, float* __restrict__ x0,
                                    float* __restrict__ y0, float* __restrict__ dx, float* __restrict__ dy,
                                    float* __restrict__ a, float* __restrict__ b, float* __restrict__ c,
                                    float* __restrict__ d, uint32_t* __restrict__ lengths) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const LineParams L = line_setup(A, i);
    orders[i] = L.order;
    x0[i] = L.x0; y0[i] = L.y0; dx[i] = L.dx; dy[i] = L.dy;
    a[i] = L.a; b[i] = L.b; c[i] = L.c; d[i] = L.d;
    lengths[i] = L.length;
}

void launch_line_records(const RasterArgs& args, uint32_t n, uint32_t* orders, float* const f[8], uint32_t* lengths,
                         cudaStream_t stream) {
    if (n) line_records_kernel<<<(n + 255) / 256, 256, 0, stream>>>(args, n, orders, f[0], f[1], f[2], f[3], f[4], f[5], f[6], f[7], lengths);
}

// ---------------------------------------------------------------------------
// Host launchers
// ---------------------------------------------------------------------------
void launch_flatten_eval(const SplineRec* splines, const PointRec* points, const uint8_t* kinds, const QuadRec* quads,
                         const FlattenJob* jobs, const JobXf* xfs, uint32_t n_jobs, uint32_t n_points, uint32_t dst_base,
                         float* x, float* y, uint32_t* gid, cudaStream_t stream) {
    if (!n_points || !n_jobs) return;
    flatten_eval_kernel<<<(n_points + 255) / 256, 256, 0, stream>>>(splines, points, kinds, quads, jobs, xfs, n_jobs, n_points,
                                                                    dst_base, x, y, gid);
}

// The count and emit passes are plain launches: the stream hands each of them a memset (max_tile)
// or the count read-back right before, which a chained launch cannot overlap either, and as plain
// launches they keep their read-only (LDG.CONSTANT) loads of the segment buffer and the layer
// tables. The scan after the count pass is chained (launch_chained).
uint32_t raster_num_blocks(uint32_t n_points) { return n_points ? (n_points + kRasterThreads - 1) / kRasterThreads : 0; }

void launch_line_count(const RasterArgs& args, uint32_t* block_sums, uint32_t* total, uint32_t* max_tile,
                       cudaStream_t stream, const CountCheck* check) {
    uint32_t nb = raster_num_blocks(args.n_points);
    cudaMemsetAsync(max_tile, 0, 2 * sizeof(uint32_t), stream);
    if (!nb) {
        cudaMemsetAsync(total, 0, sizeof(uint32_t), stream);
        return;
    }
    line_count_kernel<<<nb, kRasterThreads, 0, stream>>>(args, block_sums, max_tile);
    if (check) launch_chained(scan_block_sums_kernel<true>, 1, 1024, 0, stream, block_sums, nb, total, *check, (const uint32_t*)max_tile);
    else launch_scan_block_sums(block_sums, nb, total, stream);
}

void launch_raster_emit(const RasterArgs& args, const uint32_t* block_offsets, uint64_t* out, uint32_t cap, cudaStream_t stream,
                        const CountArgs* counts) {
    uint32_t nb = raster_num_blocks(args.n_points);
    if (!nb) return;
    if (counts) raster_emit_kernel<true><<<nb, kRasterThreads, 0, stream>>>(args, block_offsets, out, cap, *counts);
    else raster_emit_kernel<false><<<nb, kRasterThreads, 0, stream>>>(args, block_offsets, out, cap, CountArgs{});
}

void launch_line_count_views(const RasterArgs& args, const ViewArgs& views, uint32_t n_views, uint32_t* block_sums, uint32_t* total,
                             uint32_t* max_tile, cudaStream_t stream) {
    uint32_t nb = raster_num_blocks(args.n_points);
    cudaMemsetAsync(max_tile, 0, 2 * sizeof(uint32_t), stream);
    if (!nb || !n_views) {
        cudaMemsetAsync(total, 0, sizeof(uint32_t), stream);
        return;
    }
    line_count_views_kernel<<<dim3(nb, n_views), kRasterThreads, 0, stream>>>(args, views, block_sums, max_tile);
    launch_scan_block_sums(block_sums, nb * n_views, total, stream);
}

void launch_raster_emit_views(const RasterArgs& args, const ViewArgs& views, uint32_t n_views, const uint32_t* block_offsets,
                              uint64_t* out, uint32_t cap, cudaStream_t stream, const CountArgs* counts) {
    uint32_t nb = raster_num_blocks(args.n_points);
    if (!nb || !n_views) return;
    if (counts)
        raster_emit_views_kernel<true><<<dim3(nb, n_views), kRasterThreads, 0, stream>>>(args, views, block_offsets, out, cap, *counts);
    else
        raster_emit_views_kernel<false><<<dim3(nb, n_views), kRasterThreads, 0, stream>>>(args, views, block_offsets, out, cap, CountArgs{});
}

void launch_line_count_poses(const RasterArgs& args, const PoseArgs& poses, uint32_t n_frames, uint32_t* block_sums, uint32_t* total,
                             uint32_t* max_tile, cudaStream_t stream) {
    uint32_t nb = raster_num_blocks(args.n_points);
    cudaMemsetAsync(max_tile, 0, 2 * sizeof(uint32_t), stream);
    if (!nb || !n_frames) {
        cudaMemsetAsync(total, 0, sizeof(uint32_t), stream);
        return;
    }
    line_count_poses_kernel<<<dim3(nb, n_frames), kRasterThreads, 0, stream>>>(args, poses, block_sums, max_tile);
    launch_scan_block_sums(block_sums, nb * n_frames, total, stream);
}

void launch_raster_emit_poses(const RasterArgs& args, const PoseArgs& poses, uint32_t n_frames, const uint32_t* block_offsets,
                              uint64_t* out, uint32_t cap, cudaStream_t stream, const CountArgs* counts) {
    uint32_t nb = raster_num_blocks(args.n_points);
    if (!nb || !n_frames) return;
    if (counts)
        raster_emit_poses_kernel<true><<<dim3(nb, n_frames), kRasterThreads, 0, stream>>>(args, poses, block_offsets, out, cap, *counts);
    else
        raster_emit_poses_kernel<false><<<dim3(nb, n_frames), kRasterThreads, 0, stream>>>(args, poses, block_offsets, out, cap, CountArgs{});
}

void launch_pose_fold(const PoseFoldArgs& args, PoseRec* recs, uint32_t n_recs, cudaStream_t stream) {
    if (n_recs) launch_chained(pose_fold_kernel, (uint32_t)(((uint64_t)n_recs + 255u) / 256u), 256, 0, stream, args, recs, n_recs);
}

void launch_instance_fold(const InstanceFoldArgs& args, PoseRec* recs, uint32_t n_recs, cudaStream_t stream) {
    if (n_recs) launch_chained(instance_fold_kernel, (uint32_t)(((uint64_t)n_recs + 255u) / 256u), 256, 0, stream, args, recs, n_recs);
}

void launch_line_count_instances(const RasterArgs& args, const InstanceArgs& inst, uint32_t n_ctas, uint32_t* block_sums, uint32_t* total,
                                 uint32_t* max_tile, cudaStream_t stream) {
    cudaMemsetAsync(max_tile, 0, 2 * sizeof(uint32_t), stream);
    if (!n_ctas) {
        cudaMemsetAsync(total, 0, sizeof(uint32_t), stream);
        return;
    }
    line_count_instances_kernel<<<n_ctas, kRasterThreads, 0, stream>>>(args, inst, block_sums, max_tile);
    launch_scan_block_sums(block_sums, n_ctas, total, stream);
}

void launch_raster_emit_instances(const RasterArgs& args, const InstanceArgs& inst, uint32_t n_ctas, const uint32_t* block_offsets,
                                  uint64_t* out, uint32_t cap, cudaStream_t stream, const CountArgs* counts) {
    if (!n_ctas) return;
    if (counts) raster_emit_instances_kernel<true><<<n_ctas, kRasterThreads, 0, stream>>>(args, inst, block_offsets, out, cap, *counts);
    else raster_emit_instances_kernel<false><<<n_ctas, kRasterThreads, 0, stream>>>(args, inst, block_offsets, out, cap, CountArgs{});
}

void launch_line_count_batch(const BatchArgs& batch, uint32_t n_ctas, uint32_t* block_sums, uint32_t* total, uint32_t* max_tile,
                             cudaStream_t stream) {
    cudaMemsetAsync(max_tile, 0, 2 * sizeof(uint32_t), stream);
    if (!n_ctas) {
        cudaMemsetAsync(total, 0, sizeof(uint32_t), stream);
        return;
    }
    line_count_batch_kernel<<<n_ctas, kRasterThreads, 0, stream>>>(batch, block_sums, max_tile);
    launch_scan_block_sums(block_sums, n_ctas, total, stream);
}

void launch_raster_emit_batch(const BatchArgs& batch, uint32_t n_ctas, const uint32_t* block_offsets, uint64_t* out, uint32_t cap,
                              cudaStream_t stream, const CountArgs* counts) {
    if (!n_ctas) return;
    if (counts) raster_emit_batch_kernel<true><<<n_ctas, kRasterThreads, 0, stream>>>(batch, block_offsets, out, cap, *counts);
    else raster_emit_batch_kernel<false><<<n_ctas, kRasterThreads, 0, stream>>>(batch, block_offsets, out, cap, CountArgs{});
}

}  // namespace forma
