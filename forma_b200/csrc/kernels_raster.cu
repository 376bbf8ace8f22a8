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

// segment.rs:298-383 for the point pair (i, i+1).
__device__ __forceinline__ LineParams line_setup(const RasterArgs& A, uint32_t i) {
    LineParams L;
    L.length = 0;
    L.order = 0;
    L.x0 = L.y0 = L.dx = L.dy = L.a = L.b = L.c = L.d = 0.0f;
    if (i + 1u >= A.n_points) return L;
    uint32_t gid = A.gid[i];
    if (gid == 0u) return L;
    int32_t slot = gid < A.n_geoms ? A.geom_slot[gid] : -1;
    if (slot < 0) return L;
    LayerRec lay;
    if (A.layers) {
        lay = A.layers[slot];
    } else {  // no layer carries a transform: 4 bytes per layer (order | enabled << 21)
        const uint32_t bits = A.layer_bits[slot];
        lay.order = bits & 0x1FFFFFu;
        lay.enabled = (bits >> 21) & 1u;
        lay.has_xf = 0u;
    }
    if (!lay.enabled) return L;
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

// Pass 1: per-CTA sum of line lengths.
// Also tracks the largest (biased) tile coordinates any pixel segment can take,
// so that the sort only spends passes on key bits that can be set.
__global__ void __launch_bounds__(kRasterThreads) line_count_kernel(RasterArgs A, uint32_t* __restrict__ block_sums,
                                                                  uint32_t* __restrict__ max_tile /*[2]: x, y*/) {
    __shared__ uint32_t warp_sums[kRasterThreads / 32];
    __shared__ uint32_t warp_max[2][kRasterThreads / 32];
    uint32_t i = blockIdx.x * kRasterThreads + threadIdx.x;
    const LineParams L = line_setup(A, i);
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
        block_sums[blockIdx.x] = s;
        // Same-address atomics serialise in L2: only raise the maximum when needed.
        if (bx > *(volatile uint32_t*)&max_tile[0]) atomicMax(&max_tile[0], bx);
        if (by > *(volatile uint32_t*)&max_tile[1]) atomicMax(&max_tile[1], by);
    }
}

// Device-wide exclusive scan of `n` u32 values by ONE CTA (n = number of CTAs
// of the producing kernel, a few thousand); writes the grand total to
// total[0]. 1024 threads, each owning a contiguous chunk. Saturating: every
// offset and the total are min(true value, 0xFFFFFFFF).
__global__ void __launch_bounds__(1024) scan_block_sums_kernel(uint32_t* __restrict__ data, uint32_t n,
                                                              uint32_t* __restrict__ total) {
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
    if (threadIdx.x == 0) total[0] = carry;
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
__global__ void __launch_bounds__(kRasterThreads)
    raster_emit_kernel(RasterArgs A, const uint32_t* __restrict__ block_offsets, uint64_t* __restrict__ out, uint32_t cap) {
    __shared__ SharedLines S;
    __shared__ uint32_t warp_sums[kRasterThreads / 32];
    const uint32_t t = threadIdx.x;
    const uint32_t warp = t >> 5, lane = t & 31u;
    uint32_t i = blockIdx.x * kRasterThreads + t;
    LineParams L = line_setup(A, i);
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
    const uint32_t block_base = block_offsets[blockIdx.x];
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
        uint64_t tx = (uint64_t)max((int32_t)(int16_t)(tile_x + 1), 0) & 0xFFFull;
        uint64_t v = (ty << 53) | (tx << 41) | ((uint64_t)(S.order[li] & 0x1FFFFFu) << 20) | ((uint64_t)local_x << 16) |
                     ((uint64_t)local_y << 12) | ((uint64_t)(dam & 0x3Fu) << 6) | ((uint64_t)((uint32_t)cover & 0x3Fu));
        out[(uint64_t)block_base + s] = v;
    }
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

uint32_t raster_num_blocks(uint32_t n_points) { return n_points ? (n_points + kRasterThreads - 1) / kRasterThreads : 0; }

void launch_line_count(const RasterArgs& args, uint32_t* block_sums, uint32_t* total, uint32_t* max_tile,
                       cudaStream_t stream) {
    uint32_t nb = raster_num_blocks(args.n_points);
    cudaMemsetAsync(max_tile, 0, 2 * sizeof(uint32_t), stream);
    if (!nb) {
        cudaMemsetAsync(total, 0, sizeof(uint32_t), stream);
        return;
    }
    line_count_kernel<<<nb, kRasterThreads, 0, stream>>>(args, block_sums, max_tile);
    scan_block_sums_kernel<<<1, 1024, 0, stream>>>(block_sums, nb, total);
}

void launch_raster_emit(const RasterArgs& args, const uint32_t* block_offsets, uint64_t* out, uint32_t cap, cudaStream_t stream) {
    uint32_t nb = raster_num_blocks(args.n_points);
    if (!nb) return;
    raster_emit_kernel<<<nb, kRasterThreads, 0, stream>>>(args, block_offsets, out, cap);
}

}  // namespace forma
