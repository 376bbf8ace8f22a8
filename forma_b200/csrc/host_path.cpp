// forma_b200 host side — PathBuilder / Path and flatten-program construction.
// See host_path.hpp. Compiled with -ffp-contract=off.
#include "host_path.hpp"

#include "quad_math.h"

#include <algorithm>

namespace forma {
namespace {

constexpr float kPi = 3.14159274101257324f;
constexpr float kHalfPi = 1.57079637050628662f;
constexpr float kEps = 1.1920928955078125e-7f;
constexpr float kMaxError = 1.0f / 16.0f;   // path.rs:40
constexpr float kMaxAngleError = 0.001f;    // path.rs:41

struct WPt {
    float x, y, w;
    Pt applied() const {  // path.rs:65-72
        float r = rcp(w);
        return {x * r, y * r};
    }
};

float length(Pt p) { return std::sqrt(p.x * p.x + p.y * p.y); }  // math/point.rs:83-85

// math/point.rs:54-78
float atan2_approx(float y, float x) {
    float ax = std::fabs(x), ay = std::fabs(y);
    float a = std::fmin(ax, ay) / std::fmax(ax, ay);
    float s = a * a;
    float r = fmaf(fmaf(fmaf(s, -0.046496473f, 0.15931422f), s, -0.32762277f), s * a, a);
    if (ay > ax) r = kHalfPi - r;
    if (x < 0.0f) r = kPi - r;
    if (y < 0.0f) r = -r;
    return r;
}

struct Angle {
    bool some;
    float v;
};
Angle angle_of(Pt d) {  // math/point.rs:87-89
    if (length(d) >= kEps) return {true, atan2_approx(d.y, d.x)};
    return {false, 0.0f};
}

WPt cubic_at(float t, const WPt q[4]) {  // path.rs:75-120
    auto bez = [t](float a, float b, float c, float d) {
        float ab = mix(t, a, b), bc = mix(t, b, c), cd = mix(t, c, d);
        return mix(t, mix(t, ab, bc), mix(t, bc, cd));
    };
    return {bez(q[0].x, q[1].x, q[2].x, q[3].x), bez(q[0].y, q[1].y, q[2].y, q[3].y),
            bez(q[0].w, q[1].w, q[2].w, q[3].w)};
}

uint64_t to_count(float v) {  // Rust `as usize`: saturating, NaN -> 0
    if (!(v > 0.0f)) return 0;
    if (v >= 18446744073709551616.0f) return ~0ull;
    return (uint64_t)v;
}

// The first evaluated point pi in 1..last whose (float)pi exceeds the running curvature t
// (where the reference's walk leaves the quad of total t behind); last + 1 if none does.
uint64_t first_point_above(float t, uint64_t last) {
    if (!(t < (float)last)) return last + 1;
    uint64_t m = to_count(t) + 1;
    while (!((float)m > t)) ++m;  // at most half an ulp of t (t < 2^30) steps
    return m;
}

// Serial spline builder (path.rs:190-445). Splines are kept only as long as
// needed to emit their point commands at the end.
class SplineBuilder {
   public:
    void new_contour() { pending_contour_ = true; }  // push_contour, path.rs:248-250

    void line(WPt a, WPt b) {  // push_line, path.rs:252-269
        Pt p0 = a.applied(), p1 = b.applied();
        Angle ang = angle_of({p1.x - p0.x, p1.y - p0.y});
        Spline& s = current_spline(ang, p0, p0, p1);
        s.p2 = p1;
        last_angle_ = ang;
    }

    void quad(WPt q0, WPt q1, WPt q2) {  // push_quad, path.rs:271-347
        Pt p0 = q0.applied(), p1 = q1.applied(), p2 = q2.applied();
        Pt a{p1.x - p0.x, p1.y - p0.y}, b{p2.x - p1.x, p2.y - p1.y};
        Angle in = angle_of(a), out = angle_of(b);
        if (!in.some && !out.some) return;
        if (!in.some || !out.some) return line(q0, q2);

        QuadRec rec;
        const WPt* src[3] = {&q0, &q1, &q2};
        for (int i = 0; i < 3; ++i) {
            rec.px[i] = src[i]->x;
            rec.py[i] = src[i]->y;
            rec.pw[i] = src[i]->w;
        }
        Spline& s = current_spline(in, p0, p0, p2);
        s.p2 = p2;

        // Levien parameters (path.rs:296-332): quad_math.h, shared with the device, which
        // recomputes them from the control points instead of receiving them over PCIe.
        const QuadParams qp = quad_params(rec.px, rec.py, rec.pw);
        const float cur = qp.cur;
        float total = s.curvature + cur;
        s.curvature = total;
        last_angle_ = out;

        rec.x0 = qp.x0;
        rec.dx_recip = qp.dx_recip;
        rec.k0 = qp.k0;
        rec.dk = qp.dk;
        rec.curv_recip = rcp(cur);
        uint32_t spline_index = (uint32_t)splines_.size() - 1;
        rec.prev_curv = (!quad_spline_.empty() && quad_spline_.back() == spline_index) ? quad_total_.back() : 0.0f;
        rec.total = total;
        quads_.push_back(rec);
        quad_spline_.push_back(spline_index);
        quad_total_.push_back(total);
    }

    void cubic(const WPt q[4]) {  // push_cubic, path.rs:349-398
        const float max_err2 = (36.0f * 36.0f / 3.0f) * kMaxError * kMaxError;
        Pt p0 = q[0].applied(), p1 = q[1].applied(), p2 = q[2].applied();
        float dx = fmaf(p2.x, 3.0f, -p0.x) - fmaf(p1.x, 3.0f, -p1.x);
        float dy = fmaf(p2.y, 3.0f, -p0.y) - fmaf(p1.y, 3.0f, -p1.y);
        float err = fmaf(dx, dx, dy * dy);
        float mult = std::fmax(std::fmax(q[1].w, q[2].w), 1.0f);
        uint64_t n = to_count(std::ceil(powf(err * rcp(max_err2), 1.0f / 6.0f) * mult));
        if (n < 1) n = 1;
        float incr = rcp((float)n);
        Pt prev = p0;
        for (uint64_t i = 1; i <= n; ++i) {
            float t = (float)i * incr;
            Pt end = cubic_at(t, q).applied();
            Pt mid = cubic_at(t - 0.5f * incr, q).applied();
            Pt ctrl{fmaf(mid.x, 2.0f, -0.5f * (prev.x + end.x)), fmaf(mid.y, 2.0f, -0.5f * (prev.y + end.y))};
            quad({prev.x, prev.y, 1.0f}, {ctrl.x, ctrl.y, 1.0f}, {end.x, end.y, 1.0f});
            prev = end;
        }
    }

    // populate_buffers (path.rs:400-445) -> resolved point commands.
    void finish(FlattenProgram& out) {
        out.quads = std::move(quads_);
        for (const QuadRec& q : out.quads)
            if (q.pw[0] != 1.0f || q.pw[1] != 1.0f || q.pw[2] != 1.0f) out.rational = true;
        // The quads of a spline are contiguous; the reference walks them with one index for the
        // whole path: `if pi > total[qi] { qi += 1 }` per evaluated point, and `qi += 1` after
        // every spline with subdivisions (path.rs:424-445). While every quad raises the running
        // curvature by more than 1 (path.rs:322-332), that is "the first quad of the spline whose
        // running curvature reaches pi": the kernel (flatten_eval_kernel) finds it by bisection,
        // no per-point command needed. In f32 it is not always so: past 2^25 a quad can add
        // nothing (less than half an ulp, or a tie rounded to even), and from 2^23 on a quad can
        // add exactly 1. The walk then lags behind the bisection, or ends a spline before its
        // last quad and evaluates the next spline's points on this spline's quads. A program
        // where that happens records the walk point by point (`walk_lags`, kind 3 below).
        std::vector<uint32_t> quads_of(splines_.size(), 0u);
        for (uint32_t si : quad_spline_) quads_of[si] += 1;
        out.splines.reserve(splines_.size());
        bool walk_lags = false;
        uint64_t qi = 0, pt = 0;
        for (size_t si = 0; si < splines_.size(); ++si) {
            const Spline& s = splines_[si];
            uint64_t subdivisions = to_count(std::ceil(s.curvature));
            float step = s.curvature / (float)subdivisions;
            bool start = si == 0 || splines_[si - 1].ends_contour ||
                         length({splines_[si - 1].p2.x - s.p0.x, splines_[si - 1].p2.y - s.p0.y}) > kMaxError;
            uint64_t evaluated = subdivisions > 0 ? subdivisions - 1 : 0;
            if (evaluated > kSplineEvalMask) evaluated = kSplineEvalMask;
            SplineRec r;
            r.p0x = s.p0.x; r.p0y = s.p0.y; r.p2x = s.p2.x; r.p2y = s.p2.y;
            r.step = step;
            r.first_quad = (uint32_t)qi;
            r.n_quads = quads_of[si];
            r.first_point = (uint32_t)pt;
            r.info = (uint32_t)evaluated | (start ? 1u << 30 : 0u) | (s.ends_contour ? 1u << 31 : 0u);
            out.splines.push_back(r);
            for (uint32_t q = 0; q < quads_of[si]; ++q) out.quads[qi + q].step = step;
            // The walk keeps up with the bisection iff the evaluated points cross the quads' running
            // curvatures one quad at a time and reach the last quad: each quad but the last is left
            // behind at its own point.
            uint64_t crossed = 0;
            for (uint32_t q = 0; q + 1 < quads_of[si] && !walk_lags; ++q) {
                uint64_t p = first_point_above(out.quads[qi + q].total, evaluated);
                walk_lags = p > evaluated || p <= crossed;
                crossed = p;
            }
            pt += (start ? 1u : 0u) + evaluated + 1u;
            qi += quads_of[si];
            if (s.ends_contour && si + 1 < splines_.size()) out.n_contour_ends += 1;
        }
        out.n_points = (uint32_t)std::min<uint64_t>(pt, 0xFFFFFFFFull);
        {  // bounds (see FlattenProgram)
            float lo_x = INFINITY, lo_y = INFINITY, hi_x = -INFINITY, hi_y = -INFINITY;
            auto take = [&](float px, float py) {
                if (!(px == px) || !(py == py)) out.bounded = false;  // NaN
                lo_x = std::fmin(lo_x, px); hi_x = std::fmax(hi_x, px);
                lo_y = std::fmin(lo_y, py); hi_y = std::fmax(hi_y, py);
            };
            for (const SplineRec& r : out.splines) {
                take(r.p0x, r.p0y);
                take(r.p2x, r.p2y);
            }
            for (const QuadRec& q : out.quads)
                for (int k = 0; k < 3; ++k) {
                    if (!(q.pw[k] > 0.0f)) out.bounded = false;
                    else take(q.px[k] / q.pw[k], q.py[k] / q.pw[k]);
                }
            if (out.splines.empty() && out.quads.empty()) lo_x = lo_y = hi_x = hi_y = 0.0f;
            out.min_x = lo_x; out.min_y = lo_y; out.max_x = hi_x; out.max_y = hi_y;
        }
        // Paths made of short line splines are smaller point by point (9 B / point
        // against 36 B / spline): expand the records on the host in that case.
        if ((walk_lags || sizeof(SplineRec) * out.splines.size() > (sizeof(PointRec) + 1) * (size_t)out.n_points) &&
            pt < (1ull << 31)) {
            out.points.reserve(out.n_points);
            out.kinds.reserve(out.n_points);
            uint32_t wq = 0;  // the reference's walk; it stays within the quads of the spline being walked
            for (const SplineRec& r : out.splines) {
                if ((r.info >> 30) & 1u) {
                    out.points.push_back({r.p0x, r.p0y});
                    out.kinds.push_back(0);
                }
                const uint32_t evaluated = r.info & kSplineEvalMask;
                uint32_t q = r.first_quad;
                for (uint32_t pi = 1; pi <= evaluated; ++pi) {
                    PointRec p;
                    if (walk_lags) {
                        if ((float)pi > out.quads[wq].total) ++wq;
                        std::memcpy(&p.a, &wq, sizeof(uint32_t));
                        p.b = fmaf(r.step, (float)pi, -out.quads[wq].prev_curv);
                        out.kinds.push_back(3);
                    } else {
                        while (q + 1 < r.first_quad + r.n_quads && (float)pi > out.quads[q].total) ++q;
                        std::memcpy(&p.a, &q, sizeof(uint32_t));
                        p.b = (float)pi;
                        out.kinds.push_back(2);
                    }
                    out.points.push_back(p);
                }
                if (r.n_quads) ++wq;  // a spline with quads has subdivisions
                out.points.push_back({r.p2x, r.p2y});
                out.kinds.push_back((r.info >> 31) ? 1 : 0);
            }
            out.splines.clear();
            out.splines.shrink_to_fit();
        }
    }

   private:
    struct Spline {
        float curvature;
        Pt p0, p2;
        bool ends_contour;  // holds the contour token (path.rs:178)
    };

    // last_spline_or_insert_with, path.rs:208-246.
    Spline& current_spline(Angle ang, Pt at, Pt new_p0, Pt new_p2) {
        bool open_new = false;
        if (pending_contour_) {
            pending_contour_ = false;
            open_new = true;
        } else if (!splines_.empty()) {
            bool angle_changed = false;
            if (last_angle_.some && ang.some) {
                float d = std::fabs(ang.v - last_angle_.v);
                if (d > kPi) d -= kPi;
                if (d > kHalfPi) d = kPi - d;
                angle_changed = d > kMaxAngleError;
            }
            Spline& last = splines_.back();
            bool needed = angle_changed || length({at.x - last.p2.x, at.y - last.p2.y}) >= kMaxError;
            if (needed && last.ends_contour) {
                last.ends_contour = false;
                open_new = true;
            }
        }
        if (open_new) splines_.push_back({0.0f, new_p0, new_p2, true});
        return splines_.back();
    }

    bool pending_contour_ = true;  // Primitives::default(), path.rs:545
    Angle last_angle_{false, 0.0f};
    std::vector<Spline> splines_;
    std::vector<QuadRec> quads_;
    std::vector<uint32_t> quad_spline_;
    std::vector<float> quad_total_;
};

}  // namespace

bool geom_pres_ok(float ux, float uy, float vx, float vy) {
    const float max_x = 1.0f + kMaxError / 65536.0f;
    const float max_y = 1.0f + kMaxError / 32768.0f;
    return !(ux * ux + uy * uy > max_x) && !(vx * vx + vy * vy > max_y);
}

void PathData::close() {
    size_t n = x.size();
    WPt last{x[n - 1], y[n - 1], w[n - 1]};
    WPt open{x[open_index], y[open_index], w[open_index]};
    Pt a = last.applied(), b = open.applied();
    if (a.x != b.x || a.y != b.y) {
        x.push_back(open.x);
        y.push_back(open.y);
        w.push_back(open.w);
        cmd.push_back(1);
    }
}

const FlattenProgram& PathData::program() {
    if (built_) return prog_;
    SplineBuilder sb;
    size_t i = 0;
    auto at = [&](size_t k) { return WPt{x[k], y[k], w[k]}; };
    for (uint8_t c : cmd) {
        switch (c) {
            case 0:
                i += 1;
                sb.new_contour();
                break;
            case 1:
                i += 1;
                sb.line(at(i - 2), at(i - 1));
                break;
            case 2:
                i += 2;
                sb.quad(at(i - 3), at(i - 2), at(i - 1));
                break;
            default: {
                i += 3;
                WPt q[4] = {at(i - 4), at(i - 3), at(i - 2), at(i - 1)};
                sb.cubic(q);
            }
        }
    }
    sb.finish(prog_);
    built_ = true;
    return prog_;
}

Path Path::transformed(const float m[9]) const {
    // GeomPresTransform::new, math/transform.rs:161-182
    if (std::fabs(m[6]) <= kEps && std::fabs(m[7]) <= kEps) {
        float a[6] = {m[0], m[1], m[2], m[3], m[4], m[5]};
        if (std::fabs(m[8] - 1.0f) > kEps) {
            float r = rcp(m[8]);
            for (float& v : a) v *= r;
        }
        // ux = a0, vx = a1, tx = a2, uy = a3, vy = a4, ty = a5
        if (geom_pres_ok(a[0], a[3], a[1], a[4])) {
            Path p;
            p.data = data;
            p.has_xf = true;
            p.xf[0] = a[0];
            p.xf[1] = a[3];
            p.xf[2] = a[1];
            p.xf[3] = a[4];
            p.xf[4] = a[2];
            p.xf[5] = a[5];
            return p;
        }
    }
    // Projective / up-scaling transform: transform control points, re-flatten.
    auto d = std::make_shared<PathData>();
    d->x = data->x;
    d->y = data->y;
    d->w = data->w;
    d->cmd = data->cmd;
    d->open_index = data->open_index;
    for (size_t i = 0; i < d->x.size(); ++i) {
        float px = d->x[i], py = d->y[i], pw = d->w[i];
        d->x[i] = fmaf(m[0], px, fmaf(m[1], py, m[2] * pw));
        d->y[i] = fmaf(m[3], px, fmaf(m[4], py, m[5] * pw));
        d->w[i] = fmaf(m[6], px, fmaf(m[7], py, m[8] * pw));
    }
    Path p;
    p.data = d;
    return p;
}

void PathBuilder::move_to(Pt p) {
    PathData& d = *data;
    if (d.cmd.back() == 0) {
        d.x.back() = p.x;
        d.y.back() = p.y;
        d.w.back() = 1.0f;
        return;
    }
    d.close();
    d.open_index = d.x.size();
    d.x.push_back(p.x);
    d.y.push_back(p.y);
    d.w.push_back(1.0f);
    d.cmd.push_back(0);
}
void PathBuilder::line_to(Pt p) {
    data->x.push_back(p.x);
    data->y.push_back(p.y);
    data->w.push_back(1.0f);
    data->cmd.push_back(1);
}
void PathBuilder::quad_to(Pt p1, Pt p2) { rat_quad_to(p1, p2, 1.0f); }
void PathBuilder::cubic_to(Pt p1, Pt p2, Pt p3) { rat_cubic_to(p1, p2, p3, 1.0f, 1.0f); }
void PathBuilder::rat_quad_to(Pt p1, Pt p2, float weight) {
    PathData& d = *data;
    d.x.push_back(p1.x * weight);
    d.y.push_back(p1.y * weight);
    d.w.push_back(weight);
    d.x.push_back(p2.x);
    d.y.push_back(p2.y);
    d.w.push_back(1.0f);
    d.cmd.push_back(2);
}
void PathBuilder::rat_cubic_to(Pt p1, Pt p2, Pt p3, float w1, float w2) {
    PathData& d = *data;
    d.x.push_back(p1.x * w1);
    d.y.push_back(p1.y * w1);
    d.w.push_back(w1);
    d.x.push_back(p2.x * w2);
    d.y.push_back(p2.y * w2);
    d.w.push_back(w2);
    d.x.push_back(p3.x);
    d.y.push_back(p3.y);
    d.w.push_back(1.0f);
    d.cmd.push_back(3);
}
Path PathBuilder::build() {
    data->close();
    Path p;
    p.data = data;
    return p;
}

}  // namespace forma
