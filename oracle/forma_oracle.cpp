// ORACLE — TEST INFRASTRUCTURE ONLY (see fmath.hpp).
//
// C entry points (prefix `fo_`) over the CPU restatement. The shape of this
// API deliberately mirrors include/forma_b200.h so the same Python binding
// class can drive either library with the same scene-building code, the way
// the reference's e2e harness renders one Composition with two back-ends
// (e2e-tests/tests/test_env.rs:262-276).
//
// Build: see oracle/Makefile (-O2 -ffp-contract=off; OpenMP optional).
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <string>

#ifdef _OPENMP
#include <omp.h>
#endif

#include "painter.hpp"

namespace fo {

// Stand-in for crumsort::ParCrumSort (cpu/rasterizer.rs:162-164): LSD radix
// sort on key bits [20, 64), 11 bits per pass, parallel histogram/scatter with
// OpenMP. Stable, which is a legal outcome of an unstable sort.
void sort_segments(std::vector<uint64_t>& segs) {
    size_t n = segs.size();
    if (n < (1u << 14)) {
        std::sort(segs.begin(), segs.end(), [](uint64_t a, uint64_t b) { return (a >> kSortShift) < (b >> kSortShift); });
        return;
    }
    // The ping-pong buffer is kept between frames, like the reference keeps its segment
    // vector (cpu/renderer.rs:57): a fresh 8 n-byte allocation per frame costs more in page
    // faults than a radix pass.
    static thread_local std::vector<uint64_t> tmp;
    if (tmp.size() < n) tmp.resize(n);
    uint64_t* src = segs.data();
    uint64_t* dst = tmp.data();
    const int kRadixBits = 11, kBuckets = 1 << kRadixBits;
    int threads = 1;
#ifdef _OPENMP
    threads = omp_get_max_threads();
#endif
    std::vector<size_t> hist((size_t)threads * kBuckets);
    for (int shift = kSortShift; shift < 64; shift += kRadixBits) {
        std::fill(hist.begin(), hist.end(), 0);
        uint64_t all_or = 0, all_and = ~0ull;
#pragma omp parallel num_threads(threads) reduction(| : all_or) reduction(& : all_and)
        {
            int t = 0;
#ifdef _OPENMP
            t = omp_get_thread_num();
#endif
            size_t lo = n * t / threads, hi = n * (t + 1) / threads;
            size_t* h = hist.data() + (size_t)t * kBuckets;
            for (size_t i = lo; i < hi; ++i) {
                uint64_t d = (src[i] >> shift) & (kBuckets - 1);
                h[d]++;
                all_or |= d;
                all_and &= d;
            }
        }
        if (all_or == (all_and & (kBuckets - 1))) continue;  // single bucket: pass is the identity
        size_t sum = 0;
        for (int b = 0; b < kBuckets; ++b)
            for (int t = 0; t < threads; ++t) {
                size_t c = hist[(size_t)t * kBuckets + b];
                hist[(size_t)t * kBuckets + b] = sum;
                sum += c;
            }
#pragma omp parallel num_threads(threads)
        {
            int t = 0;
#ifdef _OPENMP
            t = omp_get_thread_num();
#endif
            size_t lo = n * t / threads, hi = n * (t + 1) / threads;
            size_t* h = hist.data() + (size_t)t * kBuckets;
            for (size_t i = lo; i < hi; ++i) {
                uint64_t d = (src[i] >> shift) & (kBuckets - 1);
                dst[h[d]++] = src[i];
            }
        }
        std::swap(src, dst);
    }
    if (src != segs.data()) std::memcpy(segs.data(), src, n * sizeof(uint64_t));
}

struct Timings {
    double line_setup_ms = 0, rasterize_ms = 0, sort_ms = 0, paint_ms = 0;
    uint64_t n_lines = 0, n_segments = 0;
};

struct Renderer {
    Lines lines;
    std::vector<uint64_t> segments;
    uint32_t caches_in_use = 0;
    Timings last;
};

static double now_ms() {
    using namespace std::chrono;
    return duration<double, std::milli>(steady_clock::now().time_since_epoch()).count();
}

// cpu/renderer.rs:75-224
// The reason the last call failed (fo_last_error).
static thread_local std::string g_error;

static void refuse_segments(const Lines& L) {
    g_error = std::to_string(L.total) + " pixel segments exceed the " + std::to_string(kSegmentLimit) +
              " that u32 prefix sums can index";
}

// Returns false, with nothing painted, when rasterize() refuses the frame.
static bool render(Renderer& r, Composition& comp, const RenderTarget& rt, const uint32_t channels_in[4],
                   const Color& clear_color, const Rect* crop, LayerCache* cache) {
    Channel ch[4];
    for (int k = 0; k < 4; ++k) {
        ch[k] = (Channel)channels_in[k];
        if (clear_color.a == 1.0f && ch[k] == kAlpha) ch[k] = kOne;
    }
    size_t wt = (rt.width + kTile - 1) / kTile, ht = (rt.height + kTile - 1) / kTile;
    if (cache) {
        cache->tiles.resize(wt * ht);
        if (!cache->has_size || cache->width != rt.width || cache->height != rt.height) {
            cache->has_size = true;
            cache->width = rt.width;
            cache->height = rt.height;
            cache->clear();
        }
    }
    comp.compact_geom();

    double t0 = now_ms();
    comp.fill_cpu_view(rt.width, rt.height, r.lines);
    double t1 = now_ms();
    if (!rasterize(r.lines, r.segments)) {
        refuse_segments(r.lines);
        return false;
    }
    double t2 = now_ms();
    sort_segments(r.segments);
    double t3 = now_ms();

    PropsSource props;
    props.index(comp.layers);
    props.has_cache = cache != nullptr;
    props.cache_id = cache ? cache->id : 0;

    // cpu/painter/mod.rs:719-778 (for_each_row) + :577-627 (print_row)
    const uint64_t* segs = r.segments.data();
    size_t n = r.segments.size();
    size_t first = std::partition_point(segs, segs + n, [](uint64_t s) { return seg_tile_y(s) < 0; }) - segs;
    std::vector<size_t> row_start(ht + 1);
    for (size_t j = 0; j <= ht; ++j) {
        row_start[j] = std::partition_point(segs + first, segs + n, [j](uint64_t s) { return (size_t)seg_tile_y(s) < j; }) - segs;
    }
    bool has_prev_clear = cache && cache->has_clear;
    Color prev_clear = cache ? cache->clear_color : Color();
#pragma omp parallel
    {
        Painter painter;
        Workbench wb;
#pragma omp for schedule(dynamic, 1)
        for (size_t j = 0; j < ht; ++j) {
            if (crop && !(j >= crop->vert0 && j < crop->vert1)) continue;
            paint_tile_row(painter, wb, j, segs + row_start[j], row_start[j + 1] - row_start[j], props, ch, clear_color,
                           has_prev_clear, prev_clear, cache ? cache->tiles.data() + j * wt : nullptr, rt, crop);
        }
    }
    double t4 = now_ms();

    if (cache) {
        cache->has_clear = true;
        cache->clear_color = clear_color;
        for (auto& kv : comp.layers) {
            if (kv.second->is_enabled) kv.second->is_unchanged |= (1u << cache->id);
            else kv.second->is_unchanged &= ~(1u << cache->id);
        }
    }
    r.last.line_setup_ms = t1 - t0;
    r.last.rasterize_ms = t2 - t1;
    r.last.sort_ms = t3 - t2;
    r.last.paint_ms = t4 - t3;
    r.last.n_lines = r.lines.size();
    r.last.n_segments = r.segments.size();
    return true;
}

}  // namespace fo

using namespace fo;

// Mirrors forma_props in include/forma_b200.h.
struct fo_color {
    float r, g, b, a;
};
struct fo_gradient_stop {
    fo_color color;
    float stop;  // < 0: unpositioned (GradientBuilder::color, styling.rs:84 NO_STOP)
};
struct fo_props {
    uint32_t fill_rule, func, clip_layers, is_clipped, blend_mode, fill_type;
    fo_color color;
    uint32_t gradient_type;
    float start[2], end[2];
    uint32_t n_stops;
    const fo_gradient_stop* stops;
    float tex_transform[6];  // ux, uy, vx, vy, tx, ty
    uint32_t tex_width, tex_height;
    const float* tex_linear_rgba;  // width*height*4, linear
};
struct fo_rect {
    uint64_t hor_start, hor_end, vert_start, vert_end;  // pixels; approximated to tiles
};
struct fo_timings {
    double line_setup_ms, rasterize_ms, sort_ms, paint_ms;
    uint64_t n_lines, n_segments;
};

extern "C" {

int fo_num_threads() {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

void fo_set_num_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#endif
}

void* fo_path_builder_new() { return new PathBuilder(); }
void fo_path_builder_free(void* pb) { delete (PathBuilder*)pb; }
void fo_path_builder_move_to(void* pb, float x, float y) { ((PathBuilder*)pb)->move_to({x, y}); }
void fo_path_builder_line_to(void* pb, float x, float y) { ((PathBuilder*)pb)->line_to({x, y}); }
void fo_path_builder_quad_to(void* pb, float x1, float y1, float x2, float y2) {
    ((PathBuilder*)pb)->quad_to({x1, y1}, {x2, y2});
}
void fo_path_builder_cubic_to(void* pb, float x1, float y1, float x2, float y2, float x3, float y3) {
    ((PathBuilder*)pb)->cubic_to({x1, y1}, {x2, y2}, {x3, y3});
}
void fo_path_builder_rat_quad_to(void* pb, float x1, float y1, float x2, float y2, float w) {
    ((PathBuilder*)pb)->rat_quad_to({x1, y1}, {x2, y2}, w);
}
void fo_path_builder_rat_cubic_to(void* pb, float x1, float y1, float x2, float y2, float x3, float y3, float w1,
                                  float w2) {
    ((PathBuilder*)pb)->rat_cubic_to({x1, y1}, {x2, y2}, {x3, y3}, w1, w2);
}
void fo_path_builder_extend(void* pbv, const uint8_t* cmds, uint64_t n_cmds, const float* p) {
    PathBuilder* pb = (PathBuilder*)pbv;
    for (uint64_t i = 0; i < n_cmds; ++i) {
        switch (cmds[i]) {
            case 0: pb->move_to({p[0], p[1]}); p += 2; break;
            case 1: pb->line_to({p[0], p[1]}); p += 2; break;
            case 2: pb->quad_to({p[0], p[1]}, {p[2], p[3]}); p += 4; break;
            default: pb->cubic_to({p[0], p[1]}, {p[2], p[3]}, {p[4], p[5]}); p += 6; break;
        }
    }
}
void* fo_path_builder_build(void* pb) { return new Path(((PathBuilder*)pb)->build()); }
void* fo_path_transform(const void* path, const float m[9]) { return new Path(((const Path*)path)->transformed(m)); }
void fo_path_free(void* p) { delete (Path*)p; }

// Flattened points of the path (transform applied when it is geometry-preserving).
int fo_path_segments(void* path, const float** x, const float** y, const uint8_t** contour, uint64_t* n) {
    Path* p = (Path*)path;
    const Segments& s = p->inner->segments();
    static thread_local Segments tmp;
    if (p->has_transform) {
        tmp = s;
        for (size_t i = 0; i < tmp.x.size(); ++i) {
            Point q = p->transform.apply({tmp.x[i], tmp.y[i]});
            tmp.x[i] = q.x;
            tmp.y[i] = q.y;
        }
        *x = tmp.x.data();
        *y = tmp.y.data();
        *contour = tmp.start_new_contour.data();
        *n = tmp.x.size();
    } else {
        *x = s.x.data();
        *y = s.y.data();
        *contour = s.start_new_contour.data();
        *n = s.x.size();
    }
    return 0;
}

void* fo_composition_new() { return new Composition(); }
void fo_composition_free(void* c) { delete (Composition*)c; }

// Layer handles stay valid until fo_layer_drop / fo_composition_free.
void* fo_composition_create_layer(void* c) { return ((Composition*)c)->create_layer(); }
void* fo_composition_insert(void* c, uint32_t order, void* layer, int* status) {
    if (order > kLayerLimit) {
        if (status) *status = 2;
        return nullptr;
    }
    if (status) *status = 0;
    return ((Composition*)c)->insert(order, (Layer*)layer);
}
void* fo_composition_remove(void* c, uint32_t order) { return ((Composition*)c)->remove(order); }
void* fo_composition_get(void* c, uint32_t order) { return ((Composition*)c)->get(order); }
void* fo_composition_get_mut_or_insert_default(void* c, uint32_t order, int* status) {
    if (order > kLayerLimit) {
        if (status) *status = 2;
        return nullptr;
    }
    if (status) *status = 0;
    return ((Composition*)c)->get_mut_or_insert_default(order);
}
uint64_t fo_composition_len(void* c) { return ((Composition*)c)->layers.size(); }
void fo_layer_drop(void* c, void* layer) { ((Composition*)c)->drop_layer((Layer*)layer); }
uint64_t fo_layer_geom_id(void* layer) { return ((Layer*)layer)->geom_id; }
int fo_layer_insert(void* c, void* layer, void* path) {
    ((Composition*)c)->layer_insert((Layer*)layer, *(Path*)path);
    return 0;
}
int fo_layer_clear(void* c, void* layer) {
    ((Composition*)c)->layer_clear((Layer*)layer);
    return 0;
}
int fo_layer_set_is_enabled(void* c, void* layer, int enabled) {
    ((Layer*)layer)->is_enabled = enabled != 0;
    return 0;
}
int fo_layer_is_enabled(void* layer) { return ((Layer*)layer)->is_enabled ? 1 : 0; }
// t = [ux, vx, uy, vy, tx, ty] as in GeomPresTransform::try_from([f32; 6]) /
// AffineTransform::from([f32; 6]) (math/transform.rs:92-103).
int fo_layer_set_transform(void* c, void* layer, const float t[6]) {
    Affine a;
    a.ux = t[0];
    a.vx = t[1];
    a.uy = t[2];
    a.vy = t[3];
    a.tx = t[4];
    a.ty = t[5];
    if (!geom_pres_ok(a)) return 1;
    Layer& l = *(Layer*)layer;
    bool has = !a.is_identity();
    bool same = has == l.has_transform && (!has || a == l.transform);
    if (!same) {
        l.is_unchanged = 0;
        l.has_transform = has;
        l.transform = a;
    }
    return 0;
}

static bool props_equal(const Props& a, const Props& b) {
    if (a.fill_rule != b.fill_rule || a.func != b.func) return false;
    if (a.func == kClip) return a.clip_layers == b.clip_layers;
    if (a.is_clipped != b.is_clipped || a.blend_mode != b.blend_mode || a.fill_type != b.fill_type) return false;
    if (a.fill_type == kSolid) return a.color == b.color;
    if (a.fill_type == kGradient) {
        const Gradient &g = a.gradient, &h = b.gradient;
        if (g.type != h.type || g.start != h.start || g.end != h.end || g.stops.size() != h.stops.size()) return false;
        for (size_t i = 0; i < g.stops.size(); ++i)
            if (!(g.stops[i].color == h.stops[i].color) || g.stops[i].stop != h.stops[i].stop) return false;
        return true;
    }
    return a.texture.image.data == b.texture.image.data && a.texture.transform == b.texture.transform;
}

int fo_layer_set_props(void* c, void* layer, const fo_props* p) {
    Props props;
    props.fill_rule = (FillRule)p->fill_rule;
    props.func = (FuncType)p->func;
    props.clip_layers = p->clip_layers;
    props.is_clipped = p->is_clipped != 0;
    props.blend_mode = (BlendMode)p->blend_mode;
    props.fill_type = (FillType)p->fill_type;
    props.color = {p->color.r, p->color.g, p->color.b, p->color.a};
    if (props.func == kDraw && props.fill_type == kGradient) {
        if (p->n_stops < 2) return 1;  // GradientBuilder::build -> None, styling.rs:107-109
        Gradient& g = props.gradient;
        g.type = (GradientType)p->gradient_type;
        g.start = {p->start[0], p->start[1]};
        g.end = {p->end[0], p->end[1]};
        float incr = 1.0f / (float)(p->n_stops - 1);
        for (uint32_t i = 0; i < p->n_stops; ++i) {
            const fo_gradient_stop& s = p->stops[i];
            float stop = s.stop;
            if (stop == -1.0f) stop = (float)i * incr;  // styling.rs:111-116
            else if (!(stop >= 0.0f && stop <= 1.0f)) return 1;
            g.stops.push_back({{s.color.r, s.color.g, s.color.b, s.color.a}, stop});
        }
    }
    if (props.func == kDraw && props.fill_type == kTexture) {
        size_t n = (size_t)p->tex_width * p->tex_height;
        auto data = std::make_shared<std::vector<uint16_t>>(n * 4);
        for (size_t i = 0; i < n * 4; ++i) (*data)[i] = f16_from(p->tex_linear_rgba[i]);
        // The same texels set again on a layer are the same image (the C ABI has no other way to
        // name an Image, whose PartialEq is by data pointer): the layer stays unchanged.
        const Props& old = ((Layer*)layer)->props;
        if (old.func == kDraw && old.fill_type == kTexture && old.texture.image.data && old.texture.image.width == p->tex_width &&
            *old.texture.image.data == *data)
            data = old.texture.image.data;
        Texture& t = props.texture;
        t.image.data = data;
        t.image.width = p->tex_width;
        t.image.max_x = (float)p->tex_width - 1.0f;
        t.image.max_y = (float)p->tex_height - 1.0f;
        t.transform.ux = p->tex_transform[0];
        t.transform.uy = p->tex_transform[1];
        t.transform.vx = p->tex_transform[2];
        t.transform.vy = p->tex_transform[3];
        t.transform.tx = p->tex_transform[4];
        t.transform.ty = p->tex_transform[5];
    }
    Layer& l = *(Layer*)layer;
    if (!props_equal(l.props, props)) {
        l.is_unchanged = 0;
        l.props = props;
    }
    return 0;
}

void* fo_renderer_new(int) { return new Renderer(); }
void fo_renderer_free(void* r) { delete (Renderer*)r; }

void* fo_layer_cache_new(void* rv) {
    Renderer* r = (Renderer*)rv;
    for (uint8_t id = 0; id < 32; ++id) {
        if (!((r->caches_in_use >> id) & 1)) {
            r->caches_in_use |= 1u << id;
            LayerCache* c = new LayerCache();
            c->id = id;
            return c;
        }
    }
    return nullptr;
}
void fo_layer_cache_free(void* rv, void* cv) {
    LayerCache* c = (LayerCache*)cv;
    if (rv) ((Renderer*)rv)->caches_in_use &= ~(1u << c->id);
    delete c;
}
void fo_layer_cache_clear(void* cv) { ((LayerCache*)cv)->clear(); }

int fo_renderer_render(void* rv, void* cv, uint8_t* buffer, uint64_t width, uint64_t stride, uint64_t height,
                       const uint32_t channels[4], const float clear[4], const fo_rect* crop, void* cache,
                       fo_timings* timings) {
    if (width * 4 > stride) return 1;
    Renderer* r = (Renderer*)rv;
    RenderTarget rt{buffer, (size_t)width, (size_t)height, (size_t)stride};
    Rect rect;
    if (crop) {
        rect.hor0 = crop->hor_start / kTile;
        rect.hor1 = (crop->hor_end + kTile - 1) / kTile;
        rect.vert0 = crop->vert_start / kTile;
        rect.vert1 = (crop->vert_end + kTile - 1) / kTile;
    }
    Color cc{clear[0], clear[1], clear[2], clear[3]};
    if (!render(*r, *(Composition*)cv, rt, channels, cc, crop ? &rect : nullptr, (LayerCache*)cache))
        return 5;  // FORMA_ERR_CAPACITY
    if (timings) {
        timings->line_setup_ms = r->last.line_setup_ms;
        timings->rasterize_ms = r->last.rasterize_ms;
        timings->sort_ms = r->last.sort_ms;
        timings->paint_ms = r->last.paint_ms;
        timings->n_lines = r->last.n_lines;
        timings->n_segments = r->last.n_segments;
    }
    return 0;
}

// --- stage-level access for parity tests -----------------------------------

// Lines of the last render (SoA, 10 arrays), copied out like forma_renderer_lines.
uint64_t fo_renderer_lines(void* rv, uint64_t cap, uint32_t* orders, float* x0, float* y0, float* dx, float* dy,
                           float* a, float* b, float* c, float* d, uint32_t* lengths) {
    Renderer* r = (Renderer*)rv;
    size_t n = std::min<size_t>(cap, r->lines.size());
    std::memcpy(orders, r->lines.orders.data(), n * 4);
    std::memcpy(x0, r->lines.x0.data(), n * 4);
    std::memcpy(y0, r->lines.y0.data(), n * 4);
    std::memcpy(dx, r->lines.dx.data(), n * 4);
    std::memcpy(dy, r->lines.dy.data(), n * 4);
    std::memcpy(a, r->lines.a.data(), n * 4);
    std::memcpy(b, r->lines.b.data(), n * 4);
    std::memcpy(c, r->lines.c.data(), n * 4);
    std::memcpy(d, r->lines.d.data(), n * 4);
    std::memcpy(lengths, r->lines.lengths.data(), n * 4);
    return r->lines.size();
}
// Sorted pixel segments of the last render.
uint64_t fo_renderer_segments(void* rv, uint64_t cap, uint64_t* segs) {
    Renderer* r = (Renderer*)rv;
    std::memcpy(segs, r->segments.data(), std::min<size_t>(cap, r->segments.size()) * 8);
    return r->segments.size();
}
// Line setup + rasterize only (unsorted output, reference emission order).
uint64_t fo_renderer_rasterize_only(void* rv, void* cv, uint64_t width, uint64_t height, uint64_t cap, uint64_t* segs) {
    Renderer* r = (Renderer*)rv;
    ((Composition*)cv)->fill_cpu_view(width, height, r->lines);
    if (!rasterize(r->lines, r->segments)) {
        refuse_segments(r->lines);
        return 0;
    }
    std::memcpy(segs, r->segments.data(), std::min<size_t>(cap, r->segments.size()) * 8);
    return r->segments.size();
}
int fo_renderer_sort_u64(void*, uint64_t* keys, uint64_t n) {
    std::vector<uint64_t> v(keys, keys + n);
    sort_segments(v);
    std::memcpy(keys, v.data(), n * sizeof(uint64_t));
    return 0;
}
uint64_t fo_renderer_launch_count(const void*) { return 0; }
const char* fo_last_error() { return g_error.c_str(); }

// --- small known-answer hooks (reference unit tests) ------------------------
float fo_find(int32_t i, float a, float b, float c, float d) {
    double sr = 1.0 / ((double)a + (double)b);
    return find_param(i, (double)a * sr, (double)b * sr, ((double)c - (double)d) * sr, a, b, c, d);
}
uint64_t fo_pack_segment(uint32_t layer, int32_t tx, int32_t ty, uint32_t lx, uint32_t ly, uint32_t dam, int32_t cover) {
    return pack_segment(layer, (int16_t)tx, (int16_t)ty, (uint8_t)lx, (uint8_t)ly, (uint8_t)dam, (int8_t)cover);
}
void fo_unpack_segment(uint64_t s, int32_t out[7]) {
    out[0] = (int32_t)seg_layer(s);
    out[1] = seg_tile_x(s);
    out[2] = seg_tile_y(s);
    out[3] = seg_local_x(s);
    out[4] = seg_local_y(s);
    out[5] = seg_double_area(s);
    out[6] = seg_cover(s);
}
void fo_to_srgb_bytes(const float color[4], uint8_t out[4]) { to_srgb_bytes(color, out); }
uint8_t fo_to_byte(float v) { return to_byte(v); }
void fo_blend_scalar(uint32_t mode, const float dst[4], const float src[4], float out[4]) {
    Color d{dst[0], dst[1], dst[2], dst[3]}, s{src[0], src[1], src[2], src[3]};
    Color o = scalar_blend::blend((BlendMode)mode, d, s);
    out[0] = o.r;
    out[1] = o.g;
    out[2] = o.b;
    out[3] = o.a;
}
void fo_blend_lane(uint32_t mode, const float dst[3], const float src[3], float out[3]) {
    lane_blend::blend((BlendMode)mode, dst[0], dst[1], dst[2], src[0], src[1], src[2], out);
}
// #[cfg(test)] SegmentBuffer::push (segment.rs:200-235): appends one raw line
// to the segment buffer, as the reference's rasterizer/painter unit tests do.
void fo_test_push_line(void* cv, void* lv, float x0, float y0, float x1, float y1) {
    Composition& c = *(Composition*)cv;
    uint64_t id = ((Layer*)lv)->geom_id;
    bool new_point = c.x.empty() || !(c.x.back() == x0 && c.y.back() == y0);
    if (new_point) {
        c.x.push_back(x0);
        c.y.push_back(y0);
    }
    c.x.push_back(x1);
    c.y.push_back(y1);
    if (c.ids.size() >= 2) {
        uint64_t prev = c.ids[c.ids.size() - 2];
        if (prev != 0 && prev != id) {
            c.ids.push_back(id);
            c.ids.push_back(0);
        } else {
            c.ids.pop_back();
            c.ids.push_back(id);
            c.ids.push_back(0);
        }
    } else {
        c.ids.push_back(id);
        c.ids.push_back(0);
    }
    c.geom_id_to_order[id] = ((Layer*)lv)->order;
}

// Direct access to Primitives, as the reference's path.rs unit tests use it.
void* fo_prim_new() { return new Primitives(); }
void fo_prim_free(void* p) { delete (Primitives*)p; }
void fo_prim_contour(void* p) { ((Primitives*)p)->push_contour(); }
void fo_prim_line(void* p, const float v[6]) {
    ((Primitives*)p)->push_line({{v[0], v[1]}, v[2]}, {{v[3], v[4]}, v[5]});
}
void fo_prim_quad(void* p, const float v[9]) {
    ((Primitives*)p)->push_quad({{v[0], v[1]}, v[2]}, {{v[3], v[4]}, v[5]}, {{v[6], v[7]}, v[8]});
}
void fo_prim_cubic(void* p, const float v[12]) {
    WPoint q[4] = {{{v[0], v[1]}, v[2]}, {{v[3], v[4]}, v[5]}, {{v[6], v[7]}, v[8]}, {{v[9], v[10]}, v[11]}};
    ((Primitives*)p)->push_cubic(q);
}
uint64_t fo_prim_segments(void* p, uint64_t cap, float* x, float* y, uint8_t* c) {
    Segments s = ((Primitives*)p)->into_segments();
    size_t n = std::min<size_t>(cap, s.x.size());
    for (size_t i = 0; i < n; ++i) {
        x[i] = s.x[i];
        y[i] = s.y[i];
        c[i] = s.start_new_contour[i];
    }
    return s.x.size();
}

void fo_set_recip_mode(int mode) { lane_blend::recip_mode() = mode; }
float fo_approx_atan2(float y, float x) { return approx_atan2(y, x); }
float fo_coverage(int32_t doubled_area, uint32_t fill_rule) { return Painter::coverage_of(doubled_area, (FillRule)fill_rule); }

}  // extern "C"
