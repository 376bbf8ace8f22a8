// forma_b200 — the C ABI of include/forma_b200.h, except the multi-GPU and sliced renderers
// (multi_renderer.cu) and errors and options (composition.cu).
#include <cstring>
#include <new>

#include "renderer.hpp"

using namespace forma;

struct forma_path_builder { PathBuilder b; };
struct forma_path { Path p; std::vector<float> x, y; std::vector<uint8_t> c; };
struct forma_layer_cache { LayerCache c; };

static Layer* L(forma_layer* l) { return reinterpret_cast<Layer*>(l); }
static forma_layer* H(Layer* l) { return reinterpret_cast<forma_layer*>(l); }

extern "C" {

forma_path_builder* forma_path_builder_new(void) {
    return guarded((forma_path_builder*)nullptr, [] { return new forma_path_builder(); });
}
void forma_path_builder_free(forma_path_builder* pb) { delete pb; }
void forma_path_builder_move_to(forma_path_builder* pb, float x, float y) {
    guarded_void([&] { pb->b.move_to({x, y}); });
}
void forma_path_builder_line_to(forma_path_builder* pb, float x, float y) {
    guarded_void([&] { pb->b.line_to({x, y}); });
}
void forma_path_builder_quad_to(forma_path_builder* pb, float x1, float y1, float x2, float y2) {
    guarded_void([&] { pb->b.quad_to({x1, y1}, {x2, y2}); });
}
void forma_path_builder_cubic_to(forma_path_builder* pb, float x1, float y1, float x2, float y2, float x3, float y3) {
    guarded_void([&] { pb->b.cubic_to({x1, y1}, {x2, y2}, {x3, y3}); });
}
void forma_path_builder_rat_quad_to(forma_path_builder* pb, float x1, float y1, float x2, float y2, float w) {
    guarded_void([&] { pb->b.rat_quad_to({x1, y1}, {x2, y2}, w); });
}
void forma_path_builder_rat_cubic_to(forma_path_builder* pb, float x1, float y1, float x2, float y2, float x3,
                                     float y3, float w1, float w2) {
    guarded_void([&] { pb->b.rat_cubic_to({x1, y1}, {x2, y2}, {x3, y3}, w1, w2); });
}
forma_path* forma_path_builder_build(forma_path_builder* pb) {
    return guarded((forma_path*)nullptr, [&] {
        std::unique_ptr<forma_path> p(new forma_path());
        p->p = pb->b.build();
        return p.release();
    });
}
forma_path* forma_path_transform(const forma_path* src, const float m[9]) {
    return guarded((forma_path*)nullptr, [&] {
        std::unique_ptr<forma_path> p(new forma_path());
        p->p = src->p.transformed(m);
        return p.release();
    });
}
void forma_path_free(forma_path* p) { delete p; }

void forma_path_program_stats(forma_path* p, uint64_t out[6]) {
    const FlattenProgram& prog = p->p.data->program();
    out[0] = prog.n_points;
    out[1] = prog.quads.size();
    out[2] = prog.splines.size();
    out[3] = prog.points.size();
    out[4] = prog.rational ? 1 : 0;
    out[5] = prog.n_contour_ends;
}

void forma_path_program_records(forma_path* p, const void** splines, uint64_t* n_splines, const void** points,
                                const uint8_t** kinds, uint64_t* n_records, const void** quads, uint64_t* n_quads,
                                int* bounded, float bounds[4]) {
    const FlattenProgram& prog = p->p.data->program();
    *splines = prog.splines.data();
    *n_splines = prog.splines.size();
    *points = prog.points.data();
    *kinds = prog.kinds.data();
    *n_records = prog.points.size();
    *quads = prog.quads.data();
    *n_quads = prog.quads.size();
    *bounded = prog.bounded ? 1 : 0;
    bounds[0] = prog.min_x;
    bounds[1] = prog.min_y;
    bounds[2] = prog.max_x;
    bounds[3] = prog.max_y;
}

// Evaluates the path's flatten program on the current device and copies the
// points back (inspection only; rendering never copies points to the host).
static int path_segments_impl(forma_path* p, const float** x, const float** y, const uint8_t** contour, uint64_t* n) {
    const FlattenProgram& prog = p->p.data->program();
    uint32_t count = prog.n_points;
    p->x.assign(count, 0.0f);
    p->y.assign(count, 0.0f);
    p->c.assign(count, 0);
    *n = count;
    *x = p->x.data();
    *y = p->y.data();
    *contour = p->c.data();
    if (!count) return FORMA_STATUS_OK;
    int dev_count = 0;
    if (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count == 0) {
        set_error("forma_path_segments: no CUDA device (flatten evaluation has no CPU fallback)");
        return FORMA_STATUS_NO_DEVICE;
    }
    DeviceBuffer<SplineRec> dc;
    DeviceBuffer<QuadRec> dq;
    DeviceBuffer<FlattenJob> dj;
    DeviceBuffer<float> dx, dy;
    DeviceBuffer<uint32_t> dg;
    FORMA_CUDA_TRY(dc.reserve(prog.splines.size() + 1));
    FORMA_CUDA_TRY(dq.reserve(prog.quads.size() + 1));
    FORMA_CUDA_TRY(dj.reserve(1));
    FORMA_CUDA_TRY(dx.reserve(count));
    FORMA_CUDA_TRY(dy.reserve(count));
    FORMA_CUDA_TRY(dg.reserve(count));
    FlattenJob job{};
    job.first_point = 0;
    job.quad_base = 0;
    job.spline_base = 0;
    job.n_splines = (uint32_t)prog.splines.size();
    job.geom_id = 1;
    job.xf_index = p->p.has_xf ? 1u : 0u;
    JobXf job_xf{};
    std::memcpy(job_xf.xf, p->p.xf, sizeof(job_xf.xf));
    DeviceBuffer<JobXf> dxf;
    FORMA_CUDA_TRY(dxf.reserve(1));
    FORMA_CUDA_TRY(cudaMemcpy(dxf.ptr, &job_xf, sizeof(job_xf), cudaMemcpyHostToDevice));
    DeviceBuffer<PointRec> dp;
    DeviceBuffer<uint8_t> dk;
    FORMA_CUDA_TRY(dp.reserve(prog.points.size() + 1));
    FORMA_CUDA_TRY(dk.reserve(prog.kinds.size() + 1));
    if (!prog.splines.empty())
        FORMA_CUDA_TRY(cudaMemcpy(dc.ptr, prog.splines.data(), prog.splines.size() * sizeof(SplineRec), cudaMemcpyHostToDevice));
    if (!prog.points.empty()) {
        FORMA_CUDA_TRY(cudaMemcpy(dp.ptr, prog.points.data(), prog.points.size() * sizeof(PointRec), cudaMemcpyHostToDevice));
        FORMA_CUDA_TRY(cudaMemcpy(dk.ptr, prog.kinds.data(), prog.kinds.size(), cudaMemcpyHostToDevice));
    }
    if (!prog.quads.empty()) {  // same route as rendering: upload the control points, expand on the device
        std::vector<QuadUp> ups(prog.quads.size());
        for (size_t q = 0; q < ups.size(); ++q) ups[q] = quad_upload(prog.quads[q]);
        DeviceBuffer<QuadUp> du;
        FORMA_CUDA_TRY(du.reserve(ups.size()));
        FORMA_CUDA_TRY(cudaMemcpy(du.ptr, ups.data(), ups.size() * sizeof(QuadUp), cudaMemcpyHostToDevice));
        launch_quad_expand(du.ptr, dq.ptr, (uint32_t)ups.size(), 0);
        FORMA_CUDA_TRY(cudaDeviceSynchronize());
    }
    FORMA_CUDA_TRY(cudaMemcpy(dj.ptr, &job, sizeof(job), cudaMemcpyHostToDevice));
    launch_flatten_eval(dc.ptr, dp.ptr, dk.ptr, dq.ptr, dj.ptr, dxf.ptr, 1, count, 0, dx.ptr, dy.ptr, dg.ptr, 0);
    FORMA_CUDA_TRY(cudaGetLastError());
    FORMA_CUDA_TRY(cudaMemcpy(p->x.data(), dx.ptr, count * sizeof(float), cudaMemcpyDeviceToHost));
    FORMA_CUDA_TRY(cudaMemcpy(p->y.data(), dy.ptr, count * sizeof(float), cudaMemcpyDeviceToHost));
    for (const SplineRec& s : prog.splines) {  // the end point of a spline that ends a contour
        uint32_t end = s.first_point + ((s.info >> 30) & 1u) + (s.info & kSplineEvalMask);
        if ((s.info >> 31) && end < count) p->c[end] = 1;
    }
    for (size_t i = 0; i < prog.kinds.size() && i < count; ++i) p->c[i] = prog.kinds[i] == 1u;
    return FORMA_STATUS_OK;
}
int forma_path_segments(forma_path* p, const float** x, const float** y, const uint8_t** contour, uint64_t* n) {
    return guarded((int)FORMA_STATUS_CAPACITY, [&] { return path_segments_impl(p, x, y, contour, n); });
}

forma_composition* forma_composition_new(void) {
    return guarded((forma_composition*)nullptr, [] { return new forma_composition(); });
}
void forma_composition_free(forma_composition* c) { delete c; }
forma_layer* forma_composition_create_layer(forma_composition* c) {
    return guarded((forma_layer*)nullptr, [&] { return H(c->c.create_layer()); });
}
forma_layer* forma_composition_insert(forma_composition* c, uint32_t order, forma_layer* layer, int* status) {
    if (order > kLayerLimit) {
        if (status) *status = FORMA_ERR_ORDER_LIMIT;
        return nullptr;
    }
    if (status) *status = FORMA_OK;
    return guarded((forma_layer*)nullptr, [&] { return H(c->c.insert(order, L(layer))); });
}
forma_layer* forma_composition_remove(forma_composition* c, uint32_t order) {
    return guarded((forma_layer*)nullptr, [&] { return H(c->c.remove(order)); });
}
forma_layer* forma_composition_get(forma_composition* c, uint32_t order) { return H(c->c.get(order)); }
forma_layer* forma_composition_get_mut_or_insert_default(forma_composition* c, uint32_t order, int* status) {
    if (order > kLayerLimit) {
        if (status) *status = FORMA_ERR_ORDER_LIMIT;
        return nullptr;
    }
    if (status) *status = FORMA_OK;
    return guarded((forma_layer*)nullptr, [&] { return H(c->c.get_or_insert_default(order)); });
}
uint64_t forma_composition_len(forma_composition* c) { return c->c.layers.size(); }
void forma_layer_drop(forma_composition* c, forma_layer* l) {
    guarded_void([&] { c->c.drop(L(l)); });
}

uint64_t forma_layer_geom_id(forma_layer* l) { return L(l)->geom_id; }
int forma_layer_insert(forma_composition* c, forma_layer* l, forma_path* p) {
    return guarded((int)FORMA_ERR_CAPACITY, [&] {
        c->c.layer_insert(L(l), p->p);
        return (int)FORMA_OK;
    });
}
int forma_layer_clear(forma_composition* c, forma_layer* l) {
    return guarded((int)FORMA_ERR_CAPACITY, [&] {
        c->c.layer_clear(L(l));
        return (int)FORMA_OK;
    });
}
int forma_layer_set_is_enabled(forma_composition* c, forma_layer* l, int enabled) {
    L(l)->enabled = enabled != 0;
    c->c.mark_dirty();
    return FORMA_OK;
}
int forma_layer_is_enabled(forma_layer* l) { return L(l)->enabled ? 1 : 0; }

int forma_layer_set_transform(forma_composition* c, forma_layer* l, const float t[6]) {
    // AffineTransform::from([f32; 6]): ux = t0, vx = t1, uy = t2, vy = t3, tx = t4, ty = t5
    float ux = t[0], vx = t[1], uy = t[2], vy = t[3], tx = t[4], ty = t[5];
    if (!geom_pres_ok(ux, uy, vx, vy)) {
        set_error("GeomPresTransformError::ExceededScalingFactor");
        return FORMA_ERR_INVALID_ARGUMENT;
    }
    Layer* layer = L(l);
    bool has = !(ux == 1.0f && uy == 0.0f && vx == 0.0f && vy == 1.0f && tx == 0.0f && ty == 0.0f);
    float xf[6] = {ux, uy, vx, vy, tx, ty};
    bool same = has == layer->has_xf && (!has || std::memcmp(xf, layer->xf, sizeof(xf)) == 0 ||
                                         (xf[0] == layer->xf[0] && xf[1] == layer->xf[1] && xf[2] == layer->xf[2] &&
                                          xf[3] == layer->xf[3] && xf[4] == layer->xf[4] && xf[5] == layer->xf[5]));
    if (!same) {  // layer.rs:294-299
        layer->unchanged_bits = 0;
        layer->has_xf = has;
        std::memcpy(layer->xf, xf, sizeof(xf));
        c->c.mark_dirty();
    }
    return FORMA_OK;
}

// styling.rs:224-249 — forma's own f16 (no denormals, values in [0, 1]).
static uint16_t f16_from(float v) {
    if (v == 0.0f) return 0;
    uint32_t u;
    std::memcpy(&u, &v, 4);
    return (uint16_t)((u - 0x38000000u) >> 13);
}

static int layer_set_props_impl(forma_composition* c, forma_layer* l, const forma_props* p) {
    HostProps hp;
    StyleRec& s = hp.rec;
    s.fill_rule = p->fill_rule;
    s.func = p->func;
    s.clip_layers = p->clip_layers;
    s.is_clipped = p->is_clipped ? 1u : 0u;
    s.blend_mode = p->blend_mode;
    s.fill_type = p->fill_type;
    if (s.fill_rule > 1u || s.func > 1u || s.blend_mode > 15u || s.fill_type > 2u) {
        set_error("forma_layer_set_props: enum value out of range");
        return FORMA_ERR_INVALID_ARGUMENT;
    }
    s.color[0] = p->color.r; s.color[1] = p->color.g; s.color[2] = p->color.b; s.color[3] = p->color.a;
    if (s.func == FORMA_FUNC_DRAW && s.fill_type == FORMA_FILL_GRADIENT) {
        if (p->n_stops < 2 || !p->stops) {  // GradientBuilder::build -> None, styling.rs:107-109
            set_error("a gradient needs at least 2 stops");
            return FORMA_ERR_INVALID_ARGUMENT;
        }
        s.gradient_type = p->gradient_type;
        s.start[0] = p->start[0]; s.start[1] = p->start[1];
        s.end[0] = p->end[0]; s.end[1] = p->end[1];
        float incr = 1.0f / (float)(p->n_stops - 1);
        for (uint32_t i = 0; i < p->n_stops; ++i) {
            StopRec r;
            r.color[0] = p->stops[i].color.r; r.color[1] = p->stops[i].color.g;
            r.color[2] = p->stops[i].color.b; r.color[3] = p->stops[i].color.a;
            float stop = p->stops[i].stop;
            if (stop == -1.0f) stop = (float)i * incr;  // styling.rs:111-116
            else if (!(stop >= 0.0f && stop <= 1.0f)) {
                set_error("gradient stops must be between 0.0 and 1.0");
                return FORMA_ERR_INVALID_ARGUMENT;
            }
            r.stop = stop;
            hp.stops.push_back(r);
        }
    }
    if (s.func == FORMA_FUNC_DRAW && s.fill_type == FORMA_FILL_TEXTURE) {
        size_t n = (size_t)p->tex_width * p->tex_height;
        if (!n || !p->tex_linear_rgba) {
            set_error("empty texture");
            return FORMA_ERR_INVALID_ARGUMENT;
        }
        // Reuse the texel block when the same image is set again on this layer.
        auto tex = std::make_shared<std::vector<uint16_t>>(n * 4);
        for (size_t i = 0; i < n * 4; ++i) (*tex)[i] = f16_from(p->tex_linear_rgba[i]);
        Layer* layer = L(l);
        if (layer->props.texels && *layer->props.texels == *tex) tex = layer->props.texels;
        hp.texels = tex;
        for (int i = 0; i < 6; ++i) s.tex_xf[i] = p->tex_transform[i];
        s.tex_width = p->tex_width;
        s.tex_max_x = (float)p->tex_width - 1.0f;
        s.tex_max_y = (float)p->tex_height - 1.0f;
    }
    Layer* layer = L(l);
    if (!layer->props.equals(hp)) {  // layer.rs:341-348
        layer->unchanged_bits = 0;
        layer->props = std::move(hp);
        c->c.mark_dirty();
    }
    return FORMA_OK;
}
int forma_layer_set_props(forma_composition* c, forma_layer* l, const forma_props* p) {
    return guarded((int)FORMA_ERR_CAPACITY, [&] { return layer_set_props_impl(c, l, p); });
}

static forma_renderer* renderer_new_impl(int device_ordinal) {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        set_error("no CUDA device available (%s); forma_b200 has no CPU fallback",
                  e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
        return nullptr;
    }
    if (device_ordinal < 0 || device_ordinal >= count) {
        set_error("device ordinal %d out of range (0..%d)", device_ordinal, count - 1);
        return nullptr;
    }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device_ordinal) != cudaSuccess || prop.major != 9 || prop.minor != 0) {
        set_error("device %d is sm_%d%d; this library is built for sm_90a only", device_ordinal, prop.major, prop.minor);
        return nullptr;
    }
    if (cudaSetDevice(device_ordinal) != cudaSuccess) {
        set_error("cudaSetDevice(%d) failed", device_ordinal);
        return nullptr;
    }
    forma_renderer* r = new forma_renderer();
    r->r.device = device_ordinal;
    r->r.res_key = device_ordinal;
    if (cudaMallocHost(&r->r.pinned_totals, 16 * sizeof(uint32_t)) != cudaSuccess || r->r.totals.reserve(64) != cudaSuccess ||
        cudaMemset(r->r.totals.ptr, 0, r->r.totals.capacity * sizeof(uint32_t)) != cudaSuccess) {
        set_error("allocation of renderer state failed");
        delete r;
        return nullptr;
    }
    return r;
}
forma_renderer* forma_renderer_new(int device_ordinal) {
    return guarded((forma_renderer*)nullptr, [&] { return renderer_new_impl(device_ordinal); });
}
void forma_renderer_free(forma_renderer* r) { delete r; }

void forma_renderer_set_stream(forma_renderer* r, void* cuda_stream) { r->r.stream = (cudaStream_t)cuda_stream; }

forma_layer_cache* forma_layer_cache_new(forma_renderer* r) {
    for (uint8_t id = 0; id < 32; ++id)
        if (!((r->r.caches_in_use >> id) & 1u)) {
            forma_layer_cache* c = new (std::nothrow) forma_layer_cache();
            if (!c) {
                set_error("forma_layer_cache_new: out of host memory");
                return nullptr;
            }
            r->r.caches_in_use |= 1u << id;
            c->c.id = id;
            return c;
        }
    set_error("forma_layer_cache_new: all 32 cache ids of this renderer are in use");
    return nullptr;
}
void forma_layer_cache_free(forma_renderer* r, forma_layer_cache* c) {
    if (r) r->r.caches_in_use &= ~(1u << c->c.id);
    delete c;
}
void forma_layer_cache_clear(forma_layer_cache* c) {
    if (c) c->c.clear();
}

// Every render entry point fills a FrameRequest and calls render_request(): the Compositions behind the
// handles (null batch entries stay null for Renderer::render to refuse), the sliced host-frame
// pipeline first for a host RGBA frame without a layer cache, and no C++ exception across the ABI.
// ids_fn: the name of an ID entry point, which is refused without an ID buffer (the Renderer would
// take the call for an RGBA-only request).
static int render_request(forma_renderer* r, FrameRequest q, forma_composition* c, forma_composition* const* comps = nullptr,
                          const char* ids_fn = nullptr) {
    return guarded((int)FORMA_ERR_CAPACITY, [&] {
        if (ids_fn && !q.ids.ptr) {
            set_error("%s: no ID buffer", ids_fn);
            return (int)FORMA_STATUS_INVALID;
        }
        std::vector<Composition*> cs(comps ? q.n : 0u);
        for (size_t k = 0; k < cs.size(); ++k) cs[k] = comps[k] ? &comps[k]->c : nullptr;
        q.comp = c ? &c->c : nullptr;
        q.batch = comps ? cs.data() : nullptr;
        if (q.kind == FrameKind::single && q.rgba.ptr && q.rgba.bpp == 4u && !q.rgba.on_device && !q.cache) {
            const int st = sliced_host_render(r, q);
            if (st >= 0) return st;
        }
        return r->r.render(q);
    });
}
int forma_renderer_render(forma_renderer* r, forma_composition* c, uint8_t* buffer, uint64_t width, uint64_t stride,
                          uint64_t height, const uint32_t channels[4], const float clear[4], const forma_rect* crop,
                          forma_layer_cache* cache, forma_timings* timings) {
    FrameRequest q{FrameKind::single, 0, width, height, channels, clear, timings, crop, cache ? &cache->c : nullptr};
    q.rgba = {buffer, false, stride};
    return render_request(r, q, c);
}
int forma_renderer_render_device(forma_renderer* r, forma_composition* c, uint8_t* device_buffer, uint64_t width,
                                 uint64_t stride, uint64_t height, const uint32_t channels[4], const float clear[4],
                                 const forma_rect* crop, forma_layer_cache* cache, forma_timings* timings) {
    FrameRequest q{FrameKind::single, 0, width, height, channels, clear, timings, crop, cache ? &cache->c : nullptr};
    q.rgba = {device_buffer, true, stride};
    return render_request(r, q, c);
}
int forma_renderer_render_ids(forma_renderer* r, forma_composition* c, uint32_t* ids, uint64_t width, uint64_t ids_stride,
                              uint64_t height, const forma_rect* crop, float min_coverage, forma_timings* timings) {
    FrameRequest q{FrameKind::single, 0, width, height, nullptr, nullptr, timings, crop};
    q.ids = {reinterpret_cast<uint8_t*>(ids), false, ids_stride, 0, min_coverage};
    return render_request(r, q, c, nullptr, __func__);
}
int forma_renderer_render_ids_device(forma_renderer* r, forma_composition* c, uint32_t* device_ids, uint64_t width,
                                     uint64_t ids_stride, uint64_t height, const forma_rect* crop, float min_coverage,
                                     forma_timings* timings) {
    FrameRequest q{FrameKind::single, 0, width, height, nullptr, nullptr, timings, crop};
    q.ids = {reinterpret_cast<uint8_t*>(device_ids), true, ids_stride, 0, min_coverage};
    return render_request(r, q, c, nullptr, __func__);
}
int forma_renderer_render_device_with_ids(forma_renderer* r, forma_composition* c, uint8_t* device_buffer, uint64_t width,
                                          uint64_t width_stride, uint64_t height, const uint32_t channels[4],
                                          const float clear_color[4], const forma_rect* crop, uint32_t* device_ids,
                                          uint64_t ids_stride, float min_coverage, forma_timings* timings) {
    if (!device_buffer) {  // (without one, the call would be forma_renderer_render_ids_device)
        set_error("forma_renderer_render_device_with_ids: no RGBA buffer");
        return FORMA_STATUS_INVALID;
    }
    FrameRequest q{FrameKind::single, 0, width, height, channels, clear_color, timings, crop};
    q.rgba = {device_buffer, true, width_stride};
    q.ids = {reinterpret_cast<uint8_t*>(device_ids), true, ids_stride, 0, min_coverage};
    return render_request(r, q, c, nullptr, __func__);
}
uint32_t forma_renderer_max_views(uint64_t height) { return max_views(height); }
int forma_renderer_render_views_device(forma_renderer* r, forma_composition* c, const float* views, uint32_t n, uint8_t* device_buffer,
                                       uint64_t width, uint64_t width_stride, uint64_t height, uint64_t view_stride,
                                       const uint32_t channels[4], const float clear_color[4], forma_timings* timings) {
    FrameRequest q{FrameKind::views, n, width, height, channels, clear_color, timings};
    q.views = views;
    q.rgba = {device_buffer, true, width_stride, view_stride};
    return render_request(r, q, c);
}
int forma_renderer_render_views(forma_renderer* r, forma_composition* c, const float* views, uint32_t n, uint8_t* host_buffer,
                                uint64_t width, uint64_t width_stride, uint64_t height, uint64_t view_stride,
                                const uint32_t channels[4], const float clear_color[4], forma_timings* timings) {
    FrameRequest q{FrameKind::views, n, width, height, channels, clear_color, timings};
    q.views = views;
    q.rgba = {host_buffer, false, width_stride, view_stride};
    return render_request(r, q, c);
}
// Poses: the twins of the views calls, with the pose tables in place of the view transforms.
static FrameRequest poses_request(const forma_poses* poses, uint32_t n, uint64_t width, uint64_t height, const uint32_t* channels,
                                  const float* clear_color, forma_timings* timings) {
    FrameRequest q{FrameKind::poses, n, width, height, channels, clear_color, timings};
    q.poses = poses;
    return q;
}
int forma_renderer_render_poses_device(forma_renderer* r, forma_composition* c, const forma_poses* poses, uint32_t n,
                                       uint8_t* device_buffer, uint64_t width, uint64_t width_stride, uint64_t height,
                                       uint64_t view_stride, const uint32_t channels[4], const float clear_color[4],
                                       forma_timings* timings) {
    FrameRequest q = poses_request(poses, n, width, height, channels, clear_color, timings);
    q.rgba = {device_buffer, true, width_stride, view_stride};
    return render_request(r, q, c);
}
int forma_renderer_render_poses(forma_renderer* r, forma_composition* c, const forma_poses* poses, uint32_t n, uint8_t* host_buffer,
                                uint64_t width, uint64_t width_stride, uint64_t height, uint64_t view_stride,
                                const uint32_t channels[4], const float clear_color[4], forma_timings* timings) {
    FrameRequest q = poses_request(poses, n, width, height, channels, clear_color, timings);
    q.rgba = {host_buffer, false, width_stride, view_stride};
    return render_request(r, q, c);
}
int forma_renderer_render_poses_ids_device(forma_renderer* r, forma_composition* c, const forma_poses* poses, uint32_t n,
                                           uint8_t* device_buffer, uint64_t width, uint64_t width_stride, uint64_t height,
                                           uint64_t view_stride, const uint32_t channels[4], const float clear_color[4],
                                           uint32_t* device_ids, uint64_t ids_stride, uint64_t ids_view_stride, float min_coverage,
                                           forma_timings* timings) {
    FrameRequest q = poses_request(poses, n, width, height, channels, clear_color, timings);
    q.rgba = {device_buffer, true, width_stride, view_stride};
    q.ids = {reinterpret_cast<uint8_t*>(device_ids), true, ids_stride, ids_view_stride, min_coverage};
    return render_request(r, q, c, nullptr, __func__);
}
int forma_renderer_render_poses_ids(forma_renderer* r, forma_composition* c, const forma_poses* poses, uint32_t n, uint32_t* host_ids,
                                    uint64_t width, uint64_t ids_stride, uint64_t height, uint64_t ids_view_stride,
                                    float min_coverage, forma_timings* timings) {
    FrameRequest q = poses_request(poses, n, width, height, nullptr, nullptr, timings);
    q.ids = {reinterpret_cast<uint8_t*>(host_ids), false, ids_stride, ids_view_stride, min_coverage};
    return render_request(r, q, c, nullptr, __func__);
}
// Instances: the twins of the views calls, with the instance tables in place of the view transforms.
static FrameRequest instances_request(const forma_instances* instances, uint32_t n, uint64_t width, uint64_t height,
                                      const uint32_t* channels, const float* clear_color, forma_timings* timings) {
    FrameRequest q{FrameKind::instances, n, width, height, channels, clear_color, timings};
    q.instances = instances;
    return q;
}
int forma_renderer_render_instances_device(forma_renderer* r, forma_composition* c, const forma_instances* instances, uint32_t n,
                                           uint8_t* device_buffer, uint64_t width, uint64_t width_stride, uint64_t height,
                                           uint64_t view_stride, const uint32_t channels[4], const float clear_color[4],
                                           forma_timings* timings) {
    FrameRequest q = instances_request(instances, n, width, height, channels, clear_color, timings);
    q.rgba = {device_buffer, true, width_stride, view_stride};
    return render_request(r, q, c);
}
int forma_renderer_render_instances_ids_device(forma_renderer* r, forma_composition* c, const forma_instances* instances, uint32_t n,
                                               uint8_t* device_buffer, uint64_t width, uint64_t width_stride, uint64_t height,
                                               uint64_t view_stride, const uint32_t channels[4], const float clear_color[4],
                                               uint32_t* device_ids, uint64_t ids_stride, uint64_t ids_view_stride, float min_coverage,
                                               forma_timings* timings) {
    FrameRequest q = instances_request(instances, n, width, height, channels, clear_color, timings);
    q.rgba = {device_buffer, true, width_stride, view_stride};
    q.ids = {reinterpret_cast<uint8_t*>(device_ids), true, ids_stride, ids_view_stride, min_coverage};
    return render_request(r, q, c, nullptr, __func__);
}
int forma_renderer_render_batch_device(forma_renderer* r, forma_composition* const* comps, uint32_t n, uint8_t* device_buffer,
                                       uint64_t width, uint64_t width_stride, uint64_t height, uint64_t frame_stride,
                                       const uint32_t channels[4], const float clear_color[4], forma_timings* timings) {
    FrameRequest q{FrameKind::batch, n, width, height, channels, clear_color, timings};
    q.rgba = {device_buffer, true, width_stride, frame_stride};
    return render_request(r, q, nullptr, comps);
}
int forma_renderer_render_batch(forma_renderer* r, forma_composition* const* comps, uint32_t n, uint8_t* host_buffer, uint64_t width,
                                uint64_t width_stride, uint64_t height, uint64_t frame_stride, const uint32_t channels[4],
                                const float clear_color[4], forma_timings* timings) {
    FrameRequest q{FrameKind::batch, n, width, height, channels, clear_color, timings};
    q.rgba = {host_buffer, false, width_stride, frame_stride};
    return render_request(r, q, nullptr, comps);
}
int forma_renderer_render_views_ids_device(forma_renderer* r, forma_composition* c, const float* views, uint32_t n,
                                           uint8_t* device_buffer, uint64_t width, uint64_t width_stride, uint64_t height,
                                           uint64_t view_stride, const uint32_t channels[4], const float clear_color[4],
                                           uint32_t* device_ids, uint64_t ids_stride, uint64_t ids_view_stride, float min_coverage,
                                           forma_timings* timings) {
    FrameRequest q{FrameKind::views, n, width, height, channels, clear_color, timings};
    q.views = views;
    q.rgba = {device_buffer, true, width_stride, view_stride};
    q.ids = {reinterpret_cast<uint8_t*>(device_ids), true, ids_stride, ids_view_stride, min_coverage};
    return render_request(r, q, c, nullptr, __func__);
}
int forma_renderer_render_views_ids(forma_renderer* r, forma_composition* c, const float* views, uint32_t n, uint32_t* host_ids,
                                    uint64_t width, uint64_t ids_stride, uint64_t height, uint64_t ids_view_stride,
                                    float min_coverage, forma_timings* timings) {
    FrameRequest q{FrameKind::views, n, width, height, nullptr, nullptr, timings};
    q.views = views;
    q.ids = {reinterpret_cast<uint8_t*>(host_ids), false, ids_stride, ids_view_stride, min_coverage};
    return render_request(r, q, c, nullptr, __func__);
}
int forma_renderer_render_batch_ids_device(forma_renderer* r, forma_composition* const* comps, uint32_t n, uint8_t* device_buffer,
                                           uint64_t width, uint64_t width_stride, uint64_t height, uint64_t frame_stride,
                                           const uint32_t channels[4], const float clear_color[4], uint32_t* device_ids,
                                           uint64_t ids_stride, uint64_t ids_frame_stride, float min_coverage,
                                           forma_timings* timings) {
    FrameRequest q{FrameKind::batch, n, width, height, channels, clear_color, timings};
    q.rgba = {device_buffer, true, width_stride, frame_stride};
    q.ids = {reinterpret_cast<uint8_t*>(device_ids), true, ids_stride, ids_frame_stride, min_coverage};
    return render_request(r, q, nullptr, comps, __func__);
}
int forma_renderer_render_batch_ids(forma_renderer* r, forma_composition* const* comps, uint32_t n, uint32_t* host_ids, uint64_t width,
                                    uint64_t ids_stride, uint64_t height, uint64_t ids_frame_stride, float min_coverage,
                                    forma_timings* timings) {
    FrameRequest q{FrameKind::batch, n, width, height, nullptr, nullptr, timings};
    q.ids = {reinterpret_cast<uint8_t*>(host_ids), false, ids_stride, ids_frame_stride, min_coverage};
    return render_request(r, q, nullptr, comps, __func__);
}
// Layer coverage masks: the masks target from the descriptor (a null descriptor or pointer is
// refused here, the rest by Renderer::check_request), with or without the RGBA target.
static int render_masks(forma_renderer* r, FrameRequest q, const forma_masks* masks, bool on_device, uint8_t* device_buffer,
                        uint64_t width_stride, uint64_t frame_stride, forma_composition* c, forma_composition* const* comps,
                        const char* fn) {
    if (!masks || !masks->ptr) {
        set_error("%s: no %s", fn, masks ? "mask buffer" : "mask descriptor");
        return FORMA_STATUS_INVALID;
    }
    q.masks = MaskTarget{static_cast<uint8_t*>(masks->ptr), on_device, masks->first_order, masks->n_orders, masks->format,
                         masks->stride, masks->plane_stride};
    if (device_buffer) q.rgba = {device_buffer, true, width_stride, frame_stride};
    else q.channels = nullptr, q.clear = nullptr;
    return render_request(r, q, c, comps);
}
int forma_renderer_render_masks(forma_renderer* r, forma_composition* c, const forma_masks* masks, uint64_t width, uint64_t height,
                                const forma_rect* crop, forma_timings* timings) {
    FrameRequest q{FrameKind::single, 0, width, height, nullptr, nullptr, timings, crop};
    return render_masks(r, q, masks, false, nullptr, 0, 0, c, nullptr, __func__);
}
int forma_renderer_render_masks_device(forma_renderer* r, forma_composition* c, const forma_masks* masks, uint64_t width,
                                       uint64_t height, const forma_rect* crop, uint8_t* device_buffer, uint64_t width_stride,
                                       const uint32_t channels[4], const float clear_color[4], forma_timings* timings) {
    FrameRequest q{FrameKind::single, 0, width, height, channels, clear_color, timings, crop};
    return render_masks(r, q, masks, true, device_buffer, width_stride, 0, c, nullptr, __func__);
}
int forma_renderer_render_views_masks_device(forma_renderer* r, forma_composition* c, const float* views, uint32_t n,
                                             const forma_masks* masks, uint64_t width, uint64_t height, uint8_t* device_buffer,
                                             uint64_t width_stride, uint64_t view_stride, const uint32_t channels[4],
                                             const float clear_color[4], forma_timings* timings) {
    FrameRequest q{FrameKind::views, n, width, height, channels, clear_color, timings};
    q.views = views;
    return render_masks(r, q, masks, true, device_buffer, width_stride, view_stride, c, nullptr, __func__);
}
int forma_renderer_render_poses_masks_device(forma_renderer* r, forma_composition* c, const forma_poses* poses, uint32_t n,
                                             const forma_masks* masks, uint64_t width, uint64_t height, uint8_t* device_buffer,
                                             uint64_t width_stride, uint64_t view_stride, const uint32_t channels[4],
                                             const float clear_color[4], forma_timings* timings) {
    FrameRequest q = poses_request(poses, n, width, height, channels, clear_color, timings);
    return render_masks(r, q, masks, true, device_buffer, width_stride, view_stride, c, nullptr, __func__);
}
int forma_renderer_render_instances_masks_device(forma_renderer* r, forma_composition* c, const forma_instances* instances, uint32_t n,
                                                 const forma_masks* masks, uint64_t width, uint64_t height, uint8_t* device_buffer,
                                                 uint64_t width_stride, uint64_t view_stride, const uint32_t channels[4],
                                                 const float clear_color[4], forma_timings* timings) {
    FrameRequest q = instances_request(instances, n, width, height, channels, clear_color, timings);
    return render_masks(r, q, masks, true, device_buffer, width_stride, view_stride, c, nullptr, __func__);
}
int forma_renderer_render_batch_masks_device(forma_renderer* r, forma_composition* const* comps, uint32_t n,
                                             const forma_masks* masks, uint64_t width, uint64_t height, uint8_t* device_buffer,
                                             uint64_t width_stride, uint64_t frame_stride, const uint32_t channels[4],
                                             const float clear_color[4], forma_timings* timings) {
    FrameRequest q{FrameKind::batch, n, width, height, channels, clear_color, timings};
    return render_masks(r, q, masks, true, device_buffer, width_stride, frame_stride, nullptr, comps, __func__);
}
// Layer statistics: the statistics target from the descriptor (a null descriptor or pointer is
// refused here, the rest by Renderer::check_request), with or without the RGBA target.
static int render_stats(forma_renderer* r, FrameRequest q, const forma_stats* stats, bool on_device, uint8_t* device_buffer,
                        uint64_t width_stride, uint64_t frame_stride, forma_composition* c, forma_composition* const* comps,
                        const char* fn) {
    if (!stats || !stats->ptr) {
        set_error("%s: no %s", fn, stats ? "record array" : "statistics descriptor");
        return FORMA_STATUS_INVALID;
    }
    q.stats = StatsTarget{stats->ptr, on_device, stats->first_order, stats->n_orders, stats->min_coverage};
    if (device_buffer) q.rgba = {device_buffer, true, width_stride, frame_stride};
    else q.channels = nullptr, q.clear = nullptr;
    return render_request(r, q, c, comps);
}
int forma_renderer_render_stats(forma_renderer* r, forma_composition* c, const forma_stats* stats, uint64_t width, uint64_t height,
                                const forma_rect* crop, forma_timings* timings) {
    FrameRequest q{FrameKind::single, 0, width, height, nullptr, nullptr, timings, crop};
    return render_stats(r, q, stats, false, nullptr, 0, 0, c, nullptr, __func__);
}
int forma_renderer_render_stats_device(forma_renderer* r, forma_composition* c, const forma_stats* stats, uint64_t width,
                                       uint64_t height, const forma_rect* crop, uint8_t* device_buffer, uint64_t width_stride,
                                       const uint32_t channels[4], const float clear_color[4], forma_timings* timings) {
    FrameRequest q{FrameKind::single, 0, width, height, channels, clear_color, timings, crop};
    return render_stats(r, q, stats, true, device_buffer, width_stride, 0, c, nullptr, __func__);
}
int forma_renderer_render_views_stats_device(forma_renderer* r, forma_composition* c, const float* views, uint32_t n,
                                             const forma_stats* stats, uint64_t width, uint64_t height, uint8_t* device_buffer,
                                             uint64_t width_stride, uint64_t view_stride, const uint32_t channels[4],
                                             const float clear_color[4], forma_timings* timings) {
    FrameRequest q{FrameKind::views, n, width, height, channels, clear_color, timings};
    q.views = views;
    return render_stats(r, q, stats, true, device_buffer, width_stride, view_stride, c, nullptr, __func__);
}
int forma_renderer_render_poses_stats_device(forma_renderer* r, forma_composition* c, const forma_poses* poses, uint32_t n,
                                             const forma_stats* stats, uint64_t width, uint64_t height, uint8_t* device_buffer,
                                             uint64_t width_stride, uint64_t view_stride, const uint32_t channels[4],
                                             const float clear_color[4], forma_timings* timings) {
    FrameRequest q = poses_request(poses, n, width, height, channels, clear_color, timings);
    return render_stats(r, q, stats, true, device_buffer, width_stride, view_stride, c, nullptr, __func__);
}
int forma_renderer_render_instances_stats_device(forma_renderer* r, forma_composition* c, const forma_instances* instances, uint32_t n,
                                                 const forma_stats* stats, uint64_t width, uint64_t height, uint8_t* device_buffer,
                                                 uint64_t width_stride, uint64_t view_stride, const uint32_t channels[4],
                                                 const float clear_color[4], forma_timings* timings) {
    FrameRequest q = instances_request(instances, n, width, height, channels, clear_color, timings);
    return render_stats(r, q, stats, true, device_buffer, width_stride, view_stride, c, nullptr, __func__);
}
int forma_renderer_render_batch_stats_device(forma_renderer* r, forma_composition* const* comps, uint32_t n,
                                             const forma_stats* stats, uint64_t width, uint64_t height, uint8_t* device_buffer,
                                             uint64_t width_stride, uint64_t frame_stride, const uint32_t channels[4],
                                             const float clear_color[4], forma_timings* timings) {
    FrameRequest q{FrameKind::batch, n, width, height, channels, clear_color, timings};
    return render_stats(r, q, stats, true, device_buffer, width_stride, frame_stride, nullptr, comps, __func__);
}
// Linear float frames: the RGBA target with 8- or 16-byte pixels (a null buffer is refused by
// Renderer::check_request like any missing target).
static int render_linear(forma_renderer* r, FrameRequest q, uint32_t format, forma_composition* c, forma_composition* const* comps) {
    q.rgba.bpp = format == FORMA_PIXEL_RGBA16F ? 8u : format == FORMA_PIXEL_RGBA32F ? 16u : 0u;
    if (!q.rgba.bpp) {
        set_error("invalid pixel format %u", format);
        return FORMA_STATUS_INVALID;
    }
    return render_request(r, q, c, comps);
}
int forma_renderer_render_linear(forma_renderer* r, forma_composition* c, void* buffer, uint64_t width, uint64_t width_stride,
                                 uint64_t height, const uint32_t channels[4], const float clear_color[4], const forma_rect* crop,
                                 uint32_t format, forma_timings* timings) {
    FrameRequest q{FrameKind::single, 0, width, height, channels, clear_color, timings, crop};
    q.rgba = {static_cast<uint8_t*>(buffer), false, width_stride};
    return render_linear(r, q, format, c, nullptr);
}
int forma_renderer_render_linear_device(forma_renderer* r, forma_composition* c, void* device_buffer, uint64_t width,
                                        uint64_t width_stride, uint64_t height, const uint32_t channels[4], const float clear_color[4],
                                        const forma_rect* crop, uint32_t format, forma_timings* timings) {
    FrameRequest q{FrameKind::single, 0, width, height, channels, clear_color, timings, crop};
    q.rgba = {static_cast<uint8_t*>(device_buffer), true, width_stride};
    return render_linear(r, q, format, c, nullptr);
}
int forma_renderer_render_views_linear(forma_renderer* r, forma_composition* c, const float* views, uint32_t n, void* host_buffer,
                                       uint64_t width, uint64_t width_stride, uint64_t height, uint64_t view_stride,
                                       const uint32_t channels[4], const float clear_color[4], uint32_t format, forma_timings* timings) {
    FrameRequest q{FrameKind::views, n, width, height, channels, clear_color, timings};
    q.views = views;
    q.rgba = {static_cast<uint8_t*>(host_buffer), false, width_stride, view_stride};
    return render_linear(r, q, format, c, nullptr);
}
int forma_renderer_render_views_linear_device(forma_renderer* r, forma_composition* c, const float* views, uint32_t n,
                                              void* device_buffer, uint64_t width, uint64_t width_stride, uint64_t height,
                                              uint64_t view_stride, const uint32_t channels[4], const float clear_color[4],
                                              uint32_t format, forma_timings* timings) {
    FrameRequest q{FrameKind::views, n, width, height, channels, clear_color, timings};
    q.views = views;
    q.rgba = {static_cast<uint8_t*>(device_buffer), true, width_stride, view_stride};
    return render_linear(r, q, format, c, nullptr);
}
int forma_renderer_render_batch_linear(forma_renderer* r, forma_composition* const* comps, uint32_t n, void* host_buffer, uint64_t width,
                                       uint64_t width_stride, uint64_t height, uint64_t frame_stride, const uint32_t channels[4],
                                       const float clear_color[4], uint32_t format, forma_timings* timings) {
    FrameRequest q{FrameKind::batch, n, width, height, channels, clear_color, timings};
    q.rgba = {static_cast<uint8_t*>(host_buffer), false, width_stride, frame_stride};
    return render_linear(r, q, format, nullptr, comps);
}
int forma_renderer_render_batch_linear_device(forma_renderer* r, forma_composition* const* comps, uint32_t n, void* device_buffer,
                                              uint64_t width, uint64_t width_stride, uint64_t height, uint64_t frame_stride,
                                              const uint32_t channels[4], const float clear_color[4], uint32_t format,
                                              forma_timings* timings) {
    FrameRequest q{FrameKind::batch, n, width, height, channels, clear_color, timings};
    q.rgba = {static_cast<uint8_t*>(device_buffer), true, width_stride, frame_stride};
    return render_linear(r, q, format, nullptr, comps);
}
// Frames over a background: the RGBA target in device memory, painted over its own pixels in any
// of the three formats (render_linear's checks and refusals, and check_request's over rules).
static int render_over(forma_renderer* r, FrameRequest q, uint32_t format, forma_composition* c, forma_composition* const* comps) {
    q.rgba.over = true;
    if (format == FORMA_PIXEL_SRGB8) {
        q.rgba.bpp = 4u;
        return render_request(r, q, c, comps);
    }
    return render_linear(r, q, format, c, comps);
}
int forma_renderer_render_over_device(forma_renderer* r, forma_composition* c, void* device_buffer, uint64_t width, uint64_t width_stride,
                                      uint64_t height, const uint32_t channels[4], const forma_rect* crop, uint32_t format,
                                      forma_timings* timings) {
    FrameRequest q{FrameKind::single, 0, width, height, channels, nullptr, timings, crop};
    q.rgba = {static_cast<uint8_t*>(device_buffer), true, width_stride};
    return render_over(r, q, format, c, nullptr);
}
int forma_renderer_render_views_over_device(forma_renderer* r, forma_composition* c, const float* views, uint32_t n, void* device_buffer,
                                            uint64_t width, uint64_t width_stride, uint64_t height, uint64_t view_stride,
                                            const uint32_t channels[4], uint32_t format, forma_timings* timings) {
    FrameRequest q{FrameKind::views, n, width, height, channels, nullptr, timings};
    q.views = views;
    q.rgba = {static_cast<uint8_t*>(device_buffer), true, width_stride, view_stride};
    return render_over(r, q, format, c, nullptr);
}
int forma_renderer_render_batch_over_device(forma_renderer* r, forma_composition* const* comps, uint32_t n, void* device_buffer,
                                            uint64_t width, uint64_t width_stride, uint64_t height, uint64_t frame_stride,
                                            const uint32_t channels[4], uint32_t format, forma_timings* timings) {
    FrameRequest q{FrameKind::batch, n, width, height, channels, nullptr, timings};
    q.rgba = {static_cast<uint8_t*>(device_buffer), true, width_stride, frame_stride};
    return render_over(r, q, format, nullptr, comps);
}
// Pose frames in the linear float formats and over a background: the twins of the views calls above.
int forma_renderer_render_poses_linear(forma_renderer* r, forma_composition* c, const forma_poses* poses, uint32_t n, void* host_buffer,
                                       uint64_t width, uint64_t width_stride, uint64_t height, uint64_t view_stride,
                                       const uint32_t channels[4], const float clear_color[4], uint32_t format, forma_timings* timings) {
    FrameRequest q = poses_request(poses, n, width, height, channels, clear_color, timings);
    q.rgba = {static_cast<uint8_t*>(host_buffer), false, width_stride, view_stride};
    return render_linear(r, q, format, c, nullptr);
}
int forma_renderer_render_poses_linear_device(forma_renderer* r, forma_composition* c, const forma_poses* poses, uint32_t n,
                                              void* device_buffer, uint64_t width, uint64_t width_stride, uint64_t height,
                                              uint64_t view_stride, const uint32_t channels[4], const float clear_color[4],
                                              uint32_t format, forma_timings* timings) {
    FrameRequest q = poses_request(poses, n, width, height, channels, clear_color, timings);
    q.rgba = {static_cast<uint8_t*>(device_buffer), true, width_stride, view_stride};
    return render_linear(r, q, format, c, nullptr);
}
int forma_renderer_render_poses_over_device(forma_renderer* r, forma_composition* c, const forma_poses* poses, uint32_t n,
                                            void* device_buffer, uint64_t width, uint64_t width_stride, uint64_t height,
                                            uint64_t view_stride, const uint32_t channels[4], uint32_t format, forma_timings* timings) {
    FrameRequest q = poses_request(poses, n, width, height, channels, nullptr, timings);
    q.rgba = {static_cast<uint8_t*>(device_buffer), true, width_stride, view_stride};
    return render_over(r, q, format, c, nullptr);
}
// --- shared frames (multi-GPU, see include/forma_b200.h) -----------------------
static_assert(sizeof(cudaIpcMemHandle_t) == sizeof(forma_ipc_handle), "CUDA IPC handles are 64 bytes");
int forma_shared_frame_create(int device, uint64_t bytes, void** device_ptr, forma_ipc_handle* handle) {
    if (!device_ptr || !handle || !bytes) {
        set_error("forma_shared_frame_create: bad arguments");
        return FORMA_STATUS_INVALID;
    }
    FORMA_CUDA_TRY(cudaSetDevice(device));
    void* p = nullptr;
    FORMA_CUDA_TRY(cudaMalloc(&p, bytes));
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) {
        cudaFree(p);
        set_error("cudaIpcGetMemHandle failed: %s", cudaGetErrorString(e));
        return FORMA_STATUS_CUDA;
    }
    std::memcpy(handle->bytes, &h, sizeof(h));
    *device_ptr = p;
    return FORMA_STATUS_OK;
}
int forma_shared_frame_open(int device, const forma_ipc_handle* handle, void** device_ptr) {
    if (!device_ptr || !handle) {
        set_error("forma_shared_frame_open: bad arguments");
        return FORMA_STATUS_INVALID;
    }
    FORMA_CUDA_TRY(cudaSetDevice(device));
    cudaIpcMemHandle_t h;
    std::memcpy(&h, handle->bytes, sizeof(h));
    FORMA_CUDA_TRY(cudaIpcOpenMemHandle(device_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return FORMA_STATUS_OK;
}
int forma_shared_frame_close(int device, void* mapped_ptr) {
    FORMA_CUDA_TRY(cudaSetDevice(device));
    FORMA_CUDA_TRY(cudaIpcCloseMemHandle(mapped_ptr));
    return FORMA_STATUS_OK;
}
int forma_shared_frame_free(int device, void* device_ptr) {
    FORMA_CUDA_TRY(cudaSetDevice(device));
    FORMA_CUDA_TRY(cudaFree(device_ptr));
    return FORMA_STATUS_OK;
}
static uint64_t row_costs_impl(forma_renderer* r, uint64_t cap, uint64_t* out) {
    Renderer& R = r->r;
    const uint32_t rows = R.last_tiles_y;
    if (!rows || !cap || !out) return rows;
    if (cudaSetDevice(R.device) != cudaSuccess) return 0;
    DeviceBuffer<unsigned long long> d;
    if (d.reserve(rows) != cudaSuccess) return 0;
    launch_row_costs(R.tile_range.ptr, R.last_tiles_x, rows, R.segs.ptr, R.last_segments, d.ptr, R.stream);
    std::vector<unsigned long long> h(rows);
    if (cudaMemcpyAsync(h.data(), d.ptr, rows * sizeof(unsigned long long), cudaMemcpyDeviceToHost, R.stream) != cudaSuccess ||
        cudaStreamSynchronize(R.stream) != cudaSuccess) {
        set_error("forma_renderer_row_costs: %s", cudaGetErrorString(cudaGetLastError()));
        return 0;
    }
    for (uint64_t i = 0; i < std::min<uint64_t>(cap, rows); ++i) out[i] = h[i];
    return rows;
}
uint64_t forma_renderer_row_costs(forma_renderer* r, uint64_t cap, uint64_t* out) {
    return guarded((uint64_t)0, [&] { return row_costs_impl(r, cap, out); });
}


// Pixel-pair fp32 self-test (see kernels_painter.cu): random and special operands (zeros,
// denormals, infinities, NaN, cancellation cases) through every pair helper of the painter.
static int selftest_impl(int device, uint64_t* mismatches) {
    if (!mismatches) return FORMA_ERR_INVALID_ARGUMENT;
    FORMA_CUDA_TRY(cudaSetDevice(device));
    const uint32_t n = 1u << 20;
    std::vector<float> h(3u * n);
    uint64_t sstate = 0x1234567ull;
    auto next = [&] {
        sstate += 0x9E3779B97F4A7C15ull;
        uint64_t z = sstate;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        return z ^ (z >> 31);
    };
    const uint32_t special[] = {0x00000000u, 0x80000000u, 0x00000001u, 0x007FFFFFu, 0x00800000u, 0x3F800000u, 0xBF800000u,
                                0x3F7FFFFFu, 0x3F800001u, 0x7F7FFFFFu, 0x7F800000u, 0xFF800000u, 0x7FC00000u, 0x33800000u};
    for (size_t i = 0; i < h.size(); ++i) {
        const uint64_t r = next();
        uint32_t bits;
        switch (r & 7u) {
            case 0: bits = special[(r >> 8) % (sizeof(special) / sizeof(special[0]))]; break;
            case 1: bits = (uint32_t)(r >> 32); break;                                  // any bit pattern
            case 2: bits = 0x3F800000u - (uint32_t)((r >> 32) & 0x3FFFFFu); break;      // just below 1
            default: {                                                                  // [0, 1) colours / coverages
                float f = (float)((r >> 40) & 0xFFFFFFu) / 16777216.0f;
                std::memcpy(&bits, &f, 4);
            }
        }
        std::memcpy(&h[i], &bits, 4);
    }
    DeviceBuffer<float> d;
    DeviceBuffer<uint32_t> out;
    FORMA_CUDA_TRY(d.reserve(h.size()));
    FORMA_CUDA_TRY(out.reserve(1));
    FORMA_CUDA_TRY(cudaMemcpy(d.ptr, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice));
    FORMA_CUDA_TRY(cudaMemset(out.ptr, 0, sizeof(uint32_t)));
    launch_f32x2_selftest(d.ptr, d.ptr + n, d.ptr + 2u * n, n, out.ptr, 0);
    FORMA_CUDA_TRY(cudaGetLastError());
    uint32_t bad = 0;
    FORMA_CUDA_TRY(cudaMemcpy(&bad, out.ptr, sizeof(uint32_t), cudaMemcpyDeviceToHost));
    *mismatches = bad;
    return FORMA_OK;
}
int forma_debug_selftest(int device, uint64_t* mismatches) {
    return guarded((int)FORMA_ERR_CAPACITY, [&] { return selftest_impl(device, mismatches); });
}

uint64_t forma_renderer_launch_count(const forma_renderer* r) { return r->r.launches; }
void forma_renderer_stage_times(const forma_renderer* r, double out_ms[8]) {
    const_cast<forma_renderer*>(r)->r.resolve_times();
    for (int i = 0; i < 8; ++i) out_ms[i] = r->r.stage_ms[i];
}
void forma_renderer_kernel_times(const forma_renderer* r, double out_ms[4], uint32_t out_launches[4]) {
    const_cast<forma_renderer*>(r)->r.resolve_times();
    for (int i = 0; i < 4; ++i) {
        out_ms[i] = r->r.kernel_ms[i];
        out_launches[i] = r->r.kernel_launches[i];
    }
}
void forma_renderer_counters(const forma_renderer* r, uint64_t out[8]) {
    out[6] = r->r.last_written_tiles;
    out[7] = r->r.last_tables_redone ? 2u : r->r.last_tables_sync_free ? 1u : 0u;
    out[0] = r->r.launches;
    out[1] = r->r.h2d_bytes;
    out[2] = r->r.d2h_bytes;
    out[3] = r->r.last_segments;
    out[4] = r->r.last_cells;
    out[5] = r->r.last_entries;
}
uint32_t forma_renderer_sort_mode(const forma_renderer* r) { return r->r.last_sort_redone ? 2u : r->r.last_sort_sync_free ? 1u : 0u; }
void forma_composition_evict(forma_composition* c) { c->c.evict(); }
uint64_t forma_composition_point_count(forma_composition* c) { return c->c.n_points; }
void forma_path_builder_extend(forma_path_builder* pb, const uint8_t* cmds, uint64_t n_cmds, const float* xy) {
    PathBuilder& b = pb->b;
    const float* p = xy;
    guarded_void([&] {
    for (uint64_t i = 0; i < n_cmds; ++i) {
        switch (cmds[i]) {
            case 0: b.move_to({p[0], p[1]}); p += 2; break;
            case 1: b.line_to({p[0], p[1]}); p += 2; break;
            case 2: b.quad_to({p[0], p[1]}, {p[2], p[3]}); p += 4; break;
            default: b.cubic_to({p[0], p[1]}, {p[2], p[3]}, {p[4], p[5]}); p += 6; break;
        }
    }
    });
}

static uint64_t renderer_lines_impl(forma_renderer* r, uint64_t cap, uint32_t* orders, float* x0, float* y0, float* dx,
                                    float* dy, float* a, float* b, float* c, float* d, uint32_t* lengths) {
    // Line records are never materialised by render(): line setup is fused into the
    // pixel-grid intersection kernel. For inspection they are produced here, by the same
    // device function (line_setup), from the arguments of the last render; the composition
    // of that render must still be alive.
    Renderer& R = r->r;
    if (!R.last_raster_valid || R.last_raster.n_points < 2) return 0;
    const uint32_t n = R.last_raster.n_points - 1u;
    if (!cap || !orders) return n;
    if (cudaSetDevice(R.device) != cudaSuccess) return 0;
    RasterArgs A = R.last_raster;
    A.band_lo = -3.0e38f;  // the reference's records know no tile bands
    A.band_hi = 3.0e38f;
    DeviceBuffer<uint32_t> d_orders, d_lengths;
    DeviceBuffer<float> d_f[8];
    if (d_orders.reserve(n) != cudaSuccess || d_lengths.reserve(n) != cudaSuccess) return 0;
    float* fp[8];
    for (int k = 0; k < 8; ++k) {
        if (d_f[k].reserve(n) != cudaSuccess) return 0;
        fp[k] = d_f[k].ptr;
    }
    launch_line_records(A, n, d_orders.ptr, fp, d_lengths.ptr, R.stream);
    const size_t m = (size_t)std::min<uint64_t>(cap, n);
    float* out[8] = {x0, y0, dx, dy, a, b, c, d};
    bool ok = cudaMemcpyAsync(orders, d_orders.ptr, m * 4, cudaMemcpyDeviceToHost, R.stream) == cudaSuccess &&
              cudaMemcpyAsync(lengths, d_lengths.ptr, m * 4, cudaMemcpyDeviceToHost, R.stream) == cudaSuccess;
    for (int k = 0; k < 8 && ok; ++k) ok = cudaMemcpyAsync(out[k], fp[k], m * 4, cudaMemcpyDeviceToHost, R.stream) == cudaSuccess;
    if (!ok || cudaStreamSynchronize(R.stream) != cudaSuccess) {
        set_error("forma_renderer_lines: %s", cudaGetErrorString(cudaGetLastError()));
        return 0;
    }
    uint32_t sum = 0;  // prefix_sum, segment.rs:90-98 (inclusive)
    for (size_t i = 0; i < m; ++i) {
        sum += lengths[i];
        lengths[i] = sum;
    }
    return n;
}
uint64_t forma_renderer_lines(forma_renderer* r, uint64_t cap, uint32_t* orders, float* x0, float* y0, float* dx, float* dy,
                              float* a, float* b, float* c, float* d, uint32_t* lengths) {
    return guarded((uint64_t)0, [&] { return renderer_lines_impl(r, cap, orders, x0, y0, dx, dy, a, b, c, d, lengths); });
}
uint64_t forma_renderer_segments(forma_renderer* r, uint64_t cap, uint64_t* out) {
    if (r->r.last_slices) {
        set_error("forma_renderer_segments: the last host frame was rendered in %u slices (option host_slices); "
                  "there is no single sorted segment array to inspect", r->r.last_slices);
        return 0;
    }
    uint64_t n = r->r.last_segments;
    if (out && cap && n) {
        cudaError_t e = cudaMemcpy(out, r->r.segs.ptr, std::min<uint64_t>(cap, n) * sizeof(uint64_t), cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) {
            set_error("forma_renderer_segments: %s", cudaGetErrorString(e));
            return 0;
        }
    }
    return n;
}
static uint64_t rasterize_only_impl(forma_renderer* r, forma_composition* c, uint64_t width, uint64_t height,
                                    uint64_t cap, uint64_t* out) {
    Renderer& R = r->r;
    if (cudaSetDevice(R.device) != cudaSuccess) return 0;
    if (R.upload_tables(c->c, -1) || R.flush_geometry(c->c)) return 0;
    uint32_t n = 0;
    if (R.rasterize(&c->c, (uint32_t)std::min<uint64_t>(width, 0xFFFFFFFFu), (uint32_t)std::min<uint64_t>(height, 0xFFFFFFFFu),
                    -3.0e38f, 3.0e38f, &n))
        return 0;
    if (cudaStreamSynchronize(R.stream) != cudaSuccess) return 0;
    if (out && cap && n &&
        cudaMemcpy(out, R.segs.ptr, std::min<uint64_t>(cap, n) * sizeof(uint64_t), cudaMemcpyDeviceToHost) != cudaSuccess)
        return 0;
    return n;
}
uint64_t forma_renderer_rasterize_only(forma_renderer* r, forma_composition* c, uint64_t width, uint64_t height,
                                       uint64_t cap, uint64_t* out) {
    return guarded((uint64_t)0, [&] { return rasterize_only_impl(r, c, width, height, cap, out); });
}
int forma_renderer_sort_u64(forma_renderer* r, uint64_t* keys, uint64_t n) {
    Renderer& R = r->r;
    if (n >= (1ull << 30)) {
        set_error("sort_u64: n too large");
        return FORMA_ERR_CAPACITY;
    }
    if (n < 2) return FORMA_OK;
    FORMA_CUDA_TRY(cudaSetDevice(R.device));
    FORMA_CUDA_TRY(Renderer::reserve_all(n + 1, R.segs, R.segs_tmp));  // one key of slack: the TMA downsweep copies an even number of keys
    FORMA_CUDA_TRY(R.sort_scratch.reserve(radix_scratch_bytes((uint32_t)n)));
    FORMA_CUDA_TRY(cudaMemcpyAsync(R.segs.ptr, keys, n * sizeof(uint64_t), cudaMemcpyHostToDevice, R.stream));
    // The caller's keys are on the host: take the field bounds from their OR.
    uint64_t all = 0;
    for (uint64_t i = 0; i < n; ++i) all |= keys[i];
    const uint64_t bound[3] = {(all >> 20) & 0x1FFFFFull, (all >> 41) & 0xFFFull, (all >> 53) & 0x7FFull};
    R.sort(R.segs, R.segs_tmp, nullptr, nullptr, (uint32_t)n, make_sort_plan(segment_key_layout(), bound));
    FORMA_CUDA_TRY(cudaGetLastError());
    FORMA_CUDA_TRY(cudaMemcpyAsync(keys, R.segs.ptr, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, R.stream));
    FORMA_CUDA_TRY(cudaStreamSynchronize(R.stream));
    return FORMA_OK;
}
int forma_debug_sort_plan(int layout, const uint64_t bound[3], uint8_t out[2 + 10 * kMaxSortPasses]) {
    if (layout != 0 && layout != 1) {
        set_error("sort_plan: layout %d is neither 0 (segments) nor 1 (carry)", layout);
        return FORMA_ERR_INVALID_ARGUMENT;
    }
    const SortPlan plan = make_sort_plan(layout ? carry_key_layout() : segment_key_layout(), bound);
    out[0] = (uint8_t)plan.n_passes;
    out[1] = (uint8_t)plan.total_bits;
    static_assert(sizeof(DigitSpec) == 10, "shift[3], width[3], lsh[3], bits");
    std::memcpy(out + 2, plan.pass, sizeof(plan.pass));
    return FORMA_OK;
}
uint64_t forma_renderer_sort_counts(forma_renderer* r, int keep, uint32_t info[3], uint32_t* out, uint64_t cap) {
    Renderer& R = r->r;
    if (keep >= 0) R.keep_sort_counts = keep != 0;
    info[0] = (uint32_t)R.last_count_source;
    info[1] = R.kept_passes;
    info[2] = R.kept_tiles;
    const uint64_t words = (uint64_t)R.kept_passes * R.kept_tiles * 256u;
    if (out && cap && words) {
        cudaError_t e = cudaSetDevice(R.device);
        if (e == cudaSuccess) e = cudaStreamSynchronize(R.stream);
        if (e == cudaSuccess)
            e = cudaMemcpy(out, R.kept_counts.ptr, std::min<uint64_t>(cap, words) * sizeof(uint32_t), cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) {
            set_error("forma_renderer_sort_counts: %s", cudaGetErrorString(e));
            return 0;
        }
    }
    return words;
}
void forma_renderer_sort_bounds(const forma_renderer* r, uint64_t out[4]) {
    for (int f = 0; f < 3; ++f) out[f] = r->r.segment_bound[f];
    out[3] = r->r.segment_plan.total_bits;
}
int forma_renderer_sort_pairs(forma_renderer* r, int layout, int mode, uint64_t* keys, uint32_t* vals, uint64_t count,
                              uint64_t cap) {
    Renderer& R = r->r;
    const bool dev_count = (mode & 1) != 0, hist_ready = (mode & 2) != 0;
    if ((layout != 0 && layout != 1) || (mode & ~3)) {
        set_error("sort_pairs: layout %d / mode %d", layout, mode);
        return FORMA_ERR_INVALID_ARGUMENT;
    }
    if (count >= (1ull << 30) || (dev_count && cap >= (1ull << 30))) {
        set_error("sort_pairs: n too large");
        return FORMA_ERR_CAPACITY;
    }
    const uint32_t n = (uint32_t)(dev_count ? cap : count);    // what the launches are sized by
    const uint64_t held = dev_count ? std::min(count, cap) : count;  // elements of keys / vals
    if (n < 2 || held == 0) return FORMA_OK;
    FORMA_CUDA_TRY(cudaSetDevice(R.device));
    const KeyLayout lay = layout ? carry_key_layout() : segment_key_layout();
    uint64_t all = 0, bound[3];
    for (uint64_t i = 0; i < held; ++i) all |= keys[i];
    for (int f = 0; f < 3; ++f) bound[f] = (all >> lay.pos[f]) & ((1ull << lay.maxw[f]) - 1u);
    const SortPlan plan = make_sort_plan(lay, bound);
    // Scratch: the count | (hist_ready) hist[kMaxSortPasses][256], then the zeroed look-back block |
    // (otherwise) the sort's own scratch, which it zeroes itself.
    const size_t hist_bytes = (size_t)kMaxSortPasses * 256 * sizeof(uint32_t);
    const size_t work = hist_ready ? hist_bytes + sort_lookback_bytes(n, plan) : radix_scratch_bytes(n);
    FORMA_CUDA_TRY(R.sort_scratch.reserve(256 + work));
    FORMA_CUDA_TRY(Renderer::reserve_all((size_t)n + 1, R.key2, R.key2_tmp, R.perm, R.perm_tmp));
    uint32_t* d_count = reinterpret_cast<uint32_t*>(R.sort_scratch.ptr);
    uint8_t* d_work = R.sort_scratch.ptr + 256;
    const uint32_t count32 = (uint32_t)count;
    FORMA_CUDA_TRY(cudaMemcpyAsync(d_count, &count32, sizeof(uint32_t), cudaMemcpyHostToDevice, R.stream));
    FORMA_CUDA_TRY(cudaMemcpyAsync(R.key2.ptr, keys, held * sizeof(uint64_t), cudaMemcpyHostToDevice, R.stream));
    FORMA_CUDA_TRY(cudaMemcpyAsync(R.perm.ptr, vals, held * sizeof(uint32_t), cudaMemcpyHostToDevice, R.stream));
    const uint32_t* n_dev = dev_count ? d_count : nullptr;
    const uint32_t* hist = nullptr;
    if (hist_ready) {
        FORMA_CUDA_TRY(cudaMemsetAsync(d_work, 0, work, R.stream));
        launch_radix_hist(R.key2.ptr, n, plan, reinterpret_cast<uint32_t*>(d_work), n_dev, R.stream);
        hist = reinterpret_cast<const uint32_t*>(d_work);
    }
    // A refused sort (count > cap) leaves its input where it was, whichever buffer the passes end in.
    const bool refused = dev_count && count > cap;
    const uint64_t* in_keys = R.key2.ptr;
    const uint32_t* in_vals = R.perm.ptr;
    R.sort(R.key2, R.key2_tmp, &R.perm, &R.perm_tmp, n, plan, nullptr, n_dev, hist, hist_ready ? d_work + hist_bytes : d_work);
    FORMA_CUDA_TRY(cudaGetLastError());
    FORMA_CUDA_TRY(cudaMemcpyAsync(keys, refused ? in_keys : R.key2.ptr, held * sizeof(uint64_t), cudaMemcpyDeviceToHost, R.stream));
    FORMA_CUDA_TRY(cudaMemcpyAsync(vals, refused ? in_vals : R.perm.ptr, held * sizeof(uint32_t), cudaMemcpyDeviceToHost, R.stream));
    FORMA_CUDA_TRY(cudaStreamSynchronize(R.stream));
    return FORMA_OK;
}

}  // extern "C"
