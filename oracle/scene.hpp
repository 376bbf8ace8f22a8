// ORACLE — TEST INFRASTRUCTURE ONLY (see fmath.hpp).
//
// Data model (Props/Style/Fill/Gradient), Composition/Layer bookkeeping, the
// global SegmentBuffer and the per-frame line setup. Restates
// forma/src/styling.rs, forma/src/composition/{mod,layer}.rs and
// forma/src/segment.rs.
#pragma once

#include <map>
#include <unordered_map>
#include <vector>

#include "path.hpp"

namespace fo {

constexpr uint32_t kLayerLimit = (1u << 21) - 1;  // consts.rs:106-108

struct Color {
    float r = 0.0f, g = 0.0f, b = 0.0f, a = 1.0f;
    bool operator==(const Color& o) const { return r == o.r && g == o.g && b == o.b && a == o.a; }
};

enum FillRule : uint32_t { kNonZero = 0, kEvenOdd = 1 };
enum GradientType : uint32_t { kLinear = 0, kRadial = 1 };
enum FillType : uint32_t { kSolid = 0, kGradient = 1, kTexture = 2 };
enum FuncType : uint32_t { kDraw = 0, kClip = 1 };
// styling.rs:378-395 — same order as the Rust enum.
enum BlendMode : uint32_t {
    kOver = 0, kMultiply, kScreen, kOverlay, kDarken, kLighten, kColorDodge, kColorBurn,
    kHardLight, kSoftLight, kDifference, kExclusion, kHue, kSaturation, kColorMode, kLuminosity,
};
enum Channel : uint32_t { kRed = 0, kGreen = 1, kBlue = 2, kAlpha = 3, kZero = 4, kOne = 5 };

struct GradientStop {
    Color color;
    float stop;
};

struct Gradient {
    GradientType type = kLinear;
    Point start, end;
    std::vector<GradientStop> stops;
};

// styling.rs:224-366 — custom f16 (no denormals, [0,1]).
inline uint16_t f16_from(float v) { return v != 0.0f ? (uint16_t)((f2u(v) - 0x38000000u) >> 13) : 0; }
inline float f16_to(uint16_t h) { return h != 0 ? u2f(0x38000000u + ((uint32_t)h << 13)) : 0.0f; }

struct Image {
    std::shared_ptr<std::vector<uint16_t>> data;  // RGBA f16, 4 per pixel
    float max_x = 0.0f, max_y = 0.0f;
    uint32_t width = 0;
};

struct Texture {
    Affine transform;
    Image image;
};

struct Props {
    FillRule fill_rule = kNonZero;
    FuncType func = kDraw;
    uint32_t clip_layers = 0;
    bool is_clipped = false;
    FillType fill_type = kSolid;
    Color color;  // Fill::Solid
    Gradient gradient;
    Texture texture;
    BlendMode blend_mode = kOver;
};

// composition/layer.rs:20-46
struct Layer {
    bool is_enabled = true;
    bool has_transform = false;
    Affine transform;
    uint64_t geom_id = 0;
    Props props;
    uint32_t is_unchanged = 0;  // SmallBitSet over cache ids
    size_t lines_count = 0;
    int64_t order = -1;  // Option<Order>
};

// segment.rs:530-545 (the x/y/ids part) and the per-frame line arrays.
struct Lines {
    std::vector<uint32_t> orders, lengths;  // lengths: inclusive prefix sums, wrapping in u32 like the reference's
    std::vector<float> x0, y0, dx, dy, a, b, c, d;
    uint64_t total = 0;  // the true pixel-segment count (a saturated integers_between counts as 2^32 - 1)
    size_t size() const { return orders.size(); }
    void resize(size_t n) {
        orders.resize(n);
        lengths.resize(n);
        for (auto* v : {&x0, &y0, &dx, &dy, &a, &b, &c, &d}) v->resize(n);
    }
};

// segment.rs:54-59
inline uint32_t integers_between(float a, float b) {
    float mn = rmin(a, b), mx = rmax(a, b);
    return sat_u32(std::ceil(mx) - std::floor(mn) - 1.0f);
}

struct Composition {
    // Attached layers keyed by Order::as_u32(); every Layer (attached or not)
    // is owned by `pool` until dropped (Layer::drop, composition/layer.rs:355-363).
    std::map<uint32_t, Layer*> layers;
    std::vector<std::unique_ptr<Layer>> pool;
    std::unordered_map<uint64_t, int64_t> geom_id_to_order;  // -1 == None
    uint64_t next_geom_id = 1;
    // SegmentBuffer view: ids 0 == None.
    std::vector<float> x, y;
    std::vector<uint64_t> ids;

    uint64_t new_geom_id() { return next_geom_id++; }

    // composition/mod.rs:65-83
    Layer* create_layer() {
        pool.emplace_back(new Layer());
        Layer* l = pool.back().get();
        l->geom_id = new_geom_id();
        return l;
    }

    // composition/layer.rs:148-158
    void set_order(Layer* l, int64_t order) {
        if (order >= 0 && l->order != order) {
            l->order = order;
            l->is_unchanged = 0;
        }
        geom_id_to_order[l->geom_id] = order;
    }

    // composition/mod.rs:121-138 — returns the displaced layer (now detached) or null.
    Layer* insert(uint32_t order, Layer* layer) {
        set_order(layer, order);
        Layer* old = nullptr;
        auto it = layers.find(order);
        if (it != layers.end()) {
            old = it->second;
            it->second = layer;
        } else {
            layers.emplace(order, layer);
        }
        if (old == layer) return nullptr;
        if (old) set_order(old, -1);
        return old;
    }

    // composition/mod.rs:141-149
    Layer* remove(uint32_t order) {
        auto it = layers.find(order);
        if (it == layers.end()) return nullptr;
        Layer* l = it->second;
        layers.erase(it);
        set_order(l, -1);
        return l;
    }

    // Layer::drop
    void drop_layer(Layer* l) {
        for (auto it = layers.begin(); it != layers.end(); ++it)
            if (it->second == l) {
                layers.erase(it);
                break;
            }
        geom_id_to_order.erase(l->geom_id);
        for (auto it = pool.begin(); it != pool.end(); ++it)
            if (it->get() == l) {
                pool.erase(it);
                break;
            }
    }

    Layer* get(uint32_t order) {
        auto it = layers.find(order);
        return it == layers.end() ? nullptr : it->second;
    }

    // composition/mod.rs:175-182
    Layer* get_mut_or_insert_default(uint32_t order) {
        Layer* l = get(order);
        if (!l) {
            l = create_layer();
            insert(order, l);
        }
        return l;
    }

    size_t segment_len(size_t from = 0) const {
        size_t n = 0;
        for (size_t i = from; i < ids.size(); ++i) n += ids[i] != 0;
        return n;
    }

    // composition/layer.rs:90-111 + segment.rs:181-198 + path.rs:677-723
    void layer_insert(Layer* lp, Path& path) {
        Layer& layer = *lp;
        size_t from_index = ids.size() ? ids.size() - 1 : 0;  // only the tail can change (SegmentBuffer::len caches, segment.rs:163-178)
        size_t old_len = segment_len(from_index);
        const Segments& s = path.inner->segments();
        for (size_t i = 0; i < s.x.size(); ++i) {
            Point p{s.x[i], s.y[i]};
            if (path.has_transform) p = path.transform.apply(p);
            x.push_back(p.x);
            y.push_back(p.y);
            ids.push_back(s.start_new_contour[i] ? 0 : layer.geom_id);
        }
        ids.resize(x.size() > 0 ? x.size() - 1 : 0, layer.geom_id);
        if (!ids.empty() && ids.back() != 0) ids.push_back(0);
        layer.lines_count += segment_len(from_index) - old_len;
        geom_id_to_order[layer.geom_id] = layer.order;
        layer.is_unchanged = 0;
    }

    // composition/layer.rs:131-146
    void layer_clear(Layer* lp) {
        Layer& layer = *lp;
        geom_id_to_order.erase(layer.geom_id);
        layer.geom_id = new_geom_id();
        geom_id_to_order[layer.geom_id] = layer.order;
        layer.lines_count = 0;
        layer.is_unchanged = 0;
    }

    // segment.rs:237-273 + composition/mod.rs:219-231
    void compact_geom() {
        size_t actual = 0;
        for (auto& kv : layers) actual += kv.second->lines_count;
        if (segment_len() < actual * 2) return;
        size_t len = x.size(), del = 0;
        uint64_t prev = 0;
        for (size_t i = 0; i < len; ++i) {
            uint64_t id = ids[i];
            uint64_t key = id ? id : prev;
            bool keep = geom_id_to_order.count(key) != 0;
            prev = id;
            if (!keep) {
                del += 1;
                continue;
            }
            if (del > 0) {
                std::swap(x[i - del], x[i]);
                std::swap(y[i - del], y[i]);
                std::swap(ids[i - del], ids[i]);
            }
        }
        if (del > 0) {
            x.resize(len - del);
            y.resize(len - del);
            ids.resize(len - del);
        }
    }

    // segment.rs:275-402
    void fill_cpu_view(size_t width_px, size_t height_px, Lines& out) const {
        float width = (float)width_px, height = (float)height_px;
        size_t n = ids.empty() ? 0 : ids.size() - 1;
        if (x.size() < 2) n = 0;
        out.resize(n);
        uint64_t wrapped = 0;  // lines whose own length wraps u32
#pragma omp parallel
        {
        // id -> order -> layer (segment.rs:141-149: two FxHashMap look-ups per point). `layers` is an
        // ordered map here, so the result is remembered while consecutive points share their id;
        // otherwise this loop would pay a tree walk per point that the reference does not.
        uint64_t memo_id = 0;
        const Layer* memo_layer = nullptr;
        uint32_t memo_order = 0;
#pragma omp for schedule(static) reduction(+ : wrapped)
        for (size_t i = 0; i < n; ++i) {
            auto empty = [&] {
                out.orders[i] = 0;
                out.x0[i] = out.y0[i] = out.dx[i] = out.dy[i] = 0.0f;
                out.a[i] = out.b[i] = out.c[i] = out.d[i] = 0.0f;
                out.lengths[i] = 0;
            };
            uint64_t id = ids[i];
            if (id == 0) { empty(); continue; }
            if (id != memo_id) {
                memo_id = id;
                memo_layer = nullptr;
                auto oit = geom_id_to_order.find(id);
                if (oit != geom_id_to_order.end() && oit->second >= 0) {
                    auto lit = layers.find((uint32_t)oit->second);
                    if (lit != layers.end()) {
                        memo_layer = lit->second;
                        memo_order = lit->first;
                    }
                }
            }
            if (!memo_layer) { empty(); continue; }
            const Layer& layer = *memo_layer;
            if (!layer.is_enabled) { empty(); continue; }
            uint32_t order = memo_order;

            Point p0{x[i], y[i]}, p1{x[i + 1], y[i + 1]};
            if (layer.has_transform) {
                p0 = layer.transform.apply(p0);
                p1 = layer.transform.apply(p1);
            }
            // skip_line, segment.rs:41-52
            bool skip = p0.y == p1.y || (p0.y >= height && p1.y >= height) ||
                        (p0.x >= width && p1.x >= width) || (p0.y <= 0.0f && p1.y <= 0.0f);
            if (skip) { empty(); continue; }

            float dx = p1.x - p0.x, dy = p1.y - p0.y;
            float dx_recip = recip(dx), dy_recip = recip(dy);
            float tox = dx != 0.0f ? rmax((std::ceil(p0.x) - p0.x) * dx_recip, (std::floor(p0.x) - p0.x) * dx_recip) : 0.0f;
            float toy = dy != 0.0f ? rmax((std::ceil(p0.y) - p0.y) * dy_recip, (std::floor(p0.y) - p0.y) * dy_recip) : 0.0f;
            out.orders[i] = order;
            out.x0[i] = p0.x * 16.0f;
            out.y0[i] = p0.y * 16.0f;
            out.dx[i] = dx * 16.0f;
            out.dy[i] = dy * 16.0f;
            out.a[i] = std::fabs(dx_recip);
            out.b[i] = std::fabs(dy_recip);
            out.c[i] = tox;
            out.d[i] = toy;
            const uint64_t len = (uint64_t)integers_between(p0.x, p1.x) + integers_between(p0.y, p1.y) + 1u;
            out.lengths[i] = (uint32_t)len;
            wrapped += len >> 32;
        }
        }
        // prefix_sum, segment.rs:90-98: the reference's u32 sums wrap (release builds) or panic
        // (debug builds). Here they are kept in u64 and stored wrapped, so that rasterize() can
        // refuse a frame whose true count does not fit instead of indexing past its output.
        uint64_t sum = 0;
        for (size_t i = 0; i < n; ++i) {
            sum += out.lengths[i];
            out.lengths[i] = (uint32_t)sum;
        }
        out.total = sum + (wrapped << 32);
    }
};

}  // namespace fo
