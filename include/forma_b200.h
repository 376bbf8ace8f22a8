/*
 * forma_b200 — C ABI of the H100-native replacement for google/forma's
 * rendering hot path (flatten -> pixel-grid intersection -> 64-bit
 * pixel-segment sort -> per-tile paint).
 *
 * The reference has no Renderer trait (SURVEY.md F1); the drop-in boundary is
 * the inherent method forma/src/cpu/renderer.rs:75-82
 *
 *     cpu::Renderer::render(&mut self, composition, buffer, channels,
 *                           clear_color, crop)
 *
 * together with the scene-building API its callers use
 * (forma/src/lib.rs:128-154: Composition, Layer, PathBuilder, Path, Order,
 * Props/Style/Fill/Gradient/BlendMode/FillRule/Func, Buffer/LinearLayout,
 * Channel constants). Every function below names the reference item it
 * replaces. Plain pointers and sizes only; no C++ or torch types.
 *
 * Status codes replace the reference's panics / Results.
 */
#ifndef FORMA_B200_H
#define FORMA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------ */
/* Status                                                                   */
/* ------------------------------------------------------------------------ */
enum {
    FORMA_OK = 0,
    FORMA_ERR_INVALID_ARGUMENT = 1, /* assert!/panic in the reference                     */
    FORMA_ERR_ORDER_LIMIT = 2,      /* OrderError::ExceededLayerLimit, utils/order.rs:56-65 */
    FORMA_ERR_CUDA = 3,             /* a CUDA call failed; see forma_last_error()          */
    FORMA_ERR_NO_DEVICE = 4,        /* no usable sm_90 device: there is NO CPU fallback    */
    FORMA_ERR_CAPACITY = 5          /* an internal device buffer could not be grown, or a
                                       frame needs 2^30 or more pixel segments (refused
                                       before anything is painted; no count wraps)         */
};

/* Human-readable description of the last failure on the calling thread. */
const char* forma_last_error(void);

/* consts.rs:25-26,106-108 */
#define FORMA_MAX_WIDTH 65536u
#define FORMA_MAX_HEIGHT 32768u
#define FORMA_LAYER_LIMIT 2097151u
#define FORMA_TILE_WIDTH 16u
#define FORMA_TILE_HEIGHT 16u

/* ------------------------------------------------------------------------ */
/* Data model (forma/src/styling.rs)                                        */
/* ------------------------------------------------------------------------ */
typedef struct forma_color { float r, g, b, a; } forma_color; /* styling.rs:28-33 (linear) */

enum { FORMA_FILL_RULE_NON_ZERO = 0, FORMA_FILL_RULE_EVEN_ODD = 1 };          /* styling.rs:64-67   */
enum { FORMA_GRADIENT_LINEAR = 0, FORMA_GRADIENT_RADIAL = 1 };                /* styling.rs:76-79   */
enum { FORMA_FILL_SOLID = 0, FORMA_FILL_GRADIENT = 1, FORMA_FILL_TEXTURE = 2 }; /* styling.rs:368-372 */
enum { FORMA_FUNC_DRAW = 0, FORMA_FUNC_CLIP = 1 };                            /* styling.rs:417-424 */
enum {                                                                        /* styling.rs:378-395 */
    FORMA_BLEND_OVER = 0, FORMA_BLEND_MULTIPLY, FORMA_BLEND_SCREEN, FORMA_BLEND_OVERLAY,
    FORMA_BLEND_DARKEN, FORMA_BLEND_LIGHTEN, FORMA_BLEND_COLOR_DODGE, FORMA_BLEND_COLOR_BURN,
    FORMA_BLEND_HARD_LIGHT, FORMA_BLEND_SOFT_LIGHT, FORMA_BLEND_DIFFERENCE, FORMA_BLEND_EXCLUSION,
    FORMA_BLEND_HUE, FORMA_BLEND_SATURATION, FORMA_BLEND_COLOR, FORMA_BLEND_LUMINOSITY
};
enum {                                                                        /* cpu/channel.rs:35-43 */
    FORMA_CHANNEL_RED = 0, FORMA_CHANNEL_GREEN, FORMA_CHANNEL_BLUE, FORMA_CHANNEL_ALPHA,
    FORMA_CHANNEL_ZERO, FORMA_CHANNEL_ONE
};

/* One (color, stop) pair of GradientBuilder (styling.rs:84-139). stop == -1
 * means "unpositioned" (GradientBuilder::color): it is spread evenly exactly
 * like GradientBuilder::build does. */
typedef struct forma_gradient_stop { forma_color color; float stop; } forma_gradient_stop;

/* Flat form of Props { fill_rule, func: Draw(Style{is_clipped, fill,
 * blend_mode}) | Clip(n) } (styling.rs:397-442). */
typedef struct forma_props {
    uint32_t fill_rule;
    uint32_t func;        /* FORMA_FUNC_*                                        */
    uint32_t clip_layers; /* n of Func::Clip(n)                                  */
    uint32_t is_clipped;
    uint32_t blend_mode;
    uint32_t fill_type;
    forma_color color;    /* Fill::Solid                                         */
    uint32_t gradient_type;
    float start[2], end[2];
    uint32_t n_stops;
    const forma_gradient_stop* stops;
    float tex_transform[6]; /* Texture.transform: ux, uy, vx, vy, tx, ty         */
    uint32_t tex_width, tex_height;
    const float* tex_linear_rgba; /* Image::from_linear_rgba, styling.rs:320-327 */
} forma_props;

/* cpu::Rect::new(horizontal, vertical) in pixels; approximated to the tile
 * grid exactly like cpu/renderer.rs:43-52. */
typedef struct forma_rect { uint64_t hor_start, hor_end, vert_start, vert_end; } forma_rect;

/* Per-stage device times of the last render (the reference's gpu::Timings,
 * gpu/renderer/mod.rs:25-30) plus the sizes the roofline needs. */
typedef struct forma_timings {
    double line_setup_ms, rasterize_ms, sort_ms, paint_ms;
    uint64_t n_lines, n_segments;
} forma_timings;

/* ------------------------------------------------------------------------ */
/* PathBuilder / Path (forma/src/path.rs:670-925)                           */
/* ------------------------------------------------------------------------ */
typedef struct forma_path_builder forma_path_builder;
typedef struct forma_path forma_path;

forma_path_builder* forma_path_builder_new(void);                 /* PathBuilder::new  :783 */
void forma_path_builder_free(forma_path_builder*);
void forma_path_builder_move_to(forma_path_builder*, float x, float y);            /* :788 */
void forma_path_builder_line_to(forma_path_builder*, float x, float y);            /* :816 */
void forma_path_builder_quad_to(forma_path_builder*, float x1, float y1, float x2, float y2); /* :831 */
void forma_path_builder_cubic_to(forma_path_builder*, float x1, float y1, float x2, float y2,
                                 float x3, float y3);                              /* :850 */
void forma_path_builder_rat_quad_to(forma_path_builder*, float x1, float y1, float x2, float y2,
                                    float weight);                                 /* :873 */
void forma_path_builder_rat_cubic_to(forma_path_builder*, float x1, float y1, float x2, float y2,
                                     float x3, float y3, float w1, float w2);      /* :892 */
forma_path* forma_path_builder_build(forma_path_builder*);                         /* :915 */
forma_path* forma_path_transform(const forma_path*, const float m[9]);   /* Path::transform :726 */
void forma_path_free(forma_path*);

/* Flattened polyline of the path (what Path::push_segments_to appends,
 * path.rs:677-723): n points, start_new_contour[i] != 0 marks a contour end.
 * Pointers stay valid until the next call on the same thread. */
int forma_path_segments(forma_path*, const float** x, const float** y,
                        const uint8_t** start_new_contour, uint64_t* n);
/* Host-side facts of the path's flatten program (no GPU needed): [0] output
 * points, [1] quadratics, [2] spline records, [3] point records (one of [2]/[3]
 * is 0: the smaller encoding is kept), [4] 1 if some quadratic is rational,
 * [5] contour ends before the last point. */
void forma_path_program_stats(forma_path*, uint64_t out[6]);
/* Inspection only (tests): the records of the path's flatten program as the host built
 * them, with the layouts of csrc/device_types.h: SplineRec (36 B), PointRec (8 B) with one
 * kind byte per record, QuadRec (68 B). One of n_splines / n_records is 0. bounds = min x,
 * min y, max x, max y of every point the program can emit; *bounded is 0 when no such bound
 * exists (a weight that is not positive). Host only: no device, no upload. The pointers stay
 * valid while the path (or a path transformed from it that shares its data) lives. */
void forma_path_program_records(forma_path*, const void** splines, uint64_t* n_splines, const void** points,
                                const uint8_t** kinds, uint64_t* n_records, const void** quads, uint64_t* n_quads,
                                int* bounded, float bounds[4]);

/* ------------------------------------------------------------------------ */
/* Composition / Layer (forma/src/composition/{mod,layer}.rs)               */
/* ------------------------------------------------------------------------ */
typedef struct forma_composition forma_composition;
/* A Layer handle is owned by its Composition and stays valid until
 * forma_layer_drop() or forma_composition_free(). */
typedef struct forma_layer forma_layer;

forma_composition* forma_composition_new(void);                   /* Composition::new mod.rs:60 */
void forma_composition_free(forma_composition*);
forma_layer* forma_composition_create_layer(forma_composition*);  /* mod.rs:65  (detached)      */
/* Composition::insert(Order::new(order)?, layer) mod.rs:121: returns the
 * displaced layer (now detached) or NULL; *status receives FORMA_ERR_ORDER_LIMIT. */
forma_layer* forma_composition_insert(forma_composition*, uint32_t order, forma_layer*, int* status);
forma_layer* forma_composition_remove(forma_composition*, uint32_t order);          /* mod.rs:141 */
forma_layer* forma_composition_get(forma_composition*, uint32_t order);             /* mod.rs:160 */
forma_layer* forma_composition_get_mut_or_insert_default(forma_composition*, uint32_t order,
                                                         int* status);              /* mod.rs:175 */
uint64_t forma_composition_len(forma_composition*);                                 /* mod.rs:115 */
void forma_layer_drop(forma_composition*, forma_layer*);               /* Drop for Layer, layer.rs:355 */

uint64_t forma_layer_geom_id(forma_layer*);                                        /* layer.rs:160 */
int forma_layer_insert(forma_composition*, forma_layer*, forma_path*);             /* layer.rs:90  */
int forma_layer_clear(forma_composition*, forma_layer*);                           /* layer.rs:131 */
int forma_layer_set_is_enabled(forma_composition*, forma_layer*, int enabled);     /* layer.rs:234 */
int forma_layer_is_enabled(forma_layer*);                                          /* layer.rs:207 */
/* GeomPresTransform::try_from([ux, vx, uy, vy, tx, ty]) + Layer::set_transform
 * (math/transform.rs:196-221, layer.rs:289); INVALID_ARGUMENT if it scales up. */
int forma_layer_set_transform(forma_composition*, forma_layer*, const float t[6]);
/* layer.rs:341. Equal props leave the layer unchanged for every layer cache; a texture whose
 * texels (as f16) equal the layer's current texture is the same image. */
int forma_layer_set_props(forma_composition*, forma_layer*, const forma_props*);

/* ------------------------------------------------------------------------ */
/* Renderer (forma/src/cpu/renderer.rs:56-224)                              */
/* ------------------------------------------------------------------------ */
typedef struct forma_renderer forma_renderer;
typedef struct forma_layer_cache forma_layer_cache;

/* Renderer::new (:62). Binds to CUDA device `device_ordinal`. Returns NULL and
 * sets forma_last_error() when no sm_90 device is usable. */
forma_renderer* forma_renderer_new(int device_ordinal);
void forma_renderer_free(forma_renderer*);

/* Renderer::create_buffer_layer_cache (:67); NULL when all 32 ids are in use. */
forma_layer_cache* forma_layer_cache_new(forma_renderer*);
void forma_layer_cache_free(forma_renderer*, forma_layer_cache*);
void forma_layer_cache_clear(forma_layer_cache*);                 /* BufferLayerCache::clear */

/* Renderer::render (:75-224) into a caller-owned HOST buffer laid out like
 * LinearLayout::new(width, width_stride, height) (cpu/buffer/layout/mod.rs:168).
 * Uploads what changed in the composition, runs all stages on the device and
 * copies the framebuffer (or, with a cache, only written tiles) back.
 * `timings` may be NULL: the call then does not read its stage events (a dozen event
 * queries); forma_renderer_stage_times still returns them afterwards. */
int forma_renderer_render(forma_renderer*, forma_composition*, uint8_t* buffer, uint64_t width,
                          uint64_t width_stride, uint64_t height, const uint32_t channels[4],
                          const float clear_color[4], const forma_rect* crop /* nullable */,
                          forma_layer_cache* cache /* nullable */, forma_timings* timings /* nullable */);

/* Same contract, but `device_buffer` is a CUDA device pointer on the
 * renderer's device (e.g. a torch tensor's data_ptr()): no device->host copy.
 * With a cache, the tiles the frame does not write keep the caller's bytes, as in
 * a host buffer, and so do the bytes between rows and outside the crop. A frame
 * with a cache builds its painter tables with the counts read back: it never takes
 * the sync-free path (option sync_free), whose first attempt could write the clear
 * colour into tiles the cache then finds unchanged.
 * Cache ids are per renderer (Renderer::create_buffer_layer_cache) while the
 * unchanged bits live on the layers: caches of two renderers that have the same
 * id share those bits, as in the reference. */
int forma_renderer_render_device(forma_renderer*, forma_composition*, uint8_t* device_buffer,
                                 uint64_t width, uint64_t width_stride, uint64_t height,
                                 const uint32_t channels[4], const float clear_color[4],
                                 const forma_rect* crop, forma_layer_cache* cache,
                                 forma_timings* timings);

/* ID frames (no reference counterpart): which layer made each pixel. One uint32 per pixel,
 * row-major, `ids_stride` BYTES between rows (a multiple of 4, at least 4 * width). The value
 * at pixel p is the order of the top-most Func::Draw layer that hits p, or FORMA_ID_NONE.
 * A layer hits p where the painter would blend it at p with coverage x clip mask >
 * min_coverage (the clip mask only where a clip applies to the layer): the painter's own tile
 * walk and optimiser passes decide, fill colour, alpha, gradient, texture and blend mode do not.
 * Clip layers, clipped layers without an active clip and disabled layers never hit; in a tile
 * the optimiser folds into one solid colour every pixel gets the top-most Draw layer of the
 * fold. Coverages are multiples of 1/512, so IDs are exact.
 * Only the crop's tile rectangle (clipped to width x height) is written, as with RGBA frames.
 * min_coverage must be finite and in [0, 1): otherwise INVALID_ARGUMENT and nothing is
 * written. An ID frame takes no layer cache and leaves every cache as it was.
 * render_ids copies the rectangle back into a HOST buffer; render_ids_device writes a device
 * buffer on the renderer's device. */
#define FORMA_ID_NONE 0xFFFFFFFFu
int forma_renderer_render_ids(forma_renderer*, forma_composition*, uint32_t* ids, uint64_t width,
                              uint64_t ids_stride, uint64_t height, const forma_rect* crop /* nullable */,
                              float min_coverage, forma_timings* timings /* nullable */);
int forma_renderer_render_ids_device(forma_renderer*, forma_composition*, uint32_t* device_ids, uint64_t width,
                                     uint64_t ids_stride, uint64_t height, const forma_rect* crop /* nullable */,
                                     float min_coverage, forma_timings* timings /* nullable */);
/* An RGBA frame (forma_renderer_render_device without a cache: the same bytes) and its ID frame
 * (forma_renderer_render_ids_device: the same IDs) from one pass through the stages: one
 * upload, rasterization, sort and set of painter tables, then the paint and the ID kernel.
 * Both buffers are in the renderer's device memory. */
int forma_renderer_render_device_with_ids(forma_renderer*, forma_composition*, uint8_t* device_buffer,
                                          uint64_t width, uint64_t width_stride, uint64_t height,
                                          const uint32_t channels[4], const float clear_color[4],
                                          const forma_rect* crop /* nullable */, uint32_t* device_ids,
                                          uint64_t ids_stride, float min_coverage, forma_timings* timings /* nullable */);

/* Views (no reference counterpart): `n` frames of one composition, each seen through its own
 * transform, from one pass through the stages. `views` holds n x 6 floats, each view in
 * forma_layer_set_transform order [ux, vx, uy, vy, tx, ty]. All frames share width x height,
 * width_stride, channels and clear colour; frame b starts at b * view_stride bytes, and
 * view_stride >= (height - 1) * width_stride + 4 * width, so frames never overlap. Only the
 * frames' width x height pixels are written: row padding and the bytes between frames stay.
 * Frame b is the bytes forma_renderer_render_device makes with every layer's transform
 * replaced by C = V_b ∘ T (V_b for a layer without a transform T), composed in f32 as
 *   C.ux = fmaf(V.ux, T.ux, V.vx * T.uy)   C.vx = fmaf(V.ux, T.vx, V.vx * T.vy)
 *   C.uy = fmaf(V.uy, T.ux, V.vy * T.uy)   C.vy = fmaf(V.uy, T.vx, V.vy * T.vy)
 *   C.tx = fmaf(V.ux, T.tx, fmaf(V.vx, T.ty, V.tx))   C.ty = fmaf(V.uy, T.tx, fmaf(V.vy, T.ty, V.ty))
 * with every product rounded on its own; a C equal to the identity is no transform. (Frames whose
 * lines all lie more than 2^19 px left of the frame are the exception: forma_renderer_render_device
 * mis-sorts their wrapped tile columns, the views do not.) Path
 * transforms apply first; gradients and textures stay in frame coordinates.
 * Every V_b must be finite and pass forma_layer_set_transform's check (no scaling up); the
 * composed C is not checked again, so two transforms that each pass may render with a C one
 * rounding past the limit. 1 <= n <= forma_renderer_max_views(height). A call that breaks one
 * of these rules returns FORMA_ERR_INVALID_ARGUMENT and writes nothing. FORMA_ERR_CAPACITY
 * applies to the pixel segments of all views together.
 * No layer cache is taken and every cache is left as it was. Afterwards counters, segments,
 * stage times and row costs describe the call's stacked frame (n * ceil(height / 16) tile
 * rows, view b's rows after view b - 1's), and forma_renderer_lines returns no records.
 * render_views_device writes a device buffer on the renderer's device (a [n, H, W, 4] uint8
 * tensor's data_ptr() with width_stride = 4 W, view_stride = 4 W H); render_views a host buffer. */
uint32_t forma_renderer_max_views(uint64_t height); /* floor(2046 / ceil(height / 16)); 0 when height is 0 or too tall;
                                                       also the most frames of one render_batch call */
int forma_renderer_render_views_device(forma_renderer*, forma_composition*, const float* views, uint32_t n,
                                       uint8_t* device_buffer, uint64_t width, uint64_t width_stride, uint64_t height,
                                       uint64_t view_stride, const uint32_t channels[4], const float clear_color[4],
                                       forma_timings* timings /* nullable */);
int forma_renderer_render_views(forma_renderer*, forma_composition*, const float* views, uint32_t n,
                                uint8_t* host_buffer, uint64_t width, uint64_t width_stride, uint64_t height,
                                uint64_t view_stride, const uint32_t channels[4], const float clear_color[4],
                                forma_timings* timings /* nullable */);

/* Batches (no reference counterpart): `n` frames of `n` compositions from one pass through the
 * stages, frame c showing comps[c] alone. The layout is that of the views: all frames share
 * width x height, width_stride, channels and clear colour; frame c starts at c * frame_stride
 * bytes, frame_stride >= (height - 1) * width_stride + 4 * width, and only the frames'
 * width x height pixels are written. Frame c is the bytes forma_renderer_render_device makes of
 * comps[c] without crop or cache (frames whose lines all lie more than 2^19 px left of the frame
 * excepted, as for the views). A composition may appear more than once; every occurrence is a
 * frame of its own.
 * Layer orders: the distinct compositions, in order of first appearance, get consecutive slices
 * of the 21-bit layer field. Composition k's slice starts at base_k, the sum of n_orders (its
 * largest attached order + 1, or 0 without layers) of the distinct compositions before it, and
 * its segments carry base_k + order. Clip ranges stay in the composition's own orders: a
 * Func::Clip(n) at order o covers o .. o + n, and only itself where o + n does not fit in 32 bits,
 * for every n in [0, 2^32) and whatever base_k is. The sum over all distinct compositions must not exceed
 * 2^21: otherwise FORMA_ERR_ORDER_LIMIT. Null comps or a null entry, n outside
 * 1 ... forma_renderer_max_views(height), a short frame_stride, or an invalid target or channel
 * return FORMA_ERR_INVALID_ARGUMENT. All of these are refused before anything is written.
 * FORMA_ERR_CAPACITY: more gradient stops or texels than the tables' 32-bit indices hold, or 2^30
 * pixel segments or more in all frames together.
 * Every composition is made resident whole (no band filter). No layer cache is taken and every
 * cache is left as it was. Afterwards counters, segments, stage times and row costs describe the
 * stacked frame (n * ceil(height / 16) tile rows), and forma_renderer_lines returns no records.
 * The renderer keeps the gathered tables of the last batch and gathers them again only when the
 * list of compositions or one of their tables changed.
 * render_batch_device writes a device buffer on the renderer's device (a [n, H, W, 4] uint8
 * tensor's data_ptr() with width_stride = 4 W, frame_stride = 4 W H); render_batch a host buffer. */
int forma_renderer_render_batch_device(forma_renderer*, forma_composition* const* comps, uint32_t n,
                                       uint8_t* device_buffer, uint64_t width, uint64_t width_stride, uint64_t height,
                                       uint64_t frame_stride, const uint32_t channels[4], const float clear_color[4],
                                       forma_timings* timings /* nullable */);
int forma_renderer_render_batch(forma_renderer*, forma_composition* const* comps, uint32_t n, uint8_t* host_buffer,
                                uint64_t width, uint64_t width_stride, uint64_t height, uint64_t frame_stride,
                                const uint32_t channels[4], const float clear_color[4], forma_timings* timings /* nullable */);

/* ID frames of views and batches: the ID frame (see forma_renderer_render_ids) of every frame of a
 * views or batch call, alone or together with the RGBA frames, from one pass through the stages.
 * The ID stack is laid out like the RGBA stack: ID frame b starts at b * ids_view_stride
 * (ids_frame_stride) bytes, its rows are ids_stride bytes apart. Both are multiples of 4,
 * ids_stride >= 4 * width and ids_view_stride >= (height - 1) * ids_stride + 4 * width. Only the
 * frames' width x height words are written: row padding and the bytes between frames stay.
 * The _device calls write the ID stack and, when device_buffer is not null, the RGBA stack as
 * well: one upload, line setup, sort and set of painter tables, then the paint kernel and the ID
 * kernel. The RGBA bytes are those of forma_renderer_render_views_device /
 * forma_renderer_render_batch_device with the same arguments. With a null device_buffer,
 * width_stride, view_stride / frame_stride, channels and clear_color are not read. The host
 * calls (render_views_ids, render_batch_ids) make ID frames only.
 * Views: ID frame b holds what forma_renderer_render_ids_device gives, without a crop, for the
 * composition with every layer's transform replaced by C = V_b ∘ T (the formula above); the
 * values are layer orders of the composition.
 * Batches: ID frame c holds what forma_renderer_render_ids_device gives for comps[c] alone: the
 * values are comps[c]'s own orders, not base_k + order (which slice of the layer field a
 * composition gets stays inside the call), and FORMA_ID_NONE where no layer hits. That holds for
 * every Func::Clip(n), n in [0, 2^32): a clip at order o covers the orders o .. o + n of its own
 * composition, and only itself when o + n does not fit in 32 bits, whatever its slice.
 * (Frames whose lines all lie more than 2^19 px left of the frame are the exception of views and
 * batches again: the stacked calls are right, forma_renderer_render_ids_device is not.)
 * min_coverage must be finite and in [0, 1); 1 <= n <= forma_renderer_max_views(height); the
 * order-sum, stop / texel and 2^30-segment limits of the RGBA calls apply. Every refusal
 * (FORMA_ERR_INVALID_ARGUMENT, also for a null ID buffer; FORMA_ERR_ORDER_LIMIT;
 * FORMA_ERR_CAPACITY) comes before anything is written to either buffer.
 * No layer cache is taken and every cache is left as it was. Afterwards counters, segments,
 * stage times and row costs describe the stacked frame; stage time [5] is the paint kernel
 * followed by the ID kernel, as after forma_renderer_render_device_with_ids.
 * With the defaults of a [n, H, W] int32 / uint32 tensor: ids_stride = 4 W, ids_view_stride = 4 W H. */
int forma_renderer_render_views_ids_device(forma_renderer*, forma_composition*, const float* views, uint32_t n,
                                           uint8_t* device_buffer /* nullable */, uint64_t width, uint64_t width_stride,
                                           uint64_t height, uint64_t view_stride, const uint32_t channels[4],
                                           const float clear_color[4], uint32_t* device_ids, uint64_t ids_stride,
                                           uint64_t ids_view_stride, float min_coverage, forma_timings* timings /* nullable */);
int forma_renderer_render_views_ids(forma_renderer*, forma_composition*, const float* views, uint32_t n, uint32_t* host_ids,
                                    uint64_t width, uint64_t ids_stride, uint64_t height, uint64_t ids_view_stride,
                                    float min_coverage, forma_timings* timings /* nullable */);
int forma_renderer_render_batch_ids_device(forma_renderer*, forma_composition* const* comps, uint32_t n,
                                           uint8_t* device_buffer /* nullable */, uint64_t width, uint64_t width_stride,
                                           uint64_t height, uint64_t frame_stride, const uint32_t channels[4],
                                           const float clear_color[4], uint32_t* device_ids, uint64_t ids_stride,
                                           uint64_t ids_frame_stride, float min_coverage, forma_timings* timings /* nullable */);
int forma_renderer_render_batch_ids(forma_renderer*, forma_composition* const* comps, uint32_t n, uint32_t* host_ids,
                                    uint64_t width, uint64_t ids_stride, uint64_t height, uint64_t ids_frame_stride,
                                    float min_coverage, forma_timings* timings /* nullable */);

/* Linear float frames (the reference's gpu::Renderer::render_to_texture writes an Rgba16Float
 * texture; see INTEGRATION.md): the painter's linear colour before the sRGB encode. Per pixel of
 * the written rectangle four values in the order of `channels`:
 *   - a painted tile: the planes (r, g, b, a) the painter holds after the tile's last blend, the
 *     values compute_srgb receives; no sRGB encode, no clamp, no rounding to bytes;
 *   - a tile the optimiser folds into one colour: that colour (BlendMode::blend's result);
 *   - a tile without layers: the clear colour;
 *   - FORMA_CHANNEL_ZERO gives 0.0, FORMA_CHANNEL_ONE 1.0, and ALPHA becomes ONE when
 *     clear_color[3] == 1, as for sRGB8 frames.
 * FORMA_PIXEL_RGBA32F stores the f32 values as they are (16 bytes per pixel); FORMA_PIXEL_RGBA16F
 * stores each rounded to the nearest half, ties to even (8 bytes per pixel): beyond the half range
 * a value becomes +-inf, a NaN stays a NaN. Encoding an RGBA32F frame with compute_srgb gives the
 * bytes forma_renderer_render_device writes for the same call.
 * Each call has the arguments of its sRGB8 twin (forma_renderer_render{,_device},
 * forma_renderer_render_views{,_device}, forma_renderer_render_batch{,_device}) without the layer
 * cache and with `format`; `buffer` may hold any type, and every stride is in BYTES:
 * width_stride >= bpp * width and view_stride / frame_stride >= (height - 1) * width_stride +
 * bpp * width, bpp = 8 or 16. The buffer and every stride must be multiples of 4 bytes; 16 lets
 * the paint kernel store 16-byte vectors. Refused with FORMA_ERR_INVALID_ARGUMENT before anything
 * is written: a null buffer, a format other than the two below, a stride or alignment that breaks
 * these rules, and everything the sRGB8 twin refuses (n, views, null batch entries, ...); the
 * order-sum, stop / texel and 2^30-segment limits of the twins apply as well. Only the crop's
 * tile rectangle (single frames) or the frames' width x height pixels (stacks) are written.
 * A float frame takes no layer cache and leaves every cache as it was. With the defaults of a
 * [H, W, 4] / [n, H, W, 4] float32 or float16 tensor: width_stride = bpp * W, view_stride /
 * frame_stride = bpp * W * H. */
enum { FORMA_PIXEL_RGBA16F = 1, FORMA_PIXEL_RGBA32F = 2 };
int forma_renderer_render_linear(forma_renderer*, forma_composition*, void* buffer, uint64_t width, uint64_t width_stride,
                                 uint64_t height, const uint32_t channels[4], const float clear_color[4],
                                 const forma_rect* crop /* nullable */, uint32_t format, forma_timings* timings /* nullable */);
int forma_renderer_render_linear_device(forma_renderer*, forma_composition*, void* device_buffer, uint64_t width,
                                        uint64_t width_stride, uint64_t height, const uint32_t channels[4],
                                        const float clear_color[4], const forma_rect* crop /* nullable */, uint32_t format,
                                        forma_timings* timings /* nullable */);
int forma_renderer_render_views_linear(forma_renderer*, forma_composition*, const float* views, uint32_t n, void* host_buffer,
                                       uint64_t width, uint64_t width_stride, uint64_t height, uint64_t view_stride,
                                       const uint32_t channels[4], const float clear_color[4], uint32_t format,
                                       forma_timings* timings /* nullable */);
int forma_renderer_render_views_linear_device(forma_renderer*, forma_composition*, const float* views, uint32_t n,
                                              void* device_buffer, uint64_t width, uint64_t width_stride, uint64_t height,
                                              uint64_t view_stride, const uint32_t channels[4], const float clear_color[4],
                                              uint32_t format, forma_timings* timings /* nullable */);
int forma_renderer_render_batch_linear(forma_renderer*, forma_composition* const* comps, uint32_t n, void* host_buffer,
                                       uint64_t width, uint64_t width_stride, uint64_t height, uint64_t frame_stride,
                                       const uint32_t channels[4], const float clear_color[4], uint32_t format,
                                       forma_timings* timings /* nullable */);
int forma_renderer_render_batch_linear_device(forma_renderer*, forma_composition* const* comps, uint32_t n, void* device_buffer,
                                              uint64_t width, uint64_t width_stride, uint64_t height, uint64_t frame_stride,
                                              const uint32_t channels[4], const float clear_color[4], uint32_t format,
                                              forma_timings* timings /* nullable */);

/* Frames over a background: draw onto pixels a device buffer already holds (video frames, photos,
 * a batch of training images). The calls take no clear colour: the buffer's current contents are
 * the background. The value written at pixel p is exactly the value the twin call writes at p when
 * its clear colour is decode(background[p]): byte for byte in FORMA_PIXEL_SRGB8, bit for bit in
 * the float formats. That includes the optimiser's fold of full layers (per pixel from the pixel's
 * background, unless an opaque layer is the bottom) and the Alpha -> One upgrade (per pixel, where
 * the decoded alpha is exactly 1). The twins: forma_renderer_render_device /
 * forma_renderer_render_linear_device, forma_renderer_render_views{,_linear}_device and
 * forma_renderer_render_batch{,_linear}_device; each call has its twin's arguments without the clear
 * colour and the layer cache, and with `format`.
 * decode, per channel:
 *   - FORMA_PIXEL_RGBA32F: the stored value; FORMA_PIXEL_RGBA16F: __half2float (exact);
 *   - FORMA_PIXEL_SRGB8: alpha = (float)byte / 255.0f; r, g, b = D[byte], a table of 256 f32
 *     (forma_b200/csrc/srgb_decode.h): the f32 nearest the standard sRGB EOTF of byte / 255 when
 *     compute_srgb's encode turns it back into the byte, else the nearest f32 that it does (byte 11:
 *     the EOTF gives 0.0033465, which encodes to 12; D[11] = 0.0033159761). Every byte round-trips,
 *     so a pixel that nothing covers comes back unchanged.
 * Rules:
 *   - `channels` is a permutation of R, G, B, A (ZERO and ONE cannot be decoded); for
 *     FORMA_PIXEL_SRGB8 with A last (RGBA, BGRA, ...): the twin writes a solid tile's bytes by
 *     position, alpha unencoded at position 3, and only then does such a tile decode to its colour;
 *   - the buffer and every stride are multiples of 4 bytes, strides as for the twin of the same
 *     format (bpp = 4, 8 or 16);
 *   - only the crop's tile rectangle (single frames) or the frames' width x height pixels (stacks)
 *     are read or written; row padding and the bytes between frames stay as they were. A tile no
 *     layer reaches is not written at all (its pixels are what the twin would write there);
 *   - no layer cache is taken, and every cache is left as it was;
 *   - every refusal returns FORMA_ERR_INVALID_ARGUMENT before anything is read or written: a null
 *     buffer, an unknown format, bad strides or alignment, a channel order that is not one of the
 *     above, and everything the twin refuses; the twin's order-sum, stop / texel and 2^30-segment
 *     limits apply as well;
 *   - counters, segments, stage times and row costs afterwards are those of the twin; a stack that is
 *     not painted in place (frames not whole tile rows laid out as the stacked frame's rows) has one
 *     more launch: its background is copied into the renderer's scratch before painting.
 * With the defaults of a [H, W, 4] / [n, H, W, 4] uint8, float16 or float32 tensor: width_stride =
 * bpp * W, view_stride / frame_stride = bpp * W * H. */
enum { FORMA_PIXEL_SRGB8 = 0 };
int forma_renderer_render_over_device(forma_renderer*, forma_composition*, void* device_buffer, uint64_t width,
                                      uint64_t width_stride, uint64_t height, const uint32_t channels[4],
                                      const forma_rect* crop /* nullable */, uint32_t format, forma_timings* timings /* nullable */);
int forma_renderer_render_views_over_device(forma_renderer*, forma_composition*, const float* views, uint32_t n,
                                            void* device_buffer, uint64_t width, uint64_t width_stride, uint64_t height,
                                            uint64_t view_stride, const uint32_t channels[4], uint32_t format,
                                            forma_timings* timings /* nullable */);
int forma_renderer_render_batch_over_device(forma_renderer*, forma_composition* const* comps, uint32_t n, void* device_buffer,
                                            uint64_t width, uint64_t width_stride, uint64_t height, uint64_t frame_stride,
                                            const uint32_t channels[4], uint32_t format, forma_timings* timings /* nullable */);

/* Layer coverage masks (no reference counterpart): each layer's anti-aliased coverage as a plane of
 * its own, for instance mattes, amodal masks and per-shape losses. A request names a window of
 * layer orders [first_order, first_order + n_orders), n_orders = K >= 1; plane k holds order
 * o = first_order + k. Its value at pixel p:
 *   - o an enabled Func::Draw layer without is_clipped: c_o(p), the coverage the painter's
 *     paint_layer computes for o at p under its fill rule from its cells and carried cover
 *     (doubled_area_to_coverage), a multiple of 1/512 in [0, 1];
 *   - o a Func::Draw layer with is_clipped: c_o(p) x m(p), m the clip mask that applies to o in p's
 *     tile in the painter's walk of the composition cut off above o (clip_at, cpu/painter/mod.rs:
 *     302-323, 449-464): the tile's layers are walked bottom-up from its first layer after the
 *     skip_trivial_clips pass with every layer painted, so the mask is amodal (the parts other
 *     layers hide are kept), and the clip state restarts at every layer the painter could start
 *     from (skip_fully_covered_layers: painted, not clipped, full in the tile, a solid opaque Over
 *     fill). Where no clip applies to o (no clip active, or the pass masks o out), 0; where the
 *     pass finds o's clip full, the clip is 1 and the value c_o(p). So wherever o is painted, its
 *     value is exactly the coverage x clip mask the painter paints it with;
 *   - o a Func::Clip layer: its own coverage c_o(p);
 *   - anything else (no such layer, a disabled layer, a layer without props): 0.
 * Colour, alpha, gradient, texture and blend mode play no part, nor does any other layer than the
 * clips. A plane of an unclipped Draw layer is the alpha of a linear frame (clear colour 0) of the
 * composition with every other Draw layer disabled and o solid white, opaque and Over.
 * Formats: FORMA_MASK_F32 stores the value (exact: k / 512 or a product of two such values);
 * FORMA_MASK_U8 stores compute_srgb's encode of alpha, the low byte of
 * bits(clamp(255 v, 0, 255) + 2^23).
 * Layout: plane (frame b, k) starts at ptr + (b K + k) plane_stride, its rows `stride` bytes apart
 * (a [n, K, H, W] tensor, or [K, H, W] for a single frame: stride = bpp W, plane_stride = bpp W H,
 * bpp = 4 or 1). Only each plane's width x height pixels are written, and for a single frame only
 * the crop's tile rectangle; row padding and the bytes between planes stay as they were. For a
 * batch, frame c's planes are comps[c]'s own orders; every view uses the same orders.
 * With a non-null device_buffer the call also writes the sRGB8 RGBA frame or stack from the same
 * pass (one upload, line setup, sort and set of painter tables): exactly the bytes of
 * forma_renderer_render_device (without a layer cache), forma_renderer_render_views_device or
 * forma_renderer_render_batch_device with the same arguments. With a null device_buffer,
 * width_stride, view_stride / frame_stride, channels and clear_color are not read.
 * Refusals return FORMA_ERR_INVALID_ARGUMENT before anything is written to either buffer: a null
 * descriptor or pointer; K = 0 or first_order + K > 2^21; an unknown format; stride < bpp width;
 * plane_stride < (height - 1) stride + bpp width; F32 pointers or strides that are not multiples of
 * 4; a plane stack whose size overflows 64 bits; and everything the RGBA calls refuse for the
 * target, views and batches. Their order-sum, stop / texel and 2^30-segment limits apply as well.
 * A mask call takes no layer cache and leaves every cache as it was. Afterwards counters,
 * segments, stage times and row costs describe the call's frame; stage time [5] covers the paint
 * kernel and the mask kernels (a zero fill of the planes' written rectangles, then the masks).
 * render_masks paints into device scratch and copies the planes' rectangles into a HOST buffer;
 * the _device calls write device memory on the renderer's device. */
enum { FORMA_MASK_F32 = 0, FORMA_MASK_U8 = 1 };
typedef struct forma_masks {
    void* ptr;
    uint32_t first_order, n_orders, format;
    uint64_t stride, plane_stride; /* bytes */
} forma_masks;
int forma_renderer_render_masks(forma_renderer*, forma_composition*, const forma_masks* masks, uint64_t width, uint64_t height,
                                const forma_rect* crop /* nullable */, forma_timings* timings /* nullable */);
int forma_renderer_render_masks_device(forma_renderer*, forma_composition*, const forma_masks* masks, uint64_t width,
                                       uint64_t height, const forma_rect* crop /* nullable */,
                                       uint8_t* device_buffer /* nullable */, uint64_t width_stride, const uint32_t channels[4],
                                       const float clear_color[4], forma_timings* timings /* nullable */);
int forma_renderer_render_views_masks_device(forma_renderer*, forma_composition*, const float* views, uint32_t n,
                                             const forma_masks* masks, uint64_t width, uint64_t height,
                                             uint8_t* device_buffer /* nullable */, uint64_t width_stride, uint64_t view_stride,
                                             const uint32_t channels[4], const float clear_color[4],
                                             forma_timings* timings /* nullable */);
int forma_renderer_render_batch_masks_device(forma_renderer*, forma_composition* const* comps, uint32_t n,
                                             const forma_masks* masks, uint64_t width, uint64_t height,
                                             uint8_t* device_buffer /* nullable */, uint64_t width_stride, uint64_t frame_stride,
                                             const uint32_t channels[4], const float clear_color[4],
                                             forma_timings* timings /* nullable */);

/* Layer statistics (no reference counterpart): a handful of exact integers per layer instead of
 * its planes, for the boxes, areas and occlusion ratios of instance and amodal datasets. A request
 * names a window of layer orders [first_order, first_order + n_orders), n_orders = K >= 1, as the
 * mask calls do, and a min_coverage in [0, 1) as the ID calls do. For every frame b and every
 * order o of the window there is one 48-byte record, frame b's at ptr + b K:
 *   - area:    sum over the counted pixels p of v_o(p) x 2^18, v_o(p) exactly the F32 value of
 *              forma_renderer_render_masks for o at p (clipped and clip layers included; 0 for
 *              orders that are absent, disabled or without props). v is k / 512 or a product of
 *              two such values, so the sum is an exact integer;
 *   - pixels:  the counted pixels with v_o(p) > min_coverage;
 *   - visible: the counted pixels whose ID (forma_renderer_render_ids at min_coverage) is o;
 *   - box, visible_box: x0, y0, x1, y1 (half-open, in frame pixels) of the `pixels` and the
 *              `visible` set; all four 0 when the set is empty.
 * A pixel's ID is o only where v_o(p) > min_coverage (the painter paints o there with v_o), so
 * visible <= pixels and visible_box lies inside box: visible / pixels is the share of a layer that
 * no layer above it hides, the occlusion ratio.
 * Counted pixels: for a single frame, the frame's pixels inside the crop's tile rectangle (the
 * rectangle mask and ID calls write); for views and batches, each frame's own width x height
 * pixels in its own coordinates (rows of the last tile row at or below `height` never count).
 * For a batch, frame c's records are comps[c]'s own orders; every view reports the same orders.
 * The records are integers, so the result does not depend on the order the device adds them in:
 * two identical calls give identical bytes.
 * With a non-null device_buffer the device calls also write the sRGB8 RGBA frame or stack from
 * the same pass: exactly the bytes of forma_renderer_render_device (without a layer cache),
 * forma_renderer_render_views_device or forma_renderer_render_batch_device with the same
 * arguments. With a null device_buffer, width_stride, view_stride / frame_stride, channels and
 * clear_color are not read.
 * Refusals return FORMA_ERR_INVALID_ARGUMENT before anything is written to either buffer: a null
 * descriptor or pointer; a pointer that is not 8-byte aligned; K = 0 or first_order + K > 2^21;
 * min_coverage not finite or outside [0, 1); a record array whose size overflows 64 bits; and
 * everything the mask calls refuse for the target, views and batches. Their order-sum, stop /
 * texel and 2^30-segment limits apply as well. Statistics go alone or with an sRGB8 RGBA target,
 * never with IDs or masks; they take no layer cache and leave every cache as it was. Afterwards
 * counters, segments, stage times and row costs describe the call's frame; stage time [5] covers
 * the paint kernel and the statistics kernels (the records' initialisation, the amodal walk, the
 * visible walk and the empty boxes' fix-up).
 * render_stats reduces into device scratch and copies the records into a HOST array; the _device
 * calls write device memory on the renderer's device. */
typedef struct forma_layer_stats {
    uint64_t area;           /* sum over p of v_o(p) * 2^18: exact (v is k/512 or a product of two such) */
    uint32_t pixels;         /* pixels p with v_o(p) > min_coverage                                      */
    uint32_t visible;        /* pixels p whose ID (forma_renderer_render_ids at min_coverage) is o       */
    uint32_t box[4];         /* x0, y0, x1, y1 (half-open, frame pixels) of the `pixels` set; 0s if empty */
    uint32_t visible_box[4]; /* the same for the `visible` set                                           */
} forma_layer_stats;
typedef struct forma_stats {
    forma_layer_stats* ptr; /* frame b's records at ptr + b * n_orders; 8-byte aligned */
    uint32_t first_order, n_orders;
    float min_coverage;
} forma_stats;
int forma_renderer_render_stats(forma_renderer*, forma_composition*, const forma_stats* stats, uint64_t width, uint64_t height,
                                const forma_rect* crop /* nullable */, forma_timings* timings /* nullable */);
int forma_renderer_render_stats_device(forma_renderer*, forma_composition*, const forma_stats* stats, uint64_t width,
                                       uint64_t height, const forma_rect* crop /* nullable */,
                                       uint8_t* device_buffer /* nullable */, uint64_t width_stride, const uint32_t channels[4],
                                       const float clear_color[4], forma_timings* timings /* nullable */);
int forma_renderer_render_views_stats_device(forma_renderer*, forma_composition*, const float* views, uint32_t n,
                                             const forma_stats* stats, uint64_t width, uint64_t height,
                                             uint8_t* device_buffer /* nullable */, uint64_t width_stride, uint64_t view_stride,
                                             const uint32_t channels[4], const float clear_color[4],
                                             forma_timings* timings /* nullable */);
int forma_renderer_render_batch_stats_device(forma_renderer*, forma_composition* const* comps, uint32_t n,
                                             const forma_stats* stats, uint64_t width, uint64_t height,
                                             uint8_t* device_buffer /* nullable */, uint64_t width_stride, uint64_t frame_stride,
                                             const uint32_t channels[4], const float clear_color[4],
                                             forma_timings* timings /* nullable */);

/* Poses (no reference counterpart): n frames of one composition, from one pass through the
 * stages. In frame b, each layer attached at an order o of the window [first_order,
 * first_order + K), k = o - first_order, gets its own transform and visibility: frame b is
 * exactly the bytes forma_renderer_render_device writes (no crop, no cache) for the composition
 * after
 *   forma_layer_set_transform(layer, transforms + 6 (b K + k))      when transforms is not null,
 *   forma_layer_set_is_enabled(layer, visible[b K + k] != 0)         when visible is not null
 *   forma_layer_set_props(layer, props with the fill Solid(colors[b K + k]))
 *                                when colors is not null and the layer's func is Draw(style)
 * (the state is set outright: a disabled layer can be shown in some frames). Layers outside the
 * window, orders of the window without a layer, path transforms, gradients and textures stay as
 * they are; gradients and textures stay in frame coordinates. A pose transform equal to
 * the identity is no transform, as forma_layer_set_transform has it. (Frames whose lines all lie
 * more than 2^19 px left of the frame are the exception of views and batches again: the stacked
 * call is right, forma_renderer_render_device mis-sorts their wrapped tile columns.)
 * The call does not change the composition: afterwards every layer's transform, enabled state and
 * per-cache unchanged bits are what they were, and the next ordinary render uploads nothing
 * because of it. The geometry is flattened and made resident once; per call, K 32-byte records of
 * the window's layers cross PCIe, and of the tables in host memory their bytes: n K 24-byte
 * transforms, n K visibility bytes, n K 16-byte colours. Tables in device memory do not cross.
 * Where the tables live: each non-null table may be in host memory (pageable, page-locked or
 * managed) or in device memory of the renderer's device, in any combination, with the same frames,
 * IDs, masks, statistics and refusals either way. The library asks CUDA
 * (cudaPointerGetAttributes) where each one is. A device table
 *   - is read on the renderer's stream (forma_renderer_set_stream): it must be complete in stream
 *     order on that stream, as the background of the _over_device calls must be;
 *   - must stay valid until the call returns, which is after the call's final synchronisation;
 *   - must hold n K rows: its size is the caller's responsibility, as for frame buffers;
 *   - of transforms or colours must be 4-byte aligned (FORMA_ERR_INVALID_ARGUMENT otherwise,
 *     before anything is launched); visibility bytes may start at any byte.
 * A table in device memory of another device is refused with FORMA_ERR_INVALID_ARGUMENT naming
 * both devices. Device transforms are checked on the device, which costs their calls a 4-byte
 * read-back and a wait before line setup (calls without them wait for nothing new); a refused
 * transform leaves buffers and composition as every refusal listed below does.
 * Pose fills (colors not null): the props set in frame b are the layer's own with the fill alone
 * replaced; its fill_rule, is_clipped, blend_mode (the non-separable modes included) and the
 * layer's clip range stay, so a gradient or texture layer of the window becomes solid. A Clip
 * layer has no fill: its colours are not read. Every float is taken as it is, NaN and infinities
 * included, as forma_layer_set_props takes them; an alpha that makes a full layer opaque, or stops
 * it being opaque, moves what the frame's IDs, masks and statistics see beneath it, as it would
 * after forma_layer_set_props. The call builds a pose style table in renderer-owned device memory,
 * 112 (S + n K) bytes for a composition of S style records (at most one per layer): about 90 MB for
 * 16 frames of 50 620 recoloured layers. It is kept for the next call, as the other per-frame
 * buffers are.
 * ABI: colors is the last member, so every other member keeps its offset, and a descriptor that
 * was zero-initialised before colors existed (colors = NULL) renders as it did.
 * Each call is the twin of a views call, with `const forma_poses* poses, uint32_t n` in place of
 * `const float* views, uint32_t n`: the same arguments, layouts, rules, limits, refusals and state
 * afterwards (counters, segments, stage times and row costs of the stacked frame, no line records):
 *   render_poses{,_device}       forma_renderer_render_views{,_device}
 *   render_poses_ids{,_device}   forma_renderer_render_views_ids{,_device} (RGBA optional, as there)
 *   render_poses_masks_device    forma_renderer_render_views_masks_device
 *   render_poses_stats_device    forma_renderer_render_views_stats_device
 *   render_poses_linear{,_device} forma_renderer_render_views_linear{,_device}
 *   render_poses_over_device     forma_renderer_render_views_over_device
 * In the ID, mask and statistics calls the values are the composition's own orders.
 * Besides the twin's refusals, FORMA_ERR_INVALID_ARGUMENT is returned before anything is written
 * to any buffer, with the composition untouched, for: a null poses; all three tables null; K = 0
 * or first_order + K > 2^21; n K 6 floats overflowing 64 bits; any pose transform that
 * forma_layer_set_transform refuses (forma_last_error() names the frame and the order). Unlike a
 * view, a pose transform need not be finite: a NaN or infinite translation renders as
 * forma_renderer_render_device renders it. FORMA_ERR_CAPACITY, also before anything is written:
 * the pose records or the pose style table cannot be allocated; with colors, S + n K >= 2^31 (the
 * style slots are 32-bit signed); or the twin's limits. */
typedef struct forma_poses {
    uint32_t first_order, n_orders; /* the window, K = n_orders >= 1, first_order + K <= 2^21        */
    const float* transforms;        /* nullable: n x K x 6 floats [ux, vx, uy, vy, tx, ty] per       */
                                    /*   (frame b, order first_order + k) at 6 (b K + k), in          */
                                    /*   forma_layer_set_transform order                              */
    const uint8_t* visible;         /* nullable: n x K bytes at b K + k; 0 = disabled in frame b      */
    const float* colors;            /* nullable: n x K x 4 floats, linear RGBA as in forma_color, at  */
                                    /*   4 (b K + k): the solid fill of a Draw layer in frame b       */
} forma_poses;
int forma_renderer_render_poses_device(forma_renderer*, forma_composition*, const forma_poses* poses, uint32_t n,
                                       uint8_t* device_buffer, uint64_t width, uint64_t width_stride, uint64_t height,
                                       uint64_t view_stride, const uint32_t channels[4], const float clear_color[4],
                                       forma_timings* timings /* nullable */);
int forma_renderer_render_poses(forma_renderer*, forma_composition*, const forma_poses* poses, uint32_t n,
                                uint8_t* host_buffer, uint64_t width, uint64_t width_stride, uint64_t height,
                                uint64_t view_stride, const uint32_t channels[4], const float clear_color[4],
                                forma_timings* timings /* nullable */);
int forma_renderer_render_poses_ids_device(forma_renderer*, forma_composition*, const forma_poses* poses, uint32_t n,
                                           uint8_t* device_buffer /* nullable */, uint64_t width, uint64_t width_stride,
                                           uint64_t height, uint64_t view_stride, const uint32_t channels[4],
                                           const float clear_color[4], uint32_t* device_ids, uint64_t ids_stride,
                                           uint64_t ids_view_stride, float min_coverage, forma_timings* timings /* nullable */);
int forma_renderer_render_poses_ids(forma_renderer*, forma_composition*, const forma_poses* poses, uint32_t n, uint32_t* host_ids,
                                    uint64_t width, uint64_t ids_stride, uint64_t height, uint64_t ids_view_stride,
                                    float min_coverage, forma_timings* timings /* nullable */);
int forma_renderer_render_poses_masks_device(forma_renderer*, forma_composition*, const forma_poses* poses, uint32_t n,
                                             const forma_masks* masks, uint64_t width, uint64_t height,
                                             uint8_t* device_buffer /* nullable */, uint64_t width_stride, uint64_t view_stride,
                                             const uint32_t channels[4], const float clear_color[4],
                                             forma_timings* timings /* nullable */);
int forma_renderer_render_poses_stats_device(forma_renderer*, forma_composition*, const forma_poses* poses, uint32_t n,
                                             const forma_stats* stats, uint64_t width, uint64_t height,
                                             uint8_t* device_buffer /* nullable */, uint64_t width_stride, uint64_t view_stride,
                                             const uint32_t channels[4], const float clear_color[4],
                                             forma_timings* timings /* nullable */);
int forma_renderer_render_poses_linear(forma_renderer*, forma_composition*, const forma_poses* poses, uint32_t n,
                                       void* host_buffer, uint64_t width, uint64_t width_stride, uint64_t height,
                                       uint64_t view_stride, const uint32_t channels[4], const float clear_color[4],
                                       uint32_t format, forma_timings* timings /* nullable */);
int forma_renderer_render_poses_linear_device(forma_renderer*, forma_composition*, const forma_poses* poses, uint32_t n,
                                              void* device_buffer, uint64_t width, uint64_t width_stride, uint64_t height,
                                              uint64_t view_stride, const uint32_t channels[4], const float clear_color[4],
                                              uint32_t format, forma_timings* timings /* nullable */);
int forma_renderer_render_poses_over_device(forma_renderer*, forma_composition*, const forma_poses* poses, uint32_t n,
                                            void* device_buffer, uint64_t width, uint64_t width_stride, uint64_t height,
                                            uint64_t view_stride, const uint32_t channels[4], uint32_t format,
                                            forma_timings* timings /* nullable */);

/* Instance scenes (no reference counterpart): n frames, each drawing its own list of copies of the
 * composition's layers, from one pass through the stages. The composition serves as a library of
 * geometry and props: frame b has M = n_instances slots, and slot m draws the layer attached at
 * order p = prototypes[b M + m] (FORMA_NO_INSTANCE: nothing). Frame b is exactly the bytes
 * forma_renderer_render_device writes (no crop, no cache) for a composition T_b that has, for every
 * slot m with a prototype p, a layer at order m with
 *   - the geometry of the layer at order p: every live insert of it (not those a Layer::clear
 *     dropped), in insertion order, with their path transforms;
 *   - p's props; with colors, a Draw layer's fill replaced by Solid(colors[b M + m]) (its fill rule,
 *     is_clipped, blend mode and a Clip layer's range stay; a Clip layer's colour is not read);
 *   - the transform transforms[b M + m] when that table is given (an identity is no transform), p's
 *     own transform otherwise;
 *   - enabled, whatever p's own enabled state is (a library is usually kept disabled, so that its
 *     ordinary frames show nothing).
 * Empty slots have no layer. A prototype may fill any number of slots of any frame, in any order.
 * (Frames whose lines all lie more than 2^19 px left of the frame are the exception of views and
 * batches again: the stacked call is right, forma_renderer_render_device is not.)
 * IDs, mask planes and statistics records are indexed by the slot m (T_b's orders): the ID frame
 * is an instance-segmentation label and the statistics are per-instance boxes and areas.
 * The call does not change the composition: no layer state, unchanged bit, table or geometry.
 * The geometry is flattened and made resident once; per call the host builds one 16-byte line
 * record per (frame, slot, live insert) and one 64-byte frame record per frame, which cross PCIe
 * with the host tables' bytes (4 n M prototypes, 24 n M transforms, 16 n M colours) and 32 bytes
 * per order up to the largest prototype (the prototypes' own transforms).
 * Where the tables live: each table may be in host memory or in device memory of the renderer's
 * device, under the rules of forma_poses (cudaPointerGetAttributes; another device's memory is
 * refused; device float tables 4-byte aligned; read on the renderer's stream). A device
 * `prototypes` table is copied to the host (4 n M bytes and one wait) because it decides the launch
 * sizes; device transforms are checked on the device, at the cost of a 4-byte read-back and a wait.
 * Each call is the twin of a views call, with `const forma_instances* instances, uint32_t n` in
 * place of `const float* views, uint32_t n`: the same arguments, layouts, rules, limits, refusals
 * and state afterwards (counters, segments, stage times and row costs of the stacked frame, no line
 * records):
 *   render_instances_device        forma_renderer_render_views_device
 *   render_instances_ids_device    forma_renderer_render_views_ids_device (RGBA optional, as there)
 *   render_instances_masks_device  forma_renderer_render_views_masks_device (window in slots m)
 *   render_instances_stats_device  forma_renderer_render_views_stats_device (window in slots m)
 * Besides the twin's refusals, FORMA_ERR_INVALID_ARGUMENT is returned before anything is written,
 * with the composition untouched, for: a null descriptor or null prototypes; M = 0; a prototype
 * order without an attached layer (forma_last_error() names the frame, the slot and the order); a
 * slot's transform that forma_layer_set_transform refuses (the frame and the slot are named; the
 * transforms of empty slots are not checked);
 * device float tables that are not 4-byte aligned. FORMA_ERR_ORDER_LIMIT: n M > 2^21 (frame b's
 * instances take the orders b M ... b M + M - 1 of the layer field). FORMA_ERR_CAPACITY: the
 * 2^30-segment limit of the twin, a frame of 2^31 or more point pairs, or instance records or
 * the instance style table (112 (S + n M) bytes with colors, S the composition's style records)
 * that cannot be allocated. Transforms need not be finite: a NaN or infinite translation renders
 * as forma_renderer_render_device renders it. */
#define FORMA_NO_INSTANCE 0xFFFFFFFFu
typedef struct forma_instances {
    uint32_t n_instances;        /* M >= 1 instance slots per frame                                   */
    const uint32_t* prototypes;  /* n x M layer orders at b M + m; FORMA_NO_INSTANCE = empty slot      */
    const float* transforms;     /* nullable: n x M x 6 floats at 6 (b M + m), set_transform order     */
    const float* colors;         /* nullable: n x M x 4 floats at 4 (b M + m), linear RGBA solid fill */
} forma_instances;
int forma_renderer_render_instances_device(forma_renderer*, forma_composition*, const forma_instances* instances, uint32_t n,
                                           uint8_t* device_buffer, uint64_t width, uint64_t width_stride, uint64_t height,
                                           uint64_t view_stride, const uint32_t channels[4], const float clear_color[4],
                                           forma_timings* timings /* nullable */);
int forma_renderer_render_instances_ids_device(forma_renderer*, forma_composition*, const forma_instances* instances, uint32_t n,
                                               uint8_t* device_buffer /* nullable */, uint64_t width, uint64_t width_stride,
                                               uint64_t height, uint64_t view_stride, const uint32_t channels[4],
                                               const float clear_color[4], uint32_t* device_ids, uint64_t ids_stride,
                                               uint64_t ids_view_stride, float min_coverage, forma_timings* timings /* nullable */);
int forma_renderer_render_instances_masks_device(forma_renderer*, forma_composition*, const forma_instances* instances, uint32_t n,
                                                 const forma_masks* masks, uint64_t width, uint64_t height,
                                                 uint8_t* device_buffer /* nullable */, uint64_t width_stride, uint64_t view_stride,
                                                 const uint32_t channels[4], const float clear_color[4],
                                                 forma_timings* timings /* nullable */);
int forma_renderer_render_instances_stats_device(forma_renderer*, forma_composition*, const forma_instances* instances, uint32_t n,
                                                 const forma_stats* stats, uint64_t width, uint64_t height,
                                                 uint8_t* device_buffer /* nullable */, uint64_t width_stride, uint64_t view_stride,
                                                 const uint32_t channels[4], const float clear_color[4],
                                                 forma_timings* timings /* nullable */);

/* Launch on `cuda_stream` (a cudaStream_t, e.g. torch.cuda.current_stream().cuda_stream)
 * instead of the default stream. */
void forma_renderer_set_stream(forma_renderer*, void* cuda_stream);

/* Several GPUs behind one renderer, single process (Renderer::new for a multi-GPU box):
 * `render` has the contract of forma_renderer_render, `render_device` that of
 * forma_renderer_render_device with the frame in the FIRST listed device's memory (the other
 * devices store their rows into it over NVLink; needs peer access). The frame is split into
 * bands of tile rows, one per device, rebalanced every frame on the previous frame's row
 * costs; each device keeps only its band's geometry resident. Layer caches are not
 * supported here (cache = NULL semantics). Every listed device must be an sm_90 GPU. */
typedef struct forma_renderer_multi forma_renderer_multi;
forma_renderer_multi* forma_renderer_multi_new(const int* device_ordinals, int n);
void forma_renderer_multi_free(forma_renderer_multi*);
int forma_renderer_multi_device_count(const forma_renderer_multi*);
int forma_renderer_multi_render(forma_renderer_multi*, forma_composition*, uint8_t* buffer, uint64_t width,
                                uint64_t width_stride, uint64_t height, const uint32_t channels[4],
                                const float clear_color[4], const forma_rect* crop, forma_timings* timings);
int forma_renderer_multi_render_device(forma_renderer_multi*, forma_composition*, uint8_t* buffer_on_first_device,
                                       uint64_t width, uint64_t width_stride, uint64_t height,
                                       const uint32_t channels[4], const float clear_color[4],
                                       const forma_rect* crop, forma_timings* timings);
/* bounds[n + 1]: tile-row boundaries of the bands the next frame will use; band_ms[n]:
 * device-timeline ms of every band in the last frame. Returns n. */
int forma_renderer_multi_bands(const forma_renderer_multi*, uint32_t* bounds, double* band_ms);

/* Multi-GPU frame assembly without a copy (one process per GPU, tile-row bands,
 * SURVEY.md §8e): the process that owns the frame allocates it with
 * forma_shared_frame_create and passes the 64-byte handle to the others (any
 * channel, e.g. torch.distributed); they map it with forma_shared_frame_open
 * (CUDA IPC, peer access over NVLink) and hand the mapped pointer to
 * forma_renderer_render_device with their band as `crop`: the paint kernel's
 * stores then land directly in the owner's HBM. The caller synchronises the
 * ranks (a barrier / 1-element all-reduce on the render streams) before the
 * owner reads the frame. */
typedef struct forma_ipc_handle { unsigned char bytes[64]; } forma_ipc_handle;
int forma_shared_frame_create(int device, uint64_t bytes, void** device_ptr, forma_ipc_handle* handle);
int forma_shared_frame_open(int device, const forma_ipc_handle* handle, void** device_ptr);
int forma_shared_frame_close(int device, void* mapped_ptr); /* a pointer from _open   */
int forma_shared_frame_free(int device, void* device_ptr);  /* a pointer from _create */

/* --- extensions (no reference counterpart) --------------------------------- */
/* Bulk form of move_to/line_to/quad_to/cubic_to: cmds[i] in {0 Move, 1 Line,
 * 2 Quad, 3 Cubic}, xy = the points they consume (1, 1, 2, 3 points each). */
void forma_path_builder_extend(forma_path_builder*, const uint8_t* cmds, uint64_t n_cmds, const float* xy);
/* Drops the composition's device residency: the next render re-uploads every
 * flatten program and table from pinned host memory (cold end-to-end path). */
void forma_composition_evict(forma_composition*);
uint64_t forma_composition_point_count(forma_composition*);
/* Device-timeline milliseconds of the last render: [0] uploads, [1] line-setup
 * count pass, [2] pixel-grid intersection, [3] sort, [4] painter tables,
 * [5] paint kernel (ID frames: the ID kernel, after the paint kernel in the combined call),
 * [6] device->host copy, [7] whole call. */
void forma_renderer_stage_times(const forma_renderer*, double out_ms[8]);
/* CUDA-event time of single kernels inside the last render, summed over their
 * launches: [0] radix downsweep (main sort, one launch per pass), [1] radix
 * upsweep + tile scan (one pair per pass), [2] paint kernel, [3] unused. */
void forma_renderer_kernel_times(const forma_renderer*, double out_ms[4], uint32_t out_launches[4]);
/* [0] kernel launches, [1] host->device bytes, [2] device->host bytes (all
 * since creation), [3] pixel segments, [4] cells, [5] entries of the last render,
 * [6] tiles the last layer-cache render copied back to a host buffer, [7] how the last
 * render built its painter tables: 0 = with the cell / entry counts read back on the way,
 * 1 = without a read-back (kernels sized by the previous frame's counts, option sync_free),
 * 2 = attempted without, counts exceeded the bounds, tables and paint repeated as 0. */
void forma_renderer_counters(const forma_renderer*, uint64_t out[8]);
/* How the last render's segment sort learnt the segment count: 0 = read back after the count
 * pass; 1 = not at all (option sync_free_sort: a single device frame launched over the previous
 * frame's count and sort plan, checked on the device); 2 = attempted as 1, the count or the tile
 * bounds did not fit, the frame repeated as 0 (the attempt wrote nothing to the caller's buffer). */
uint32_t forma_renderer_sort_mode(const forma_renderer*);
/* Host frames (forma_renderer_render without a layer cache) of compositions whose layers carry no
 * transform are rendered as a pipeline of tile-row slices on the renderer's device (option
 * host_slices): slice k + 1 uploads its band's geometry while slice k computes and slice k - 1
 * copies its rows back. Returns the number of slices of the last host frame (0 = one piece);
 * out_ms (may be null, room for 16) receives each slice's device-timeline ms (from the start of the
 * frame: a slice's upload waits for those of the slices before it), out_stage_ms (may be null,
 * room for 16 x 8) each slice's stage times as in forma_renderer_stage_times. After a sliced
 * frame the counters above are sums over the slices (pixel segments and entries: every slice
 * counts its own rows, so they are the frame's; cells: an upper bound, a slice also sees the
 * segments boundary-crossing lines leave in its neighbours' rows) and the stage times those of
 * the slowest slice. */
int forma_renderer_host_slices(const forma_renderer*, double* out_ms, double* out_stage_ms);

/* Cost of every tile row of the last render (32 x its (tile, layer) entries + its pixel
 * segments; rows outside the rendered crop cost 0): what a caller balances the tile-row
 * bands of the next multi-GPU frame on (SURVEY.md 8e). Returns the number of tile rows;
 * call with cap = 0 to size `out`. */
uint64_t forma_renderer_row_costs(forma_renderer*, uint64_t cap, uint64_t* out);

/* Schedule switches of the library (process-wide; none changes results): "speculate",
 * "band_copy", "copy_bands", "sort_full_key", "sort_big_log2", "sort_scan_log2", "sort_counts", "paint_lpt",
 * "paint_wide", "band_filter", "sync_free", "host_slices", "slice_bands", "slice_min_points", "slice_chain",
 * "pdl", "sync_free_sort", "test_gap_cap", "test_fast_shrink", "test_sort_bound".
 * Defaults come from the environment (FORMA_SPECULATE, ...); see DESIGN.md section 6. */
int forma_set_option(const char* name, int value);
int forma_get_option(const char* name, int* value);

/* Device self-test of the painter's pixel-pair fp32 arithmetic against the scalar IEEE
 * operations it stands for (2^20 operand triples incl. zeros, denormals, infinities, NaN);
 * *mismatches must come back 0. */
int forma_debug_selftest(int device, uint64_t* mismatches);

/* Number of CUDA kernels the renderer launched since it was created. */
uint64_t forma_renderer_launch_count(const forma_renderer*);

/* --- stage-level access (parity tests; the reference's own tests reach the
 *     same data through Rasterizer::segments(), cpu/rasterizer.rs:88) -------- */

/* The line records of the last render (SegmentBufferView of segment.rs:530-545: one
 * record per point pair, `lengths` as inclusive prefix sums) in host arrays of capacity
 * `cap`; returns the count (call with cap = 0 to size the arrays). render() never
 * materialises them; they are recomputed here from the last render's composition, which
 * must still be alive. */
uint64_t forma_renderer_lines(forma_renderer*, uint64_t cap, uint32_t* orders, float* x0, float* y0,
                              float* dx, float* dy, float* a, float* b, float* c, float* d,
                              uint32_t* lengths);
/* Copy the SORTED pixel segments of the last render; returns the count. */
uint64_t forma_renderer_segments(forma_renderer*, uint64_t cap, uint64_t* segments);
/* Line setup + pixel-grid intersection only; copies the UNSORTED segments (in
 * the reference's emission order) to `segments`; returns the count. */
uint64_t forma_renderer_rasterize_only(forma_renderer*, forma_composition*, uint64_t width,
                                       uint64_t height, uint64_t cap, uint64_t* segments);
/* Stage 3 alone: sort `n` host keys on bits [20, 64) on the device
 * (replaces crumsort at cpu/rasterizer.rs:162-164). */
int forma_renderer_sort_u64(forma_renderer*, uint64_t* keys, uint64_t n);
/* The sort plan for `bound` (the largest value of each key field, least significant field first)
 * under layout 0 (segments: layer | tile_x | tile_y) or 1 (the painter's carry keys: tile_x |
 * layer | tile_y): out[0] = n_passes, out[1] = total_bits, then 10 bytes per pass (shift[3],
 * width[3], lsh[3], bits); the bytes of unused passes are 0. Host only: no device. */
int forma_debug_sort_plan(int layout, const uint64_t bound[3], uint8_t out[2 + 10 * 6]);
/* Sorts (key, value) pairs with the single-sweep pair passes of the painter tables. layout: as
 * above; the plan's bounds are taken from the OR of the keys.
 * mode bit 0: the count is passed to the kernels in device memory and `cap` as its bound; keys /
 *             vals then hold min(count, cap) elements. Without it `count` elements are sorted and
 *             `cap` is ignored.
 * mode bit 1: the digit histogram is counted before the sort and passed in, as a kernel that
 *             writes the keys would.
 * With bit 0 and count > cap nothing is sorted and keys / vals come back unchanged. */
int forma_renderer_sort_pairs(forma_renderer*, int layout, int mode, uint64_t* keys, uint32_t* vals, uint64_t count,
                              uint64_t cap);
/* The bounds the last frame's segment sort was planned from: out[0..2] = layer, tile_x, tile_y
 * (the largest value each field was taken to have), out[3] = the key bits the plan sorts. */
void forma_renderer_sort_bounds(const forma_renderer*, uint64_t out[4]);
/* The per-tile digit counts of the last frame's segment sort (option "sort_counts"): the counts
 * its reduce-then-scan passes were given by the kernels that wrote their keys. keep: 1 = the
 * following frames of this renderer keep a copy of every pass's counts, 0 = they do not, -1 =
 * unchanged. info[0]: where pass 0's counts came from: 0 no tile counts (option off, or a sort
 * without reduce-then-scan passes), 1 the emit pass launched before the count read-back, with the
 * previous frame's pass-0 digit, 2 the emit pass launched after it (no speculation, or segments
 * beyond the speculative capacity), 3 an upsweep pass of the sort (first frame, the digit changed,
 * the previous frame had no tile counts); info[1] = passes and info[2] = 4096-key tiles of the
 * kept counts (0 when none were kept). `out` (may be null) gets min(cap, passes * tiles * 256) u32:
 * pass p's count of digit d in tile t at [(p * tiles + t) * 256 + d]. Returns passes * tiles * 256. */
uint64_t forma_renderer_sort_counts(forma_renderer*, int keep, uint32_t info[3], uint32_t* out, uint64_t cap);

#ifdef __cplusplus
}
#endif
#endif /* FORMA_B200_H */
