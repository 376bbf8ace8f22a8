// The body of paint_kernel, paint_views_kernel and their linear twins (kernels_painter.cu), included into each so that
// each kernel is compiled from the same text as a function of its own. Expects S, in and n_tiles,
// and FORMA_PAINT_FRAME_TY(ty): the tile row in frame coordinates at which gradients and textures
// are sampled (ty itself for a single frame, the row inside its view for a stack of views).
// A kernel that stores something other than sRGB8 defines both store hooks:
//   FORMA_PAINT_STORE_SOLID(dst): the tile folded to the one colour dst (Rgba, no layer cache);
//   FORMA_PAINT_STORE_PIXELS():   the lane's painted pixels, planes dr / dg / db / da at (x0, ty * 16 + row).
// A kernel for frames whose layers are all solid `Over` fills without clips (Composition::solid_over_only)
// defines FORMA_PAINT_SOLID_OVER: clip state, pass B, gradient prefetch and the blend paths of every
// other style fold away, and what remains is the same code as for such layers in the general build.
// A kernel that paints over the pixels already in the frame (forma_renderer_render_over_device)
// defines FORMA_PAINT_LOAD_PIXELS() as well as FORMA_PAINT_STORE_PIXELS():
//   FORMA_PAINT_LOAD_PIXELS(): the lane's eight pixels at (x0, ty * 16 + row), decoded into the
//   planes dr / dg / db / da, and bit j of bg_opaque set where pixel j's alpha is 1.
// The background is then each pixel's clear colour: a tile without entries is not written (its
// pixels are what the clear colour would give them back), the solid fold runs per pixel from the
// background unless an opaque layer is its bottom, and every tile is stored through
// FORMA_PAINT_STORE_PIXELS(), which applies the Alpha -> One upgrade per pixel (bg_opaque).
#ifdef FORMA_PAINT_SOLID_OVER
    constexpr bool kSolidOver = true;
#else
    constexpr bool kSolidOver = false;
#endif
    __shared__ __align__(16) WarpSmem s_warp[kPaintWarpsPerBlock];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    WarpSmem& W = s_warp[warp];
    const Rgba clear{S.clear[0], S.clear[1], S.clear[2], S.clear[3]};
    const bool rgba_order = S.channels[0] == 0u && S.channels[1] == 1u && S.channels[2] == 2u && S.channels[3] == 3u;
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(in.framebuffer) | (uintptr_t)S.stride) & 15u) == 0u;
    const uint32_t ntx = S.tx_hi - S.tx_lo;
    const uint32_t row = lane >> 1, hx = lane & 1u;
    // The cells of this warp start (and are kept) zeroed.
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        W.cells[0][k * 32 + lane] = 0u;
        W.cells[1][k * 32 + lane] = 0u;
    }
    __syncwarp();

    // Ticket -> tile. Tickets [0, H) walk the heavy-tile lists (largest class first), the
    // remaining n_tiles tickets the tile rectangle in row-major order; a tile that is on a
    // list is skipped there. Lists hold tiles of the whole frame: those outside this
    // launch's rows / columns are skipped here.
    uint32_t hcount[kHeavyClasses], H = 0;
#pragma unroll
    for (int c = 0; c < kHeavyClasses; ++c) {
        hcount[c] = in.heavy ? in.heavy_count[c] : 0u;
        H += hcount[c];
    }
    const uint32_t n_tickets = H + n_tiles;
    auto resolve = [&](uint32_t ticket, uint32_t& tid, uint32_t& b, uint32_t& e) -> bool {
        if (ticket >= n_tickets) return false;
        if (ticket < H) {
            uint32_t t = ticket;
            int c = kHeavyClasses - 1;
#pragma unroll
            for (int q = kHeavyClasses - 1; q > 0; --q)
                if (c == q && t >= hcount[q]) {
                    t -= hcount[q];
                    c = q - 1;
                }
            tid = in.heavy[(size_t)c * in.n_tiles_total + t];
            const uint32_t ty = tid / S.tiles_x, tx = tid - ty * S.tiles_x;
            if (ty < S.ty_lo || ty >= S.ty_hi || tx < S.tx_lo || tx >= S.tx_hi) {
                tid = 0xFFFFFFFFu;  // not this launch's tile
                return true;
            }
            const uint2 r = in.tile_range[tid];
            b = r.x;
            e = r.y;
            return true;
        }
        const uint32_t lin = ticket - H;
        tid = (S.ty_lo + lin / ntx) * S.tiles_x + S.tx_lo + lin % ntx;
        const uint2 r = in.tile_range[tid];
        b = r.x;
        e = r.y;
        if (in.heavy && e - b >= kHeavyMin) tid = 0xFFFFFFFFu;  // painted from its list
        return true;
    };

    // Tickets are drawn two tiles ahead and the entry range of the next tile is loaded while
    // the current one is painted.
    uint32_t next_ticket = 0, cur_tid = 0, cur_b = 0, cur_e = 0;
    bool have = false;
    {
        uint32_t t0 = 0;
        if (lane == 0) t0 = atomicAdd(in.tile_counter, 1u);
        t0 = __shfl_sync(kFullMask, t0, 0);
        if (lane == 0) next_ticket = atomicAdd(in.tile_counter, 1u);
        have = resolve(t0, cur_tid, cur_b, cur_e);
    }
    while (have) {
        const uint32_t tid = cur_tid, b = cur_b, e = cur_e;
        {
            const uint32_t nxt = __shfl_sync(kFullMask, next_ticket, 0);
            have = resolve(nxt, cur_tid, cur_b, cur_e);
            if (lane == 0) next_ticket = atomicAdd(in.tile_counter, 1u);
        }
        if (tid == 0xFFFFFFFFu) continue;
        const uint32_t ty = tid / S.tiles_x, tx = tid - ty * S.tiles_x;
#ifdef FORMA_PAINT_LOAD_PIXELS
        // No entries: the background stays. This also keeps the first attempt of a sync-free frame
        // whose tables are redone from writing: its tile ranges are all empty (build_tables).
        if (b == e) continue;
#endif

        // ---- optimizer passes (layer_workbench/passes/*.rs) ------------------
        // Pass A: per-entry facts, 32 entries at a time.
        // (has-segments / full / unchanged facts were computed when the entries were built.)
        bool any_clip = false, all_unchanged = true;
        for (uint32_t p0 = b; p0 < e; p0 += 32u) {
            uint32_t p = p0 + lane;
            uint32_t f = p < e ? (uint32_t)in.eflags[p] : kFlagUnchanged;
            if (!kSolidOver) any_clip |= __any_sync(kFullMask, (f & kFlagClipish) != 0u);
            all_unchanged = all_unchanged && !__any_sync(kFullMask, (f & kFlagUnchanged) == 0u);
        }

        // tile_unchanged pass (passes/tile_unchanged.rs:24-57) — only with a layer cache.
        const bool use_cache = S.cache_tiles != nullptr;
        uint32_t cache_x = 0, cache_solid = 0;
        bool layers_were_removed = true;  // PassesSharedState::reset
        if (use_cache) {
            uint2 c = S.cache_tiles[tid];
            const uint32_t layers = (e - b) & 0xFFFFFFu;
            const bool had = (c.x >> 31) != 0u;
            const uint32_t previous = c.x & 0xFFFFFFu;
            cache_solid = c.y;
            cache_x = (1u << 31) | (c.x & (1u << 30)) | layers;  // update_layer_count(Some(layers))
            bool is_unchanged = false;
            if (had) {
                layers_were_removed = layers < previous;
                is_unchanged = previous == layers && all_unchanged;
            }
            if (S.clear_unchanged && is_unchanged) {  // TileWriteOp::None
                if (lane == 0) S.cache_tiles[tid] = make_uint2(cache_x, cache_solid);
                continue;
            }
        }

        // Pass B: skip_trivial_clips (sequential; only tiles that contain clips).
        if (!kSolidOver && any_clip) {
            if (lane == 0) {
                bool has_clip = false, clip_full = false, clip_used = false;
                uint32_t clip_last = 0, clip_i = 0;
                for (uint32_t p = b; p < e; ++p) {
                    uint32_t f = in.eflags[p];
                    if (!(f & kFlagClipish)) {  // neither a clip nor a clipped layer
                        if (has_clip && in.recs[p].layer > clip_last) {
                            has_clip = false;
                            if (!clip_used) in.eflags[clip_i] |= (uint8_t)kFlagMaskedOut;
                        }
                        continue;
                    }
                    const uint32_t id = in.recs[p].layer;
                    if (!(f & kFlagClippedDraw)) {  // Func::Clip
                        clip_full = (f & kFlagFull) != 0;
                        clip_last = id + in.recs[p].clip_layers;
                        clip_i = p;
                        clip_used = false;
                        has_clip = true;
                        if (clip_full) f |= kFlagMaskedOut;
                    }
                    if (f & kFlagClippedDraw) {
                        if (has_clip && id <= clip_last) {
                            if (clip_full) f |= kFlagSkipClip;
                            else clip_used = true;
                        } else {
                            f |= kFlagMaskedOut;
                        }
                    }
                    in.eflags[p] = (uint8_t)f;
                    if (has_clip && id > clip_last) {
                        has_clip = false;
                        if (!clip_used) in.eflags[clip_i] |= (uint8_t)kFlagMaskedOut;
                    }
                }
                if (has_clip && !clip_used) in.eflags[clip_i] |= (uint8_t)kFlagMaskedOut;
            }
            __syncwarp();
        }

        // Pass C: skip_fully_covered_layers — the top-most full, unclipped, opaque
        // `Over` solid layer culls everything below it.
        uint32_t first_paint = b;  // MaskedVec::skip_until
        bool incomplete = false;   // an "interesting" incomplete cover at or above the opaque layer
        bool have_opaque = false;
        bool visible_unchanged = !layers_were_removed;  // skip_fully_covered_layers.rs:38-47
        for (uint32_t hi = e; hi > b && !have_opaque;) {
            uint32_t lo = hi - b >= 32u ? hi - 32u : b;
            uint32_t p = lo + lane;
            bool inc = false, cand = false, changed = false;
            if (p < hi) {
                uint32_t f = in.eflags[p];
                if (!(f & kFlagMaskedOut)) {
                    bool clipped = (f & kFlagClippedDraw) && !(f & kFlagSkipClip);
                    if (clipped || !(f & kFlagFull)) inc = true;
                    else if (f & kFlagOpaque) cand = true;
                    changed = !(f & kFlagUnchanged);
                }
            }
            uint32_t cand_mask = __ballot_sync(kFullMask, cand);
            uint32_t inc_mask = __ballot_sync(kFullMask, inc);
            uint32_t changed_mask = __ballot_sync(kFullMask, changed);
            if (cand_mask) {
                uint32_t top = 31u - (uint32_t)__clz((int)cand_mask);
                have_opaque = true;
                first_paint = lo + top;
                if (top < 31u && (inc_mask >> (top + 1u)) != 0u) incomplete = true;
                if ((changed_mask >> top) != 0u) visible_unchanged = false;  // layers visited before the break
            } else {
                if (inc_mask) incomplete = true;
                if (changed_mask) visible_unchanged = false;
            }
            hi = lo;
        }
        if (use_cache && have_opaque && !incomplete && visible_unchanged) {
            // Everything visible is unchanged: nothing to draw (skip_fully_covered_layers.rs:86-89).
            if (lane == 0) S.cache_tiles[tid] = make_uint2(cache_x, cache_solid);
            continue;
        }

#ifdef FORMA_PAINT_LOAD_PIXELS
        (void)clear;
        f2 dr[4], dg[4], db[4], da[4];
        uint32_t bg_opaque = 0;
        const uint32_t x0 = tx * 16u + hx * 8u;  // first pixel column of the lane
        FORMA_PAINT_LOAD_PIXELS();
        if (!incomplete) {
            // The fold of skip_fully_covered_layers (rs:81-118) with each pixel's background as its
            // clear colour: from an opaque bottom layer once, as the other kernels fold, or else per
            // pixel from the background. The planes then hold the solid tile's colour.
            const uint32_t p_first = first_paint + (have_opaque ? 1u : 0u);
            bool solid = true;
            for (uint32_t p = p_first; p < e; ++p) {
                if (in.eflags[p] & kFlagMaskedOut) continue;
                const uint32_t m = in.recs[p].meta;
                if (meta_func(m) != 0u || meta_fill_type(m) != 0u) {
                    solid = false;
                    break;
                }
            }
            if (solid) {
                if (have_opaque) {
                    const EntryRec& r0 = in.recs[first_paint];
                    Rgba dst{r0.color[0], r0.color[1], r0.color[2], r0.color[3]};
                    for (uint32_t p = p_first; p < e; ++p) {
                        if (in.eflags[p] & kFlagMaskedOut) continue;
                        const EntryRec& r = in.recs[p];
                        dst = blend_solid(meta_blend(r.meta), dst, Rgba{r.color[0], r.color[1], r.color[2], r.color[3]});
                    }
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        dr[q] = f2_splat(dst.r); dg[q] = f2_splat(dst.g); db[q] = f2_splat(dst.b); da[q] = f2_splat(dst.a);
                    }
                } else {
                    for (uint32_t p = p_first; p < e; ++p) {
                        if (in.eflags[p] & kFlagMaskedOut) continue;
                        const EntryRec& r = in.recs[p];
                        const Rgba src{r.color[0], r.color[1], r.color[2], r.color[3]};
                        const uint32_t mode = meta_blend(r.meta);
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            const Rgba d0 = blend_solid(mode, Rgba{dr[q].x, dg[q].x, db[q].x, da[q].x}, src);
                            const Rgba d1 = blend_solid(mode, Rgba{dr[q].y, dg[q].y, db[q].y, da[q].y}, src);
                            dr[q] = f2{d0.r, d1.r}; dg[q] = f2{d0.g, d1.g}; db[q] = f2{d0.b, d1.b}; da[q] = f2{d0.a, d1.a};
                        }
                    }
                }
                first_paint = e;  // nothing to paint: straight to the store
            }
        }
        bool clip_active = false;
        uint32_t clip_last = 0;
#else
        if (!incomplete) {
            // Every visible layer is full: fold with the scalar blend and emit a
            // solid tile (skip_fully_covered_layers.rs:81-118, mod.rs:686-704).
            Rgba dst = clear;
            uint32_t p = first_paint;
            if (have_opaque) {
                const EntryRec& r = in.recs[p];
                dst = Rgba{r.color[0], r.color[1], r.color[2], r.color[3]};
                ++p;
            }
            bool solid = true;
            for (; p < e; ++p) {
                if (in.eflags[p] & kFlagMaskedOut) continue;
                const EntryRec& r = in.recs[p];
                if (meta_func(r.meta) == 0u && meta_fill_type(r.meta) == 0u) {
                    dst = blend_solid(meta_blend(r.meta), dst, Rgba{r.color[0], r.color[1], r.color[2], r.color[3]});
                } else {
                    solid = false;
                    break;
                }
            }
            if (solid) {
#ifdef FORMA_PAINT_STORE_SOLID
                FORMA_PAINT_STORE_SOLID(dst);
                continue;
#else
                const uint32_t bytes = solid_to_srgb_bytes(dst, S.channels);
                // CachedTile::convert_optimizer_op (cpu/painter/mod.rs:686-704): the same
                // solid colour as last frame is not written again.
                const bool same = use_cache && ((cache_x >> 30) & 1u) && cache_solid == bytes;
                if (!same) store_tile_solid(S, in.framebuffer, tx, ty, lane, bytes, vec_ok);
                if (lane == 0) {
                    if (use_cache) S.cache_tiles[tid] = make_uint2(cache_x | (1u << 30), bytes);
                    if (!same && S.written_list) S.written_list[atomicAdd(S.written_count, 1u)] = tid;
                }
                continue;
#endif
            }
        }
        if (lane == 0) {
            // update_solid_color(None): the tile is painted
            if (use_cache) S.cache_tiles[tid] = make_uint2(cache_x & ~(1u << 30), cache_solid);
            if (S.written_list) S.written_list[atomicAdd(S.written_count, 1u)] = tid;
        }

        // ---- paint (layer_workbench/mod.rs:301-337, cpu/painter/mod.rs:290-347) ---
        // Pixel pair q = pixels 2 q, 2 q + 1 of the lane; (r, g, b, a) planes.
        f2 dr[4], dg[4], db[4], da[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            dr[q] = f2_splat(clear.r); dg[q] = f2_splat(clear.g); db[q] = f2_splat(clear.b); da[q] = f2_splat(clear.a);
        }
        bool clip_active = false;
        uint32_t clip_last = 0;
        const uint32_t x0 = tx * 16u + hx * 8u;            // first pixel column of the lane
#endif
        const float fy8 = (float)(FORMA_PAINT_FRAME_TY(ty) * 16u + (row & 8u));  // y of lane 0 of the reference's f32x8 holding this row
        const int ly8 = (int)(row & 7u);                   // the row inside it
        const uint32_t grp_shift = (lane & 16u) + hx;      // ballot bits of this lane's f32x8 group: grp_shift + 2 i
        const uint4* hdr4 = reinterpret_cast<const uint4*>(W.hdr);

        for (uint32_t p0 = first_paint; p0 < e; p0 += 32u) {
            const uint32_t cnt = min(32u, e - p0);
            __syncwarp();  // the previous group's records are no longer read
            if (lane < cnt) {
                // Stage the record; its spare word carries the (possibly updated) optimizer flags,
                // and a masked-out entry gets an empty segment range: nothing to accumulate.
                const uint4* src = reinterpret_cast<const uint4*>(in.recs + p0 + lane);
                uint4* dstp = reinterpret_cast<uint4*>(&W.hdr[lane]);
                uint4 q0 = src[0];
                const uint4 q1 = src[1], q2 = src[2];
                uint4 q3 = src[3];
                q3.w = in.eflags[p0 + lane];
                if (q3.w & kFlagMaskedOut) q0.z = q0.y;
                dstp[0] = q0; dstp[1] = q1; dstp[2] = q2; dstp[3] = q3;
            }
            __syncwarp();

            // Pipeline prologue: entry 0 is accumulated now, the segments of entry 1 are requested.
            uint64_t nx0 = 0, nx1 = 0;  // first two chunks of the entry after the one being accumulated
            uint32_t grad_word = 0, grad_next = 0;
            {
                const uint4 h = hdr4[0];
                if (!kSolidOver && (h.w & kMetaSmallGradient)) grad_next = reinterpret_cast<const uint32_t*>(&S.grads[hdr4[3].x])[lane];
                const uint32_t s0 = h.y, s1 = h.z;
                uint64_t a0 = 0, a1 = 0;
                if (s0 + lane < s1) a0 = in.segs[s0 + lane];
                if (s0 + 32u + lane < s1) a1 = in.segs[s0 + 32u + lane];
                if (cnt > 1u) {
                    const uint4 g = hdr4[4];
                    if (g.y + lane < g.z) nx0 = in.segs[g.y + lane];
                    if (g.y + 32u + lane < g.z) nx1 = in.segs[g.y + 32u + lane];
                }
                if (s1 > s0) scatter_entry(in.segs, s0, s1, a0, a1, W.cells[0], lane);
                __syncwarp();
            }

            for (uint32_t k = 0; k < cnt; ++k) {
                // Request the segments of entry k + 2, accumulate entry k + 1 into the other buffer.
                {
                    const uint64_t c0 = nx0, c1 = nx1;
                    nx0 = nx1 = 0;
                    if (k + 2u < cnt) {
                        const uint4 g = hdr4[(k + 2u) * 4u];
                        if (g.y + lane < g.z) nx0 = in.segs[g.y + lane];
                        if (g.y + 32u + lane < g.z) nx1 = in.segs[g.y + 32u + lane];
                    }
                    grad_word = grad_next;  // word `lane` of this entry's gradient record (if it has one)
                    if (k + 1u < cnt) {
                        const uint4 g = hdr4[(k + 1u) * 4u];
                        if (!kSolidOver && (g.w & kMetaSmallGradient))
                            grad_next = reinterpret_cast<const uint32_t*>(&S.grads[hdr4[(k + 1u) * 4u + 3u].x])[lane];
                        if (g.z > g.y) scatter_entry(in.segs, g.y, g.z, c0, c1, W.cells[(k + 1u) & 1u], lane);
                    }
                }
                const uint4 h0 = hdr4[k * 4u], h3 = hdr4[k * 4u + 3u];  // layer, seg0, seg1, meta | slot, clip_layers, flags0, flags
                const uint32_t flags = h3.w;
                if (flags & kFlagMaskedOut) {
                    __syncwarp();
                    continue;
                }
                const uint32_t meta = h0.w, layer = h0.x;
                const uint32_t fill_rule = meta_fill_rule(meta);

                // Running cover of this lane's row left of its first pixel (i8, wrapping like the
                // reference's lanes): the carry-in, plus the left half's covers for the right half.
                const uint32_t cw = reinterpret_cast<const uint32_t*>(&W.hdr[k].carry)[row >> 2];
                int32_t run = (int32_t)(int8_t)((cw >> (8u * (row & 3u))) & 0xFFu);
                f2 cov[4];  // coverage of the lane's pixel pairs
                if (h0.z > h0.y) {
                    // (the __syncwarp that ended the previous iteration made this buffer's atomics visible)
                    uint4* c4 = reinterpret_cast<uint4*>(W.cells[k & 1u]);
                    const uint4 w0 = c4[2u * lane], w1 = c4[2u * lane + 1u];
                    c4[2u * lane] = make_uint4(0u, 0u, 0u, 0u);
                    c4[2u * lane + 1u] = make_uint4(0u, 0u, 0u, 0u);
                    const uint32_t w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
                    int32_t area[8], cv[8], total = 0;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        cv[j] = (int32_t)(int16_t)(w[j] & 0xFFFFu);
                        area[j] = (int32_t)(w[j] + 0x8000u) >> 16;  // == (w - cover) >> 16: the high half as i16
                        total += cv[j];
                    }
                    const int32_t left = __shfl_xor_sync(kFullMask, total, 1);
                    if (hx) run += left;
                    // compute_doubled_areas, mod.rs:388-404: 32 * cover of the columns to the left + area
                    int32_t dbl[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        dbl[j] = 32 * (int32_t)(int8_t)run + area[j];
                        run += cv[j];
                    }
                    if (fill_rule == 0u) {
#pragma unroll
                        for (int q = 0; q < 4; ++q)
                            cov[q] = f2{coverage_non_zero(dbl[2 * q]), coverage_non_zero(dbl[2 * q + 1])};
                    } else {
#pragma unroll
                        for (int q = 0; q < 4; ++q)
                            cov[q] = f2{coverage_even_odd(dbl[2 * q]), coverage_even_odd(dbl[2 * q + 1])};
                    }
                } else {
                    const float c = fill_rule == 0u ? coverage_non_zero(32 * run) : coverage_even_odd(32 * run);
#pragma unroll
                    for (int q = 0; q < 4; ++q) cov[q] = f2_splat(c);
                }

                if (clip_active && clip_last < layer) clip_active = false;  // mod.rs:302-306

                if (!kSolidOver && meta_func(meta) == 1u) {  // clip_at, mod.rs:449-464
                    if (!clip_active) {
                        clip_active = true;
                        clip_last = layer + h3.y;
                    }
                    float4* m4 = reinterpret_cast<float4*>(W.clip);
                    m4[2u * lane] = make_float4(cov[0].x, cov[0].y, cov[1].x, cov[1].y);
                    m4[2u * lane + 1u] = make_float4(cov[2].x, cov[2].y, cov[3].x, cov[3].y);
                    __syncwarp();
                    continue;
                }
                const bool apply_clip = !kSolidOver && meta_is_clipped(meta) && !(flags & kFlagSkipClip);
                bool nonzero = false;
#pragma unroll
                for (int q = 0; q < 4; ++q) nonzero = nonzero || cov[q].x != 0.0f || cov[q].y != 0.0f;
                if (!__any_sync(kFullMask, nonzero) || (apply_clip && !clip_active)) {  // mod.rs:317-323
                    __syncwarp();
                    continue;
                }
                f2 clip2[4];  // clip mask of the pairs; only read when apply_clip
                if (apply_clip) {
                    const float4* m4 = reinterpret_cast<const float4*>(W.clip);
                    const float4 m0 = m4[2u * lane], m1 = m4[2u * lane + 1u];
                    clip2[0] = f2{m0.x, m0.y}; clip2[1] = f2{m0.z, m0.w}; clip2[2] = f2{m1.x, m1.y}; clip2[3] = f2{m1.z, m1.w};
                } else {
                    clip2[0] = clip2[1] = clip2[2] = clip2[3] = f2_splat(0.0f);
                }

                const uint32_t mode = meta_blend(meta);
                const uint32_t fill_type = meta_fill_type(meta);
                const uint4 h2 = hdr4[k * 4u + 2u];  // the solid colour
                if (fill_type == 0u && mode == 0u) {
                    // blend_at (mod.rs:406-447) for a solid `Over` layer: blended == src. Zero
                    // coverage is not the identity (a non-finite colour gives NaN, a -0 plane
                    // becomes +0), so the f32x8 rule holds here too: bit j of `act` is set iff
                    // pixel j of the lane's f32x8 group (the 8 lanes that differ in lane bits 1-3)
                    // has non-zero coverage somewhere.
                    uint32_t act = 0;
#pragma unroll
                    for (int q = 0; q < 4; ++q)
                        act |= (cov[q].x != 0.0f ? 1u : 0u) << (2 * q) | (cov[q].y != 0.0f ? 2u : 0u) << (2 * q);
                    act |= __shfl_xor_sync(kFullMask, act, 2);
                    act |= __shfl_xor_sync(kFullMask, act, 4);
                    act |= __shfl_xor_sync(kFullMask, act, 8);
                    const f2 cr = f2_splat(__uint_as_float(h2.x)), cg = f2_splat(__uint_as_float(h2.y));
                    const f2 cb = f2_splat(__uint_as_float(h2.z)), ca = f2_splat(__uint_as_float(h2.w));
                    if (apply_clip) {  // src_a = fill.a * coverage * mask (mod.rs:425-429)
#pragma unroll
                        for (int q = 0; q < 4; ++q) cov[q] = mul2(mul2(ca, cov[q]), clip2[q]);
                    } else {
#pragma unroll
                        for (int q = 0; q < 4; ++q) cov[q] = mul2(ca, cov[q]);
                    }
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const f2 sa = cov[q];
                        const f2 inv_dst_a = sub2(f2_splat(1.0f), da[q]);
                        const f2 inv_dst_a_src_a = mul2(inv_dst_a, sa);
                        const f2 inv_src_a = sub2(f2_splat(1.0f), sa);
                        const f2 dst_a_src_a = mul2(da[q], sa);
                        const uint32_t a2 = act >> (2 * q);
                        dr[q] = keep2(a2, compose2(dr[q], cr, cr, inv_dst_a_src_a, dst_a_src_a, inv_src_a), dr[q]);
                        dg[q] = keep2(a2, compose2(dg[q], cg, cg, inv_dst_a_src_a, dst_a_src_a, inv_src_a), dg[q]);
                        db[q] = keep2(a2, compose2(db[q], cb, cb, inv_dst_a_src_a, dst_a_src_a, inv_src_a), db[q]);
                        da[q] = keep2(a2, fma2(da[q], inv_src_a, sa), da[q]);
                    }
                    __syncwarp();
                    continue;
                }
                if (kSolidOver) {  // (no other layer in such a frame)
                    __syncwarp();
                    continue;
                }

                // Everything else follows the reference's f32x8 rule exactly: a pixel is blended iff
                // some pixel of its f32x8 (same column, same half of the tile) has non-zero coverage.
                uint32_t active = 0;
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const uint32_t b0 = __ballot_sync(kFullMask, cov[q].x != 0.0f), b1 = __ballot_sync(kFullMask, cov[q].y != 0.0f);
                    if ((b0 >> grp_shift) & 0x5555u) active |= 1u << (2 * q);
                    if ((b1 >> grp_shift) & 0x5555u) active |= 2u << (2 * q);
                }
                const int32_t slot = (int32_t)h3.x;
                const bool small_gradient = (meta & kMetaSmallGradient) != 0u;
                if (mode < 12u && (fill_type == 0u || small_gradient)) {
                    // Separable blend of a solid colour or a gradient of up to four stops: one
                    // out-of-line call per pixel pair that has a pixel to blend.
                    if (small_gradient) {
                        // The layer's gradient record (128 bytes, requested one entry ago) -> shared memory.
                        __syncwarp();
                        reinterpret_cast<uint32_t*>(&W.grad)[lane] = grad_word;
                        __syncwarp();
                    }
                    const float4 solid = make_float4(__uint_as_float(h2.x), __uint_as_float(h2.y), __uint_as_float(h2.z), __uint_as_float(h2.w));
                    const uint32_t ctl = mode | (apply_clip ? 0x100u : 0u) | (small_gradient ? 0x200u : 0u);
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const uint32_t act = (active >> (2 * q)) & 3u;
                        if (act) {
                            const PairPlanes d = blend_pair_separable(PairPlanes{dr[q], dg[q], db[q], da[q]}, cov[q], clip2[q], ctl | (act << 16),
                                                                      (float)(x0 + 2u * (uint32_t)q), fy8, ly8, &W.grad, solid);
                            dr[q] = d.r; dg[q] = d.g; db[q] = d.b; da[q] = d.a;
                        }
                    }
                } else {
                    // Textures, gradients with more than four stops, non-separable modes: one
                    // out-of-line call per blended pixel.
                    const StyleRec* st = &S.styles[slot];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const float fx = (float)(x0 + 2u * (uint32_t)q);
                        if ((active >> (2 * q)) & 1u) {
                            const float4 d = blend_pixel_generic(st, S.stops, S.texels, fx, fy8, ly8, cov[q].x, apply_clip ? clip2[q].x : -1.0f,
                                                                 make_float4(dr[q].x, dg[q].x, db[q].x, da[q].x));
                            dr[q].x = d.x; dg[q].x = d.y; db[q].x = d.z; da[q].x = d.w;
                        }
                        if ((active >> (2 * q + 1)) & 1u) {
                            const float4 d = blend_pixel_generic(st, S.stops, S.texels, fx + 1.0f, fy8, ly8, cov[q].y,
                                                                 apply_clip ? clip2[q].y : -1.0f, make_float4(dr[q].y, dg[q].y, db[q].y, da[q].y));
                            dr[q].y = d.x; dg[q].y = d.y; db[q].y = d.z; da[q].y = d.w;
                        }
                    }
                }
                __syncwarp();
            }
        }

#ifdef FORMA_PAINT_STORE_PIXELS
        FORMA_PAINT_STORE_PIXELS();
#else
        // compute_srgb + LinearLayout::write (mod.rs:466-483, layout/mod.rs:265-282).
        const uint32_t py = ty * 16u + row;
        if (py < S.height && x0 < S.width) {
            uint32_t out[8];
            if (rgba_order) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    uint32_t r0, r1, g0, g1, b0, b1, a0, a1;
                    to_byte2(srgb2(dr[q]), r0, r1);
                    to_byte2(srgb2(dg[q]), g0, g1);
                    to_byte2(srgb2(db[q]), b0, b1);
                    to_byte2(da[q], a0, a1);
                    out[2 * q] = r0 | (g0 << 8) | (b0 << 16) | (a0 << 24);
                    out[2 * q + 1] = r1 | (g1 << 8) | (b1 << 16) | (a1 << 24);
                }
            } else {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    out[2 * q] = srgb_bytes_any_order(dr[q].x, dg[q].x, db[q].x, da[q].x, S.channels);
                    out[2 * q + 1] = srgb_bytes_any_order(dr[q].y, dg[q].y, db[q].y, da[q].y, S.channels);
                }
            }
            uint8_t* rowp = in.framebuffer + (size_t)py * S.stride + (size_t)x0 * 4u;
            if (vec_ok && x0 + 8u <= S.width) {
                reinterpret_cast<uint4*>(rowp)[0] = make_uint4(out[0], out[1], out[2], out[3]);
                reinterpret_cast<uint4*>(rowp)[1] = make_uint4(out[4], out[5], out[6], out[7]);
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    if (x0 + (uint32_t)j < S.width) reinterpret_cast<uint32_t*>(rowp)[j] = out[j];
            }
        }
#endif
    }
