// The body of paint_ids_kernel and paint_ids_stacked_kernel (kernels_ids.cu), included into both so
// that each kernel is compiled from the same text as a function of its own. Expects S, in and
// n_tiles, and FORMA_IDS_REBASE(out, ty): what happens to the lane's eight IDs of a tile of row ty
// before they are stored (nothing for a single frame or views; a batch takes the frame's order
// base off them). A kernel that defines FORMA_IDS_SINK(out, ty, tx, row, hx) hands the lane's eight
// IDs of every tile to it instead of storing them (FORMA_IDS_REBASE is then not used).
    __shared__ __align__(16) IdWarpSmem s_warp[kIdWarpsPerBlock];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    IdWarpSmem& W = s_warp[warp];
    const uint32_t ntx = S.tx_hi - S.tx_lo;
    const uint32_t row = lane >> 1, hx = lane & 1u;
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(in.ids) | (uintptr_t)in.ids_stride) & 15u) == 0u;
    const float min_cov = in.min_coverage;
#pragma unroll
    for (int k = 0; k < 8; ++k) W.cells[k * 32 + lane] = 0u;
    __syncwarp();

    uint32_t hcount[kHeavyClasses], H = 0;
#pragma unroll
    for (int c = 0; c < kHeavyClasses; ++c) {
        hcount[c] = in.heavy ? in.heavy_count[c] : 0u;
        H += hcount[c];
    }
    const uint32_t n_tickets = H + n_tiles;
    for (;;) {
        // Ticket -> tile, as in paint_kernel: tickets [0, H) walk the heavy lists (largest class
        // first), the rest the tile rectangle row-major, skipping the listed tiles.
        uint32_t ticket = 0;
        if (lane == 0) ticket = atomicAdd(in.tile_counter, 1u);
        ticket = __shfl_sync(kFullMask, ticket, 0);
        if (ticket >= n_tickets) break;
        uint32_t tid;
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
            if (ty < S.ty_lo || ty >= S.ty_hi || tx < S.tx_lo || tx >= S.tx_hi) continue;
        } else {
            const uint32_t lin = ticket - H;
            tid = (S.ty_lo + lin / ntx) * S.tiles_x + S.tx_lo + lin % ntx;
        }
        const uint2 range = in.tile_range[tid];
        const uint32_t b = range.x, e = range.y;
        if (ticket >= H && in.heavy && e - b >= kHeavyMin) continue;  // done from its list
        const uint32_t ty = tid / S.tiles_x, tx = tid - ty * S.tiles_x;

        bool clip_tile = false;
        for (uint32_t p0 = b; p0 < e && !clip_tile; p0 += 32u) {
            const uint32_t p = p0 + lane;
            clip_tile = __any_sync(kFullMask, p < e && (in.recs[p].flags0 & kFlagClipish) != 0u);
        }

        uint32_t* out = W.ids + 8u * lane;  // this lane's eight pixels
#pragma unroll
        for (int j = 0; j < 8; ++j) out[j] = FORMA_ID_NONE;
        float cov[8];
        if (!clip_tile) {
            uint32_t open = 0xFFu;  // this lane's pixels without a hit yet
            bool done = e == b;
            for (uint32_t hi = e; hi > b && !done;) {
                const uint32_t lo = hi - b >= 32u ? hi - 32u : b;
                stage_group(W, in, lo, hi - lo, false, lane);
                for (uint32_t k = hi - lo; k-- > 0u;) {
                    const EntryRec& h = W.hdr[k];
                    const uint32_t flags = h.pad;
                    if (flags & kFlagMaskedOut) continue;
                    if (flags & kFlagFull) {  // an unclipped Draw entry of coverage 1 everywhere
#pragma unroll
                        for (int j = 0; j < 8; ++j)
                            if ((open >> j) & 1u) out[j] = h.layer;
                        done = true;
                        break;
                    }
                    entry_coverage(W, h, in.segs, lane, cov);
#pragma unroll
                    for (int j = 0; j < 8; ++j)
                        if (((open >> j) & 1u) && cov[j] > min_cov) {
                            out[j] = h.layer;
                            open &= ~(1u << j);
                        }
                    if (__all_sync(kFullMask, open == 0u)) {
                        done = true;
                        break;
                    }
                }
                hi = lo;
            }
        } else {
            if (lane == 0) skip_trivial_clips_ids(in.recs, in.id_flags, b, e);
            __syncwarp();
            // The painter's first layer (skip_fully_covered_layers): the top-most visible full,
            // unclipped, opaque entry.
            uint32_t first = b;
            for (uint32_t hi = e; hi > b;) {
                const uint32_t lo = hi - b >= 32u ? hi - 32u : b;
                bool cand = false;
                if (lo + lane < hi) {
                    const uint32_t f = in.id_flags[lo + lane];
                    const bool clipped = (f & kFlagClippedDraw) && !(f & kFlagSkipClip);
                    cand = !(f & kFlagMaskedOut) && !clipped && (f & kFlagFull) && (f & kFlagOpaque);
                }
                const uint32_t m = __ballot_sync(kFullMask, cand);
                if (m) {
                    first = lo + 31u - (uint32_t)__clz((int)m);
                    break;
                }
                hi = lo;
            }
            bool clip_active = false;
            uint32_t clip_last = 0;
            for (uint32_t p0 = first; p0 < e; p0 += 32u) {
                const uint32_t cnt = min(32u, e - p0);
                stage_group(W, in, p0, cnt, true, lane);
                for (uint32_t k = 0; k < cnt; ++k) {
                    const EntryRec& h = W.hdr[k];
                    const uint32_t flags = h.pad;
                    if (flags & kFlagMaskedOut) continue;
                    const uint32_t layer = h.layer, meta = h.meta;
                    if (clip_active && clip_last < layer) clip_active = false;  // mod.rs:302-306
                    const bool is_clip = ((meta >> 1) & 1u) != 0u;
                    const bool apply_clip = !is_clip && ((meta >> 2) & 1u) && !(flags & kFlagSkipClip);
                    if (!is_clip && !apply_clip && (flags & kFlagFull)) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) out[j] = layer;
                        continue;
                    }
                    if (apply_clip && !clip_active) continue;  // mod.rs:317-323
                    entry_coverage(W, h, in.segs, lane, cov);
                    if (is_clip) {  // clip_at, mod.rs:449-464
                        if (!clip_active) {
                            clip_active = true;
                            clip_last = layer + h.clip_layers;
                        }
                        float4* m4 = reinterpret_cast<float4*>(W.clip);
                        m4[2u * lane] = make_float4(cov[0], cov[1], cov[2], cov[3]);
                        m4[2u * lane + 1u] = make_float4(cov[4], cov[5], cov[6], cov[7]);
                        __syncwarp();
                        continue;
                    }
                    if (apply_clip) {
                        const float4* m4 = reinterpret_cast<const float4*>(W.clip);
                        const float4 m0 = m4[2u * lane], m1 = m4[2u * lane + 1u];
                        const float m[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
#pragma unroll
                        for (int j = 0; j < 8; ++j) cov[j] = __fmul_rn(cov[j], m[j]);
                    }
#pragma unroll
                    for (int j = 0; j < 8; ++j)
                        if (cov[j] > min_cov) out[j] = layer;
                }
            }
        }

#ifdef FORMA_IDS_SINK
        (void)vec_ok;
        FORMA_IDS_SINK(out, ty, tx, row, hx);
#else
        FORMA_IDS_REBASE(out, ty);
        const uint32_t py = ty * 16u + row, x0 = tx * 16u + hx * 8u;
        if (py < S.height && x0 < S.width) {
            uint32_t* rowp = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(in.ids) + (size_t)py * in.ids_stride) + x0;
            if (vec_ok && x0 + 8u <= S.width) {
                reinterpret_cast<uint4*>(rowp)[0] = reinterpret_cast<const uint4*>(out)[0];
                reinterpret_cast<uint4*>(rowp)[1] = reinterpret_cast<const uint4*>(out)[1];
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    if (x0 + (uint32_t)j < S.width) rowp[j] = out[j];
            }
        }
#endif
    }
