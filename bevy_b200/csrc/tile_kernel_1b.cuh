// tile_kernel_1b.cuh -- kernel 1b (k_propagate_cull_tma), included by kernels.cu once per variant:
//   B200VIS_TILE_1B      the kernel's name
//   B200VIS_TILE_1B_EXT  false: the kernel every frame runs;
//                        true: the kernel of frames with pending GlobalTransforms written by other systems
//                        (b200vis_write_global_transforms_scattered).  A row then hands its children
//                        changed || (visited && S_GT_EXT) instead of changed -- p_global_transform.is_changed() of
//                        propagate_descendants_unchecked (systems.rs:706-724) -- in shared memory to children in its tile and as
//                        S_GT_HANDED to children in later passes; the row's own Changed<GlobalTransform> stays `changed`.  The pass
//                        consumes the marks.
// One source for both keeps the unmarked kernel's code exactly what it is without the feature.
//
// Row-0 staging (the unmarked PROP instantiations, gt_hint != nullptr).  set_if_neq reads the old GlobalTransform only to
// decide `changed` and to keep the old bits when nothing changed.  A differing row 0 (X.x, Y.x, Z.x, T.x) proves a change by
// IEEE != on its own (NaN compares unequal, so it lands there too); only when row 0 is equal (including a +0 / -0
// difference) do rows 1-2 decide.  So a tile can be staged with old row 0 alone: 32 B/row less TMA traffic, 136 instead of
// 168 B/row in all.  In such a tile every row that row 0 does not prove changed -- a row no level visited, an unwritten root,
// a row whose new row 0 equals the old one -- reads its old rows 1-2 from HBM into its own slots, before its level hand-over
// (its children read them), the cull and the bulk store (which read all three rows).  Thread 0 picks the staging per tile
// from gt_hint[tile]: non-zero when the tile's last run had such a row (static tiles then cost what full staging costs), and
// every run writes it back.  It is only a hint: either staging gives the same bits.
template <bool PROP, bool CULL, bool SIMPLE>
__global__ void __launch_bounds__(kTileRows, 4)
B200VIS_TILE_1B(Rows R, const Tile *__restrict__ tiles, uint32_t n_tiles, const __grid_constant__ CullViews cvw,
                VisibleBufs vb, DevStats *__restrict__ stats, uint32_t static_opt, uint32_t parity,
                uint32_t *__restrict__ ticket, uint32_t ticket_base, uint32_t rev, uint8_t *__restrict__ gt_hint) {
    constexpr bool EXT = B200VIS_TILE_1B_EXT;
    constexpr bool ROW0 = PROP && !EXT;      // instantiations that may stage old GlobalTransform row 0 alone
    extern __shared__ __align__(128) uint8_t smem_raw[];
    TmaSmem &s = *reinterpret_cast<TmaSmem *>(smem_raw);
    const uint32_t lr = threadIdx.x;
    if (lr == 0) {
        mbar_init(&s.bar[0], 1); mbar_init(&s.bar[1], 1);
        s.gt_fb[0] = 0u; s.gt_fb[1] = 0u;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    TP_BEGIN();
    // launched with programmatic stream serialization: everything above overlapped the previous kernel's tail
    asm volatile("griddepcontrol.wait;" ::: "memory");
    PROBE_SCOPE(0u, ticket_base);
    // rev: the pass walks its tiles from the last one (t below is the position in the walk, tile_at() the descriptor it takes).
    // The tiles of one pass are independent of each other (out-of-tile parents sit in earlier passes), so the order changes
    // no result.
    auto tile_idx = [&](uint32_t i) { return rev ? n_tiles - 1u - i : i; };
    auto tile_at = [&](uint32_t i) -> const Tile & { return tiles[tile_idx(i)]; };
    // thread 0 picks the staging of a tile when it issues its loads, and publishes it in s.gt_full before the mbarrier arrive
    auto stage_full = [&](uint32_t i) -> bool { return !ROW0 || gt_hint == nullptr || gt_hint[tile_idx(i)] != 0; };
    uint32_t t = blockIdx.x;
    if (lr == 0 && t < n_tiles) {
        const bool full = stage_full(t);
        if (ROW0) s.gt_full[0] = full;
        issue_tile_loads<PROP, CULL>(R, tile_at(t), s.st[0], &s.bar[0], full);
    }
    uint32_t n_gt_total = 0, n_vv_total = 0;
    // Tile hand-out: a CTA starts on tile blockIdx.x and then takes the tiles the grid has not started yet in ticket order
    // (one atomic per tile, drawn by thread 0 when it prefetches, i.e. one tile ahead).  A fixed stride would leave a CTA with
    // ceil(n/g) tiles running next to finished neighbours with floor(n/g) -- a fifth of the pass at 3.3 tiles per CTA.  The
    // ticket counter is never reset: every launch draws exactly n_tiles tickets, and the host passes the running base.
    for (uint32_t it = 0; t < n_tiles; ++it) {
        TP(0);
        const uint32_t sidx = it & 1u;
        const Tile tile = tile_at(t);
        TP(1);
        mbar_wait(&s.bar[sidx], (it >> 1) & 1u);
        TP(2);
        TileStage &S = s.st[sidx];
        const bool row0 = ROW0 && !s.gt_full[sidx];      // this tile's old rows 1-2 are not staged
        const uint32_t off = tile.base & 15u;
        const uint32_t li = off + lr;                 // index into the staged window
        const bool active = lr < tile.n_rows;
        const uint32_t row = tile.base + lr;
        const uint32_t f = active ? S.flags[li] : 0u;
        const uint32_t st8 = active ? S.state[li] : 0u;
        // bounds are only needed after the hierarchy walk (keeping them out of the staged window lets a fourth CTA fit in shared
        // memory).  Without a walk: plain coalesced loads issued now, consumed in phase 3.
        float4 bA = make_float4(0, 0, 0, 0); float2 bB = make_float2(0, 0);
        if (!PROP && CULL && active) { bA = R.bndA[row]; bB = R.bndB[row]; }

        bool visited = false, changed = false;
        const bool ext_mark = EXT && (st8 & S_GT_EXT);
        if (PROP) {
            const uint32_t topo = active ? S.topo[li] : T_DETACHED;
            const uint32_t depth = (topo >> 9) & 0x1FFu, plocal = topo & 0x1FFu;
            const bool tchanged = f & F_TCHANGED;
            const bool has_children = topo & T_HAS_CHILDREN;
            bool dirty = tchanged;
            if (static_opt && R.dirty != nullptr) {
                dirty = active && R.dirty[row];
            } else if (static_opt && tile.n_levels > 1 && __syncthreads_or(tchanged && depth > 0)) {
                // only when a non-root row of the tile changed does anything have to climb: otherwise every row's
                // TransformTreeChanged bit equals its own Changed<Transform> bit (one barrier instead of two + a climb)
                s.parent[lr] = (uint16_t)((depth > 0) ? plocal : 0xFFFFu);
                s.dirty[lr] = 0;
                __syncthreads();
                if (active && tchanged) {
                    uint32_t c = lr;
                    while (!s.dirty[c]) {
                        s.dirty[c] = 1;
                        const uint32_t p = s.parent[c];
                        if (p == 0xFFFFu) break;
                        c = p;
                    }
                }
                __syncthreads();
                dirty = s.dirty[lr];
            }
            TP(3);
            const Aff l = affine_from_trs(S.trsA[li], S.trsB[li], S.trsC[li]);
            // With a walk, the row's bounds come in by cp.async into its own Transform slots, which nothing reads again in this
            // tile: the loads run under the walk without holding six registers through it (at the 64-register budget those
            // registers were spilled in the hot loop), and the cull reads them back from shared memory
            if (CULL && active) { cp_async_16(&S.trsA[li], R.bndA + row); cp_async_8(&S.trsC[li], R.bndB + row); }
            const uint32_t my_level = (active && !(topo & T_DETACHED)) ? depth : 0xFFFFFFFFu;
            if (active && (topo & T_DETACHED) && has_children) s.pst[lr] = 0;
            // set_if_neq of a visited row: row 0 first (see the top of this file); when it is equal, rows 1-2 decide, read
            // from HBM into the row's own slots in a row-0 tile, where they stay as the kept bits if nothing changed
            auto set_if_neq = [&](const Aff &n) -> bool {
                bool c = row_neq(n.r0, S.gt0[li]);
                if (!c) {
                    s.gt_fb[sidx] = 1u;
                    if (row0) { S.gt1[li] = R.gt1[row]; S.gt2[li] = R.gt2[row]; }
                    c = row_neq(n.r1, S.gt1[li]) | row_neq(n.r2, S.gt2[li]);
                }
                if (c) { S.gt0[li] = n.r0; S.gt1[li] = n.r1; S.gt2[li] = n.r2; }
                return c;
            };
            if (my_level == 0) {
                if (topo & T_ROOT) {
                    visited = has_children ? (!static_opt || dirty) : tchanged;
                    changed = visited;
                    if (changed) { S.gt0[li] = l.r0; S.gt1[li] = l.r1; S.gt2[li] = l.r2; }
                } else {
                    const uint32_t pr = R.parent[row];
                    const uint32_t ps = R.state[pr];
                    visited = (ps & S_VISITED) && !(static_opt && !dirty && !(ps & (EXT ? S_GT_HANDED : S_GT_CHANGED)));
                    if (visited) {
                        Aff n;
                        n.r0 = affine_mul_row(R.gt0[pr], l); n.r1 = affine_mul_row(R.gt1[pr], l); n.r2 = affine_mul_row(R.gt2[pr], l);
                        changed = set_if_neq(n);
                    }
                }
                if (has_children) s.pst[lr] = (uint8_t)((visited ? 1u : 0u) | ((changed || (visited && ext_mark)) ? 2u : 0u));
            }
            TP(4);
            // one level of the walk for this thread's row: the parent's rows are the tile's own (in-place) GlobalTransform entries
            auto walk_row = [&]() {
                const uint32_t pst = s.pst[plocal];
                const uint32_t pi = off + plocal;
                visited = (pst & 1u) && !(static_opt && !dirty && !(pst & 2u));
                if (visited) {
                    Aff n;
                    n.r0 = affine_mul_row(S.gt0[pi], l); n.r1 = affine_mul_row(S.gt1[pi], l); n.r2 = affine_mul_row(S.gt2[pi], l);
                    changed = set_if_neq(n);
                }
                if (has_children) s.pst[lr] = (uint8_t)((visited ? 1u : 0u) | ((changed || (visited && ext_mark)) ? 2u : 0u));
            };
            if (tile.lvl_warps != 0ull) {
                // Per-warp level schedule (2..8 levels).  A warp only takes part in the hand-over of the levels its own rows
                // produce (level l-1) or consume (level l), through hardware named barrier l with exactly the warps the planner
                // counted (Tile::lvl_warps): consumers bar.sync, pure producers bar.arrive and go on; a leaf warp waits once
                // instead of once per level, and nobody pays the loop for levels that are not theirs.  (The tile still ends in a
                // CTA-wide barrier, so one set of barrier ids is enough here.)
                // (a detached row takes no part in the walk but publishes pst = 0 for its children: it counts as a level-0 row)
                const uint32_t lmask = __reduce_or_sync(0xFFFFFFFFu, active ? (1u << (depth & 15u)) : 0u);
                uint32_t need = (lmask | (lmask << 1)) & ((1u << tile.n_levels) - 2u);
                while (need) {
                    const uint32_t lvl = (uint32_t)__ffs((int)need) - 1u;
                    need &= need - 1u;
                    const bool consumer = (lmask >> lvl) & 1u;
                    if ((tile.warp_sync_mask >> lvl) & 1u) {       // every edge into this level stays inside a warp
                        if (!consumer) continue;
                        __syncwarp();
                    } else {
                        const uint32_t cnt = ((uint32_t)(tile.lvl_warps >> (4u * lvl)) & 15u) * 32u;
                        if (!consumer) {
                            __threadfence_block();
                            asm volatile("bar.arrive %0, %1;" ::"r"(lvl), "r"(cnt) : "memory");
                            continue;
                        }
                        asm volatile("bar.sync %0, %1;" ::"r"(lvl), "r"(cnt) : "memory");
                    }
                    if (my_level == lvl) walk_row();
                }
            } else {
                for (uint32_t lvl = 1; lvl < tile.n_levels; ++lvl) {
                    if (lvl < 32u && ((tile.warp_sync_mask >> lvl) & 1u)) __syncwarp(); else __syncthreads();
                    if (my_level == lvl) walk_row();
                }
            }
            // a row no level visited keeps its old matrix, which the cull and the bulk store read (children of an unvisited
            // row are not visited, so nothing reads it earlier); the cp.async lands behind the cp.async.wait_all below
            if (active && !visited) {
                s.gt_fb[sidx] = 1u;
                if (row0) { cp_async_16(&S.gt1[li], R.gt1 + row); cp_async_16(&S.gt2[li], R.gt2 + row); }
            }
            if (active && tchanged) R.flags[row] = (uint8_t)(f & ~F_TCHANGED);
        }
        TP(5);
        // Prefetch the NEXT tile into the other stage.  That stage was last read by the previous tile's bulk store,
        // issued most of an iteration ago, so the wait below is (almost always) already satisfied: putting the
        // prefetch here instead of at the top of the loop keeps the store drain off every warp's critical path.
        if (lr == 0) {
            const uint32_t tn = ticket ? gridDim.x + (atomicAdd(ticket, 1u) - ticket_base) : t + gridDim.x;
            if (tn < n_tiles) {
                const bool full = stage_full(tn);
                asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the stage's generic writes (bounds) -> TMA loads
                if (ROW0) s.gt_full[sidx ^ 1u] = full;
                issue_tile_loads<PROP, CULL>(R, tile_at(tn), s.st[sidx ^ 1u], &s.bar[sidx ^ 1u], full);
            }
            s.next_tile[sidx] = tn;      // read by everybody behind the tile's closing barrier
        }
        TP(6);
        uint32_t out = st8 & (S_VV | S_HAS_CLASS);     // (drops S_GT_EXT: the pass consumes the marks)
        if (PROP) out |= (changed ? S_GT_CHANGED : 0u) | (visited ? S_VISITED : 0u);
        else out |= st8 & (S_GT_CHANGED | S_VISITED);
        if (EXT && PROP && (changed || (visited && ext_mark))) out |= S_GT_HANDED;

        bool vv_changed = false;
        if (CULL) {
            if (PROP) {      // this thread's bounds copies (above) have landed
                asm volatile("cp.async.wait_all;" ::: "memory");
                if (active) { bA = S.trsA[li]; bB = S.trsC[li]; }
            }
            Aff g; g.r0 = S.gt0[li]; g.r1 = S.gt1[li]; g.r2 = S.gt2[li];   // own row: written by this thread or untouched
            const bool in_query = active && !(f & F_NO_CPU_CULL);
            const bool base = in_query && (f & F_INHERITED);
        const bool rej_base = base;
            const uint32_t prev = st8 & 1u;
            const uint32_t lane = lr & 31u;
            const bool has_aabb = f & F_AABB;
            const bool do_test = (f & (F_AABB | F_SPHERE)) && !(f & F_NO_FRUSTUM);
            float cx, cy, cz, radius;
            const float hx = bA.w, hy = bB.x, hz = bB.y;
            if (has_aabb) {
                cx = ((g.r0.x * bA.x + g.r0.y * bA.y) + g.r0.z * bA.z) + g.r0.w;
                cy = ((g.r1.x * bA.x + g.r1.y * bA.y) + g.r1.z * bA.z) + g.r1.w;
                cz = ((g.r2.x * bA.x + g.r2.y * bA.y) + g.r2.z * bA.z) + g.r2.w;
                const float vx = (g.r0.x * hx + g.r0.y * hy) + g.r0.z * hz;
                const float vy = (g.r1.x * hx + g.r1.y * hy) + g.r1.z * hz;
                const float vz = (g.r2.x * hx + g.r2.y * hy) + g.r2.z * hz;
                radius = sqrtf((vx * vx + vy * vy) + vz * vz);
            } else {
                const bool from_gt = f & F_SPHERE_GT;
                cx = from_gt ? g.r0.w : bA.x; cy = from_gt ? g.r1.w : bA.y; cz = from_gt ? g.r2.w : bA.z;
                radius = bA.w;
            }
            unsigned long long elayers = 1ull; uint32_t erange = 0xFFFFFFFFu, rnk = row;
            if (!SIMPLE && active) {
                if (R.layers != nullptr) elayers = R.layers[row];
                if ((f & F_RANGE) && R.range != nullptr) erange = range_mask_of(R, row, has_aabb, cx, cy, cz, g);
                if (R.rank != nullptr) rnk = R.rank[row];
            }
            // warp-level shortcut: views whose frustum the whole warp's rows are outside of (see warp_view_reject)
            const uint32_t rejmask = warp_view_reject(cvw, rej_base && do_test, rej_base && !do_test, cx, cy, cz, radius);
            bool any = false;
            uint32_t my_ballot = 0;
#pragma unroll
            for (uint32_t v = 0; v < kMaxViews; ++v) {
                if (v >= cvw.n_views) break;
                const uint32_t von = cvw.on[v];
                if (!(von & 1u)) continue;
                if (SIMPLE && !(von & 4u)) continue;   // bit2: the view includes the default layer
                if (((rejmask >> v) & 1u) && !(von & 2u)) continue;         // every row of this warp is outside this view's frustum
                bool vis = base;
                if (!SIMPLE) {
                    vis = vis && layers_intersect(R, cvw, row, v, elayers);
                    if ((f & F_RANGE) && R.range != nullptr) {
                        const int32_t ri = cvw.range_index[v];
                        vis = vis && ri >= 0 && ((erange >> ri) & 1u);
                    }
                }
                if (do_test && !(von & 2u)) {
                    const float d0 = plane_dot_point(cvw.planes[v][0], cx, cy, cz), d1 = plane_dot_point(cvw.planes[v][1], cx, cy, cz);
                    const float d2 = plane_dot_point(cvw.planes[v][2], cx, cy, cz), d3 = plane_dot_point(cvw.planes[v][3], cx, cy, cz);
                    const float d4 = plane_dot_point(cvw.planes[v][4], cx, cy, cz);
                    const bool out_s = (d0 + radius <= 0.0f) | (d1 + radius <= 0.0f) | (d2 + radius <= 0.0f) |
                                       (d3 + radius <= 0.0f) | (d4 + radius <= 0.0f);
                    vis = vis && !out_s;
                    if (vis && has_aabb) {
                        const float d[5] = {d0, d1, d2, d3, d4};
                        bool out_o = false;
#pragma unroll
                        for (int k = 0; k < 5; ++k) {
                            const float4 n = cvw.planes[v][k];
                            const float dx = fabsf(dot3(n.x, n.y, n.z, g.r0.x, g.r1.x, g.r2.x));
                            const float dy = fabsf(dot3(n.x, n.y, n.z, g.r0.y, g.r1.y, g.r2.y));
                            const float dz = fabsf(dot3(n.x, n.y, n.z, g.r0.z, g.r1.z, g.r2.z));
                            const float rr = (dx * hx + dy * hy) + dz * hz;
                            out_o |= (d[k] + rr <= 0.0f);
                        }
                        vis = !out_o;
                    }
                }
                any |= vis;
                const bool listed = vis && (st8 & S_HAS_CLASS);
                if (SIMPLE || R.rank == nullptr) {
                    const uint32_t b = __ballot_sync(0xFFFFFFFFu, listed);
                    if (lane == v) my_ballot = b;
                } else if (listed) {
                    uint32_t *mask = vb.mask + (size_t)v * vb.words_stride;
                    uint32_t *cc = vb.chunk_count + ((size_t)parity * kMaxViews + v) * vb.chunks_stride;
                    atomicOr(mask + (rnk >> 5), 1u << (rnk & 31u));
                    atomicAdd(cc + ((rnk >> 5) / kChunkWords), 1u);
                }
            }
            if (my_ballot) {
                uint32_t vl = lane;
                asm volatile("" : "+r"(vl));     // keeps the two row offsets below out of registers held through the tile loop
                uint32_t *mask = vb.mask + (size_t)vl * vb.words_stride;
                uint32_t *cc = vb.chunk_count + ((size_t)parity * kMaxViews + vl) * vb.chunks_stride;
                const uint32_t row0 = row - lane, w0 = row0 >> 5, sh = row0 & 31u;
                const uint32_t lo = my_ballot << sh, hi = sh ? (my_ballot >> (32u - sh)) : 0u;
                if (lo) { atomicOr(mask + w0, lo); atomicAdd(cc + (w0 / kChunkWords), __popc(lo)); }
                if (hi) { atomicOr(mask + w0 + 1, hi); atomicAdd(cc + ((w0 + 1) / kChunkWords), __popc(hi)); }
            }
            if (in_query) {
                out = (out & ~S_VV) | (any ? (1u | (prev << 1)) : 0u);
                vv_changed = (any ? 1u : 0u) != prev;
                if (vv_changed) out |= S_VV_CHANGED;
            }
        } else {
            out |= st8 & S_VV_CHANGED;
        }
        if (active && out != st8) R.state[row] = (uint8_t)out;
        // a light row publishes what assign_objects_to_clusters needs of it (GlobalTransform::translation,
        // ViewVisibility::get) so that the cluster kernels never touch the row arrays again
        if (CULL && R.light_snap != nullptr && (f & F_SPHERE_GT) && active) {
            const uint32_t ord = R.light_ord[row];     // 0xFFFFFFFF: a sphere-from-GT row that is not a current light
            if (ord < R.n_lights) R.light_snap[ord] = make_float4(S.gt0[li].w, S.gt1[li].w, S.gt2[li].w, (out & 1u) ? 1.0f : 0.0f);
        }

        // end of tile: everybody is done with this stage; count changes; write the tile's matrices back
        n_gt_total += (PROP && changed) ? 1u : 0u;      // per-thread tallies, reduced once at the end of the kernel
        n_vv_total += vv_changed ? 1u : 0u;
        if (ROW0 && !CULL && row0) asm volatile("cp.async.wait_all;" ::: "memory");   // old rows 1-2 of unvisited rows
        TP(7);
        const int any_gt = __syncthreads_or(PROP && changed);
        TP(8);
        if (ROW0 && lr == 0) {      // the tile's staging for its next run
            const uint32_t fb = s.gt_fb[sidx];
            if (gt_hint != nullptr && fb != s.gt_full[sidx]) gt_hint[tile_idx(t)] = (uint8_t)fb;
            s.gt_fb[sidx] = 0u;
        }
        t = s.next_tile[sidx];
        if (lr == 0) {
            if (PROP && any_gt) {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic smem writes -> async proxy
                const uint32_t bytes = (uint32_t)tile.n_rows * 16u;
                bulk_s2g(R.gt0 + tile.base, S.gt0 + off, bytes); bulk_s2g(R.gt1 + tile.base, S.gt1 + off, bytes);
                bulk_s2g(R.gt2 + tile.base, S.gt2 + off, bytes);
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
        }
        TP(9);
    }
    TP_END();
    if (lr == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    // block-reduce the per-thread tallies (warp shuffle, then one shared-memory atomic per warp)
    __shared__ uint32_t s_cnt[2];
    if (lr < 2) s_cnt[lr] = 0;
    __syncthreads();
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { n_gt_total += __shfl_xor_sync(0xFFFFFFFFu, n_gt_total, o); n_vv_total += __shfl_xor_sync(0xFFFFFFFFu, n_vv_total, o); }
    if ((lr & 31u) == 0) { if (n_gt_total) atomicAdd(&s_cnt[0], n_gt_total); if (n_vv_total) atomicAdd(&s_cnt[1], n_vv_total); }
    __syncthreads();
    if (lr == 0) {
        if (s_cnt[0]) atomicAdd(&stats->changed[parity][0], s_cnt[0]);
        if (s_cnt[1]) atomicAdd(&stats->changed[parity][1], s_cnt[1]);
    }
}
