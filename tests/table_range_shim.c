/*
 * table_range_shim.c -- the cull system's VisibilityRange sequence of rust/b200vis_plugin.rs, through include/b200vis.h in
 * plain C, on Bevy-native archetype tables (malloc'd, filled in spawn order), checked against the CPU oracle every frame.
 *
 * The "ECS": a forest of complete binary trees, spawned level by level across all trees.  Four archetype tables -- roots,
 * inner nodes, leaves, and leaves with a VisibilityRange -- each with Bevy's column layouts:
 *     GlobalTransform 64 B, ViewVisibility 1 B, Aabb 32 B (two Vec3A), InheritedVisibility 1 B, each with changed_ticks;
 *     VisibilityRange 20 B { start_margin: Range<f32>, end_margin: Range<f32>, use_aabb: bool } in the ranged table.
 * Range views: 31 ShadowLodOrigin entities, then the two cameras, in that query order; `.take(32)` keeps the origins
 * and camera 0, so camera 0 reads bit 31 and camera 1 has range_view_index -1 (every ranged entity culled for it,
 * range.rs:214-222).
 *
 * The plugin's sequence:
 *   sync:  b200vis_set_tables (again whenever a table's len changes), b200vis_set_table_cull_inputs (F_RANGE on the
 *          ranged table), b200vis_set_table_visibility_ranges with the layout from size_of / offset_of! -- no detach
 *          in between, so tables whose entries did not change are not read in full again;
 *   cull:  b200vis_set_visibility_range_views (the 32 positions), b200vis_set_views (range_view_index = the camera's
 *          place in that list, or -1), b200vis_upload_bounds only at the start with a NULL range mask,
 *          b200vis_read_tables(RD_CULL_INPUTS, last_run, this_run), b200vis_run(PROPAGATE | CULL).
 * Between frames the "game": every root moves; some ranged slots get a new VisibilityRange with this frame's tick;
 * leaves move between the plain and the ranged table (swap_remove, the inserted VisibilityRange stamped with the frame's
 * tick); after the moves, other ranged slots are overwritten without a tick (bypass_change_detection), which a
 * tick-driven read does not see.
 * Checked every frame: the range masks against orc_check_visibility_ranges, and every view's visible rows against
 * orc_cull with those masks.
 *
 * Build (tests/test_table_range_shim.py does this): gcc -O2 -std=gnu11 -Wall -Wextra -Werror -Iinclude
 *        tests/table_range_shim.c -Lbevy_b200 -lb200vis -Loracle -lbevy_oracle -lm ; run: ./table_range_shim [n_trees]
 *        [levels] [frames], or ./table_range_shim --sizeof to print the layouts (no GPU needed).
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "b200vis.h"

int orc_propagate(uint32_t n, const uint32_t *parent, const float *trs, float *gt, const uint8_t *tchanged,
                  const uint8_t *gt_ext_changed, int static_opt, uint8_t *changed);
int orc_cull(uint32_t n, const float *gt, const float *bounds, const uint8_t *flags, const uint64_t *layer_mask,
             const uint32_t *range_mask, const uint8_t *class_mask, const uint64_t *entity_bits, uint8_t *vv, uint8_t *vv_changed,
             uint32_t n_views, const float *view_planes, const uint64_t *view_layers, const uint8_t *view_flags,
             const int8_t *view_range_index, uint32_t *visible_rows, uint32_t *visible_count);
void orc_check_visibility_ranges(uint32_t n, const float *gt, const float *bounds, const uint8_t *flags, const float *range,
                                 const uint8_t *use_aabb, uint32_t n_views, const float *view_pos, uint32_t *mask_out);

/* Bevy's components as rustc lays them out for this test's "ECS" */
typedef struct { float m[16]; } BevyGlobalTransform;                                   /* Affine3A, 64 B */
typedef struct { float center[4], half_extents[4]; } BevyAabb;                         /* two Vec3A, 32 B */
typedef struct { float start_margin[2], end_margin[2]; uint8_t use_aabb; uint8_t pad[3]; } BevyVisibilityRange;   /* 20 B */

enum { ROOTS, INNER, LEAVES, RANGED, N_TABLES };
typedef struct {
    BevyGlobalTransform *gt; uint32_t *gt_ticks;
    uint8_t *vv; uint32_t *vv_ticks;
    BevyAabb *aabb; uint32_t *aabb_ticks;
    uint8_t *iv; uint32_t *iv_ticks;
    BevyVisibilityRange *range; uint32_t *range_ticks;   /* the ranged table only */
    uint32_t *entities;
    uint32_t len, capacity;
} Table;

#define CHECK(call)                                                                                     \
    do {                                                                                                \
        int32_t rc_ = (call);                                                                           \
        if (rc_ != B200VIS_OK) {                                                                        \
            fprintf(stderr, "%s failed: %d (%s)\n", #call, rc_, b200vis_last_error(ctx));               \
            return 2;                                                                                   \
        }                                                                                               \
    } while (0)

static uint64_t rng_state = 11;
static float frand(float lo, float hi) {                /* SplitMix64 */
    uint64_t z = (rng_state += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; z ^= z >> 31;
    return lo + (hi - lo) * (float)((z >> 40) * (1.0 / 16777216.0));
}
static void random_range(BevyVisibilityRange *r, uint32_t k) {
    const float start = frand(0.0f, 150.0f), end = start + frand(20.0f, 300.0f);
    r->start_margin[0] = start; r->start_margin[1] = start + 5.0f;     /* the margins' inner ends: never read */
    r->end_margin[0] = end - 5.0f; r->end_margin[1] = end;
    r->use_aabb = (uint8_t)(k % 3u == 0 ? 0 : k % 3u == 1 ? 1 : 2);    /* bool bytes other than 0 and 1 count as true */
    memset(r->pad, 0, sizeof r->pad);
}

static int cmp_u32(const void *a, const void *b) {
    const uint32_t x = *(const uint32_t *)a, y = *(const uint32_t *)b;
    return x < y ? -1 : x > y;
}

int main(int argc, char **argv) {
    if (argc > 1 && strcmp(argv[1], "--sizeof") == 0) {
        printf("{\"visibility_range\": %zu, \"layout\": [%zu, %zu, %zu, %zu]}\n", sizeof(BevyVisibilityRange),
               sizeof(b200vis_visibility_range_layout), offsetof(b200vis_visibility_range_layout, start),
               offsetof(b200vis_visibility_range_layout, end), offsetof(b200vis_visibility_range_layout, use_aabb));
        return 0;
    }
    const uint32_t n_trees = argc > 1 ? (uint32_t)atoi(argv[1]) : 120, levels = argc > 2 ? (uint32_t)atoi(argv[2]) : 6;
    const uint32_t frames = argc > 3 ? (uint32_t)atoi(argv[3]) : 5, V = 2, N_ORIGINS = 31, N_RANGE_VIEWS = 32;
    const uint32_t per = (1u << levels) - 1, n = n_trees * per;
    b200vis_ctx *ctx = NULL;

    /* ---- spawn: level by level across the trees ---- */
    uint32_t *child_of = malloc((size_t)n * 4), *node_entity = malloc((size_t)n * 4);
    for (uint32_t e = 0, lvl = 0; lvl < levels; ++lvl)
        for (uint32_t tr = 0; tr < n_trees; ++tr)
            for (uint32_t k = (1u << lvl) - 1; k < (2u << lvl) - 1; ++k) node_entity[tr * per + k] = e++;
    uint8_t *has_kids = calloc(n, 1);
    for (uint32_t tr = 0; tr < n_trees; ++tr)
        for (uint32_t k = 0; k < per; ++k) {
            const uint32_t e = node_entity[tr * per + k];
            child_of[e] = k ? node_entity[tr * per + (k - 1) / 2] : B200VIS_NO_PARENT;
            if (k) has_kids[child_of[e]] = 1;
        }
    float *trs_e = malloc((size_t)n * 40);
    BevyAabb *aabb_e = malloc((size_t)n * sizeof(BevyAabb));
    BevyVisibilityRange *range_e = malloc((size_t)n * sizeof(BevyVisibilityRange));
    uint8_t *arch = malloc(n);
    Table tab[N_TABLES];
    memset(tab, 0, sizeof tab);
    for (uint32_t e = 0; e < n; ++e) {
        float *t = trs_e + (size_t)e * 10;
        const int root = child_of[e] == B200VIS_NO_PARENT;
        float q[4] = {frand(-1, 1), frand(-1, 1), frand(-1, 1), frand(-1, 1)};
        const float qn = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
        const float spread = root ? 250.0f : 3.0f;
        for (int i = 0; i < 3; ++i) { t[i] = frand(-spread, spread); t[7 + i] = frand(0.5f, 1.5f); }
        for (int i = 0; i < 4; ++i) t[3 + i] = q[i] / qn;
        memset(&aabb_e[e], 0, sizeof aabb_e[e]);
        for (int i = 0; i < 3; ++i) { aabb_e[e].center[i] = frand(-1.0f, 1.0f); aabb_e[e].half_extents[i] = frand(0.25f, 0.75f); }
        random_range(&range_e[e], e);
        arch[e] = root ? ROOTS : has_kids[e] ? INNER : (e & 1u) ? RANGED : LEAVES;
        tab[arch[e]].len++;
    }
    /* ---- the archetype tables, each in spawn order, with room for the moves ---- */
    for (int t = 0; t < N_TABLES; ++t) {
        uint32_t cap = 8;
        while (cap < tab[t].len + 64) cap *= 2;
        Table *T = &tab[t];
        T->capacity = cap;
        T->gt = aligned_alloc(64, (size_t)cap * 64); T->gt_ticks = calloc(cap, 4);
        T->vv = calloc(cap, 1); T->vv_ticks = calloc(cap, 4);
        T->aabb = aligned_alloc(16, (size_t)cap * sizeof(BevyAabb)); T->aabb_ticks = calloc(cap, 4);
        T->iv = calloc(cap, 1); T->iv_ticks = calloc(cap, 4);
        if (t == RANGED) { T->range = calloc(cap, sizeof(BevyVisibilityRange)); T->range_ticks = calloc(cap, 4); }
        T->entities = malloc((size_t)cap * 4);
        memset(T->gt, 0, (size_t)cap * 64); memset(T->aabb, 0, (size_t)cap * sizeof(BevyAabb));
        T->len = 0;
    }
    for (uint32_t e = 0; e < n; ++e) {                   /* spawn: every component with tick 990 */
        Table *T = &tab[arch[e]];
        const uint32_t s = T->len++;
        T->aabb[s] = aabb_e[e]; T->aabb_ticks[s] = 990;
        T->iv[s] = 1; T->iv_ticks[s] = 990;
        if (T->range) { T->range[s] = range_e[e]; T->range_ticks[s] = 990; }
        T->entities[s] = e;
    }

    /* ---- device rows: the planned order ---- */
    uint32_t *new_to_old = malloc((size_t)n * 4), *row_of = malloc((size_t)n * 4);
    if (b200vis_plan_row_order(n, child_of, new_to_old) != B200VIS_OK) { fprintf(stderr, "plan_row_order failed\n"); return 2; }
    for (uint32_t r = 0; r < n; ++r) row_of[new_to_old[r]] = r;
    uint32_t *parent = malloc((size_t)n * 4);
    uint64_t *entity_bits = malloc((size_t)n * 8);
    float *trs = malloc((size_t)n * 40), *bounds = malloc((size_t)n * 24), *range_se = malloc((size_t)n * 8);
    uint8_t *flags = malloc(n), *cls = malloc(n), *use_aabb = malloc(n);
    for (uint32_t r = 0; r < n; ++r) {                   /* the oracle's view of each row (upload_bounds' too) */
        const uint32_t e = new_to_old[r];
        parent[r] = child_of[e] == B200VIS_NO_PARENT ? B200VIS_NO_PARENT : row_of[child_of[e]];
        entity_bits[r] = e;
        memcpy(trs + (size_t)r * 10, trs_e + (size_t)e * 10, 40);
        for (int i = 0; i < 3; ++i) { bounds[r * 6 + i] = aabb_e[e].center[i]; bounds[r * 6 + 3 + i] = aabb_e[e].half_extents[i]; }
        flags[r] = B200VIS_F_INHERITED_VISIBLE | B200VIS_F_HAS_AABB | (arch[e] == RANGED ? B200VIS_F_HAS_VIS_RANGE : 0);
        cls[r] = 1;
        range_se[r * 2] = range_e[e].start_margin[0]; range_se[r * 2 + 1] = range_e[e].end_margin[1];
        use_aabb[r] = range_e[e].use_aabb != 0;
    }
    b200vis_config cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.max_entities = n; cfg.max_lights = 1; cfg.max_views = V;
    if (b200vis_create(&cfg, &ctx) != B200VIS_OK) { fprintf(stderr, "b200vis_create: %s\n", b200vis_last_error(NULL)); return 3; }
    CHECK(b200vis_set_topology(ctx, n, parent, entity_bits));
    CHECK(b200vis_upload_transforms(ctx, 0, n, trs));
    {
        float *gt12 = calloc((size_t)n * 12, 4);
        for (uint32_t r = 0; r < n; ++r) gt12[r * 12] = gt12[r * 12 + 4] = gt12[r * 12 + 8] = 1.0f;
        CHECK(b200vis_upload_global_transforms(ctx, 0, n, gt12));
        free(gt12);
    }
    /* the cull system after a renumbering: every row once, and no VisibleEntityRanges mask */
    CHECK(b200vis_upload_bounds(ctx, 0, n, bounds, flags, cls, NULL, NULL));

    /* ---- b200_sync_tables: the registry, the cull inputs and the VisibilityRange columns ---- */
    const b200vis_bounds_layout blay = {sizeof(BevyAabb), offsetof(BevyAabb, center), offsetof(BevyAabb, half_extents), 32, 0, 16};
    const b200vis_visibility_range_layout rlay = {sizeof(BevyVisibilityRange),
                                                  offsetof(BevyVisibilityRange, start_margin) + 0 * sizeof(float),
                                                  offsetof(BevyVisibilityRange, end_margin) + 1 * sizeof(float),
                                                  offsetof(BevyVisibilityRange, use_aabb)};
    uint32_t *slot_rows = malloc((size_t)n * 4);
#define SYNC_TABLES(send_maps)                                                                                         \
    do {                                                                                                               \
        b200vis_table desc_[N_TABLES];                                                                                 \
        b200vis_table_cull_inputs cull_[N_TABLES];                                                                     \
        b200vis_table_visibility_ranges rg_[N_TABLES];                                                                 \
        for (int t_ = 0; t_ < N_TABLES; ++t_) {                                                                        \
            const Table *T_ = &tab[t_];                                                                                \
            desc_[t_] = (b200vis_table){T_->gt, T_->gt_ticks, T_->vv, T_->vv_ticks, T_->len, T_->capacity};             \
            memset(&cull_[t_], 0, sizeof cull_[t_]);                                                                   \
            cull_[t_].aabbs = T_->aabb; cull_[t_].aabb_changed_ticks = T_->aabb_ticks;                                 \
            cull_[t_].inherited_visibility = T_->iv; cull_[t_].iv_changed_ticks = T_->iv_ticks;                        \
            cull_[t_].flags = T_->range ? B200VIS_F_HAS_VIS_RANGE : 0u;                                                \
            rg_[t_].ranges = T_->range; rg_[t_].changed_ticks = T_->range_ticks;                                       \
        }                                                                                                              \
        CHECK(b200vis_set_tables(ctx, N_TABLES, desc_));                                                              \
        CHECK(b200vis_set_table_cull_inputs(ctx, N_TABLES, cull_, &blay));                                            \
        CHECK(b200vis_set_table_visibility_ranges(ctx, N_TABLES, rg_, &rlay));                                        \
        for (int t_ = 0; t_ < N_TABLES && (send_maps); ++t_) {                                                         \
            for (uint32_t s_ = 0; s_ < tab[t_].len; ++s_) slot_rows[s_] = row_of[tab[t_].entities[s_]];                \
            CHECK(b200vis_set_table_rows(ctx, (uint32_t)t_, 0, tab[t_].len, slot_rows));                               \
        }                                                                                                              \
    } while (0)
    SYNC_TABLES(1);

    /* ---- the range views: 31 ShadowLodOrigin entities, then the cameras ---- */
    float view_pos[(31 + 2) * 3];
    for (uint32_t i = 0; i < N_ORIGINS * 3; ++i) view_pos[i] = frand(-300.0f, 300.0f);

    float *o_gt = calloc((size_t)n * 12, 4);
    for (uint32_t r = 0; r < n; ++r) o_gt[r * 12] = o_gt[r * 12 + 4] = o_gt[r * 12 + 8] = 1.0f;
    uint8_t *o_vv = calloc(n, 1), *o_vvch = calloc(n, 1), *o_gtch = calloc(n, 1), *tchanged = malloc(n);
    uint32_t *o_mask = malloc((size_t)n * 4), *d_mask = malloc((size_t)n * 4);
    uint32_t *o_rows = malloc((size_t)V * n * 4), o_count[B200VIS_MAX_VIEWS], *d_rows = malloc((size_t)V * n * 4);
    memset(tchanged, 1, n);
    int ok = 1;
    uint32_t last_run = 995, total_in_range = 0, total_ranged_visible = 0, moved_in = 0, bypassed = 0, stamped = 0;
    for (uint32_t frame = 1; frame <= frames && ok; ++frame) {
        const uint32_t this_run = 1000u + 10u * frame;
        /* ---- the game ---- */
        if (frame > 1)
            for (uint32_t tr = 0; tr < n_trees; ++tr) {   /* every root moves */
                const uint32_t r = row_of[node_entity[tr * per]];
                trs[(size_t)r * 10 + 0] += 0.5f * sinf(0.1f * (float)(frame + tr));
                tchanged[r] = 1;
                CHECK(b200vis_upload_transforms(ctx, r, 1, trs + (size_t)r * 10));
            }
        Table *RT = &tab[RANGED], *LT = &tab[LEAVES];
        if (frame == 2 || frame == 4) {
            for (uint32_t s = frame; s < RT->len; s += 7) {
                const uint32_t e = RT->entities[s], r = row_of[e];
                if (s % 2u || frame < 4) {               /* a new VisibilityRange, stamped with this frame's tick */
                    random_range(&RT->range[s], e + frame);
                    RT->range_ticks[s] = this_run - 1u;
                    range_se[r * 2] = RT->range[s].start_margin[0]; range_se[r * 2 + 1] = RT->range[s].end_margin[1];
                    use_aabb[r] = RT->range[s].use_aabb != 0;
                    ++stamped;
                } else {                                 /* bypass_change_detection, after the moves: no tick, so the
                                                            cull keeps the value it read (nothing reads the slot in full) */
                    RT->range[s].start_margin[0] = 1e6f; RT->range[s].end_margin[1] = 2e6f;
                    ++bypassed;
                }
            }
        }
        if (frame == 3) {                                /* archetype moves, both ways, with swap_remove */
            for (int dir = 0; dir < 2; ++dir)
                for (uint32_t k = 0; k < 12; ++k) {
                    Table *src = dir ? RT : LT, *dst = dir ? LT : RT;
                    const uint32_t s = (k * 13u + 1u) % src->len, e = src->entities[s], d = dst->len++, last = --src->len;
                    dst->entities[d] = e; dst->gt[d] = src->gt[s]; dst->gt_ticks[d] = src->gt_ticks[s];
                    dst->vv[d] = src->vv[s]; dst->vv_ticks[d] = src->vv_ticks[s];
                    dst->aabb[d] = src->aabb[s]; dst->aabb_ticks[d] = src->aabb_ticks[s];
                    dst->iv[d] = src->iv[s]; dst->iv_ticks[d] = src->iv_ticks[s];
                    const uint32_t r = row_of[e];
                    if (dst->range) {                    /* insert VisibilityRange */
                        random_range(&dst->range[d], e + 77u);
                        dst->range_ticks[d] = this_run - 2u;
                        range_se[r * 2] = dst->range[d].start_margin[0]; range_se[r * 2 + 1] = dst->range[d].end_margin[1];
                        use_aabb[r] = dst->range[d].use_aabb != 0;
                        flags[r] |= B200VIS_F_HAS_VIS_RANGE;
                        ++moved_in;
                    } else {
                        flags[r] &= (uint8_t)~B200VIS_F_HAS_VIS_RANGE;
                    }
                    if (s != last) {
                        src->entities[s] = src->entities[last]; src->gt[s] = src->gt[last]; src->gt_ticks[s] = src->gt_ticks[last];
                        src->vv[s] = src->vv[last]; src->vv_ticks[s] = src->vv_ticks[last];
                        src->aabb[s] = src->aabb[last]; src->aabb_ticks[s] = src->aabb_ticks[last];
                        src->iv[s] = src->iv[last]; src->iv_ticks[s] = src->iv_ticks[last];
                        if (src->range) { src->range[s] = src->range[last]; src->range_ticks[s] = src->range_ticks[last]; }
                    }
                }
            SYNC_TABLES(1);                              /* len changed: the registry and every attachment again */
        }
        /* ---- the cameras and the range views ---- */
        b200vis_view views[2];
        float planes[2][6][4];
        uint64_t view_layers[2] = {1, 1};
        uint8_t view_flags[2] = {B200VIS_VIEW_ACTIVE, B200VIS_VIEW_ACTIVE};
        int8_t vri[2];
        for (uint32_t v = 0; v < V; ++v) {
            const float yaw = 0.2f * (float)frame + 3.1415927f * (float)v, cy = cosf(yaw), sy = sinf(yaw);
            const float gt[12] = {cy, 0, -sy, 0, 1, 0, sy, 0, cy, 10.0f * (float)v, 0, -5.0f * (float)v};
            float cfv[16];
            b200vis_host_perspective(0.9f, 16.0f / 9.0f, 0.1f, cfv);
            b200vis_host_compute_frustum(cfv, gt, 1000.0f, planes[v]);
            memcpy(&view_pos[(N_ORIGINS + v) * 3], &gt[9], 12);
            memset(&views[v], 0, sizeof views[v]);
            memcpy(views[v].half_spaces, planes[v], sizeof planes[v]);
            views[v].layer_mask = 1; views[v].flags = B200VIS_VIEW_ACTIVE;
            /* the camera's place among the first 32 range views, or -1 */
            vri[v] = N_ORIGINS + v < N_RANGE_VIEWS ? (int8_t)(N_ORIGINS + v) : (int8_t)-1;
            views[v].range_view_index = vri[v];
        }
        const uint32_t n_listed = N_ORIGINS + V < N_RANGE_VIEWS ? N_ORIGINS + V : N_RANGE_VIEWS;
        /* ---- b200_check_visibility ---- */
        CHECK(b200vis_set_visibility_range_views(ctx, n_listed, view_pos));
        CHECK(b200vis_set_views(ctx, V, views));
        CHECK(b200vis_read_tables(ctx, B200VIS_RD_CULL_INPUTS, last_run, this_run));
        CHECK(b200vis_run(ctx, B200VIS_STAGE_PROPAGATE | B200VIS_STAGE_CULL));
        b200vis_frame_stats stats;
        CHECK(b200vis_download_frame(ctx, &stats, d_rows, n, NULL, NULL, 0));
        CHECK(b200vis_download_visibility_ranges(ctx, 0, n, d_mask));
        last_run = this_run;
        /* ---- the oracle ---- */
        if (orc_propagate(n, parent, trs, o_gt, tchanged, NULL, 1, o_gtch) != 0) { fprintf(stderr, "oracle propagate failed\n"); return 4; }
        orc_check_visibility_ranges(n, o_gt, bounds, flags, range_se, use_aabb, n_listed, view_pos, o_mask);
        orc_cull(n, o_gt, bounds, flags, NULL, o_mask, cls, entity_bits, o_vv, o_vvch, V, &planes[0][0][0], view_layers,
                 view_flags, vri, o_rows, o_count);
        memset(tchanged, 0, n);
        uint32_t in_range = 0, bad_mask = 0;
        for (uint32_t r = 0; r < n; ++r) {
            in_range += o_mask[r] != 0;
            if (d_mask[r] != o_mask[r] && bad_mask++ < 4)
                fprintf(stderr, "frame %u row %u: range mask 0x%08x vs the oracle's 0x%08x\n", frame, r, d_mask[r], o_mask[r]);
        }
        ok &= bad_mask == 0;
        uint32_t ranged_visible = 0;
        for (uint32_t v = 0; v < V && ok; ++v) {
            uint32_t *d = d_rows + (size_t)v * n, *o = o_rows + (size_t)v * n;
            if (stats.visible_count[v] != o_count[v]) {
                fprintf(stderr, "frame %u view %u: %u visible rows vs the oracle's %u\n", frame, v, stats.visible_count[v], o_count[v]);
                ok = 0; break;
            }
            qsort(d, o_count[v], 4, cmp_u32); qsort(o, o_count[v], 4, cmp_u32);
            if (memcmp(d, o, (size_t)o_count[v] * 4) != 0) { fprintf(stderr, "frame %u view %u: visible rows differ\n", frame, v); ok = 0; }
            for (uint32_t i = 0; i < o_count[v]; ++i) {
                const int ranged = (flags[o[i]] & B200VIS_F_HAS_VIS_RANGE) != 0;
                ranged_visible += ranged;
                if (ranged && vri[v] < 0) { fprintf(stderr, "frame %u view %u: a ranged row is visible without a range bit\n", frame, v); ok = 0; }
            }
        }
        total_in_range += in_range; total_ranged_visible += ranged_visible;
        printf("frame %u: %u rows in range of some view, %u ranged rows visible: %s\n", frame, in_range, ranged_visible, ok ? "OK" : "MISMATCH");
    }
    printf("{\"entities\": %u, \"in_range\": %u, \"ranged_visible\": %u, \"moved_in\": %u, \"stamped\": %u, \"bypassed\": %u}\n",
           n, total_in_range, total_ranged_visible, moved_in, stamped, bypassed);
    CHECK(b200vis_set_tables(ctx, 0, NULL));
    b200vis_destroy(ctx);
    printf(ok ? "TABLE_RANGE_SHIM OK\n" : "TABLE_RANGE_SHIM FAILED\n");
    return ok ? 0 : 1;
}
