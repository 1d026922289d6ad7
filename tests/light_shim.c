/*
 * light_shim.c -- the light-visibility frame of rust/b200vis_plugin.rs (b200_check_light_visibility), through
 * include/b200vis.h in plain C, on Bevy-native archetype tables (malloc'd, filled in spawn order), checked against the CPU
 * oracle every frame.
 *
 * The "ECS": a forest of complete binary trees spawned level by level, then the point and spot lights.  Archetype tables,
 * each with Bevy's column layouts (Transform 40 B with rotation first, GlobalTransform 64 B, ViewVisibility 1 B, Aabb 32 B,
 * InheritedVisibility 1 B, VisibilityRange 20 B, each with changed_ticks):
 *     ROOTS       no Mesh3d (not a shadow caster)
 *     INNER       Mesh3d (caster)
 *     LEAVES      Mesh3d (caster)
 *     NOT_CASTER  Mesh3d + NotShadowCaster
 *     NO_FC       Mesh3d + NoFrustumCulling (caster)
 *     RANGED      Mesh3d + VisibilityRange (caster)
 *     LIGHTS      PointLight / SpotLight (not a caster)
 * Range views: one ShadowLodOrigin entity, then the two cameras (bits 0, 1, 2).  Point and spot items use bit 0, a
 * cascade its camera's bit.  One directional light has CascadesFrusta over both cameras x 4 hand-built boxes.
 *
 * Per frame, as the plugin runs it:
 *   CPU reset_view_visibility on the table bytes (no tick); b200vis_read_tables(RD_TRANSFORM | RD_CULL_INPUTS);
 *   b200vis_run(PROPAGATE | CULL); b200vis_writeback_tables(WB_GLOBAL_TRANSFORM | WB_SET_VISIBLE, cam_tick);
 *   the light step: the items (points and spots with shadow maps, every (view, cascade) of a visible directional light with
 *   shadow maps), b200vis_set_shadow_items (the sink's max_items grown first when it is too small),
 *   b200vis_set_shadow_item_render_layers_ext when some light has a layer in 64..255, b200vis_run_shadow_culling,
 *   b200vis_writeback_tables(WB_SET_VISIBLE, light_tick), b200vis_synchronize; a sink too small for the run grows to
 *   max(total, 2 x capacity) and b200vis_emit_shadow_entities + b200vis_synchronize fill it; the components are filled
 *   for active items only, CascadesVisibleEntities with the reference's view bookkeeping;
 *   CPU mark_newly_hidden_entities_invisible on the table bytes (mark_tick).
 * Across frames: roots and lights move; point light 0 leaves every view at frame 3 (its item inactive, its lists kept)
 * and comes back at frame 5; spot light 0 moves to RenderLayers layer 70 only at frame 4; the directional light is
 * invisible at frame 3, loses camera 1 at frame 4 and has three cascades at frame 5; frames 1, 2 and 4 start from a
 * 64-entry sink for 4 items, so both growth paths (items before set_shadow_items, entries through the emit) run.
 * Checked every frame against the oracle (orc_cull with mark_newly_hidden deferred, the three light passes,
 * orc_mark_newly_hidden): every list of every component, the CascadesVisibleEntities keys, every ViewVisibility byte,
 * and that the byte's changed tick is cam_tick, light_tick or mark_tick exactly where the oracle's Changed fires in
 * that pass (unchanged elsewhere).
 *
 * Build (tests/test_light_shim.py does this): gcc -O2 -std=gnu11 -Wall -Wextra -Werror -Iinclude tests/light_shim.c
 *        -Lbevy_b200 -lb200vis -Loracle -lbevy_oracle -lm ; run: ./light_shim [n_trees] [levels] [frames] [points]
 *        [spots], or ./light_shim --sizeof to print the layouts (no GPU needed).
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "b200vis.h"

int orc_propagate(uint32_t n, const uint32_t *parent, const float *trs, float *gt, const uint8_t *tchanged,
                  const uint8_t *gt_ext_changed, int static_opt, uint8_t *changed);
int orc_cull(uint32_t n, const float *gt, const float *bounds, const uint8_t *flags, const uint64_t *layer_mask,
             const uint32_t *range_mask, const uint8_t *class_mask, const uint64_t *entity_bits, uint8_t *vv, uint8_t *vv_changed,
             uint32_t n_views, const float *view_planes, const uint64_t *view_layers, const uint8_t *view_flags,
             const int8_t *view_range_index, uint32_t *visible_rows, uint32_t *visible_count);
void orc_set_defer_mark_newly_hidden(int on);
void orc_mark_newly_hidden(uint32_t n, const uint8_t *flags, uint8_t *vv, uint8_t *vv_changed);
void orc_check_visibility_ranges(uint32_t n, const float *gt, const float *bounds, const uint8_t *flags, const float *range,
                                 const uint8_t *use_aabb, uint32_t n_views, const float *view_pos, uint32_t *mask_out);
int orc_check_point_light_mesh_visibility(uint32_t n, const float *gt, const float *bounds, const uint8_t *flags, const uint8_t *caster,
                                          const uint64_t *layer_mask, const uint32_t *range_mask, int lod_origin_index,
                                          const uint64_t *entity_bits, uint8_t *vv, uint8_t *vv_changed, uint32_t n_lights,
                                          const float *light_sphere, const uint64_t *light_layers, const float *frusta,
                                          uint32_t *visible_rows, uint32_t *visible_count);
int orc_check_spot_light_mesh_visibility(uint32_t n, const float *gt, const float *bounds, const uint8_t *flags, const uint8_t *caster,
                                         const uint64_t *layer_mask, const uint32_t *range_mask, int lod_origin_index,
                                         const uint64_t *entity_bits, uint8_t *vv, uint8_t *vv_changed, uint32_t n_lights,
                                         const float *light_sphere, const uint64_t *light_layers, const float *frusta,
                                         uint32_t *visible_rows, uint32_t *visible_count);
int orc_check_dir_light_mesh_visibility(uint32_t n, const float *gt, const float *bounds, const uint8_t *flags, const uint8_t *caster,
                                        const uint64_t *layer_mask, const uint32_t *range_mask, const uint64_t *entity_bits,
                                        uint8_t *vv, uint8_t *vv_changed, uint32_t n_items, const int32_t *view_range_index,
                                        const uint64_t *light_layers, const uint32_t *n_cascades, const float *frusta,
                                        uint32_t *visible_rows, uint32_t *visible_count);

/* Bevy's components as rustc lays them out for this test's "ECS" */
typedef struct { float rotation[4], translation[3], scale[3]; } BevyTransform;           /* 40 B */
typedef struct { float m[16]; } BevyGlobalTransform;                                   /* Affine3A, 64 B */
typedef struct { float center[4], half_extents[4]; } BevyAabb;                         /* two Vec3A, 32 B */
typedef struct { float start_margin[2], end_margin[2]; uint8_t use_aabb; uint8_t pad[3]; } BevyVisibilityRange;   /* 20 B */

enum { ROOTS, INNER, LEAVES, NOT_CASTER, NO_FC, RANGED, LIGHTS, N_TABLES };
static const uint8_t IS_CASTER[N_TABLES] = {0, 1, 1, 0, 1, 1, 0};
typedef struct {
    BevyTransform *tr; uint32_t *tr_ticks;
    BevyGlobalTransform *gt; uint32_t *gt_ticks;
    uint8_t *vv; uint32_t *vv_ticks;
    BevyAabb *aabb; uint32_t *aabb_ticks;
    uint8_t *iv; uint32_t *iv_ticks;
    BevyVisibilityRange *range; uint32_t *range_ticks;
    uint32_t *entities;
    uint32_t len, capacity;
} Table;

/* a Vec<Entity> of the components the plugin fills */
typedef struct { uint64_t *e; uint32_t n, cap; } List;
static void list_set(List *l, const uint64_t *src, uint32_t n) {      /* clear + extend_from_slice */
    if (n > l->cap) { l->cap = n; l->e = realloc(l->e, (size_t)n * 8); }
    if (n) memcpy(l->e, src, (size_t)n * 8);
    l->n = n;
}
/* CascadesVisibleEntities: view entity -> one list per cascade */
#define MAX_CASC 8
typedef struct { uint32_t n_views, view[4], n_casc[4]; List lists[4][MAX_CASC]; } CascadesVisible;

#define CHECK(call)                                                                                     \
    do {                                                                                                \
        int32_t rc_ = (call);                                                                           \
        if (rc_ != B200VIS_OK) {                                                                        \
            fprintf(stderr, "%s failed: %d (%s)\n", #call, rc_, b200vis_last_error(ctx));               \
            return 2;                                                                                   \
        }                                                                                               \
    } while (0)

static uint64_t rng_state = 23;
static float frand(float lo, float hi) {                /* SplitMix64 */
    uint64_t z = (rng_state += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; z ^= z >> 31;
    return lo + (hi - lo) * (float)((z >> 40) * (1.0 / 16777216.0));
}
static double now_ms(void) { struct timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return t.tv_sec * 1e3 + t.tv_nsec * 1e-6; }
/* an axis-aligned box as a Frustum (half spaces n . p + d >= 0; index 4 is the near plane, which cascades skip) */
static void box_frustum(const float lo[3], const float hi[3], float hs[6][4]) {
    const float p[6][4] = {{1, 0, 0, -lo[0]}, {-1, 0, 0, hi[0]}, {0, 1, 0, -lo[1]}, {0, -1, 0, hi[1]}, {0, 0, 1, -lo[2]}, {0, 0, -1, hi[2]}};
    memcpy(hs, p, sizeof p);
}
/* the directional light's CascadesFrusta this frame: cameras and cascade counts */
static uint32_t dir_views(uint32_t frame, uint32_t views[2], uint32_t casc[2]) {
    if (frame == 4) { views[0] = 0; casc[0] = 4; return 1; }                  /* camera 1 has left */
    if (frame == 5) { views[0] = 0; casc[0] = 3; return 1; }                  /* three cascades */
    views[0] = 0; views[1] = 1; casc[0] = casc[1] = 4; return 2;
}

int main(int argc, char **argv) {
    if (argc > 1 && strcmp(argv[1], "--sizeof") == 0) {
        printf("{\"shadow_item\": {\"sizeof\": %zu, \"kind\": %zu, \"light_row\": %zu, \"range\": %zu, \"range_view_index\": %zu, "
               "\"layer_mask\": %zu, \"frusta\": %zu}, \"shadow_entities_sink\": {\"sizeof\": %zu, \"entities\": %zu, \"capacity\": %zu, "
               "\"max_items\": %zu, \"offsets\": %zu, \"active\": %zu}}\n",
               sizeof(b200vis_shadow_item), offsetof(b200vis_shadow_item, kind), offsetof(b200vis_shadow_item, light_row),
               offsetof(b200vis_shadow_item, range), offsetof(b200vis_shadow_item, range_view_index),
               offsetof(b200vis_shadow_item, layer_mask), offsetof(b200vis_shadow_item, frusta),
               sizeof(b200vis_shadow_entities_sink), offsetof(b200vis_shadow_entities_sink, entities),
               offsetof(b200vis_shadow_entities_sink, capacity), offsetof(b200vis_shadow_entities_sink, max_items),
               offsetof(b200vis_shadow_entities_sink, offsets), offsetof(b200vis_shadow_entities_sink, active));
        return 0;
    }
    const uint32_t n_trees = argc > 1 ? (uint32_t)atoi(argv[1]) : 60, levels = argc > 2 ? (uint32_t)atoi(argv[2]) : 6;
    const uint32_t frames = argc > 3 ? (uint32_t)atoi(argv[3]) : 6;
    const uint32_t n_point = argc > 4 ? (uint32_t)atoi(argv[4]) : 6, n_spot = argc > 5 ? (uint32_t)atoi(argv[5]) : 4;
    const uint32_t V = 2, per = (1u << levels) - 1, n_forest = n_trees * per, n_lights = n_point + n_spot, n = n_forest + n_lights;
    const float S = 8.0f * sqrtf((float)n_trees), light_range = 0.6f * S;     /* the forest's half width, the lights' reach */
    b200vis_ctx *ctx = NULL;

    /* ---- spawn: the trees level by level, then the lights ---- */
    uint32_t *child_of = malloc((size_t)n * 4), *node_entity = malloc((size_t)n_forest * 4);
    for (uint32_t e = 0, lvl = 0; lvl < levels; ++lvl)
        for (uint32_t tr = 0; tr < n_trees; ++tr)
            for (uint32_t k = (1u << lvl) - 1; k < (2u << lvl) - 1; ++k) node_entity[tr * per + k] = e++;
    uint8_t *has_kids = calloc(n, 1), *arch = malloc(n);
    for (uint32_t tr = 0; tr < n_trees; ++tr)
        for (uint32_t k = 0; k < per; ++k) {
            const uint32_t e = node_entity[tr * per + k];
            child_of[e] = k ? node_entity[tr * per + (k - 1) / 2] : B200VIS_NO_PARENT;
            if (k) has_kids[child_of[e]] = 1;
        }
    BevyTransform *tr_e = malloc((size_t)n * sizeof(BevyTransform));
    BevyAabb *aabb_e = calloc(n, sizeof(BevyAabb));
    BevyVisibilityRange *range_e = calloc(n, sizeof(BevyVisibilityRange));
    Table tab[N_TABLES];
    memset(tab, 0, sizeof tab);
    for (uint32_t e = 0; e < n; ++e) {
        const int light = e >= n_forest, root = light || child_of[e] == B200VIS_NO_PARENT;
        if (light) child_of[e] = B200VIS_NO_PARENT;
        float q[4] = {frand(-1, 1), frand(-1, 1), frand(-1, 1), frand(-1, 1)};
        const float qn = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
        const float spread = light ? 0.5f * S : root ? S : 3.0f;
        for (int i = 0; i < 3; ++i) { tr_e[e].translation[i] = frand(-spread, spread); tr_e[e].scale[i] = light ? 1.0f : frand(0.5f, 1.5f); }
        if (light) tr_e[e].translation[1] *= 0.2f;
        for (int i = 0; i < 4; ++i) tr_e[e].rotation[i] = light ? (i == 3) : q[i] / qn;
        for (int i = 0; i < 3; ++i) { aabb_e[e].center[i] = light ? 0.0f : frand(-1.0f, 1.0f); aabb_e[e].half_extents[i] = light ? 0.5f : frand(0.25f, 0.75f); }
        const float start = frand(0.0f, 0.5f * S), end = start + frand(0.5f * S, 2.0f * S);
        range_e[e].start_margin[0] = start; range_e[e].start_margin[1] = start + 1.0f;
        range_e[e].end_margin[0] = end - 1.0f; range_e[e].end_margin[1] = end; range_e[e].use_aabb = (uint8_t)(e & 1u);
        arch[e] = light ? LIGHTS : root ? ROOTS : has_kids[e] ? INNER
                : (e % 5u == 0) ? NOT_CASTER : (e % 5u == 1) ? NO_FC : (e % 5u == 2) ? RANGED : LEAVES;
        tab[arch[e]].len++;
    }
    for (int t = 0; t < N_TABLES; ++t) {
        Table *T = &tab[t];
        uint32_t cap = 8;
        while (cap < T->len + 8) cap *= 2;
        T->capacity = cap;
        T->tr = calloc(cap, sizeof(BevyTransform)); T->tr_ticks = calloc(cap, 4);
        T->gt = aligned_alloc(64, (size_t)cap * 64); memset(T->gt, 0, (size_t)cap * 64); T->gt_ticks = calloc(cap, 4);
        T->vv = calloc(cap, 1); T->vv_ticks = calloc(cap, 4);
        T->aabb = aligned_alloc(16, (size_t)cap * sizeof(BevyAabb)); memset(T->aabb, 0, (size_t)cap * sizeof(BevyAabb));
        T->aabb_ticks = calloc(cap, 4); T->iv = calloc(cap, 1); T->iv_ticks = calloc(cap, 4);
        if (t == RANGED) { T->range = calloc(cap, sizeof(BevyVisibilityRange)); T->range_ticks = calloc(cap, 4); }
        T->entities = malloc((size_t)cap * 4);
        T->len = 0;
    }
    uint32_t *slot_of = malloc((size_t)n * 4);
    for (uint32_t e = 0; e < n; ++e) {                   /* spawn: every component with tick 990 */
        Table *T = &tab[arch[e]];
        const uint32_t s = T->len++;
        T->tr[s] = tr_e[e]; T->tr_ticks[s] = 990;
        T->aabb[s] = aabb_e[e]; T->aabb_ticks[s] = 990;
        T->iv[s] = 1; T->iv_ticks[s] = 990;
        if (T->range) { T->range[s] = range_e[e]; T->range_ticks[s] = 990; }
        T->entities[s] = e; slot_of[e] = s;
    }

    /* ---- device rows: the planned order; the oracle's view of each row ---- */
    uint32_t *new_to_old = malloc((size_t)n * 4), *row_of = malloc((size_t)n * 4);
    if (b200vis_plan_row_order(n, child_of, new_to_old) != B200VIS_OK) { fprintf(stderr, "plan_row_order failed\n"); return 2; }
    for (uint32_t r = 0; r < n; ++r) row_of[new_to_old[r]] = r;
    uint32_t *parent = malloc((size_t)n * 4);
    uint64_t *entity_bits = malloc((size_t)n * 8);
    float *trs = malloc((size_t)n * 40), *bounds = malloc((size_t)n * 24), *range_se = malloc((size_t)n * 8);
    uint8_t *flags = malloc(n), *cls = malloc(n), *use_aabb = malloc(n), *caster = malloc(n);
    for (uint32_t r = 0; r < n; ++r) {
        const uint32_t e = new_to_old[r];
        parent[r] = child_of[e] == B200VIS_NO_PARENT ? B200VIS_NO_PARENT : row_of[child_of[e]];
        entity_bits[r] = ((uint64_t)1 << 32) | e;        /* generation 1, index e */
        const BevyTransform *t = &tr_e[e];
        const float p[10] = {t->translation[0], t->translation[1], t->translation[2], t->rotation[0], t->rotation[1], t->rotation[2],
                             t->rotation[3], t->scale[0], t->scale[1], t->scale[2]};
        memcpy(trs + (size_t)r * 10, p, 40);
        for (int i = 0; i < 3; ++i) { bounds[r * 6 + i] = aabb_e[e].center[i]; bounds[r * 6 + 3 + i] = aabb_e[e].half_extents[i]; }
        flags[r] = B200VIS_F_INHERITED_VISIBLE | B200VIS_F_HAS_AABB | (arch[e] == RANGED ? B200VIS_F_HAS_VIS_RANGE : 0) |
                   (arch[e] == NO_FC ? B200VIS_F_NO_FRUSTUM_CULLING : 0);
        cls[r] = 1;
        range_se[r * 2] = range_e[e].start_margin[0]; range_se[r * 2 + 1] = range_e[e].end_margin[1];
        use_aabb[r] = range_e[e].use_aabb != 0;
        caster[r] = IS_CASTER[arch[e]];
    }
    b200vis_config cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.max_entities = n; cfg.max_lights = 1; cfg.max_views = V;
    if (b200vis_create(&cfg, &ctx) != B200VIS_OK) { fprintf(stderr, "b200vis_create: %s\n", b200vis_last_error(NULL)); return 3; }
    CHECK(b200vis_set_topology(ctx, n, parent, entity_bits));
    CHECK(b200vis_upload_transforms(ctx, 0, n, trs));      /* the plugin's rebuild: every row once */
    {
        float *gt12 = calloc((size_t)n * 12, 4);
        for (uint32_t r = 0; r < n; ++r) gt12[r * 12] = gt12[r * 12 + 4] = gt12[r * 12 + 8] = 1.0f;
        CHECK(b200vis_upload_global_transforms(ctx, 0, n, gt12));
        free(gt12);
    }
    CHECK(b200vis_upload_bounds(ctx, 0, n, bounds, flags, cls, NULL, NULL));

    /* ---- b200_sync_tables: registry, cull inputs, shadow casters (before the first cull read), ranges, slot maps ---- */
    const b200vis_transform_layout tlay = {sizeof(BevyTransform), offsetof(BevyTransform, translation), offsetof(BevyTransform, rotation),
                                           offsetof(BevyTransform, scale)};
    const b200vis_bounds_layout blay = {sizeof(BevyAabb), offsetof(BevyAabb, center), offsetof(BevyAabb, half_extents), 32, 0, 16};
    const b200vis_visibility_range_layout rlay = {sizeof(BevyVisibilityRange), offsetof(BevyVisibilityRange, start_margin),
                                                  offsetof(BevyVisibilityRange, end_margin) + sizeof(float),
                                                  offsetof(BevyVisibilityRange, use_aabb)};
    {
        b200vis_table desc[N_TABLES];
        b200vis_table_inputs in[N_TABLES];
        b200vis_table_cull_inputs cull[N_TABLES];
        b200vis_table_visibility_ranges rg[N_TABLES];
        for (int t = 0; t < N_TABLES; ++t) {
            const Table *T = &tab[t];
            desc[t] = (b200vis_table){T->gt, T->gt_ticks, T->vv, T->vv_ticks, T->len, T->capacity};
            in[t] = (b200vis_table_inputs){T->tr, T->tr_ticks};
            memset(&cull[t], 0, sizeof cull[t]);
            cull[t].aabbs = T->aabb; cull[t].aabb_changed_ticks = T->aabb_ticks;
            cull[t].inherited_visibility = T->iv; cull[t].iv_changed_ticks = T->iv_ticks;
            cull[t].flags = (t == RANGED ? B200VIS_F_HAS_VIS_RANGE : 0u) | (t == NO_FC ? B200VIS_F_NO_FRUSTUM_CULLING : 0u);
            rg[t].ranges = T->range; rg[t].changed_ticks = T->range_ticks;
        }
        CHECK(b200vis_set_tables_ex(ctx, N_TABLES, desc, in, &tlay));
        CHECK(b200vis_set_table_cull_inputs(ctx, N_TABLES, cull, &blay));
        CHECK(b200vis_set_table_shadow_casters(ctx, N_TABLES, IS_CASTER));
        CHECK(b200vis_set_table_visibility_ranges(ctx, N_TABLES, rg, &rlay));
        uint32_t *rows = malloc((size_t)n * 4);
        for (int t = 0; t < N_TABLES; ++t) {
            for (uint32_t s = 0; s < tab[t].len; ++s) rows[s] = row_of[tab[t].entities[s]];
            CHECK(b200vis_set_table_rows(ctx, (uint32_t)t, 0, tab[t].len, rows));
        }
        free(rows);
    }

    /* ---- the shadow entity sink: 64 entries for 4 items to start with, so both growth paths run ---- */
    uint32_t sink_cap = 0, sink_items = 0;
    uint64_t *sink_ent = NULL;
    uint32_t *sink_off = NULL;
    uint8_t *sink_act = NULL;
#define SET_SINK(cap_, items_)                                                                                          \
    do {                                                                                                               \
        sink_cap = (cap_); sink_items = (items_);                                                                      \
        sink_ent = malloc((size_t)sink_cap * 8); sink_off = malloc(((size_t)sink_items * 6 + 1) * 4);                  \
        sink_act = malloc(sink_items);                     /* replaced buffers stay alive: the library keeps them mapped */ \
        const b200vis_shadow_entities_sink s_ = {sink_ent, sink_cap, sink_items, sink_off, sink_act};                  \
        CHECK(b200vis_set_shadow_entities_sink(ctx, &s_));                                                             \
    } while (0)
    SET_SINK(64, 4);

    /* ---- the lights' components (what the plugin fills) and the expected contents ---- */
    List *cube = calloc((size_t)n_point * 6, sizeof(List)), *want_cube = calloc((size_t)n_point * 6, sizeof(List));
    List *spot = calloc(n_spot, sizeof(List)), *want_spot = calloc(n_spot, sizeof(List));
    CascadesVisible cascades;
    memset(&cascades, 0, sizeof cascades);
    const uint32_t light_row0 = n_forest;                /* light k is entity n_forest + k: points first, then spots */
    uint8_t *shadows_on = malloc(n_lights);
    for (uint32_t k = 0; k < n_lights; ++k) shadows_on[k] = !(k < n_point && k % 3u == 2u);   /* some point lights: off */
    uint64_t *light_block0 = malloc((size_t)n_lights * 8), (*light_ext)[3] = calloc(n_lights, 24);
    for (uint32_t k = 0; k < n_lights; ++k) light_block0[k] = 1;

    float view_pos[3 * 3] = {0.1f * S, 2.0f, -0.2f * S};  /* the ShadowLodOrigin, then the cameras */
    float *o_gt = calloc((size_t)n * 12, 4);
    for (uint32_t r = 0; r < n; ++r) o_gt[r * 12] = o_gt[r * 12 + 4] = o_gt[r * 12 + 8] = 1.0f;
    uint8_t *o_vv = calloc(n, 1), *o_vvch = calloc(n, 1), *o_gtch = calloc(n, 1), *tchanged = malloc(n), *cam_ch = malloc(n);
    uint8_t *light_ch = malloc(n), *marked = malloc(n), *listed = malloc(n);
    uint32_t *o_mask = malloc((size_t)n * 4), *o_rows = malloc((size_t)V * n * 4), o_count[B200VIS_MAX_VIEWS];
    uint32_t *l_rows = malloc((size_t)MAX_CASC * n * 4), l_count[64];
    uint32_t *want_tick = calloc(n, 4);
    uint64_t *keys = malloc((size_t)n * 8);
    b200vis_shadow_item *items = malloc((size_t)(n_lights + 2 * MAX_CASC) * sizeof(b200vis_shadow_item));
    uint64_t (*items_ext)[3] = calloc(n_lights + 2 * MAX_CASC, 24);
    float *point_frusta = malloc((size_t)n_lights * 144 * 4), *spot_frusta = malloc((size_t)n_lights * 24 * 4);
    float casc_frusta[2][MAX_CASC][6][4];
    memset(tchanged, 1, n);
    int ok = 1;
    uint32_t last_run = 995, grown = 0, inactive_kept = 0, entries = 0, emits = 0;
    double ms_items = 0, ms_sync = 0, ms_fill = 0;
    for (uint32_t frame = 1; frame <= frames && ok; ++frame) {
        const uint32_t cam_tick = 1000u + 10u * frame, light_tick = cam_tick + 2u, mark_tick = cam_tick + 3u;
        /* ---- the game: roots and lights move (Transform written with a tick between the cull system's runs) ---- */
        for (uint32_t e = 0; e < n; ++e) {
            if (child_of[e] != B200VIS_NO_PARENT || (frame == 1)) continue;
            Table *T = &tab[arch[e]];
            const uint32_t s = slot_of[e], r = row_of[e];
            BevyTransform *t = &T->tr[s];
            t->translation[0] += 0.4f * sinf(0.3f * (float)(frame + e));
            if (e == light_row0) t->translation[1] = frame == 3 || frame == 4 ? 50.0f * S : 0.0f;   /* point light 0: out of view */
            T->tr_ticks[s] = cam_tick - 5u;
            const float p[10] = {t->translation[0], t->translation[1], t->translation[2], t->rotation[0], t->rotation[1], t->rotation[2],
                                 t->rotation[3], t->scale[0], t->scale[1], t->scale[2]};
            memcpy(trs + (size_t)r * 10, p, 40);
            tchanged[r] = 1;
        }
        if (frame == 4) { light_block0[n_point] = 0; light_ext[n_point][0] = 1ull << 6; }   /* spot 0: layer 70 only */
        /* ---- reset_view_visibility (CPU, bypassing change detection) ---- */
        for (int t = 0; t < N_TABLES; ++t)
            for (uint32_t s = 0; s < tab[t].len; ++s) tab[t].vv[s] = (uint8_t)((tab[t].vv[s] & 1u) << 1);
        /* ---- the cameras, the range views, the cull ---- */
        b200vis_view views[2];
        float planes[2][6][4];
        uint64_t view_layers[2] = {1, 1};
        uint8_t view_flags[2] = {B200VIS_VIEW_ACTIVE, B200VIS_VIEW_ACTIVE};
        int8_t vri[2] = {1, 2};
        for (uint32_t v = 0; v < V; ++v) {
            const float yaw = 0.15f * (float)frame + 3.1415927f * (float)v, cy = cosf(yaw), sy = sinf(yaw), d = 1.6f * S;
            const float gt[12] = {cy, 0, -sy, 0, 1, 0, sy, 0, cy, d * sy, 0, d * cy};
            float cfv[16];
            b200vis_host_perspective(1.2f, 16.0f / 9.0f, 0.1f, cfv);
            b200vis_host_compute_frustum(cfv, gt, 10.0f * S, planes[v]);
            memcpy(&view_pos[(1 + v) * 3], &gt[9], 12);
            memset(&views[v], 0, sizeof views[v]);
            memcpy(views[v].half_spaces, planes[v], sizeof planes[v]);
            views[v].layer_mask = 1; views[v].flags = B200VIS_VIEW_ACTIVE; views[v].range_view_index = vri[v];
        }
        CHECK(b200vis_set_visibility_range_views(ctx, 3, view_pos));
        CHECK(b200vis_set_views(ctx, V, views));
        CHECK(b200vis_read_tables(ctx, B200VIS_RD_TRANSFORM | B200VIS_RD_CULL_INPUTS, last_run, cam_tick));
        CHECK(b200vis_run(ctx, B200VIS_STAGE_PROPAGATE | B200VIS_STAGE_CULL));
        CHECK(b200vis_writeback_tables(ctx, B200VIS_WB_GLOBAL_TRANSFORM | B200VIS_WB_SET_VISIBLE, cam_tick, cam_tick));
        CHECK(b200vis_synchronize(ctx));
        last_run = cam_tick;
        /* ---- the oracle: propagate, ranges, cull with mark_newly_hidden deferred ---- */
        if (orc_propagate(n, parent, trs, o_gt, tchanged, NULL, 1, o_gtch) != 0) { fprintf(stderr, "oracle propagate failed\n"); return 4; }
        memset(tchanged, 0, n);
        orc_check_visibility_ranges(n, o_gt, bounds, flags, range_se, use_aabb, 3, view_pos, o_mask);
        orc_set_defer_mark_newly_hidden(1);
        orc_cull(n, o_gt, bounds, flags, NULL, o_mask, cls, entity_bits, o_vv, o_vvch, V, &planes[0][0][0], view_layers, view_flags,
                 vri, o_rows, o_count);
        orc_set_defer_mark_newly_hidden(0);
        memcpy(cam_ch, o_vvch, n);
        memset(listed, 0, n);
        for (uint32_t v = 0; v < V; ++v)
            for (uint32_t i = 0; i < o_count[v]; ++i) listed[o_rows[(size_t)v * n + i]] = 1;
        /* the lights' frusta from this frame's GlobalTransforms (update_point_light_frusta / update_spot_light_frusta) */
        for (uint32_t k = 0; k < n_lights; ++k) {
            const float *g = o_gt + (size_t)row_of[light_row0 + k] * 12;
            if (k < n_point) b200vis_host_point_light_frusta(g, light_range, 0.1f, (float (*)[6][4])(point_frusta + (size_t)k * 144));
            else {
                float cfv[16];
                b200vis_host_perspective(1.0f, 1.0f, 0.1f, cfv);
                b200vis_host_compute_frustum(cfv, g, light_range, (float (*)[4])(spot_frusta + (size_t)k * 24));
            }
        }
        uint32_t dv[2], dc[2];
        const uint32_t n_dv = dir_views(frame, dv, dc);
        const int dir_visible = frame != 3;
        for (uint32_t i = 0; i < n_dv; ++i)
            for (uint32_t c = 0; c < dc[i]; ++c) {
                const float h = 0.15f * S * (float)(c + 1), off = (dv[i] ? -0.2f : 0.2f) * S;
                const float lo[3] = {off - h, -h, -h}, hi[3] = {off + h, h, h};
                box_frustum(lo, hi, casc_frusta[i][c]);
            }

        /* ==== b200_check_light_visibility ==== */
        double t0 = now_ms();
        uint32_t n_items = 0, any_ext = 0;
        uint32_t item_light[64];                         /* light k, or 1000 + view slot * 16 + cascade */
        for (uint32_t k = 0; k < n_lights; ++k) {
            if (!shadows_on[k]) continue;
            b200vis_shadow_item *it = &items[n_items];
            memset(it, 0, sizeof *it);
            it->kind = k < n_point ? B200VIS_SHADOW_POINT : B200VIS_SHADOW_SPOT;
            it->light_row = row_of[light_row0 + k]; it->range = light_range; it->range_view_index = 0;
            it->layer_mask = light_block0[k];
            if (k < n_point) memcpy(it->frusta, point_frusta + (size_t)k * 144, 144 * 4);
            else memcpy(it->frusta[0], spot_frusta + (size_t)k * 24, 24 * 4);
            memcpy(items_ext[n_items], light_ext[k], 24);
            any_ext |= (light_ext[k][0] | light_ext[k][1] | light_ext[k][2]) != 0;
            item_light[n_items++] = k;
        }
        if (dir_visible)
            for (uint32_t i = 0; i < n_dv; ++i)
                for (uint32_t c = 0; c < dc[i]; ++c) {
                    b200vis_shadow_item *it = &items[n_items];
                    memset(it, 0, sizeof *it);
                    it->kind = B200VIS_SHADOW_DIRECTIONAL_CASCADE; it->range_view_index = vri[dv[i]]; it->layer_mask = 1;
                    memcpy(it->frusta[0], casc_frusta[i][c], 24 * 4);
                    memset(items_ext[n_items], 0, 24);
                    item_light[n_items++] = 1000u + i * 16u + c;
                }
        if (n_items > sink_items) SET_SINK(sink_cap, n_items > 2 * sink_items ? n_items : 2 * sink_items);
        ms_items += now_ms() - t0;
        CHECK(b200vis_set_shadow_items(ctx, n_items, items, 1));
        if (any_ext) CHECK(b200vis_set_shadow_item_render_layers_ext(ctx, n_items, &items_ext[0][0]));
        CHECK(b200vis_run_shadow_culling(ctx));
        CHECK(b200vis_writeback_tables(ctx, B200VIS_WB_SET_VISIBLE, 0, light_tick));
        t0 = now_ms();
        CHECK(b200vis_synchronize(ctx));
        ms_sync += now_ms() - t0;
        uint32_t total = sink_off[n_items * 6];
        if (total > sink_cap) {
            SET_SINK(total > 2 * sink_cap ? total : 2 * sink_cap, sink_items);
            CHECK(b200vis_emit_shadow_entities(ctx));
            t0 = now_ms();
            CHECK(b200vis_synchronize(ctx));
            ms_sync += now_ms() - t0;
            ++emits;
        }
        t0 = now_ms();
        for (uint32_t i = 0; i < n_items; ++i) {          /* active items only; an inactive light keeps its lists */
            if (!sink_act[i] || item_light[i] >= 1000u) continue;
            const uint32_t k = item_light[i];
            if (k < n_point)
                for (uint32_t f = 0; f < 6; ++f) list_set(&cube[k * 6 + f], sink_ent + sink_off[i * 6 + f], sink_off[i * 6 + f + 1] - sink_off[i * 6 + f]);
            else list_set(&spot[k - n_point], sink_ent + sink_off[i * 6], sink_off[i * 6 + 1] - sink_off[i * 6]);
        }
        {   /* CascadesVisibleEntities: resize / drop / add views, clear when invisible, replace each cascade's list */
            CascadesVisible *cv = &cascades;
            for (uint32_t j = 0; j < cv->n_views;) {
                uint32_t i = 0;
                while (i < n_dv && dv[i] != cv->view[j]) ++i;
                if (i == n_dv) {                          /* the view left CascadesFrusta */
                    for (uint32_t c = 0; c < MAX_CASC; ++c) cv->lists[j][c].n = 0;
                    cv->view[j] = cv->view[cv->n_views - 1]; cv->n_casc[j] = cv->n_casc[cv->n_views - 1];
                    memcpy(cv->lists[j], cv->lists[cv->n_views - 1], sizeof cv->lists[j]);
                    memset(cv->lists[cv->n_views - 1], 0, sizeof cv->lists[j]);
                    --cv->n_views;
                    continue;
                }
                for (uint32_t c = dc[i]; c < cv->n_casc[j]; ++c) cv->lists[j][c].n = 0;
                cv->n_casc[j] = dc[i];
                ++j;
            }
            for (uint32_t i = 0; i < n_dv; ++i) {
                uint32_t j = 0;
                while (j < cv->n_views && cv->view[j] != dv[i]) ++j;
                if (j == cv->n_views) { cv->view[j] = dv[i]; cv->n_casc[j] = dc[i]; cv->n_views++; }
            }
            if (!dir_visible) { for (uint32_t j = 0; j < cv->n_views; ++j) for (uint32_t c = 0; c < MAX_CASC; ++c) cv->lists[j][c].n = 0; cv->n_views = 0; }
            for (uint32_t i = 0; i < n_items; ++i) {
                if (item_light[i] < 1000u) continue;
                const uint32_t vs = (item_light[i] - 1000u) / 16u, c = (item_light[i] - 1000u) % 16u;
                uint32_t j = 0;
                while (j < cv->n_views && cv->view[j] != dv[vs]) ++j;
                list_set(&cv->lists[j][c], sink_ent + sink_off[i * 6], sink_off[i * 6 + 1] - sink_off[i * 6]);
            }
        }
        ms_fill += now_ms() - t0;
        entries += total;
        /* ==== mark_newly_hidden_entities_invisible (CPU, on the table bytes) ==== */
        for (int t = 0; t < N_TABLES; ++t)
            for (uint32_t s = 0; s < tab[t].len; ++s)
                if ((tab[t].vv[s] & 3u) == 2u) { tab[t].vv[s] = 0; tab[t].vv_ticks[s] = mark_tick; }

        /* ---- the oracle's light passes (directional, then point and spot lights in some view), then mark ---- */
        if (dir_visible && n_dv) {
            int32_t dvri[2]; uint64_t dl[2] = {1, 1};
            float fr[2 * MAX_CASC * 24];
            uint32_t m = 0;
            for (uint32_t i = 0; i < n_dv; ++i) { dvri[i] = vri[dv[i]]; for (uint32_t c = 0; c < dc[i]; ++c) memcpy(fr + (size_t)(m++) * 24, casc_frusta[i][c], 96); }
            orc_check_dir_light_mesh_visibility(n, o_gt, bounds, flags, caster, NULL, o_mask, entity_bits, o_vv, o_vvch, n_dv, dvri, dl, dc, fr,
                                                l_rows, l_count);
            for (uint32_t i = 0, q = 0; i < n_dv; ++i)
                for (uint32_t c = 0; c < dc[i]; ++c, ++q) {
                    for (uint32_t x = 0; x < l_count[q]; ++x) keys[x] = entity_bits[l_rows[(size_t)q * n + x]];
                    uint32_t j = 0;
                    while (j < cascades.n_views && cascades.view[j] != dv[i]) ++j;
                    const List *got = j < cascades.n_views ? &cascades.lists[j][c] : NULL;
                    if (!got || got->n != l_count[q] || (l_count[q] && memcmp(got->e, keys, (size_t)l_count[q] * 8))) {
                        fprintf(stderr, "frame %u: cascade list (view %u, cascade %u) differs (%u vs %u entries)\n", frame, dv[i], c,
                                got ? got->n : 0u, l_count[q]);
                        ok = 0;
                    }
                }
        }
        {   /* the CascadesVisibleEntities keys */
            const uint32_t want_views = dir_visible ? n_dv : 0;
            int keys_ok = cascades.n_views == want_views;
            for (uint32_t i = 0; i < want_views && keys_ok; ++i) {
                uint32_t j = 0;
                while (j < cascades.n_views && cascades.view[j] != dv[i]) ++j;
                keys_ok = j < cascades.n_views && cascades.n_casc[j] == dc[i];
            }
            if (!keys_ok) { fprintf(stderr, "frame %u: CascadesVisibleEntities keys differ\n", frame); ok = 0; }
        }
        for (uint32_t k = 0; k < n_lights; ++k) {
            const uint32_t lr = row_of[light_row0 + k];
            if (!shadows_on[k] || !listed[lr]) { inactive_kept += shadows_on[k] && frame > 1; continue; }
            const float *g = o_gt + (size_t)lr * 12;
            const float sphere[4] = {g[9], g[10], g[11], light_range};
            const uint64_t ll = light_block0[k];
            if (k < n_point) {
                orc_check_point_light_mesh_visibility(n, o_gt, bounds, flags, caster, NULL, o_mask, 0, entity_bits, o_vv, o_vvch, 1, sphere, &ll,
                                                      point_frusta + (size_t)k * 144, l_rows, l_count);
                for (uint32_t f = 0; f < 6; ++f) {
                    for (uint32_t x = 0; x < l_count[f]; ++x) keys[x] = entity_bits[l_rows[(size_t)f * n + x]];
                    list_set(&want_cube[k * 6 + f], keys, l_count[f]);
                }
            } else {
                orc_check_spot_light_mesh_visibility(n, o_gt, bounds, flags, caster, NULL, o_mask, 0, entity_bits, o_vv, o_vvch, 1, sphere, &ll,
                                                     spot_frusta + (size_t)k * 24, l_rows, l_count);
                for (uint32_t x = 0; x < l_count[0]; ++x) keys[x] = entity_bits[l_rows[x]];
                list_set(&want_spot[k - n_point], keys, l_count[0]);
            }
        }
        for (uint32_t r = 0; r < n; ++r) { light_ch[r] = o_vvch[r] && !cam_ch[r]; marked[r] = (o_vv[r] & 3u) == 2u; }
        orc_mark_newly_hidden(n, flags, o_vv, o_vvch);
        /* ---- compare: every list of every component, every ViewVisibility byte and its tick ---- */
        for (uint32_t l = 0; l < n_point * 6; ++l)
            if (cube[l].n != want_cube[l].n || (cube[l].n && memcmp(cube[l].e, want_cube[l].e, (size_t)cube[l].n * 8))) {
                fprintf(stderr, "frame %u: point light %u face %u: %u entries vs the oracle's %u\n", frame, l / 6, l % 6, cube[l].n, want_cube[l].n);
                ok = 0;
            }
        for (uint32_t k = 0; k < n_spot; ++k)
            if (spot[k].n != want_spot[k].n || (spot[k].n && memcmp(spot[k].e, want_spot[k].e, (size_t)spot[k].n * 8))) {
                fprintf(stderr, "frame %u: spot light %u: %u entries vs the oracle's %u\n", frame, k, spot[k].n, want_spot[k].n);
                ok = 0;
            }
        uint32_t bad = 0, light_only = 0;
        for (uint32_t e = 0; e < n; ++e) {
            const uint32_t r = row_of[e];
            const Table *T = &tab[arch[e]];
            const uint32_t s = slot_of[e];
            if (cam_ch[r]) want_tick[r] = cam_tick;
            else if (light_ch[r]) { want_tick[r] = light_tick; ++light_only; }
            else if (marked[r]) want_tick[r] = mark_tick;
            if ((T->vv[s] != o_vv[r] || T->vv_ticks[s] != want_tick[r]) && bad++ < 4)
                fprintf(stderr, "frame %u entity %u: ViewVisibility %u tick %u vs the oracle's %u tick %u\n", frame, e, T->vv[s], T->vv_ticks[s],
                        o_vv[r], want_tick[r]);
        }
        ok &= bad == 0;
        grown += emits;
        printf("frame %u: %u items, %u entries, %u rows made visible by lights alone, sink %u entries: %s\n", frame, n_items, total, light_only,
               sink_cap, ok ? "OK" : "MISMATCH");
        emits = 0;
        if (frame == 1 || frame == 3) SET_SINK(64, sink_items);   /* frames 2 and 4 start from a 64-entry sink again */
    }
    FILE *p = popen("nvidia-smi --query-gpu=name,power.limit --format=csv,noheader 2>/dev/null", "r");
    char card[256] = "unknown";
    if (p) { if (!fgets(card, sizeof card, p)) strcpy(card, "unknown"); pclose(p); }
    card[strcspn(card, "\n")] = 0;
    printf("{\"metric\": \"light_shim\", \"card\": \"%s\", \"entities\": %u, \"point\": %u, \"spot\": %u, \"cascades\": \"1 x 2 x 4\", "
           "\"frames\": %u, \"entries\": %u, \"grown\": %u, \"inactive_kept\": %u, \"host_ms_per_frame\": {\"build_items\": %.4f, "
           "\"synchronize\": %.4f, \"fill_lists\": %.4f}}\n",
           card, n, n_point, n_spot, frames, entries, grown, inactive_kept, ms_items / frames, ms_sync / frames, ms_fill / frames);
    CHECK(b200vis_set_shadow_entities_sink(ctx, NULL));
    CHECK(b200vis_set_tables(ctx, 0, NULL));
    b200vis_destroy(ctx);
    printf(ok ? "LIGHT_SHIM OK\n" : "LIGHT_SHIM FAILED\n");
    return ok ? 0 : 1;
}
