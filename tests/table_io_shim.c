/*
 * table_io_shim.c -- a whole frame through include/b200vis.h in plain C with no per-entity host work in either direction:
 * the GPU reads Transform and other systems' GlobalTransforms straight from Bevy-native archetype tables, and writes
 * GlobalTransform, ViewVisibility and both changed_ticks columns back into them.
 *
 * The "ECS": a forest of complete binary trees plus point lights, spawned level by level across all trees, then the lights.
 * Four archetype tables -- roots, inner nodes, leaves, lights -- hold their entities in spawn order, with Bevy's layouts:
 *     Transform        48 B  { rotation: Quat, translation: Vec3, scale: Vec3 } (rustc puts the 16-byte aligned Quat
 *                            first), changed_ticks 4 B
 *     GlobalTransform  64 B  glam Affine3A, changed_ticks 4 B
 *     ViewVisibility    1 B, changed_ticks 4 B
 * Per frame, with the propagate system's (last_run, this_run):
 *   - a "game system" moves every root by writing its Transform and stamping the tick, and rewrites every other
 *     Transform with bypass_change_detection (bytes the device must not pick up, tick untouched);
 *   - a "physics system" writes the GlobalTransform of a few leaves and stamps their ticks;
 *   - b200vis_read_tables(RD_TRANSFORM | RD_GLOBAL_TRANSFORM, last_run, this_run), b200vis_step with no changed rows,
 *     b200vis_writeback_tables(this_run), one b200vis_synchronize.
 * Every slot is checked against the CPU oracle (oracle/libbevy_oracle.so, orc_propagate with tchanged / gt_ext_changed).
 *
 * Build (tests/test_table_io_shim.py does this): gcc -O2 -std=gnu11 -Wall -Wextra -Werror -Iinclude tests/table_io_shim.c
 *        -Lbevy_b200 -lb200vis -Loracle -lbevy_oracle -lm ; run: ./table_io_shim [n_trees] [levels] [frames], or
 *        ./table_io_shim --sizeof to print the layouts of b200vis_transform_layout and b200vis_table_inputs (no GPU needed).
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

typedef struct { float rotation[4], translation[3], scale[3], pad[2]; } BevyTransform;   /* 48 B */
typedef struct { float m[16]; } BevyGlobalTransform;                                      /* 64 B */
enum { ROOTS, INNER, LEAVES, LIGHTS, N_TABLES };
typedef struct {
    BevyTransform *transform; uint32_t *t_ticks;
    BevyGlobalTransform *global; uint32_t *gt_ticks;
    uint8_t *view_visibility; uint32_t *vv_ticks;
    uint32_t *entities;                                 /* Table::entities */
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
static void to_bevy(const float *t10, BevyTransform *b) {   /* packed translation.xyz, rotation.xyzw, scale.xyz */
    memset(b, 0, sizeof *b);
    memcpy(b->translation, t10, 12); memcpy(b->rotation, t10 + 3, 16); memcpy(b->scale, t10 + 7, 12);
}

int main(int argc, char **argv) {
    if (argc > 1 && strcmp(argv[1], "--sizeof") == 0) {
        printf("{\"layout\": {\"sizeof\": %zu, \"stride\": %zu, \"translation\": %zu, \"rotation\": %zu, \"scale\": %zu}, "
               "\"inputs\": {\"sizeof\": %zu, \"transforms\": %zu, \"transform_changed_ticks\": %zu}}\n",
               sizeof(b200vis_transform_layout), offsetof(b200vis_transform_layout, stride),
               offsetof(b200vis_transform_layout, translation), offsetof(b200vis_transform_layout, rotation),
               offsetof(b200vis_transform_layout, scale), sizeof(b200vis_table_inputs),
               offsetof(b200vis_table_inputs, transforms), offsetof(b200vis_table_inputs, transform_changed_ticks));
        return 0;
    }
    const uint32_t n_trees = argc > 1 ? (uint32_t)atoi(argv[1]) : 200, levels = argc > 2 ? (uint32_t)atoi(argv[2]) : 6;
    const uint32_t frames = argc > 3 ? (uint32_t)atoi(argv[3]) : 4, n_lights = 48, V = 2;
    const uint32_t per = (1u << levels) - 1, n_mesh = n_trees * per, n = n_mesh + n_lights;
    b200vis_ctx *ctx = NULL;

    /* ---- spawn: level by level across the trees, then the lights ---- */
    uint32_t *child_of = malloc((size_t)n * 4), *node_entity = malloc((size_t)n_mesh * 4);
    for (uint32_t e = 0, lvl = 0; lvl < levels; ++lvl)
        for (uint32_t tr = 0; tr < n_trees; ++tr)
            for (uint32_t k = (1u << lvl) - 1; k < (2u << lvl) - 1; ++k) node_entity[tr * per + k] = e++;
    for (uint32_t tr = 0; tr < n_trees; ++tr)
        for (uint32_t k = 0; k < per; ++k)
            child_of[node_entity[tr * per + k]] = k ? node_entity[tr * per + (k - 1) / 2] : B200VIS_NO_PARENT;
    for (uint32_t e = n_mesh; e < n; ++e) child_of[e] = B200VIS_NO_PARENT;
    float *trs_e = malloc((size_t)n * 40), *bounds_e = malloc((size_t)n * 24);
    uint8_t *flags_e = malloc(n);
    for (uint32_t e = 0; e < n; ++e) {
        float *t = trs_e + (size_t)e * 10, *b = bounds_e + (size_t)e * 6;
        const int light = e >= n_mesh, root = !light && child_of[e] == B200VIS_NO_PARENT;
        float q[4] = {frand(-1, 1), frand(-1, 1), frand(-1, 1), frand(-1, 1)};
        const float qn = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
        const float spread = (light || root) ? 200.0f : 2.0f;
        for (int i = 0; i < 3; ++i) { t[i] = frand(-spread, spread); t[7 + i] = light ? 1.0f : frand(0.5f, 1.5f); }
        for (int i = 0; i < 4; ++i) t[3 + i] = light ? (float)(i == 3) : q[i] / qn;
        memset(b, 0, 24);
        if (light) { b[3] = frand(5.0f, 40.0f); flags_e[e] = B200VIS_F_INHERITED_VISIBLE | B200VIS_F_HAS_SPHERE | B200VIS_F_SPHERE_FROM_GT; }
        else { for (int i = 3; i < 6; ++i) b[i] = frand(0.25f, 0.75f); flags_e[e] = B200VIS_F_INHERITED_VISIBLE | B200VIS_F_HAS_AABB; }
    }
    /* ---- the archetype tables, each in spawn order; spawn ticks = the first frame's last_run (not newer) ---- */
    const uint32_t tick0 = 1000;
    uint8_t *has_kids = calloc(n, 1), *arch = malloc(n);
    for (uint32_t e = 0; e < n; ++e) if (child_of[e] != B200VIS_NO_PARENT) has_kids[child_of[e]] = 1;
    Table tab[N_TABLES];
    memset(tab, 0, sizeof tab);
    for (uint32_t e = 0; e < n; ++e) {
        arch[e] = e >= n_mesh ? LIGHTS : child_of[e] == B200VIS_NO_PARENT ? ROOTS : has_kids[e] ? INNER : LEAVES;
        tab[arch[e]].len++;
    }
    for (int t = 0; t < N_TABLES; ++t) {
        uint32_t cap = 1;
        while (cap < tab[t].len) cap *= 2;
        tab[t].capacity = cap;
        tab[t].transform = aligned_alloc(64, (size_t)cap * sizeof(BevyTransform));
        tab[t].global = aligned_alloc(64, (size_t)cap * 64);   /* plain heap memory: the library registers it */
        tab[t].t_ticks = malloc((size_t)cap * 4); tab[t].gt_ticks = malloc((size_t)cap * 4);
        tab[t].view_visibility = malloc(cap); tab[t].vv_ticks = malloc((size_t)cap * 4);
        tab[t].entities = malloc((size_t)cap * 4);
        memset(tab[t].transform, 0xAB, (size_t)cap * sizeof(BevyTransform)); memset(tab[t].t_ticks, 0xAB, (size_t)cap * 4);
        memset(tab[t].global, 0xAB, (size_t)cap * 64); memset(tab[t].gt_ticks, 0xAB, (size_t)cap * 4);
        memset(tab[t].view_visibility, 0xAB, cap); memset(tab[t].vv_ticks, 0xAB, (size_t)cap * 4);
        tab[t].len = 0;
    }
    for (uint32_t e = 0; e < n; ++e) {
        Table *T = &tab[arch[e]];
        const uint32_t s = T->len++;
        to_bevy(trs_e + (size_t)e * 10, &T->transform[s]);
        memset(&T->global[s], 0, 64);
        T->global[s].m[0] = T->global[s].m[5] = T->global[s].m[10] = 1.0f;
        T->t_ticks[s] = T->gt_ticks[s] = tick0; T->view_visibility[s] = 0; T->vv_ticks[s] = tick0;
        T->entities[s] = e;
    }

    /* ---- device rows: the planned order (the rebuild path: every column uploaded once) ---- */
    uint32_t *new_to_old = malloc((size_t)n * 4), *row_of = malloc((size_t)n * 4);
    if (b200vis_plan_row_order(n, child_of, new_to_old) != B200VIS_OK) { fprintf(stderr, "plan_row_order failed\n"); return 2; }
    for (uint32_t r = 0; r < n; ++r) row_of[new_to_old[r]] = r;
    uint32_t *parent = malloc((size_t)n * 4);
    uint64_t *entity_bits = malloc((size_t)n * 8);
    float *trs = malloc((size_t)n * 40), *bounds = malloc((size_t)n * 24);
    uint8_t *flags = malloc(n), *cls = malloc(n);
    for (uint32_t r = 0; r < n; ++r) {
        const uint32_t e = new_to_old[r];
        parent[r] = child_of[e] == B200VIS_NO_PARENT ? B200VIS_NO_PARENT : row_of[child_of[e]];
        entity_bits[r] = e;
        memcpy(trs + (size_t)r * 10, trs_e + (size_t)e * 10, 40); memcpy(bounds + (size_t)r * 6, bounds_e + (size_t)e * 6, 24);
        flags[r] = flags_e[e]; cls[r] = 1;
    }
    b200vis_config cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.max_entities = n; cfg.max_lights = n_lights; cfg.max_views = V;
    if (b200vis_create(&cfg, &ctx) != B200VIS_OK) { fprintf(stderr, "b200vis_create: %s\n", b200vis_last_error(NULL)); return 3; }
    CHECK(b200vis_set_topology(ctx, n, parent, entity_bits));
    CHECK(b200vis_upload_transforms(ctx, 0, n, trs));
    {
        float *gt12 = calloc((size_t)n * 12, 4);
        for (uint32_t r = 0; r < n; ++r) gt12[r * 12] = gt12[r * 12 + 4] = gt12[r * 12 + 8] = 1.0f;
        CHECK(b200vis_upload_global_transforms(ctx, 0, n, gt12));
        free(gt12);
    }
    CHECK(b200vis_upload_bounds(ctx, 0, n, bounds, flags, cls, NULL, NULL));
    uint8_t *zeros = calloc(n, 1);
    CHECK(b200vis_upload_view_visibility(ctx, 0, n, zeros));
    uint32_t light_row[48];
    float light_range[48];
    for (uint32_t i = 0; i < n_lights; ++i) { light_row[i] = row_of[n_mesh + i]; light_range[i] = bounds_e[(size_t)(n_mesh + i) * 6 + 3]; }
    CHECK(b200vis_set_lights(ctx, n_lights, light_row, light_range, NULL));
    /* ---- register the tables with their input columns, and the slot -> row maps ---- */
    b200vis_table desc[N_TABLES];
    b200vis_table_inputs in[N_TABLES];
    const b200vis_transform_layout layout = {sizeof(BevyTransform), offsetof(BevyTransform, translation),
                                             offsetof(BevyTransform, rotation), offsetof(BevyTransform, scale)};
    for (int t = 0; t < N_TABLES; ++t) {
        desc[t].global_transforms = tab[t].global; desc[t].gt_changed_ticks = tab[t].gt_ticks;
        desc[t].view_visibility = tab[t].view_visibility; desc[t].vv_changed_ticks = tab[t].vv_ticks;
        desc[t].len = tab[t].len; desc[t].capacity = tab[t].capacity;
        in[t].transforms = tab[t].transform; in[t].transform_changed_ticks = tab[t].t_ticks;
    }
    CHECK(b200vis_set_tables_ex(ctx, N_TABLES, desc, in, &layout));
    uint32_t *slot_rows = malloc((size_t)n * 4);
    for (int t = 0; t < N_TABLES; ++t) {
        for (uint32_t s = 0; s < tab[t].len; ++s) slot_rows[s] = row_of[tab[t].entities[s]];
        CHECK(b200vis_set_table_rows(ctx, (uint32_t)t, 0, tab[t].len, slot_rows));
    }
    b200vis_cluster_config ccfg;
    b200vis_host_default_cluster_config(&ccfg, 1920, 1080);

    /* ---- oracle (row order) ---- */
    float *o_gt = calloc((size_t)n * 12, 4);
    for (uint32_t r = 0; r < n; ++r) o_gt[r * 12] = o_gt[r * 12 + 4] = o_gt[r * 12 + 8] = 1.0f;
    uint8_t *o_vv = calloc(n, 1), *o_vvch = calloc(n, 1), *o_gtch = calloc(n, 1), *tchanged = malloc(n), *ext = calloc(n, 1);
    uint32_t *o_rows = malloc((size_t)V * n * 4), o_count[B200VIS_MAX_VIEWS];
    memset(tchanged, 1, n);                              /* the first frame: Added<GlobalTransform> everywhere */
    CHECK(b200vis_mark_transforms_changed(ctx, 0, n));
    int ok = 1;
    uint32_t last_run = tick0;
    for (uint32_t frame = 1; frame <= frames && ok; ++frame) {
        const uint32_t this_run = tick0 + 10u * frame;
        uint32_t moved = 0, written = 0;
        if (frame > 1) {
            /* the game system: every root moves (tick stamped), every other Transform rewritten without a tick */
            for (int t = 0; t < N_TABLES; ++t)
                for (uint32_t s = 0; s < tab[t].len; ++s) {
                    const uint32_t e = tab[t].entities[s], r = row_of[e];
                    float *t10 = trs + (size_t)r * 10;
                    if (t == ROOTS) {
                        t10[2] += 0.02f * sinf(0.001f * (float)(frame + s));
                        to_bevy(t10, &tab[t].transform[s]);
                        tab[t].t_ticks[s] = this_run - 5u;
                        tchanged[r] = 1; ++moved;
                    } else {
                        float junk[10];
                        for (int i = 0; i < 10; ++i) junk[i] = t10[i] + 100.0f;
                        to_bevy(junk, &tab[t].transform[s]);
                    }
                }
            /* the physics system: the GlobalTransform of every 97th leaf */
            for (uint32_t s = frame % 97u; s < tab[LEAVES].len; s += 97u) {
                const uint32_t r = row_of[tab[LEAVES].entities[s]];
                float *g = o_gt + (size_t)r * 12, *m = tab[LEAVES].global[s].m;
                for (int i = 0; i < 12; ++i) g[i] += frand(-0.5f, 0.5f);
                if (s % 2u) g[4] = -0.0f;
                for (int k = 0; k < 4; ++k) { for (int i = 0; i < 3; ++i) m[4 * k + i] = g[3 * k + i]; m[4 * k + 3] = 0.0f; }
                tab[LEAVES].gt_ticks[s] = this_run - 3u;
                ext[r] = 1; ++written;
            }
        }
        b200vis_camera cam[2];
        float planes[2][6][4];
        uint64_t view_layers[2] = {1, 1};
        uint8_t view_flags[2] = {B200VIS_VIEW_ACTIVE, B200VIS_VIEW_ACTIVE};
        for (uint32_t v = 0; v < V; ++v) {
            memset(&cam[v], 0, sizeof cam[v]);
            const float yaw = 0.01f * (float)frame + 1.5707963f * (float)v, cy = cosf(yaw), sy = sinf(yaw);
            const float gt[12] = {cy, 0, -sy, 0, 1, 0, sy, 0, cy, 0, 0, 0};
            memcpy(cam[v].global_transform, gt, sizeof gt);
            cam[v].fov_y = 0.78539816f; cam[v].aspect = 16.0f / 9.0f; cam[v].near_z = 0.1f; cam[v].far_z = 1000.0f;
            cam[v].layer_mask = 1; cam[v].flags = B200VIS_VIEW_ACTIVE; cam[v].range_view_index = -1;
            float cfv[16];
            b200vis_host_perspective(cam[v].fov_y, cam[v].aspect, cam[v].near_z, cfv);
            b200vis_host_compute_frustum(cfv, gt, cam[v].far_z, planes[v]);
        }
        /* the frame: no entity loop on the host in either direction */
        CHECK(b200vis_read_tables(ctx, B200VIS_RD_TRANSFORM | B200VIS_RD_GLOBAL_TRANSFORM, last_run, this_run));
        CHECK(b200vis_step(ctx, 0, NULL, NULL, V, cam, &ccfg, 0));
        CHECK(b200vis_writeback_tables(ctx, B200VIS_WB_GLOBAL_TRANSFORM | B200VIS_WB_VIEW_VISIBILITY, this_run, this_run));
        CHECK(b200vis_synchronize(ctx));
        last_run = this_run;
        /* ---- check against the oracle, through the tables only ---- */
        if (orc_propagate(n, parent, trs, o_gt, tchanged, ext, 1, o_gtch) != 0) { fprintf(stderr, "oracle propagate failed\n"); return 4; }
        orc_cull(n, o_gt, bounds, flags, NULL, NULL, cls, entity_bits, o_vv, o_vvch, V, &planes[0][0][0], view_layers, view_flags, NULL,
                 o_rows, o_count);
        uint32_t gt_changed = 0;
        for (int t = 0; t < N_TABLES && ok; ++t) {
            const Table *T = &tab[t];
            for (uint32_t s = 0; s < T->len && ok; ++s) {
                const uint32_t r = row_of[T->entities[s]];
                const float *g = o_gt + (size_t)r * 12;
                const float want[16] = {g[0], g[1], g[2], 0, g[3], g[4], g[5], 0, g[6], g[7], g[8], 0, g[9], g[10], g[11], 0};
                if (memcmp(want, T->global[s].m, 64) != 0) { fprintf(stderr, "frame %u table %d slot %u: GlobalTransform differs\n", frame, t, s); ok = 0; }
                if ((T->gt_ticks[s] == this_run) != (o_gtch[r] != 0)) { fprintf(stderr, "frame %u table %d slot %u: Changed<GlobalTransform>\n", frame, t, s); ok = 0; }
                if (T->view_visibility[s] != o_vv[r]) { fprintf(stderr, "frame %u table %d slot %u: ViewVisibility %u vs %u\n", frame, t, s, T->view_visibility[s], o_vv[r]); ok = 0; }
                if ((T->vv_ticks[s] == this_run) != (o_vvch[r] != 0)) { fprintf(stderr, "frame %u table %d slot %u: Changed<ViewVisibility>\n", frame, t, s); ok = 0; }
                gt_changed += T->gt_ticks[s] == this_run;
            }
        }
        memset(tchanged, 0, n); memset(ext, 0, n);
        printf("frame %u: %u Transforms and %u GlobalTransforms written by other systems, %u GlobalTransforms stamped: %s\n",
               frame, moved, written, gt_changed, ok ? "OK" : "MISMATCH");
    }
    printf("{\"entities\": %u}\n", n);
    CHECK(b200vis_set_tables(ctx, 0, NULL));
    b200vis_destroy(ctx);
    printf(ok ? "TABLE_IO_SHIM OK\n" : "TABLE_IO_SHIM FAILED\n");
    return ok ? 0 : 1;
}
