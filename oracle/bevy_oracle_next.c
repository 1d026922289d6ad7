/*
 * bevy_oracle_next.c -- CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT CODE), SURVEY.md section 8(f) rows
 *
 * Plain-C restatements of the systems either side of the propagate -> cull -> cluster path
 * (bevyengine/bevy 0.20.0-dev) that the CUDA library also covers:
 *   N1  RenderVisibleEntitiesClass::update_cpu_culled_entities / collect_visible_cpu_culled_entities_for_subview
 *       crates/bevy_render/src/view/visibility/mod.rs:194-249, 395-430
 *   N2  extract_clusters_for_cpu_clustering / prepare_clusters_for_cpu_clustering / ViewClusterBindings packing
 *       crates/bevy_pbr/src/cluster/mod.rs:394-582, 584-800, 855-859
 *   N4  check_visibility_ranges        crates/bevy_camera/src/visibility/range.rs:230-284
 *       visibility_propagate_system    crates/bevy_camera/src/visibility/mod.rs:638-729
 * Same rules as bevy_oracle.c: only tests/, __graft_entry__.smoke() and bench.py's CPU legs may load this.
 *
 * PINNING STATUS
 *   N1: pinned by cpu_visible_entity_pair_lookup_uses_main_entity_sort_order (view/visibility/mod.rs:436-481).
 *   N4 visibility_propagate_system: pinned by the InheritedVisibility truth tables and the change-detection
 *       sequence (visibility/mod.rs:950-1282).
 *   N2 and check_visibility_ranges: the reference holds no test with literal answers -> "parity unpinned";
 *       they are integer packing / one distance compare and are cross-checked against independent numpy
 *       restatements in tests/test_oracle_next.py.
 * Floating point model: as bevy_oracle.c (binary32, no FMA contraction, glam SSE2 operation order).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------------------ */
/* N1: render-world visible-entity diff                                                                    */
/* ------------------------------------------------------------------------------------------------------ */
typedef struct { uint64_t render, main; } pair_t;
static int cmp_pair_main(const void *a, const void *b) {
    const uint64_t x = ((const pair_t *)a)->main, y = ((const pair_t *)b)->main;
    return x < y ? -1 : x > y;
}
/* render_view_entities.entities.sort_unstable_by_key(|(_, main_entity)| *main_entity)  (mod.rs:425-427).
 * MainEntity orders like Entity, i.e. by Entity::to_bits(). */
ORC_API void orc_sort_pairs_by_main(uint64_t *render, uint64_t *main_bits, uint32_t n) {
    pair_t *p = (pair_t *)malloc((size_t)(n ? n : 1) * sizeof *p);
    for (uint32_t i = 0; i < n; ++i) { p[i].render = render[i]; p[i].main = main_bits[i]; }
    qsort(p, n, sizeof *p, cmp_pair_main);
    for (uint32_t i = 0; i < n; ++i) { render[i] = p[i].render; main_bits[i] = p[i].main; }
    free(p);
}
/* update_cpu_culled_entities (mod.rs:194-249): lock-step march over the old and the new sorted list.
 * Outputs: added (new \ old) and removed (old \ new), both in list order; the new list becomes
 * entities_cpu_culling (the caller keeps it). */
ORC_API void orc_update_cpu_culled_entities(const uint64_t *old_render, const uint64_t *old_main, uint32_t n_old,
                                            const uint64_t *new_render, const uint64_t *new_main, uint32_t n_new,
                                            uint64_t *added_render, uint64_t *added_main, uint32_t *n_added,
                                            uint64_t *removed_render, uint64_t *removed_main, uint32_t *n_removed) {
    uint32_t io = 0, na = 0, nr = 0;
    for (uint32_t i = 0; i < n_new; ++i) {
        /* mark entities as removed until we see the one we are looking at (:213-219) */
        while (io < n_old && old_main[io] < new_main[i]) {
            removed_render[nr] = old_render[io]; removed_main[nr] = old_main[io]; ++nr; ++io;
        }
        /* same entity at the head of the old list: still visible; otherwise newly visible (:227-236) */
        if (io < n_old && old_main[io] == new_main[i]) ++io;
        else { added_render[na] = new_render[i]; added_main[na] = new_main[i]; ++na; }
    }
    /* whatever is left in the old list was not seen: removed (:240-247) */
    while (io < n_old) { removed_render[nr] = old_render[io]; removed_main[nr] = old_main[io]; ++nr; ++io; }
    *n_added = na; *n_removed = nr;
}
/* entity_pair_is_visible, CPU-culled half (mod.rs:271-282): binary search by main entity, then compare render entity */
ORC_API int orc_entity_pair_is_visible(const uint64_t *render, const uint64_t *main_bits, uint32_t n, uint64_t entity,
                                       uint64_t main_entity) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) { const uint32_t mid = lo + (hi - lo) / 2; if (main_bits[mid] < main_entity) lo = mid + 1; else hi = mid; }
    return lo < n && main_bits[lo] == main_entity && render[lo] == entity;
}

/* ------------------------------------------------------------------------------------------------------ */
/* N2: Clusters -> ViewClusterBindings wire format (point lights)                                          */
/* ------------------------------------------------------------------------------------------------------ */
#define VCB_MAX_OFFSETS (16384 / 4)                 /* cluster/mod.rs:585 */
#define VCB_MAX_UNIFORM_ITEMS (VCB_MAX_OFFSETS / 4) /* :586 */
#define VCB_MAX_INDICES 16384                       /* :587 */
#define CLUSTER_COUNT_SIZE 9u                       /* :43 */
#define CLUSTER_OFFSET_MASK ((1u << (32u - CLUSTER_COUNT_SIZE * 2u)) - 1u) /* :45 */
#define CLUSTER_COUNT_MASK ((1u << CLUSTER_COUNT_SIZE) - 1u)               /* :46 */
static uint32_t pack_offset_and_counts(size_t offset, uint32_t point_count, uint32_t spot_count) { /* :855-859 */
    return (((uint32_t)offset & CLUSTER_OFFSET_MASK) << (CLUSTER_COUNT_SIZE * 2u)) |
           ((point_count & CLUSTER_COUNT_MASK) << CLUSTER_COUNT_SIZE) | (spot_count & CLUSTER_COUNT_MASK);
}
/* Input: one view's Clusters in CSR form (cluster c holds light ordinals indices[offsets[c] .. offsets[c+1])), in
 * the reference's push order), gpu_index_of_light = GlobalClusterableObjectMeta::entity_to_index for the ordinals
 * 0 .. n_map-1 (NULL = identity); an ordinal with no entry gets push_dummy_index's !0 (:527-533).  The record
 * stream of extract_clusters_for_cpu_clustering (:419-470) is ClusterHeader(counts), Light(e)...;
 * prepare_clusters_for_cpu_clustering (:494-520) consumes it.
 * storage != 0: offsets_and_counts[n][8] = (offset, point, spot, rect | probes, volumes, decals, 0) (:636-652),
 *               index_lists[n_indices] (:688-693)
 * storage == 0: offsets_and_counts[4096] packed (:622-634), index_lists[4096] = 16384 u8 slots OR-ed in (:676-686);
 *               both zeroed first (clear(), :598-606); the record loop BREAKS at the first Light seen with
 *               n_indices >= MAX_INDICES (:505-514), leaving every later cluster header unwritten.  The
 *               dummy push skips that check; past MAX_INDICES its slot lies outside the uniform array, where
 *               the reference's indexing panics: the oracle stops the loop there too. */
ORC_API void orc_cluster_bindings(uint32_t n_clusters, const uint32_t *offsets, const uint32_t *indices,
                                  const uint32_t *gpu_index_of_light, uint32_t n_map, int storage, uint32_t *offsets_and_counts,
                                  uint32_t *index_lists, uint32_t *n_offsets_out, uint32_t *n_indices_out) {
    size_t n_indices = 0, n_offsets = 0;
    if (!storage) {
        memset(offsets_and_counts, 0, VCB_MAX_UNIFORM_ITEMS * 4 * sizeof(uint32_t));
        memset(index_lists, 0, VCB_MAX_UNIFORM_ITEMS * 4 * sizeof(uint32_t));
    }
    int stop = 0;
    for (uint32_t c = 0; c < n_clusters && !stop; ++c) {
        const uint32_t point_lights = offsets[c + 1] - offsets[c];   /* ObjectsInClusterCpu::counts.point_lights */
        /* ClusterHeader record -> push_offset_and_counts(n_indices, counts) */
        if (storage) {
            uint32_t *o = offsets_and_counts + n_offsets * 8;
            o[0] = (uint32_t)n_indices; o[1] = point_lights; o[2] = 0; o[3] = 0; o[4] = 0; o[5] = 0; o[6] = 0; o[7] = 0;
        } else {
            const size_t array_index = n_offsets >> 2;
            if (array_index < VCB_MAX_UNIFORM_ITEMS)
                offsets_and_counts[array_index * 4 + (n_offsets & 3)] = pack_offset_and_counts(n_indices, point_lights, 0);
        }
        n_offsets++;
        /* Light records */
        for (uint32_t k = offsets[c]; k < offsets[c + 1]; ++k) {
            if (n_indices >= VCB_MAX_INDICES && !storage) { stop = 1; break; }
            const uint32_t index = !gpu_index_of_light ? indices[k]
                                   : indices[k] < n_map ? gpu_index_of_light[indices[k]] : 0xFFFFFFFFu;
            if (storage) index_lists[n_indices] = index;
            else {
                const size_t array_index = n_indices >> 4, component = (n_indices >> 2) & 3, sub_index = n_indices & 3;
                index_lists[array_index * 4 + component] |= index << (8 * sub_index);
            }
            n_indices++;
        }
    }
    *n_offsets_out = (uint32_t)n_offsets; *n_indices_out = (uint32_t)n_indices;
}

/* ------------------------------------------------------------------------------------------------------ */
/* N4a: check_visibility_ranges (range.rs:230-284)                                                          */
/* ------------------------------------------------------------------------------------------------------ */
#define F_HAS_AABB 0x02
#define F_HAS_VIS_RANGE 0x10
#define F_NO_CPU_CULLING 0x20
/* gt[n][12] = Affine3A x_axis, y_axis, z_axis, translation; bounds[n][6] (Aabb centre first);
 * range[n][2] = start_margin.start, end_margin.end (the two values is_visible_at_all reads, range.rs:157-159);
 * use_aabb[n]; view_pos[n_views][3] = view GlobalTransform translations in view-query order (only the first 32
 * are used, :247).  mask_out[n]: VisibleEntityRanges::entities value, 0 = no entry. */
ORC_API void orc_check_visibility_ranges(uint32_t n, const float *gt, const float *bounds, const uint8_t *flags,
                                         const float *range, const uint8_t *use_aabb, uint32_t n_views,
                                         const float *view_pos, uint32_t *mask_out) {
    if (n_views > 32) n_views = 32;
    for (uint32_t i = 0; i < n; ++i) {
        mask_out[i] = 0;
        if (!(flags[i] & F_HAS_VIS_RANGE) || (flags[i] & F_NO_CPU_CULLING)) continue;   /* not in entity_query */
        const float *g = gt + (size_t)i * 12, *b = bounds + (size_t)i * 6;
        float mx, my, mz;
        if (use_aabb[i] && (flags[i] & F_HAS_AABB)) {   /* transform_point3a(center) = ((X*c.x + Y*c.y) + Z*c.z) + t */
            mx = ((g[0] * b[0] + g[3] * b[1]) + g[6] * b[2]) + g[9];
            my = ((g[1] * b[0] + g[4] * b[1]) + g[7] * b[2]) + g[10];
            mz = ((g[2] * b[0] + g[5] * b[1]) + g[8] * b[2]) + g[11];
        } else { mx = g[9]; my = g[10]; mz = g[11]; }
        uint32_t visibility = 0;
        for (uint32_t v = 0; v < n_views; ++v) {
            const float dx = view_pos[v * 3] - mx, dy = view_pos[v * 3 + 1] - my, dz = view_pos[v * 3 + 2] - mz;
            const float d = sqrtf((dx * dx + dy * dy) + dz * dz);   /* Vec3A::length = sqrt(dot) */
            if (d >= range[i * 2] && d < range[i * 2 + 1]) visibility |= 1u << v;
        }
        mask_out[i] = visibility;
    }
}

/* ------------------------------------------------------------------------------------------------------ */
/* N4b: visibility_propagate_system (visibility/mod.rs:638-729), literal change-driven form                 */
/* ------------------------------------------------------------------------------------------------------ */
enum { VIS_INHERITED = 0, VIS_HIDDEN = 1, VIS_VISIBLE = 2, VIS_NO_COMPONENTS = 4 };
typedef struct {
    const uint32_t *child_off, *child_idx;
    const uint8_t *vis;
    uint8_t *inh, *changed;
} vp_ctx;
/* propagate_recursive (:701-729) with an explicit stack */
static void propagate_recursive(const vp_ctx *c, int parent_is_visible, uint32_t entity, uint32_t *stack, uint8_t *stack_vis) {
    uint32_t sp = 0;
    stack[sp] = entity; stack_vis[sp] = (uint8_t)parent_is_visible; ++sp;
    while (sp) {
        --sp;
        const uint32_t e = stack[sp]; const int pv = stack_vis[sp];
        if (c->vis[e] & VIS_NO_COMPONENTS) continue;   /* visibility_query.get_mut(entity) fails: return early */
        const int is_visible = (c->vis[e] & 3) == VIS_VISIBLE ? 1 : (c->vis[e] & 3) == VIS_HIDDEN ? 0 : pv;
        if (c->inh[e] != is_visible) {
            c->inh[e] = (uint8_t)is_visible; c->changed[e] = 1;
            for (uint32_t k = c->child_off[e + 1]; k-- > c->child_off[e];) {   /* children_query.get(entity) */
                stack[sp] = c->child_idx[k]; stack_vis[sp] = (uint8_t)is_visible; ++sp;
            }
        }
    }
}
/* parent[n] (0xFFFFFFFF = no ChildOf), vis[n] (Visibility | VIS_NO_COMPONENTS), inh[n] in/out, changed[n] out (1 where
 * the system wrote InheritedVisibility, i.e. its change tick fires); changed_rows = the `changed` query's rows in
 * iteration order, removed_rows = RemovedComponents<ChildOf> rows. */
ORC_API int orc_visibility_propagate(uint32_t n, const uint32_t *parent, const uint8_t *vis, uint8_t *inh, uint8_t *changed,
                                     uint32_t n_changed, const uint32_t *changed_rows, uint32_t n_removed,
                                     const uint32_t *removed_rows) {
    uint32_t *off = (uint32_t *)calloc((size_t)n + 2, 4), *idx = (uint32_t *)malloc((size_t)(n ? n : 1) * 4);
    uint32_t *stack = (uint32_t *)malloc((size_t)(n ? n : 1) * 4);
    uint8_t *stack_vis = (uint8_t *)malloc(n ? n : 1);
    if (!off || !idx || !stack || !stack_vis) { free(off); free(idx); free(stack); free(stack_vis); return 1; }
    for (uint32_t i = 0; i < n; ++i) if (parent[i] < n) off[parent[i] + 2]++;
    for (uint32_t i = 0; i < n; ++i) off[i + 2] += off[i + 1];
    for (uint32_t i = 0; i < n; ++i) if (parent[i] < n) idx[off[parent[i] + 1]++] = i;   /* off[e+1] ends at the end of e's list */
    memset(changed, 0, n);
    vp_ctx c = {off, idx, vis, inh, changed};
    for (uint32_t k = 0; k < n_changed; ++k) {
        const uint32_t e = changed_rows[k];
        if (vis[e] & VIS_NO_COMPONENTS) continue;   /* With<InheritedVisibility> + &Visibility */
        int is_visible;
        switch (vis[e] & 3) {
        case VIS_VISIBLE: is_visible = 1; break;
        case VIS_HIDDEN: is_visible = 0; break;
        default: {   /* fall back to true if no parent is found or the parent lacks components (:655-659) */
            const uint32_t p = parent[e];
            is_visible = (p < n && !(vis[p] & VIS_NO_COMPONENTS)) ? inh[p] : 1;
        }
        }
        if (inh[e] != is_visible) {   /* only update if it has changed (:667-675) */
            inh[e] = (uint8_t)is_visible; changed[e] = 1;
            for (uint32_t j = off[e]; j < off[e + 1]; ++j) propagate_recursive(&c, is_visible, idx[j], stack, stack_vis);
        }
    }
    for (uint32_t k = 0; k < n_removed; ++k) {   /* entities that just lost their ChildOf (:679-698) */
        const uint32_t e = removed_rows[k];
        if (vis[e] & VIS_NO_COMPONENTS) continue;
        const int is_visible = (vis[e] & 3) != VIS_HIDDEN;
        if (inh[e] != is_visible) {
            inh[e] = (uint8_t)is_visible; changed[e] = 1;
            for (uint32_t j = off[e]; j < off[e + 1]; ++j) propagate_recursive(&c, is_visible, idx[j], stack, stack_vis);
        }
    }
    free(off); free(idx); free(stack); free(stack_vis);
    return 0;
}
