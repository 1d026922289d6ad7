/*
 * b200vis.h -- C ABI of libb200vis.so: the H100-native replacement for the
 * per-frame visibility pipeline of bevyengine/bevy 0.20.0-dev
 * (propagate -> cull -> cluster).
 *
 * The reference has NO FFI seam for these stages: they are plain Rust systems.
 * Each entry point below therefore cites the reference system / type whose
 * work it takes over; the Rust-side binding a maintainer adds (a
 * `B200VisibilityPlugin` calling these through `extern "C"`) is shown in
 * INTEGRATION.md and rust/b200vis_plugin.rs.
 *
 * Conventions: every call returns an int32 status (0 = B200VIS_OK); no
 * unwinding, no global state; the caller owns all host memory, the library
 * owns all device memory; a context is thread-compatible (one caller at a
 * time), like a Bevy system holding `ResMut`.  Plain pointers and sizes only.
 * Rows are the caller's mirror of ECS archetype rows (one row per entity that
 * has Transform + GlobalTransform); ranges are [first_row, first_row+count).
 */
#ifndef B200VIS_H
#define B200VIS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200VIS_ABI_VERSION 2
#if defined(__GNUC__)
#define B200VIS_API __attribute__((visibility("default")))
#else
#define B200VIS_API
#endif

/* ---- status codes -------------------------------------------------------- */
enum {
    B200VIS_OK = 0,
    B200VIS_ERR_INVALID_ARG = 1,
    B200VIS_ERR_CUDA = 2,            /* CUDA runtime error or no CUDA device: see b200vis_last_error */
    B200VIS_ERR_OUT_OF_MEMORY = 3,
    B200VIS_ERR_HIERARCHY_CYCLE = 4, /* the shim must panic!(): crates/bevy_transform/src/systems.rs:715, test :1101 */
    B200VIS_ERR_PARENT_OUT_OF_RANGE = 5,
    B200VIS_ERR_CAPACITY = 6,        /* more rows / lights / views / indices than the context was created for */
    B200VIS_ERR_NOT_READY = 7,       /* a stage was run before its inputs were uploaded */
    B200VIS_ERR_UNSUPPORTED = 8
};

/* parent_row sentinels (b200vis_set_topology) */
#define B200VIS_NO_PARENT 0xFFFFFFFFu /* no ChildOf: a hierarchy root or a flat entity */
#define B200VIS_DETACHED  0xFFFFFFFEu /* has ChildOf, but the parent lacks Transform/GlobalTransform: never
                                         reached by propagation (NodeQuery, systems.rs:752-764) */

/* per-row flag byte (b200vis_upload_bounds) */
#define B200VIS_F_INHERITED_VISIBLE  0x01u /* InheritedVisibility::get() (visibility/mod.rs:164) */
#define B200VIS_F_HAS_AABB           0x02u /* Option<&Aabb> is Some (primitives.rs:63-68) */
#define B200VIS_F_HAS_SPHERE         0x04u /* Option<&Sphere> is Some (primitives.rs:197-211) */
#define B200VIS_F_NO_FRUSTUM_CULLING 0x08u /* Has<NoFrustumCulling> */
#define B200VIS_F_HAS_VIS_RANGE      0x10u /* Has<VisibilityRange> (visibility/range.rs) */
#define B200VIS_F_NO_CPU_CULLING     0x20u /* With<NoCpuCulling>: row is outside the visibility queries */
#define B200VIS_F_SPHERE_FROM_GT     0x40u /* Sphere.center is the row's own GlobalTransform translation, i.e. the
                                              steady state of update_point_light_bounding_spheres
                                              (crates/bevy_light/src/point_light.rs:195-209) */
/* bit 0x80 is owned by the library: "Transform changed since the last propagate" */

/* per-view flag byte */
#define B200VIS_VIEW_ACTIVE          0x01u /* camera.is_active (visibility/mod.rs:780) */
#define B200VIS_VIEW_NO_CPU_CULLING  0x02u /* Has<NoCpuCulling> on the camera (visibility/mod.rs:823) */

/* stages for b200vis_run */
#define B200VIS_STAGE_PROPAGATE      0x1u  /* TransformSystems::Propagate */
#define B200VIS_STAGE_CULL           0x2u  /* reset_view_visibility + check_visibility_cpu_culling +
                                              mark_newly_hidden_entities_invisible */
#define B200VIS_STAGE_CLUSTER_ASSIGN 0x4u  /* assign_objects_to_clusters: lights -> cluster x light bitmask slab */
#define B200VIS_STAGE_CLUSTER_LISTS  0x8u  /* bitmask (after the optional all-gather) -> ordered index lists */
#define B200VIS_STAGE_CLUSTER        (B200VIS_STAGE_CLUSTER_ASSIGN | B200VIS_STAGE_CLUSTER_LISTS)
#define B200VIS_STAGE_ALL            0xFu

#define B200VIS_MAX_VIEWS     8u     /* views b200vis_frame_stats reports, and views per rank with world_size > 1 */
#define B200VIS_MAX_CAMERAS   32u    /* views one context may hold (b200vis_config::max_views, world_size 1): views past the
                                        eighth are culled in extra passes of eight views each (DESIGN.md section 4) */
#define B200VIS_MAX_CLUSTERS  4096u  /* assign.rs:410-413 */

typedef struct b200vis_ctx b200vis_ctx;

typedef struct b200vis_config {
    int32_t  device;              /* CUDA device ordinal */
    uint32_t max_entities;        /* row capacity */
    uint32_t max_lights;          /* point lights this context (this rank's shard) may hold */
    uint32_t max_views;           /* 1..B200VIS_MAX_CAMERAS; <= B200VIS_MAX_VIEWS when world_size > 1 */
    uint32_t max_cluster_indices; /* per-view capacity of the cluster index list (0 => 1<<20) */
    uint32_t world_size;          /* ranks sharing the cluster exchange (0/1 => single GPU) */
    uint32_t rank;
    uint32_t reserved;
} b200vis_config;

/* One camera: what check_visibility_cpu_culling reads per view
 * (view_query, crates/bevy_camera/src/visibility/mod.rs:750-757). */
typedef struct b200vis_view {
    float    half_spaces[6][4];   /* Frustum: normal.xyz, d; order L,R,T,B,Near,Far (view_frustum.rs:25-34) */
    uint64_t layer_mask;          /* RenderLayers first block; default layer 0 => 1 */
    uint8_t  flags;               /* B200VIS_VIEW_* */
    int8_t   range_view_index;    /* bit index in VisibleEntityRanges, -1 if the view is not in it */
    uint8_t  pad[6];
} b200vis_view;

/* Per-view constants of assign_objects_to_clusters, computed on the host exactly
 * where the reference computes them (assign.rs:324-485); b200vis_host_cluster_view_setup
 * fills one of these from a camera + ClusterConfig + last frame's feedback. */
typedef struct b200vis_cluster_view {
    uint32_t enabled;             /* 0 => clusters.clear() path (ClusterConfig::None / empty viewport) */
    uint32_t dims[3];             /* Clusters::dimensions */
    uint32_t tile_size[2];        /* Clusters::tile_size (reported back, unused on the device) */
    uint32_t is_orthographic;
    float    near_z, far_z;       /* Clusters::near / far */
    float    cluster_factors[2];  /* calculate_cluster_factors (assign.rs:817-832) */
    float    view_from_world[16]; /* Mat4, column major */
    float    clip_from_view[16];
    float    view_from_world_scale[3];
    float    view_from_world_scale_max;
    float    frustum[6][4];       /* the view's Frustum, all six planes are used (assign.rs:496) */
    uint64_t layer_mask;
    const float *x_planes;        /* [(dims.x+1)][4] HalfSpace normal_d, view space (assign.rs:455-475) */
    const float *y_planes;        /* [(dims.y+1)][4] */
    const float *z_planes;        /* [(dims.z+1)][4] */
} b200vis_cluster_view;

/* Small per-frame result block (one D2H copy): what the shim writes back into
 * VisibleEntities / Clusters bookkeeping. */
typedef struct b200vis_frame_stats {
    uint32_t visible_count[B200VIS_MAX_VIEWS];       /* entries in each view's visible list */
    uint32_t cluster_index_count[B200VIS_MAX_VIEWS]; /* -> Clusters::last_frame_total_cluster_index_count */
    float    cluster_farthest_z[B200VIS_MAX_VIEWS];  /* -> Clusters::last_frame_farthest_z */
    uint32_t cluster_index_overflow[B200VIS_MAX_VIEWS]; /* 1 if the list did not fit max_cluster_indices */
    uint32_t gt_changed_count;                       /* rows whose Changed<GlobalTransform> fired */
    uint32_t vv_changed_count;                       /* rows whose Changed<ViewVisibility> fired */
    uint32_t frame;                                  /* frames run so far */
    uint32_t pad;
} b200vis_frame_stats;

/* ClusterConfig + GlobalClusterSettings + viewport, and last frame's Clusters feedback: inputs of the
 * host-side per-view prologue (b200vis_update_camera / b200vis_host_cluster_view_setup). */
typedef struct b200vis_cluster_config {      /* ClusterConfig + GlobalClusterSettings + viewport */
    uint32_t kind;               /* 0 None, 1 Single, 2 XYZ, 3 FixedZ (cluster/mod.rs:107-139) */
    uint32_t dims[3];            /* XYZ */
    uint32_t total, z_slices;    /* FixedZ */
    float    first_slice_depth;  /* ClusterZConfig */
    uint32_t far_z_mode;         /* 0 MaxClusterableObjectRange, 1 Constant */
    float    far_z_constant;
    uint32_t dynamic_resizing;
    uint32_t screen_w, screen_h; /* Camera::physical_viewport_size */
    uint32_t view_cluster_bindings_max_indices;
} b200vis_cluster_config;
typedef struct b200vis_cluster_feedback {    /* Clusters::last_frame_* (cluster/mod.rs:155-161) */
    uint32_t has_farthest_z;     float farthest_z;
    uint32_t has_index_count;    uint32_t index_count;
} b200vis_cluster_feedback;

/* ---- lifetime ------------------------------------------------------------- */
B200VIS_API int32_t b200vis_abi_version(void);
/* Kernel launches this library has issued since it was loaded (all contexts); bench.py reports the difference over its
 * timed regions as `gpu_launches`. */
B200VIS_API uint64_t b200vis_kernel_launch_count(void);
/* sizeof of the ABI structs, in declaration order (config, view, cluster_view, frame_stats, cluster_config,
 * cluster_feedback): lets a foreign-language binding verify its layout at start-up. */
B200VIS_API void b200vis_struct_sizes(uint32_t out[6]);
B200VIS_API int32_t b200vis_create(const b200vis_config *cfg, b200vis_ctx **out);
B200VIS_API void b200vis_destroy(b200vis_ctx *ctx);
B200VIS_API const char *b200vis_last_error(const b200vis_ctx *ctx); /* valid until the next call on ctx; ctx may be NULL */
/* All uploads, kernels and downloads of this context are issued on `cuda_stream`
 * (a cudaStream_t; NULL => the context's own stream). */
B200VIS_API int32_t b200vis_set_stream(b200vis_ctx *ctx, void *cuda_stream);
B200VIS_API int32_t b200vis_synchronize(b200vis_ctx *ctx);
/* b200vis_run(B200VIS_STAGE_ALL) pipelines frames: the latency-bound tail of frame f (visible-list expansion,
 * cluster kernels) runs on an internal side stream and overlaps frame f+1's tile pass.  b200vis_join makes the
 * context's stream wait (asynchronously) for that tail, e.g. before recording a timing event; every download and
 * b200vis_synchronize join implicitly.  Set B200VIS_PIPELINE=0 to serialise everything on one stream. */
B200VIS_API int32_t b200vis_join(b200vis_ctx *ctx);
/* Multi-GPU: b200vis_run(PROPAGATE|CULL|CLUSTER_ASSIGN) leaves the frame's tail open on this stream; the host issues
 * its all-gather of the cluster slabs ON THIS STREAM (so it is ordered after CLUSTER_ASSIGN) and then calls
 * b200vis_run(CLUSTER_LISTS), which continues there.  Equals the context's stream when pipelining is off. */
B200VIS_API int32_t b200vis_tail_stream(b200vis_ctx *ctx, void **cuda_stream);

/* ---- mirroring the ECS columns --------------------------------------------- */
/* Hierarchy + identity: the whole world, planned from scratch, with fresh frame state (every visible entity is
 * reported added by the next visible diff).  Per-frame spawns, despawns and ChildOf changes go through
 * b200vis_edit_topology instead, and b200vis_compact_topology drops the tombstones they leave; this call is for the
 * first upload and for world_size > 1.
 * Replaces the Children/ChildOf walks of propagate_descendants_unchecked
 * (systems.rs:679-748) with a cached execution plan.  entity_bits = Entity::to_bits()
 * (crates/bevy_ecs/src/entity/mod.rs:468-476), which fixes the order of every
 * visible list (visibility/mod.rs:870-874).  Rows must be in topological order
 * (parent_row[r] < r); b200vis_plan_row_order produces such an order. */
B200VIS_API int32_t b200vis_set_topology(b200vis_ctx *ctx, uint32_t n_rows, const uint32_t *parent_row,
                             const uint64_t *entity_bits);
/* One call per frame with every structural change of that frame, applied in this order:
 *   1. despawn   despawn_rows[n_despawn]: the rows leave every query and become tombstones (the other rows keep their
 *                numbers).  Despawn is recursive: a despawned row's live children must be despawned in the same call.
 *   2. reparent  reparent_rows[n_reparent] -> new_parent[] (B200VIS_NO_PARENT, B200VIS_DETACHED or a live row < the row):
 *                Changed<ChildOf> / RemovedComponents<ChildOf>; the rows are marked as b200vis_mark_transforms_changed does.
 *   3. spawn     n_spawn rows appended at [n, n + n_spawn): spawn_parent[] (sentinel, live row, or an earlier row of this
 *                batch), spawn_entity_bits[] = Entity::to_bits(); Added<GlobalTransform> (marked changed).
 * All or nothing: on any error nothing has changed.  Errors: CAPACITY (more than max_entities rows, tombstones included);
 * INVALID_ARG (a row out of range or dead, entity bits equal to those of any row, live or dead, a despawned row with live
 * children, a despawned row that is still in the b200vis_set_lights list or a point / spot shadow item: remove it there
 * first); UNSUPPORTED (a parent at or after its child's row, a tile that would need more than 128 rows with in-tile
 * children, world_size > 1).  On UNSUPPORTED or CAPACITY, compact with b200vis_compact_topology (which also takes the
 * reparents that break the row order) and repeat the rest of the edit.
 * Dead rows: parent B200VIS_DETACHED, flags B200VIS_F_NO_CPU_CULLING only, ViewVisibility 0, no VisibilityClass, not a
 * shadow caster.  They are in no visible, shadow or cluster list; a dead row that was visible is reported removed by
 * the next visible diff; its Changed flags never fire (the write-back mirrors its ViewVisibility 0 once).
 * b200vis_set_lights and b200vis_set_shadow_items reject dead rows.
 * Spawned rows start as b200vis_create leaves a row: Transform, GlobalTransform and bounds all zero, flags 0 (no
 * InheritedVisibility), no class, RenderLayers layer 0, no VisibilityRange, Visibility::Inherited, not a shadow caster.
 * Upload their columns with the usual calls before the next run.
 * Frame history carries over: frame counter, statistics, the visible-diff sets (which b200vis_run_shadow_culling reads),
 * Clusters feedback, recorded frame constants and the result / column sinks. */
B200VIS_API int32_t b200vis_edit_topology(b200vis_ctx *ctx, uint32_t n_despawn, const uint32_t *despawn_rows,
                                          uint32_t n_reparent, const uint32_t *reparent_rows, const uint32_t *new_parent,
                                          uint32_t n_spawn, const uint32_t *spawn_parent, const uint64_t *spawn_entity_bits);
/* Renumber the world on the device: drop the tombstones b200vis_edit_topology left, apply reparents that need not keep
 * row order, and re-plan -- keeping every column and the frame history resident.
 * reparent_rows[n_reparent] -> new_parent[] use the current row numbers; a new parent is a live row anywhere in the world,
 * B200VIS_NO_PARENT or B200VIS_DETACHED.  The rows are marked changed as the reparent step of b200vis_edit_topology marks
 * them.  New row order: b200vis_plan_row_order over the surviving rows in their current order, reparents applied; the
 * plan is the one b200vis_set_topology builds for that hierarchy.  old_to_new[r] (nullable, one entry per row before the
 * call) = the new number of row r, or 0xFFFFFFFF if it was dropped: renumber the entity <-> row maps, the host mirror
 * columns and the memory given to b200vis_set_column_sinks with it before the next write-back.
 * A dead row that a held result still names -- any view slot's visible list (an inactive view keeps its list), the
 * visible diff and the visible sets it compares against, a shadow list -- survives as a tombstone and goes at a later
 * compaction.  Every output after the call (GlobalTransform, change flags, ViewVisibility, visible lists and classes,
 * visible diff, shadow lists, clusters, statistics, sinks) equals what the uncompacted world gives, renumbered through
 * old_to_new; the compaction itself sets no Changed flag.  Light ordinals and shadow-item order are kept.
 * All or nothing.  Errors: INVALID_ARG (a reparented row out of range or dead or listed twice, a new parent out of range
 * or dead), HIERARCHY_CYCLE, UNSUPPORTED (world_size > 1), NOT_READY (no b200vis_set_topology yet). */
B200VIS_API int32_t b200vis_compact_topology(b200vis_ctx *ctx, uint32_t n_reparent, const uint32_t *reparent_rows,
                                             const uint32_t *new_parent, uint32_t *old_to_new /* [rows before], nullable */);
/* out = { rows (tombstones included), live rows, tiles, passes }: what a caller weighs before calling
 * b200vis_compact_topology. */
B200VIS_API int32_t b200vis_topology_summary(const b200vis_ctx *ctx, uint32_t out[4]);
/* Helper for the shim: a permutation (new_row -> old_row) that is topological and
 * keeps every tree contiguous in BFS order (the layout the tile kernel likes). */
B200VIS_API int32_t b200vis_plan_row_order(uint32_t n_rows, const uint32_t *parent_row, uint32_t *new_to_old);
/* What b200vis_set_topology would plan for this hierarchy (no GPU needed): out = { tiles, passes (kernel launches per
 * propagate), deepest in-tile level count, rows whose parent lives in another tile }.  Same error codes. */
B200VIS_API int32_t b200vis_host_plan_summary(uint32_t n_rows, const uint32_t *parent_row, uint32_t out[4]);
/* The plan as the default tile kernel (one CTA of 8 warps per tile) sees it (no GPU needed; for tests and tools):
 * tile_desc[i] = { first row, rows, in-tile levels, warp_sync_mask (bit l: every edge into level l stays inside a warp),
 * top_levels, lvl_warps low word, lvl_warps high word (nibble l = warps that meet at the hand-over of level l; 0 = the
 * tile is walked with CTA-wide barriers), pass }, topo[row] = parent's local row | in-tile depth << 9 | flags (bits 28-31).
 * With tile_desc == NULL only *n_tiles is written. */
B200VIS_API int32_t b200vis_host_tile_plan(uint32_t n_rows, const uint32_t *parent_row, uint32_t tile_rows, uint32_t tiles_capacity,
                                           uint32_t *n_tiles, uint32_t *tile_desc, uint32_t *topo);
/* The plan as the warp-per-tile kernel (B200VIS_TILE_KERNEL=warp) sees it (no GPU needed; for tests and tools): one work item per WARP.
 * tile_desc[i] = { first row, rows, chunks | contiguous-chunk bits << 8, pass }, nonroot[i][8] = per chunk the schedule
 * slots holding a row whose parent is in the tile, sched[i][256] = schedule slot -> local row (0xFF = padding, except in
 * a 256-row tile), wtopo[row] = depth | own slot << 8 | parent's slot << 15 | has-slot << 22 | flags (bits 28-31).
 * tile_rows = 0 means the default tile size (256).  With tile_desc == NULL only *n_tiles is written. */
B200VIS_API int32_t b200vis_host_warp_plan(uint32_t n_rows, const uint32_t *parent_row, uint32_t tile_rows, uint32_t tiles_capacity,
                                           uint32_t *n_tiles, uint32_t *tile_desc, uint32_t *nonroot, uint8_t *sched, uint32_t *wtopo);
/* The plan b200vis_edit_topology keeps, after an edit script (no GPU needed; for tests and tools).  The script is a
 * sequence of steps, each { n_despawn, n_reparent, n_spawn, despawn_rows[n_despawn], reparent_rows[n_reparent],
 * new_parent[n_reparent], spawn_parent[n_spawn] }, applied like b200vis_edit_topology calls with at most max_rows rows.
 * A step { 0xFFFFFFFF, n_reparent, n_held, reparent_rows[n_reparent], new_parent[n_reparent], held_rows[n_held] } is
 * a b200vis_compact_topology call whose held results name the dead rows held_rows[] (tile_rows != 0: the new plan is cut
 * with that tile size instead of b200vis_set_topology's search).
 * Returns the first failing step's error (the outputs then hold the plan before that step).  *n_rows = rows after
 * the script; tile_desc[i][17] = { the 8 words of b200vis_host_tile_plan, chunks | contiguous-chunk bits << 8,
 * nonroot[8] of b200vis_host_warp_plan }, sched[i][256], topo[row], wtopo[row] as there; counters = { tiles re-planned
 * and rows re-planned by the last applied step, passes, steps applied }.  With tile_desc == NULL only *n_rows, *n_tiles
 * and counters are written. */
B200VIS_API int32_t b200vis_host_edit_plan(uint32_t n_rows, const uint32_t *parent_row, uint32_t tile_rows, uint32_t max_rows,
                                           uint32_t script_words, const uint32_t *script, uint32_t tiles_capacity, uint32_t *n_rows_out,
                                           uint32_t *n_tiles, uint32_t *tile_desc, uint32_t *topo, uint32_t *wtopo, uint8_t *sched,
                                           uint32_t counters[4]);

/* Transform column, dirty ranges: trs[count][10] = translation.xyz, rotation.xyzw, scale.xyz
 * (components/transform.rs:86-105).  Marks the rows Changed<Transform>. */
B200VIS_API int32_t b200vis_upload_transforms(b200vis_ctx *ctx, uint32_t first_row, uint32_t count, const float *trs);
/* Same, for the scattered row set a `Changed<Transform>` query yields: rows[count], trs[count][10]. */
B200VIS_API int32_t b200vis_upload_transforms_scattered(b200vis_ctx *ctx, uint32_t count, const uint32_t *rows,
                                                        const float *trs);
/* Rows that are Changed<ChildOf> | Added<GlobalTransform> | freshly orphaned without new Transform data
 * (mark_dirty_trees' input set, systems.rs:112-113). */
B200VIS_API int32_t b200vis_mark_transforms_changed(b200vis_ctx *ctx, uint32_t first_row, uint32_t count);
/* GlobalTransform column as it stands on the host (the initial mirror, spawn time):
 * gt[count][12] = Affine3A x_axis.xyz, y_axis.xyz, z_axis.xyz, translation.xyz.  Sets no Changed flag; GlobalTransforms
 * that other systems write between frames go through b200vis_write_global_transforms_scattered. */
B200VIS_API int32_t b200vis_upload_global_transforms(b200vis_ctx *ctx, uint32_t first_row, uint32_t count, const float *gt);
/* GlobalTransforms that another system wrote since the last run that included PROPAGATE
 * (Changed<GlobalTransform> as the propagate system sees it, systems.rs:709-710): sets the column
 * (gt[count][12] as in b200vis_upload_global_transforms) and marks p_global_transform.is_changed()
 * for the next run that includes PROPAGATE, which consumes the marks.
 * That run re-propagates the children of every marked row it visits, even when the row's recomputed value equals the
 * written one; a marked row it does not visit keeps the written value.  A mark does not dirty the row's ancestors, and
 * the row's own Changed<GlobalTransform> output is unaffected (the writer stamped its own tick).  A run without
 * PROPAGATE keeps the marks and culls at the written values.  A row listed twice takes its last value.
 * Marks are per row: b200vis_edit_topology drops a despawned row's mark, b200vis_compact_topology carries them through
 * old_to_new, b200vis_set_topology clears them.  A run that includes PROPAGATE while marks are pending returns
 * UNSUPPORTED, consuming nothing, when B200VIS_TILE_KERNEL selects an experiment tile kernel.
 * Errors: NOT_READY (no b200vis_set_topology yet), INVALID_ARG (a null array, a row out of range or despawned). */
B200VIS_API int32_t b200vis_write_global_transforms_scattered(b200vis_ctx *ctx, uint32_t count,
                                                              const uint32_t *rows, const float *gt);
/* Aabb / Sphere / flags / VisibilityClass / RenderLayers / VisibleEntityRanges columns:
 * bounds[count][6] = center.xyz, half_extents.xyz (Aabb) or center.xyz, radius,0,0 (Sphere);
 * class_mask: one bit per VisibilityClass the entity is in (0 => set_visible() but no list entry,
 * visibility/mod.rs:846-857); layer_mask / range_mask may be NULL (=> default layer / no
 * VisibleEntityRanges resource). */
B200VIS_API int32_t b200vis_upload_bounds(b200vis_ctx *ctx, uint32_t first_row, uint32_t count, const float *bounds,
                              const uint8_t *flags, const uint8_t *class_mask, const uint64_t *layer_mask,
                              const uint32_t *range_mask);
/* ViewVisibility column (bit0 current, bit1 previous; visibility/mod.rs:226-242) */
/* RenderLayers beyond the first 64 layers: the component is a SmallVec of 64-bit blocks (render_layers.rs:20-23) and
 * intersects() ORs the block-wise ANDs over the blocks both sides have (:121-135).  Block 0 is the layer_mask of
 * b200vis_upload_bounds / b200vis_view / b200vis_camera; blocks[count][3] / blocks[3] are blocks 1..3 (layers 64..255) of
 * the rows / of a view.  A view's blocks serve both its camera cull and its cluster view (the camera of view v is the
 * same camera in both stages).  Lights and shadow items take theirs from b200vis_set_light_render_layers_ext and
 * b200vis_set_shadow_item_render_layers_ext; until then they have block 0 only. */
B200VIS_API int32_t b200vis_upload_render_layers_ext(b200vis_ctx *ctx, uint32_t first_row, uint32_t count, const uint64_t *blocks);
B200VIS_API int32_t b200vis_set_view_render_layers_ext(b200vis_ctx *ctx, uint32_t view, const uint64_t blocks[3]);
B200VIS_API int32_t b200vis_upload_view_visibility(b200vis_ctx *ctx, uint32_t first_row, uint32_t count, const uint8_t *vv);

/* StaticTransformOptimizations resource (systems.rs:87-103); default Enabled (1). */
B200VIS_API int32_t b200vis_set_static_transform_optimizations(b200vis_ctx *ctx, int32_t enabled);

/* ---- per-frame constants ----------------------------------------------------- */
B200VIS_API int32_t b200vis_set_views(b200vis_ctx *ctx, uint32_t n_views, const b200vis_view *views);
/* PointLight set (point_lights_query, assign.rs:146-153): light_row = the light entity's row (its
 * GlobalTransform translation and ViewVisibility are read on the device), in query order.  layer_mask = block 0 of each
 * light's RenderLayers (NULL = the default layer); the call empties every light's blocks 1..3. */
B200VIS_API int32_t b200vis_set_lights(b200vis_ctx *ctx, uint32_t n_lights, const uint32_t *light_row, const float *range,
                           const uint64_t *layer_mask /* nullable */);
/* RenderLayers blocks 1..3 (layers 64..255) of the clustered lights: blocks[n_lights][3] in b200vis_set_lights ordinal
 * order, NULL = all empty.  Call it after b200vis_set_lights, which empties them again.  The cluster stage then tests the
 * light's whole RenderLayers against its view's (assign.rs:489, render_layers.rs:121-135): block 0 against the layer_mask
 * of the cluster view, blocks 1..3 against the view's b200vis_set_view_render_layers_ext blocks.  Frame constants recorded
 * (b200vis_record_frame_constants) while no light had blocks 1..3 replay with block 0 only.
 * Errors: INVALID_ARG (n_lights is not the current light count), UNSUPPORTED (world_size > 1: the light records that
 * travel between ranks carry block 0 only); nothing changes then. */
B200VIS_API int32_t b200vis_set_light_render_layers_ext(b200vis_ctx *ctx, uint32_t n_lights, const uint64_t *blocks);
B200VIS_API int32_t b200vis_set_cluster_view(b200vis_ctx *ctx, uint32_t view, const b200vis_cluster_view *params);
/* Cluster grid dimensions of the view as last set (b200vis_set_cluster_view / b200vis_update_camera / b200vis_step);
 * zeros when clustering is off for the view.  The shim sizes Clusters::clusterable_objects from it. */
B200VIS_API int32_t b200vis_cluster_view_dims(const b200vis_ctx *ctx, uint32_t view, uint32_t dims[3]);

/* Frame constants kept in HBM: record_frame_constants snapshots the current views / cluster views (device copy
 * of the packed tables + the host copy the kernel parameters are built from) and returns a slot;
 * use_recorded_frame_constants(slot) makes b200vis_run use that snapshot with no host maths and no upload
 * (-1 returns to the live path).  Lets a recorded frame sequence replay with every input resident. */
B200VIS_API int32_t b200vis_record_frame_constants(b200vis_ctx *ctx, uint32_t *slot);
B200VIS_API int32_t b200vis_use_recorded_frame_constants(b200vis_ctx *ctx, int32_t slot);

/* Optional per-stage device timing: when on, b200vis_run brackets its stages with CUDA events on the
 * context's stream (up to 256 runs are kept).  b200vis_collect_stage_times_ms synchronizes ONCE, returns the
 * summed durations of the tile kernel(s) (propagate+cull), the visible-list expansion and the cluster kernels
 * over the `frames` runs recorded since the last collect, and resets the recorder. */
B200VIS_API int32_t b200vis_set_profiling(b200vis_ctx *ctx, int32_t enabled);
B200VIS_API int32_t b200vis_collect_stage_times_ms(b200vis_ctx *ctx, float *tile_ms, float *expand_ms, float *cluster_ms,
                                                   uint32_t *frames);

/* One call per camera per frame: the host-side work of update_frusta (visibility/mod.rs:627-636) and of the
 * per-view prologue of assign_objects_to_clusters (assign.rs:324-485) for a perspective camera, written
 * straight into the context's frame constants.  cfg == NULL leaves the view without clusters; `out` (nullable)
 * receives the cluster view that was set (its plane pointers are only valid until the next call). */
typedef struct b200vis_camera {
    float    global_transform[12]; /* camera GlobalTransform, layout as in b200vis_upload_global_transforms */
    float    fov_y, aspect, near_z, far_z; /* PerspectiveProjection (projection.rs:419-426) */
    uint64_t layer_mask;
    uint8_t  flags;                /* B200VIS_VIEW_* */
    int8_t   range_view_index;
    uint8_t  pad[6];
} b200vis_camera;
B200VIS_API int32_t b200vis_set_view_count(b200vis_ctx *ctx, uint32_t n_views);
B200VIS_API int32_t b200vis_update_camera(b200vis_ctx *ctx, uint32_t view, const b200vis_camera *camera,
                                          const b200vis_cluster_config *cfg, const b200vis_cluster_feedback *feedback,
                                          b200vis_cluster_view *out);

/* ---- run ----------------------------------------------------------------------- */
B200VIS_API int32_t b200vis_run(b200vis_ctx *ctx, uint32_t stages);

/* One call per frame for a single-GPU host loop: upload the changed Transforms, recompute every camera's frame
 * constants (b200vis_update_camera with the library's own copy of last frame's Clusters feedback), run all stages
 * and -- with B200VIS_STEP_WAIT -- synchronise and refresh that feedback from the frame's statistics.  With a result
 * sink set, the frame's results are in the caller's pinned buffers when the call returns. */
#define B200VIS_STEP_WAIT 0x1u
B200VIS_API int32_t b200vis_step(b200vis_ctx *ctx, uint32_t n_changed, const uint32_t *rows, const float *trs,
                                 uint32_t n_cameras, const b200vis_camera *cameras, const b200vis_cluster_config *cfg,
                                 uint32_t flags);

/* ---- results --------------------------------------------------------------------- */
B200VIS_API int32_t b200vis_download_frame_stats(b200vis_ctx *ctx, b200vis_frame_stats *out);
/* The per-view part of the frame statistics for views [first_view, first_view + count) of any context, up to max_views
 * (b200vis_frame_stats holds views 0..7).  Each array receives `count` entries and may be NULL. */
B200VIS_API int32_t b200vis_download_view_stats(b200vis_ctx *ctx, uint32_t first_view, uint32_t count, uint32_t *visible_count,
                                                uint32_t *cluster_index_count, float *cluster_farthest_z,
                                                uint32_t *cluster_index_overflow);
/* gt[count][stride_floats] (stride 12, or 16 for glam's padded Affine3A layout); changed[count]:
 * 1 where the shim must stamp changed_ticks (set_if_neq semantics, systems.rs:719). Either may be NULL. */
B200VIS_API int32_t b200vis_download_global_transforms(b200vis_ctx *ctx, uint32_t first_row, uint32_t count, float *gt,
                                           uint32_t stride_floats, uint8_t *changed);
B200VIS_API int32_t b200vis_download_view_visibility(b200vis_ctx *ctx, uint32_t first_row, uint32_t count, uint8_t *vv,
                                         uint8_t *changed);
/* VisibleEntities of one view: rows of the visible entities that have a VisibilityClass, ascending by
 * Entity::to_bits() (visibility/mod.rs:861-874).  An inactive view keeps last frame's list (:780-782). */
B200VIS_API int32_t b200vis_download_visible(b200vis_ctx *ctx, uint32_t view, uint32_t *rows, uint32_t capacity,
                                 uint32_t *count);
/* VisibleEntities::entities is one sorted Vec per VisibilityClass, and an entity with k classes is pushed k times
 * (visibility/mod.rs:344-347, 852-857).  classes[i] = the class mask (as uploaded by b200vis_upload_bounds, bit k = class k
 * of the shim's TypeId registry, at most 8) of the i-th row of b200vis_download_visible's list: walking the list once and
 * pushing entity i into every class list whose bit is set yields each class's list already sorted. */
B200VIS_API int32_t b200vis_download_visible_classes(b200vis_ctx *ctx, uint32_t view, uint8_t *classes, uint32_t capacity,
                                                     uint32_t *count);
/* Clusters of one view in CSR form: offsets[n_clusters+1], light ordinals (index into the
 * b200vis_set_lights arrays; with world_size>1: global ordinal = rank-major) in the reference's
 * push order, cluster index = (y*dims.x + x)*dims.z + z (assign.rs:676-678). */
B200VIS_API int32_t b200vis_download_clusters(b200vis_ctx *ctx, uint32_t view, uint32_t *offsets, uint32_t *indices,
                                  uint32_t indices_capacity, uint32_t *total);

/* Everything the shim writes back after a frame, with two stream synchronisations instead of one per list:
 * the stats block, every view's sorted visible rows (visible_rows[v*visible_capacity ...]) and every view's
 * cluster CSR (cluster_offsets[v*4097 ...], cluster_indices[v*cluster_capacity ...]).  Array pointers may be NULL. */
B200VIS_API int32_t b200vis_download_frame(b200vis_ctx *ctx, b200vis_frame_stats *stats, uint32_t *visible_rows,
                                           uint32_t visible_capacity, uint32_t *cluster_offsets,
                                           uint32_t *cluster_indices, uint32_t cluster_capacity);

/* Result sink: caller-owned PINNED host memory that the frame's results are written into by the GPU itself (small
 * "publish" kernels doing coalesced posted writes over PCIe right after the producing kernels), so that reading a
 * frame back needs ONE stream synchronisation and no size round trip:
 *   stats            the b200vis_frame_stats block
 *   visible_rows     [max_views][visible_capacity]  sorted visible rows per view (count in stats->visible_count)
 *   cluster_offsets  [max_views][4097], cluster_indices [max_views][cluster_capacity]
 * The library registers the ranges with cudaHostRegister if they are not already pinned.  NULL removes the sink. */
typedef struct b200vis_result_sink {
    b200vis_frame_stats *stats;
    uint32_t *visible_rows;   uint32_t visible_capacity;
    uint8_t  *visible_classes; /* nullable: [max_views][visible_capacity] VisibilityClass mask of each listed row */
    uint32_t *cluster_offsets;
    uint32_t *cluster_indices; uint32_t cluster_capacity;
} b200vis_result_sink;
B200VIS_API int32_t b200vis_set_result_sink(b200vis_ctx *ctx, const b200vis_result_sink *sink);
/* Per-view statistics of every view, written with the result sink's stats block (so reading them needs no extra
 * synchronisation): per_view[max_views][4] = visible_count, cluster_index_count, cluster_farthest_z (float bits),
 * cluster_index_overflow.  Needs a result sink to be published.  Pinned or registered like the result sink; NULL removes it. */
B200VIS_API int32_t b200vis_set_view_stats_sink(b200vis_ctx *ctx, uint32_t *per_view);
/* VisibleEntities as Entity values, one sorted list per VisibilityClass (visibility/mod.rs:344-347, 852-874).  Entity is
 * repr(C, align(8)) and equivalent to a u64 (crates/bevy_ecs/src/entity/mod.rs:423-432), so each entry is
 * Entity::to_bits() as given to b200vis_set_topology / b200vis_edit_topology and the shim extends each class's Vec<Entity>
 * with one slice:
 *   entities [max_views][capacity]  a view's class lists back to back, class 0 first
 *   offsets  [max_views][9]         class k of view v is entities[v*capacity + offsets[v*9+k] .. offsets[v*9+k+1])
 * For every active view below the frame's view count, class k's list is the view's b200vis_download_visible list filtered
 * to the rows whose b200vis_download_visible_classes mask has bit k, mapped through the entity bits: ascending by
 * to_bits(), an entity with several classes in each of their lists.  offsets[v*9+8] is the true total even when it
 * exceeds capacity; positions at or past capacity are not written.  An inactive view, and a view at or past the frame's
 * view count, has neither its region nor its offsets written (an inactive view keeps its lists, :780-782).
 * Written by the GPU on the frame's tail right behind the list expansion, wherever the CULL stage runs (pipelined
 * STAGE_ALL, B200VIS_PIPELINE=0, b200vis_step, more than eight views, after edits and compactions); the frame is readable
 * after the next b200vis_synchronize.  Pinned or registered like the result sink.  While the sink is set the entity keys
 * stay resident on the device (8 bytes per max_entities row).  NULL removes the sink.
 * Errors: INVALID_ARG (capacity 0, entities or offsets NULL, entities not 8-byte aligned), UNSUPPORTED (world_size > 1). */
typedef struct b200vis_visible_entities_sink {
    uint64_t *entities;
    uint32_t  capacity;           /* entries per view */
    uint32_t *offsets;
} b200vis_visible_entities_sink;
B200VIS_API int32_t b200vis_set_visible_entities_sink(b200vis_ctx *ctx, const b200vis_visible_entities_sink *sink);

/* ---- write-back of the frame's column results into the caller's ECS columns -------------------------------------------
 * The reference systems leave their results IN the ECS: GlobalTransform (+ Changed<GlobalTransform>) and ViewVisibility
 * (+ Changed<ViewVisibility>) are read downstream (e.g. crates/bevy_pbr/src/render/mesh.rs:1933-1955).  With column sinks
 * registered, b200vis_writeback_columns (or b200vis_step with B200VIS_STEP_WRITEBACK) has the GPU write, over PCIe and
 * straight into host memory -- typically the table column slices `ContiguousMut::bypass_change_detection()` hands out
 * (crates/bevy_ecs/src/change_detection/params.rs:1079-1142):
 *   global_transforms [n][gt_stride_floats]  ONLY the rows whose GlobalTransform changed this frame (set_if_neq semantics:
 *                                            the other rows keep their bytes); stride 16 = glam Affine3A (four 16-byte
 *                                            Vec3A lanes, padding lanes written as 0), stride 12 = packed X,Y,Z,T
 *   gt_changed_bits   [ceil(n/32)]           bit r%32 of word r/32: stamp changed_ticks[r] = this_run
 *   view_visibility   [n]                    the ViewVisibility byte of every row (bit0 current, bit1 previous)
 *   vv_changed_bits   [ceil(n/32)]           Changed<ViewVisibility>
 * Any pointer may be NULL (that column is not delivered).  The memory is registered with cudaHostRegister if it is not
 * pinned already.  Results are complete after b200vis_synchronize (or b200vis_step(.., WAIT)).  NULL removes the sinks. */
typedef struct b200vis_column_sinks {
    float *global_transforms; uint32_t gt_stride_floats;
    uint32_t *gt_changed_bits;
    uint8_t *view_visibility;
    uint32_t *vv_changed_bits;
} b200vis_column_sinks;
B200VIS_API int32_t b200vis_set_column_sinks(b200vis_ctx *ctx, const b200vis_column_sinks *sinks);
B200VIS_API int32_t b200vis_writeback_columns(b200vis_ctx *ctx);
/* The same for a subset of the columns: a shim that runs the stages from separate systems writes the GlobalTransform
 * column back right after PROPAGATE and the ViewVisibility column after CULL (and the light-visibility systems). */
#define B200VIS_WB_GLOBAL_TRANSFORM 0x1u
#define B200VIS_WB_VIEW_VISIBILITY  0x2u
B200VIS_API int32_t b200vis_writeback_columns_ex(b200vis_ctx *ctx, uint32_t which);
#define B200VIS_STEP_WRITEBACK 0x2u  /* b200vis_step: enqueue the column write-back right behind the tile pass */

/* ---- write-back straight into the caller's archetype tables -------------------------------------------------------------
 * In Bevy, GlobalTransform and ViewVisibility live in one column per archetype table, each in the table's own slot order
 * (crates/bevy_ecs/src/storage/table/mod.rs), and a hierarchy spans several tables (roots, inner nodes and leaves differ in
 * ChildOf / Children).  A table registry lets the GPU write every result, and the change tick itself, into those columns:
 * b200vis_writeback_tables walks each table in slot order and gathers each slot's row through a slot -> row map that lives
 * on the device.
 *   global_transforms  [capacity] glam Affine3A, 64 B per slot: ONLY slots whose row's GlobalTransform changed this frame
 *                      are written (the set_if_neq rule of the column sinks), padding lanes as 0
 *   gt_changed_ticks   [capacity] GlobalTransform's changed_ticks column: gt_tick where that write happened
 *   view_visibility    [capacity] the ViewVisibility byte, written where it differs from what the slot is known to hold
 *   vv_changed_ticks   [capacity] vv_tick exactly where Changed<ViewVisibility> fires
 * Any column may be NULL (not delivered / not stamped).  Only slots [0, len) that are mapped to a live row are ever
 * written; every other byte and tick keeps its value.  The library registers the page-rounded [0, capacity) ranges of
 * memory that is not pinned (cudaHostRegister, mapped; overlapping ranges of different tables become one registration),
 * owns those registrations and releases them when a table's columns or capacity change and in b200vis_destroy.  Memory
 * that is already pinned by its owner is used through its device alias.  A registration covers whole pages, so other
 * allocations on those pages are page-locked with it, and a CUDA copy from pageable memory that lies only partly inside a
 * registered range can fail with cudaErrorInvalidValue: small tables are best allocated from page-aligned memory that owns
 * its pages.  world_size > 1: UNSUPPORTED. */
#define B200VIS_MAX_TABLES 4096u
typedef struct b200vis_table {
    void     *global_transforms;  /* [capacity] GlobalTransform (Affine3A, 64 B per slot); NULL = not delivered */
    uint32_t *gt_changed_ticks;   /* [capacity] Tick (u32); NULL = not stamped */
    uint8_t  *view_visibility;    /* [capacity]; NULL = not delivered */
    uint32_t *vv_changed_ticks;   /* [capacity] */
    uint32_t  len;                /* Table::entity_count: only slots [0, len) are ever written */
    uint32_t  capacity;           /* Table::capacity: the extent that is registered */
} b200vis_table;
/* Replaces the registry: table t of the call is table t from then on.  The slot maps of tables that stay keep their
 * entries below the new capacity; slots at or past it, and the tables past n_tables, are unmapped.  When a table's
 * view_visibility column moves, its slots are sent their ViewVisibility byte again by the next write-back.
 * n_tables == 0 empties the registry.  Errors: INVALID_ARG (len > capacity, a global_transforms column not 16-byte aligned,
 * a ticks column not 4-byte aligned), CAPACITY (more than B200VIS_MAX_TABLES tables, or more than 2^31 slots in all), UNSUPPORTED (world_size > 1); nothing
 * changes then.  On B200VIS_ERR_CUDA (cudaHostRegister refused the memory) the registry is left empty. */
B200VIS_API int32_t b200vis_set_tables(b200vis_ctx *ctx, uint32_t n_tables, const b200vis_table *tables);
/* Maps slots [first_slot, first_slot + count) of `table` to rows[i] (B200VIS_UNMAPPED = unmapped), in order.  The call does
 * not wait for the stream: map changes are queued and reach the device as one batch at the next write-back.  Mapping row r
 * to (table, slot) removes r's previous mapping, and the row that slot held before becomes unmapped: an archetype move, or
 * the swap_remove behind it (table/mod.rs), is one or two such calls.  All or nothing.  Errors: INVALID_ARG (a table out of
 * range, slots past the table's capacity, a row out of range or despawned, a null rows with count > 0), UNSUPPORTED
 * (world_size > 1).
 * Rows move with the world: b200vis_set_topology unmaps every slot (the tables stay registered), b200vis_edit_topology unmaps
 * the rows it despawns, b200vis_compact_topology renumbers the maps itself (the caller does nothing to its tables). */
#define B200VIS_UNMAPPED 0xFFFFFFFFu
B200VIS_API int32_t b200vis_set_table_rows(b200vis_ctx *ctx, uint32_t table, uint32_t first_slot, uint32_t count,
                                           const uint32_t *rows);
/* Enqueues the write-back of `which` (B200VIS_WB_*) on the context's stream, behind the frame's tile pass, like
 * b200vis_writeback_columns_ex; the results are complete after b200vis_synchronize.  gt_tick / vv_tick = the tick stamped
 * into the changed_ticks columns (the writing system's this_run).
 *   B200VIS_WB_SET_VISIBLE  SetViewVisibility::set_visible (crates/bevy_camera/src/visibility/mod.rs:290-306) applied to the
 *                           bytes the caller's reset_view_visibility left, for builds where the device does not own the
 *                           ViewVisibility state: every slot below len mapped to a row whose device ViewVisibility bit 0
 *                           is set has its byte b READ; where b & 1 == 0 the slot gets b | 1, and where also b & 2 == 0
 *                           vv_changed_ticks gets vv_tick.  Nothing else is written.  It neither uses nor updates what the
 *                           ViewVisibility write-back knows a slot holds: every mapped slot it covers is marked unknown, so
 *                           a later B200VIS_WB_VIEW_VISIBILITY sends every byte again.  Tables without view_visibility are
 *                           skipped.
 *                           The light pass: b200vis_run_shadow_culling folds its set_visible() into the device bit 0, so
 *                           a second call behind it, with the light system's tick, applies set_visible() to the rows
 *                           only lights see; rows the cameras made visible already hold bit 0 and are left alone.  (The
 *                           forked build's B200VIS_WB_VIEW_VISIBILITY after the shadow stage does the same job.)
 * Errors: NOT_READY (no b200vis_set_tables yet), UNSUPPORTED (world_size > 1), INVALID_ARG (B200VIS_WB_SET_VISIBLE with
 * B200VIS_WB_VIEW_VISIBILITY; nothing is enqueued then). */
#define B200VIS_WB_SET_VISIBLE 0x4u
B200VIS_API int32_t b200vis_writeback_tables(b200vis_ctx *ctx, uint32_t which, uint32_t gt_tick, uint32_t vv_tick);

/* ---- reading Transform and outside-written GlobalTransform straight from the same tables ----------------------------------
 * The device finds Changed<Transform> and Changed<GlobalTransform> itself: it reads every slot's tick over PCIe, and the
 * Transform or Affine3A of the slots whose tick is newer, through the same slot -> row maps as the write-back.
 * Transform is repr(Rust), so its layout is passed in (size_of::<Transform>() and offset_of! of its three fields). */
typedef struct b200vis_transform_layout {
    uint32_t stride;                          /* bytes per slot */
    uint32_t translation, rotation, scale;    /* byte offsets of Vec3, Quat (x, y, z, w), Vec3 */
} b200vis_transform_layout;
typedef struct b200vis_table_inputs {
    const void     *transforms;               /* [capacity] Transform; NULL = the table is not read for Transform */
    const uint32_t *transform_changed_ticks;  /* [capacity] Transform's changed_ticks; NULL exactly when transforms is */
} b200vis_table_inputs;
/* b200vis_set_tables with input columns: inputs == NULL or inputs[n_tables].  The input columns are registered, kept and
 * released with the output columns (the page rules above apply to them too).  b200vis_set_tables(ctx, n, t) is
 * b200vis_set_tables_ex(ctx, n, t, NULL, NULL).  Errors, besides those of b200vis_set_tables: INVALID_ARG (a layout field
 * that is not 4-byte aligned, a field past stride, overlapping fields, no layout while some table has transforms, only one
 * of a table's two input pointers NULL, a misaligned input pointer); nothing changes then. */
B200VIS_API int32_t b200vis_set_tables_ex(b200vis_ctx *ctx, uint32_t n_tables, const b200vis_table *tables,
                                          const b200vis_table_inputs *inputs, const b200vis_transform_layout *layout);
/* Enqueues the read of `which` on the context's stream, in call order with every other upload; queued map changes are
 * sent first.  A slot is read when it is below len, mapped to a live row, and its tick is newer by Bevy's
 * Tick::is_newer_than(last_run, this_run) (change_detection/tick.rs): this_run - tick < this_run - last_run in wrapping
 * u32 arithmetic, both ages clamped to MAX_CHANGE_AGE = 0xFFFFFFFF - (2 * 518400000 - 1).  Pass the reading system's
 * SystemChangeTick pair: ticks that system's own write-back stamped last frame equal last_run and are not read.
 *   B200VIS_RD_TRANSFORM         Transform, as b200vis_upload_transforms_scattered would upload it for the row (bits copied,
 *                                the row marked Changed<Transform>)
 *   B200VIS_RD_GLOBAL_TRANSFORM  global_transforms / gt_changed_ticks of b200vis_table (tables lacking either are skipped),
 *                                as b200vis_write_global_transforms_scattered would write lanes 0-2 of the four Vec3A.
 *                                Without a synchronisation the host cannot know whether any slot was newer, so the next
 *                                run with PROPAGATE takes the marked tile-kernel instantiation (and an experiment tile
 *                                kernel returns UNSUPPORTED) whenever some table has both columns.
 * The frame is then b200vis_read_tables, b200vis_step(ctx, 0, NULL, NULL, ...) (or the runs), the write-back, one
 * b200vis_synchronize.  The caller leaves the columns alone until that synchronize.  Errors: NOT_READY (no tables
 * registered), UNSUPPORTED (world_size > 1). */
#define B200VIS_RD_TRANSFORM        0x1u
#define B200VIS_RD_GLOBAL_TRANSFORM 0x2u
#define B200VIS_RD_CULL_INPUTS      0x4u   /* b200vis_set_table_cull_inputs' columns, see below */
B200VIS_API int32_t b200vis_read_tables(b200vis_ctx *ctx, uint32_t which, uint32_t last_run, uint32_t this_run);

/* ---- reading the cull inputs (Aabb, Sphere, InheritedVisibility) straight from the same tables ------------------------------
 * Aabb (primitives.rs:65) and Sphere (primitives.rs:199) are repr(Rust): their layouts are passed in (size_of and offset_of!
 * of their fields).  Every field is f32: center and half_extents are lanes 0-2 of a Vec3A, radius one float.
 * The other inputs of check_visibility_cpu_culling (Has<NoFrustumCulling>, Has<VisibilityRange>, Without<NoCpuCulling>, a
 * point light's Sphere rebuilt from its GlobalTransform) are fixed for an archetype, so they are given once per table in
 * `flags`.  VisibilityClass and RenderLayers are not read: b200vis_upload_bounds carries them.  The VisibilityRange
 * parameters come from the tables through b200vis_set_table_visibility_ranges, or as rows through
 * b200vis_upload_visibility_ranges; without either, b200vis_upload_bounds carries the VisibleEntityRanges mask. */
typedef struct b200vis_bounds_layout {
    uint32_t aabb_stride, aabb_center, aabb_half_extents;   /* bytes; each field is 3 floats */
    uint32_t sphere_stride, sphere_center, sphere_radius;   /* center 3 floats, radius 1 float */
} b200vis_bounds_layout;
typedef struct b200vis_table_cull_inputs {
    const void     *aabbs;                 /* [capacity] Aabb; NULL = the archetype has no Aabb */
    const uint32_t *aabb_changed_ticks;    /* [capacity]; NULL exactly when aabbs is */
    const void     *spheres;               /* [capacity] Sphere; NULL = no Sphere */
    const uint32_t *sphere_changed_ticks;  /* [capacity]; NULL exactly when spheres is */
    const uint8_t  *inherited_visibility;  /* [capacity] InheritedVisibility (bool); NULL = not in the visibility query */
    const uint32_t *iv_changed_ticks;      /* [capacity]; NULL exactly when inherited_visibility is */
    uint32_t        flags;                 /* per-archetype bits only: B200VIS_F_NO_FRUSTUM_CULLING | _HAS_VIS_RANGE |
                                              _NO_CPU_CULLING | _SPHERE_FROM_GT */
} b200vis_table_cull_inputs;
/* inputs[t] belongs to table t of the current registry: n_tables must equal its size.  The call replaces the previous
 * cull inputs.  An entry with every pointer NULL and flags 0 leaves its table unread.  b200vis_set_tables / _ex replace
 * the registry and drop all cull inputs (nothing is read for them until this call attaches them again); the columns of a
 * table whose registry entry did not change stay registered until then.
 * The columns are registered, merged with the output and input columns, kept and released by the code of
 * b200vis_set_tables_ex, and the page rules above apply to them.
 * When table t's entry (its pointers, its flags, or the part of the layout it uses) differs from entry t of the previous
 * call, every slot of the table is read in full at the next RD_CULL_INPUTS read: a reallocated table, a table that had no
 * cull inputs before.
 * B200VIS_RD_CULL_INPUTS gives each row the device state b200vis_upload_bounds gives it for the row's bounds and flags
 * (class mask, RenderLayers and the range mask stay as they are).  A slot is considered when it is below len, is mapped
 * to a live row and its table is read.  It is read in full when it was (re)mapped by b200vis_set_table_rows since the
 * last RD_CULL_INPUTS read, or its table was (re)attached as above; otherwise each column is read only where its tick is
 * newer by the Tick::is_newer_than rule of b200vis_read_tables.
 *   flags    (full read) the table's flags, | HAS_AABB if it has aabbs, | HAS_SPHERE if it has spheres and no aabbs
 *            (Aabb takes precedence, visibility/mod.rs:824-843), | INHERITED_VISIBLE if the byte is nonzero; the row's
 *            Changed<Transform> mark is kept
 *   Aabb     (full read or newer tick) bounds = center.xyz, half_extents.xyz
 *   Sphere   (a table without aabbs; full read or newer tick) bounds = center.xyz, radius, 0, 0
 *   InheritedVisibility (newer tick) bit INHERITED_VISIBLE of the flags only
 * A table with neither Aabb nor Sphere leaves the rows' bounds as they are.  Rows in no read table keep what
 * b200vis_upload_bounds gave them.  The maps' "(re)mapped" marks survive an RD_TRANSFORM read and
 * b200vis_compact_topology; b200vis_set_topology unmaps every slot, so the rows mapped again are read in full.
 * Errors: INVALID_ARG (n_tables differs from the registry's size, only one pointer of a column pair NULL, a pointer not
 * 4-byte aligned, a layout field not 4-byte aligned, overlapping or past its stride, no layout while some table has aabbs
 * or spheres, flags other than the four per-archetype bits, a table whose B200VIS_F_HAS_VIS_RANGE differs from whether
 * it has an attached VisibilityRange column, see b200vis_set_table_visibility_ranges), NOT_READY (no tables registered), UNSUPPORTED
 * (world_size > 1); nothing changes then.  On B200VIS_ERR_CUDA the registry is left empty when cudaHostRegister refused
 * the memory, and otherwise every cull input and the VisibilityRange attachment are detached (the next calls read every
 * table they attach in full). */
B200VIS_API int32_t b200vis_set_table_cull_inputs(b200vis_ctx *ctx, uint32_t n_tables, const b200vis_table_cull_inputs *inputs,
                                                  const b200vis_bounds_layout *layout);

/* ---- SURVEY.md 8(f) N1: the render world's visible-entity diff ---------------------------------------------
 * RenderVisibleEntitiesClass::update_cpu_culled_entities (crates/bevy_render/src/view/visibility/mod.rs:194-249)
 * marches over last frame's and this frame's sorted list to find the newly added and newly removed entities.  With
 * the diff enabled the CULL stage produces both lists on the device (set algebra on the rank-ordered bit sets, ordered
 * emit), so the shim can feed `added_entities` / `removed_entities` directly and skip the download of the full lists.
 * Rows ascend by Entity::to_bits() like the lists themselves.  "Last frame" = the last frame the view was active; an
 * inactive view reports nothing.  Enabling the diff and b200vis_set_topology (row identities change) reset the old
 * list to empty: the next frame reports every visible row as added, and the shim drops its render-world list. */
B200VIS_API int32_t b200vis_enable_visible_diff(b200vis_ctx *ctx, int32_t enabled);
B200VIS_API int32_t b200vis_download_visible_diff(b200vis_ctx *ctx, uint32_t view, uint32_t *added_rows, uint32_t added_capacity,
                                                  uint32_t *n_added, uint32_t *removed_rows, uint32_t removed_capacity,
                                                  uint32_t *n_removed);
/* Sink form (pinned host memory written by the GPU right after the CULL stage, like b200vis_set_result_sink):
 * rows[2][max_views][capacity] (0 = added, 1 = removed), counts[max_views][2]; a list longer than `capacity` is
 * truncated (the count still says how long it was).  A result sink whose visible_rows is NULL then keeps the full
 * lists on the device.  NULL, 0, NULL removes the sink. */
B200VIS_API int32_t b200vis_set_visible_diff_sink(b200vis_ctx *ctx, uint32_t *rows, uint32_t capacity, uint32_t *counts);
/* The camera half of collect_visible_cpu_culled_entities (render view/visibility/mod.rs:389-431) as Entity values: one
 * diff per (camera, VisibilityClass), against the lists last reported for that camera.  The caller gives each view a diff
 * slot with b200vis_set_view_diff_slots: a persistent identity for one camera's RenderVisibleEntities, so the diff does
 * not depend on the order of the view query, which may change from frame to frame.  A slot holds eight sets, one per
 * class (bit k of b200vis_upload_bounds' class mask), with the lists last reported for it.  Every run that culls then,
 * on the frame's tail behind the visible-list expansion (pipelined STAGE_ALL, B200VIS_PIPELINE=0, b200vis_step, CULL-only
 * runs, more than eight views, recorded frame constants, after edits and compactions; readable after the next
 * b200vis_synchronize):
 *   - an active view with a slot: for each class k, added_k = list_k \ prev[slot][k] and removed_k = prev[slot][k] \
 *     list_k, both ascending by to_bits() (MainEntity order: the march compares main entities only, mod.rs:213-231, so
 *     pairing each entry with a render entity is the shim's job, Entity::PLACEHOLDER for meshes); then prev[slot][k] :=
 *     list_k.  list_k is the view's VisibleEntities list of class k, as b200vis_set_visible_entities_sink writes it.
 *   - an inactive view (B200VIS_VIEW_ACTIVE clear) with a slot: empty lists, and the slot is emptied.  The render world
 *     removes RenderVisibleEntities from an inactive camera (render camera.rs:515-525, 549-575): when it is active again,
 *     everything is added.
 *   - a slot no view of the run names: emptied.
 *   - a view without a slot: empty lists.
 * Written, with list l = view * 8 + k for the views 0 .. n_views-1 of the frame:
 *   added_offsets / removed_offsets[0 .. n_views*8]  exclusive prefix sums; list l of added is added[added_offsets[l] ..
 *                            added_offsets[l+1]), likewise removed.  The last offset is the true total, even past the
 *                            capacity; no entry at or past the capacity is written, nothing past list n_views*8.
 *   added / removed          Entity::to_bits() of the entries.
 * b200vis_set_topology empties every slot (the rows' identities change).  b200vis_edit_topology and
 * b200vis_compact_topology carry the slots across: a despawned entity in a slot's set is reported removed with its own
 * entity bits by the next run (a compaction keeps it as a tombstone until then), spawned entities are added when they
 * are listed.  The camera diff of b200vis_enable_visible_diff is independent of this one and unchanged by it.
 * Pinned or registered like the result sink.  Registering allocates, for max_slots slots, the eight sets per slot and
 * their per-chunk counts, plus the run's added / removed bits and per-chunk counts: max_slots x (24 x words + 9 x
 * chunks) x 4 bytes, words = max_entities / 32 and chunks = words / 1024 rounded up (about 3 MB per slot at one million
 * rows), and 2 x (max_views x 8 + 1) offsets.  Every slot starts empty and no view has a slot until the slots are set.
 * While the sink is set the entity keys stay resident on the device.  NULL removes the sink and frees the sets.
 * Errors, with nothing changed: INVALID_ARG (a NULL pointer, a zero capacity, added / removed not 8-byte aligned),
 * UNSUPPORTED (world_size > 1). */
#define B200VIS_VIEW_NO_SLOT 0xFFFFFFFFu
typedef struct b200vis_view_diff_sink {
    uint64_t *added;            /* [added_capacity] every list's added Entity::to_bits(), back to back */
    uint32_t  added_capacity;
    uint64_t *removed;          /* [removed_capacity] every list's removed entries, back to back */
    uint32_t  removed_capacity;
    uint32_t *added_offsets;    /* [max_views * 8 + 1] */
    uint32_t *removed_offsets;  /* [max_views * 8 + 1] */
    uint32_t  max_slots;        /* slots are 0 .. max_slots - 1 */
} b200vis_view_diff_sink;
B200VIS_API int32_t b200vis_set_view_diff_sink(b200vis_ctx *ctx, const b200vis_view_diff_sink *sink);
/* View i gets slot slots[i] (B200VIS_VIEW_NO_SLOT = none); views at or past n_views have no slot.  The map holds from the
 * next run that culls until it is set again; a pipelined frame's tail uses the map of its own run.  Errors, with nothing
 * changed: INVALID_ARG (n_views > max_views, slots NULL with n_views > 0, a slot >= max_slots, the same slot twice),
 * NOT_READY (no b200vis_set_view_diff_sink registered). */
B200VIS_API int32_t b200vis_set_view_diff_slots(b200vis_ctx *ctx, uint32_t n_views, const uint32_t *slots);

/* ---- SURVEY.md 8(f) N3: shadow-view culling of point lights -------------------------------------------------------
 * check_point_light_mesh_visibility (crates/bevy_light/src/lib.rs:517-668): for every point light that is in some
 * view's VisibleEntities and has shadow maps enabled, every shadow-casting mesh is tested against the light's range
 * sphere (Sphere::intersects_obb, bevy_camera/src/primitives.rs:219-226) and the six CubemapFrusta
 * (Frustum::intersects_obb with near and far planes, :272-294); survivors are set_visible() and land in the light's
 * six sorted CubemapVisibleEntities lists.
 *   caster[count]   1 = the row is in visible_entity_query (Mesh3d, no NotShadowCaster, no DirectionalLight);
 *                   NoCpuCulling, InheritedVisibility, RenderLayers, Aabb, NoFrustumCulling, VisibilityRange come from
 *                   the columns already resident
 *   shadow lights   ordinals into the b200vis_set_lights arrays (the lights with shadow_maps_enabled), their
 *                   CubemapFrusta frusta[n][6 faces][6 half spaces][4] (update_point_light_frusta,
 *                   bevy_light/src/point_light.rs:212-265; b200vis_host_point_light_frusta computes them for hosts
 *                   without glam), RenderLayers (NULL = default), and the bit of get_shadow_lod_origin's view in the
 *                   VisibleEntityRanges masks (-1 = none).  Whether a light is in some view's VisibleEntities is
 *                   decided on the device from the per-view sets of the visible-diff bookkeeping (which
 *                   b200vis_upload_shadow_casters switches on: call it before the frame's CULL stage); the light's
 *                   sphere is its row's GlobalTransform translation and its range.
 *   b200vis_run_shadow_culling  after b200vis_run(.. CULL ..) of the same frame; also folds set_visible() into the
 *                   ViewVisibility column / change flags (download them afterwards).
 *   lists           rows ascending by Entity::to_bits() (sort_unstable, lib.rs:650-661); list_capacity rows per list
 *                   are kept (0 = max_entities). */
B200VIS_API int32_t b200vis_upload_shadow_casters(b200vis_ctx *ctx, uint32_t first_row, uint32_t count, const uint8_t *caster);
B200VIS_API int32_t b200vis_set_shadow_lights(b200vis_ctx *ctx, uint32_t n_lights, const uint32_t *light_ordinals, const float *frusta,
                                              const uint64_t *layer_mask, int32_t lod_origin_range_index, uint32_t list_capacity);
/* The general form: point lights, SPOT lights (the second half of check_point_light_mesh_visibility, lib.rs:670-749: one
 * Frustum, near and far planes tested, the same range-sphere pre-test) and DIRECTIONAL-light cascades
 * (check_dir_light_mesh_visibility, lib.rs:342-510: one item per (light, view, cascade) with that cascade's Frustum; the near
 * plane is not tested, :455-458; there is no range sphere; the caller lists only lights with shadow_maps_enabled that are
 * visible, :395-399).  A point / spot item names the light's ROW (spot lights are not clustered, so they have no ordinal);
 * it takes part only while that row is in some view's VisibleEntities.  range_view_index = the bit of the
 * VisibleEntityRanges masks that gates rows with a VisibilityRange: the shadow LOD origin's for point / spot lights, the
 * cascade's own view for directional lights; -1 = that view is not in the map (ranged rows are then skipped).
 * Lists: b200vis_download_shadow_visible(item, face) with face 0 for spot lights and cascades. */
#define B200VIS_SHADOW_POINT 0u
#define B200VIS_SHADOW_SPOT 1u
#define B200VIS_SHADOW_DIRECTIONAL_CASCADE 2u
typedef struct b200vis_shadow_item {
    uint32_t kind;
    uint32_t light_row;          /* point / spot */
    float    range;              /* point / spot: PointLight::range / SpotLight::range */
    int32_t  range_view_index;
    uint64_t layer_mask;         /* the light's RenderLayers, block 0 (default layer = 1); blocks 1..3:
                                    b200vis_set_shadow_item_render_layers_ext */
    float    frusta[6][6][4];    /* point: the six CubemapFrusta faces; spot / cascade: frusta[0] */
} b200vis_shadow_item;
B200VIS_API int32_t b200vis_set_shadow_items(b200vis_ctx *ctx, uint32_t n_items, const b200vis_shadow_item *items, uint32_t list_capacity);
/* RenderLayers blocks 1..3 (layers 64..255) of the installed shadow items: blocks[n_items][3] in item order, NULL = all
 * empty.  Call it after b200vis_set_shadow_items / _ex / b200vis_set_shadow_lights, each of which empties them again.  The
 * shadow cull then tests the light's whole RenderLayers against each row's (lib.rs:437, 611, 703; render_layers.rs:121-135):
 * block 0 against the rows' layer_mask, blocks 1..3 against their b200vis_upload_render_layers_ext blocks.
 * Errors: INVALID_ARG (n_items is not the installed item count), UNSUPPORTED (world_size > 1); nothing changes then. */
B200VIS_API int32_t b200vis_set_shadow_item_render_layers_ext(b200vis_ctx *ctx, uint32_t n_items, const uint64_t *blocks);
B200VIS_API int32_t b200vis_run_shadow_culling(b200vis_ctx *ctx);
B200VIS_API int32_t b200vis_download_shadow_visible(b200vis_ctx *ctx, uint32_t shadow_light, uint32_t face, uint32_t *rows,
                                                    uint32_t capacity, uint32_t *count);
/* The shadow lists as Entity values (CubemapVisibleEntities faces, the spot light's VisibleMeshEntities, a cascade's
 * VisibleMeshEntities), every list of the run back to back in one region; list l = item * 6 + face.  Each entry is
 * Entity::to_bits() as given to b200vis_set_topology / b200vis_edit_topology, so the shim fills each list with one
 * extend_from_slice, as for b200vis_set_visible_entities_sink.  While the sink is registered, every
 * b200vis_run_shadow_culling writes, on the context's stream (readable after the next b200vis_synchronize):
 *   offsets[0 .. n_items*6]  exclusive prefix sums over the lists in item order: list l is entities[offsets[l] ..
 *                            offsets[l+1]); faces 1-5 of spot and cascade items are empty.  offsets[n_items*6] is the
 *                            true total, even when it exceeds capacity.
 *   active[0 .. n_items)     1 when item i was culled this run: a point / spot item whose light is in some view's
 *                            VisibleEntities (lib.rs:561-563), and every cascade item; 0 otherwise.  The lists of an
 *                            inactive item are empty ranges, and its CubemapVisibleEntities / VisibleMeshEntities keep
 *                            what they held (the reference `continue`s past such a light, lib.rs:568-586).
 *   entities                 each list ascending by to_bits() (sort_unstable, lib.rs:493, 666, 745); no entry at or past
 *                            capacity is written.
 * Nothing past item n_items is written.  The lists come from the bit sets, not from the row lists, so the row lists can be
 * kept at list_capacity = 1 (b200vis_download_shadow_visible then truncates, as it does today).  Pinned or registered
 * like the result sink.  While the sink is set the entity keys stay resident on the device (8 bytes per max_entities
 * row).  NULL removes the sink.
 * Errors: INVALID_ARG (capacity 0, a NULL pointer, entities not 8-byte aligned), CAPACITY (max_items below the installed
 * item count; b200vis_set_shadow_items / b200vis_set_shadow_lights with more items than a registered sink's max_items
 * give CAPACITY too, and change nothing), UNSUPPORTED (world_size > 1). */
typedef struct b200vis_shadow_entities_sink {
    uint64_t *entities;   /* [capacity] every list of the run back to back; list l = item * 6 + face */
    uint32_t  capacity;   /* entries in all lists together */
    uint32_t  max_items;  /* offsets has max_items * 6 + 1 entries, active has max_items */
    uint32_t *offsets;    /* [max_items * 6 + 1] */
    uint8_t  *active;     /* [max_items] */
} b200vis_shadow_entities_sink;
B200VIS_API int32_t b200vis_set_shadow_entities_sink(b200vis_ctx *ctx, const b200vis_shadow_entities_sink *sink);
/* Writes the lists of the last b200vis_run_shadow_culling again, into the entity sink registered now: offsets, active
 * flags and entities exactly as that run would have written them into this sink.  This is how a caller recovers from a
 * sink that was too small: run, b200vis_synchronize, see offsets[n_items*6] > capacity, register a larger sink, emit,
 * b200vis_synchronize.  Running the shadow stage again instead would not give the same result, because every run moves the
 * shadow-diff slots forward.
 * Enqueued on the context's stream.  It runs no cull and changes nothing else: not the ViewVisibility bits or change
 * flags, not the frame statistics, not the row lists of b200vis_download_shadow_visible, and not the shadow-diff slots or
 * the diff sink's outputs.  For this, every run made while an entity sink is registered keeps a device copy of its
 * bit sets (n_items x 6 x max_entities / 8 bytes, copied before the lists are expanded).
 * Errors, with nothing enqueued: NOT_READY (no entity sink registered; no run with an entity sink registered since the
 * last b200vis_set_shadow_items / _ex, b200vis_set_shadow_lights, b200vis_set_topology, b200vis_edit_topology or
 * b200vis_compact_topology, any of which may change the items, the rows or their rank order), CAPACITY (the sink's
 * max_items below the installed item count: a safeguard, since b200vis_set_shadow_entities_sink and the item setters
 * already refuse that combination), UNSUPPORTED (world_size > 1). */
B200VIS_API int32_t b200vis_emit_shadow_entities(b200vis_ctx *ctx);
/* The shadow lists' changes: what collect_visible_cpu_culled_entities computes for the light subviews (render
 * view/visibility/mod.rs:333-381 calling update_cpu_culled_entities, :194-249), as Entity values.  The caller gives each
 * item a diff slot with b200vis_set_shadow_items_ex: a persistent identity for the item's RetainedViewEntity (one per
 * (point light, face), (spot light, 0), (directional light, view, cascade); bevy_pbr render/light.rs:511-551), so the
 * diff does not depend on the items' order, which may change from frame to frame.  A slot holds six sets, one per face,
 * with the lists last reported for it; faces past an item's own are empty lists.  Every b200vis_run_shadow_culling then,
 * on the context's stream (readable after the next b200vis_synchronize):
 *   - an active item with a slot (the entity sink's active byte 1): for each face f, added = list_f \ prev[slot][f] and
 *     removed = prev[slot][f] \ list_f, both ascending by to_bits(); then prev[slot][f] := list_f.  (The render-world
 *     Entity of a mesh is Entity::PLACEHOLDER, mod.rs:78-81: the main-world key decides.)
 *   - an inactive item with a slot: empty lists, and the slot is emptied;
 *   - a slot no item of the run names: emptied.  Both follow the render world, which drops the
 *     RenderShadowMapVisibleEntities of a light it did not extract (light.rs:468, 482-487, 940-951): when the light comes
 *     back, every entity is added.  A slot survives a run only if an active item names it, so no "clear" call is needed.
 *   - an item without a slot (B200VIS_SHADOW_NO_SLOT) has no diff: its lists are empty ranges.
 * Written, with list l = item * 6 + face in item order as in the entity sink:
 *   added_offsets / removed_offsets[0 .. n_items*6]  exclusive prefix sums; list l of added is added[added_offsets[l] ..
 *                            added_offsets[l+1]), likewise removed.  The last offset is the true total, even past the
 *                            capacity; no entry at or past the capacity is written.  Nothing past item n_items is written.
 *   added / removed          Entity::to_bits() of the entries.
 * The sets are bit sets over the rank order (ascending to_bits()).  b200vis_set_topology empties every slot (the rows'
 * identities change), as it does the camera diff.  b200vis_edit_topology and b200vis_compact_topology carry the slots
 * across: a despawned row in a slot's set is reported removed with its own entity bits by the next run (a compaction keeps
 * it as a tombstone until then), spawned rows are added when they are listed.
 * The diff works with or without the entity sink and with list_capacity = 1.  Pinned or registered like the result sink.
 * Registering allocates max_slots x 6 rank-ordered sets and their per-chunk counts (max_slots x 6 x (words + chunks) x 4
 * bytes, words = max_entities / 32 rounded up: about 0.75 MB per slot at one million rows), plus the run's added / removed
 * bits (2 x max_items x 6 sets); every slot starts empty, and the installed items have no slot until items are set again.
 * While the sink is set the entity keys stay resident on the device.  NULL removes the sink and frees the sets.
 * Errors, with nothing changed: INVALID_ARG (a NULL pointer, a zero capacity, added / removed not 8-byte aligned),
 * CAPACITY (max_items below the installed item count; b200vis_set_shadow_items / _ex / b200vis_set_shadow_lights with more
 * items than a registered sink's max_items), UNSUPPORTED (world_size > 1). */
#define B200VIS_SHADOW_NO_SLOT 0xFFFFFFFFu
typedef struct b200vis_shadow_diff_sink {
    uint64_t *added;            /* [added_capacity] every list's added entries, back to back */
    uint32_t  added_capacity;
    uint64_t *removed;          /* [removed_capacity] every list's removed entries, back to back */
    uint32_t  removed_capacity;
    uint32_t *added_offsets;    /* [max_items * 6 + 1] */
    uint32_t *removed_offsets;  /* [max_items * 6 + 1] */
    uint32_t  max_items;
    uint32_t  max_slots;        /* slots are 0 .. max_slots - 1 */
} b200vis_shadow_diff_sink;
B200VIS_API int32_t b200vis_set_shadow_diff_sink(b200vis_ctx *ctx, const b200vis_shadow_diff_sink *sink);
/* b200vis_set_shadow_items with a diff slot per item (diff_slots[n_items], B200VIS_SHADOW_NO_SLOT = none); diff_slots ==
 * NULL is exactly b200vis_set_shadow_items.  Errors, with nothing changed: INVALID_ARG (a slot >= max_slots, the same
 * slot twice), NOT_READY (slots without a registered b200vis_set_shadow_diff_sink), CAPACITY (as above), and those of
 * b200vis_set_shadow_items. */
B200VIS_API int32_t b200vis_set_shadow_items_ex(b200vis_ctx *ctx, uint32_t n_items, const b200vis_shadow_item *items,
                                                uint32_t list_capacity, const uint32_t *diff_slots);
/* The shadow-caster byte from the archetype tables: is_caster[t] = 1 when table t's archetype is in the light systems'
 * visible_entity_query (With<Mesh3d>, Without<NotShadowCaster>, Without<DirectionalLight>; NoCpuCulling is a flag of
 * the cull inputs, lib.rs:526-537, 690-701).  n_tables must equal the registry's size.  Like
 * b200vis_upload_shadow_casters, the first attach allocates the caster column and switches on the visible-set
 * bookkeeping.  While attached, b200vis_read_tables(B200VIS_RD_CULL_INPUTS, ..) writes the caster byte of every slot it
 * reads in full (b200vis_set_table_cull_inputs says which), and a table whose is_caster differs from the previous attach
 * (every table, on an attach after none) is read in full at the next such read.  Rows of tables that are not read keep
 * the byte b200vis_upload_shadow_casters gave them.  b200vis_set_tables / _ex drop the attachment as they drop the cull
 * inputs; NULL, 0 detaches.
 * Errors: INVALID_ARG (n_tables differs from the registry's size, is_caster NULL with n_tables > 0), NOT_READY (no tables
 * registered), UNSUPPORTED (world_size > 1); nothing changes then. */
B200VIS_API int32_t b200vis_set_table_shadow_casters(b200vis_ctx *ctx, uint32_t n_tables, const uint8_t *is_caster);
/* update_point_light_frusta for one light (no GPU needed): light_gt12 as in upload_global_transforms */
B200VIS_API void b200vis_host_point_light_frusta(const float *light_gt12, float range, float shadow_map_near_z, float frusta[6][6][4]);

/* ---- SURVEY.md 8(f) N4: the two per-entity passes that feed the cull kernel's flag byte ---------------------------
 * (a) check_visibility_ranges (crates/bevy_camera/src/visibility/range.rs:230-284).  With the VisibilityRange columns
 *     resident -- start_end[count][2] = (start_margin.start, end_margin.end), the two values is_visible_at_all reads
 *     (range.rs:157-159), and use_aabb[count] -- the cull phase evaluates the distance test itself on this frame's
 *     GlobalTransform instead of taking an uploaded range_mask, and keeps the masks for download
 *     (VisibleEntityRanges::entities; 0 = no entry).  Range views: the translations of the views the system indexes, in
 *     its view-query order (only the first 32 count, :247); b200vis_view.range_view_index maps a culled view to its bit. */
B200VIS_API int32_t b200vis_upload_visibility_ranges(b200vis_ctx *ctx, uint32_t first_row, uint32_t count, const float *start_end,
                                                     const uint8_t *use_aabb);
B200VIS_API int32_t b200vis_set_visibility_range_views(b200vis_ctx *ctx, uint32_t n_views, const float *positions /* [n][3] */);
B200VIS_API int32_t b200vis_download_visibility_ranges(b200vis_ctx *ctx, uint32_t first_row, uint32_t count, uint32_t *mask);
/*     The same VisibilityRange columns straight from the archetype tables.  VisibilityRange (range.rs:80-112) is
 *     repr(Rust): its layout is passed in (size_of, and offset_of! of start_margin.start, end_margin.end and use_aabb).
 *     ranges[t] belongs to table t of the current registry: n_tables must equal its size.  Like
 *     b200vis_upload_visibility_ranges, the first attach allocates the resident range columns, after which
 *     b200vis_set_visibility_range_views works and the cull phase evaluates the masks itself.  The columns are
 *     registered, kept and released by the code of b200vis_set_tables_ex, and the page rules above apply to them.
 *     b200vis_set_tables / _ex drop the attachment; NULL, 0 detaches.
 *     While attached, b200vis_read_tables(B200VIS_RD_CULL_INPUTS, ..) also writes a row's range parameters:
 *       (start_margin.start, end_margin.end) and use_aabb != 0, on every full read of its slot
 *       (b200vis_set_table_cull_inputs says which), and where the slot's range tick is newer by the Tick::is_newer_than
 *       rule of b200vis_read_tables.  A table whose entry (its pointers, or the layout) differs from the previous attach
 *       is read in full at the next such read: a reallocated table, a table newly given ranges, and every table on an
 *       attach after a detach or before any attach.  b200vis_set_tables / _ex drop the attachment but, as for the
 *       cull inputs, a table whose registry entry did not change keeps its entry for that comparison (and its columns
 *       stay registered), so attaching it again unchanged reads nothing in full -- unless an RD_CULL_INPUTS read ran
 *       in between: that read may have read slots in full without their range parameters, so the kept entries are
 *       dropped and the next attach reads every ranged table in full.
 *     Rule: no row is range-tested with parameters nobody supplied.  B200VIS_F_HAS_VIS_RANGE stays a per-archetype bit of
 *     the cull inputs' flags, so while ranges are attached a table has a range column exactly when its attached cull
 *     inputs carry B200VIS_F_HAS_VIS_RANGE (a table without cull inputs has none).  An attach that breaks this, and a
 *     b200vis_set_table_cull_inputs that would break it while ranges are attached, fail with INVALID_ARG; to change which
 *     tables are ranged, detach the ranges first.  Rows in no table keep what b200vis_upload_visibility_ranges gave them.
 *     Errors: INVALID_ARG (n_tables differs from the registry's size, the rule above, only one pointer of a pair NULL, a
 *     pointer not 4-byte aligned, a float field or the stride not 4-byte aligned, a field past the stride, fields
 *     overlapping each other or the use_aabb byte, no layout while some table has ranges), NOT_READY (no tables
 *     registered), UNSUPPORTED (world_size > 1); nothing changes then.  On B200VIS_ERR_CUDA the registry is left empty
 *     when cudaHostRegister refused the memory, and otherwise both the ranges and the cull inputs are detached (the
 *     registrations may have moved under either; the next calls read every table they attach in full). */
typedef struct b200vis_visibility_range_layout {
    uint32_t stride;    /* size_of::<VisibilityRange>() */
    uint32_t start;     /* offset_of!(VisibilityRange, start_margin.start), f32 */
    uint32_t end;       /* offset_of!(VisibilityRange, end_margin.end), f32 */
    uint32_t use_aabb;  /* offset_of!(VisibilityRange, use_aabb), bool (1 byte, nonzero = true) */
} b200vis_visibility_range_layout;
typedef struct b200vis_table_visibility_ranges {
    const void     *ranges;         /* [capacity] VisibilityRange; NULL = the archetype has none */
    const uint32_t *changed_ticks;  /* [capacity]; NULL exactly when ranges is */
} b200vis_table_visibility_ranges;
B200VIS_API int32_t b200vis_set_table_visibility_ranges(b200vis_ctx *ctx, uint32_t n_tables, const b200vis_table_visibility_ranges *ranges,
                                                        const b200vis_visibility_range_layout *layout);
/* (b) visibility_propagate_system (crates/bevy_camera/src/visibility/mod.rs:638-729).  visibility[count]: 0 Inherited,
 *     1 Hidden, 2 Visible (the enum's order, :83-96), | 4 when the entity lacks Visibility / InheritedVisibility.
 *     b200vis_propagate_visibility walks the same level-ordered tiles as the transform propagation and leaves every
 *     InheritedVisibility (bit 0 of the flags column the cull phase reads) at the value the reference's change-driven
 *     system converges to; a parent that is a root's absence, lacks the components, or is B200VIS_DETACHED counts as
 *     visible (:655-659).  changed[i] = 1 where the value was rewritten (set-if-different, :667), i.e. where the shim
 *     stamps InheritedVisibility's change tick. */
#define B200VIS_VISIBILITY_INHERITED 0u
#define B200VIS_VISIBILITY_HIDDEN 1u
#define B200VIS_VISIBILITY_VISIBLE 2u
#define B200VIS_VISIBILITY_NO_COMPONENTS 4u
B200VIS_API int32_t b200vis_upload_visibility(b200vis_ctx *ctx, uint32_t first_row, uint32_t count, const uint8_t *visibility);
B200VIS_API int32_t b200vis_propagate_visibility(b200vis_ctx *ctx);
B200VIS_API int32_t b200vis_download_inherited_visibility(b200vis_ctx *ctx, uint32_t first_row, uint32_t count, uint8_t *inherited,
                                                          uint8_t *changed);

/* ---- SURVEY.md 8(f) N2: Clusters -> ViewClusterBindings ----------------------------------------------------------
 * extract_clusters_for_cpu_clustering + prepare_clusters_for_cpu_clustering (crates/bevy_pbr/src/cluster/mod.rs:394-582)
 * flatten each view's per-cluster Vec<Entity> into the two GPU buffers of ViewClusterBindings (:584-800).  With a mode
 * set, the CLUSTER_LISTS stage emits that wire format directly from the device CSR:
 *   STORAGE  offsets_and_counts[n_clusters][8] = (offset, point_lights, spot, rect | probes, volumes, decals, 0);
 *            index_lists[n_indices] u32
 *   UNIFORM  offsets_and_counts[4096] = pack_offset_and_counts (:855-859); index_lists[4096] = 16384 8-bit slots,
 *            truncated at ViewClusterBindings::MAX_INDICES exactly like the reference's record loop (:505-514)
 * gpu_index_of_light[n_map] = GlobalClusterableObjectMeta::entity_to_index for each light ordinal (NULL = the ordinal
 * itself); ordinals without an entry get the dummy index !0 (:703-705). */
#define B200VIS_BINDINGS_OFF 0u
#define B200VIS_BINDINGS_STORAGE 1u
#define B200VIS_BINDINGS_UNIFORM 2u
B200VIS_API int32_t b200vis_set_cluster_bindings(b200vis_ctx *ctx, uint32_t mode, const uint32_t *gpu_index_of_light, uint32_t n_map);
/* capacities in 32-bit words; n_offsets / n_indices = ViewClusterBindings::n_offsets / n_indices */
B200VIS_API int32_t b200vis_download_cluster_bindings(b200vis_ctx *ctx, uint32_t view, uint32_t *offsets_and_counts, uint32_t oc_capacity,
                                                      uint32_t *index_lists, uint32_t il_capacity, uint32_t *n_offsets,
                                                      uint32_t *n_indices);

/* ---- multi-GPU cluster exchange (one all-gather per frame, done by the host's collective) ------- */
/* Each rank fills `slab_bytes` at `send`; after all-gathering the slabs rank-major into `recv`
 * (world_size * slab_bytes) the LISTS stage reads `recv`.  Buffers are caller-allocated device memory
 * (e.g. torch tensors); with world_size <= 1 the library uses its own buffer and no exchange. */
/* Built-in exchange: the library dlopen()s libnccl.so.2 (the copy the host process already loaded, e.g. torch's), rank 0
 * makes a unique id, the host broadcasts those 128 bytes by any means, every rank calls b200vis_comm_init (a collective),
 * and from then on b200vis_run(B200VIS_STAGE_ALL) issues the ncclAllGather of the slabs itself, on the frame's tail
 * stream, between CLUSTER_ASSIGN and CLUSTER_LISTS -- one call per frame, pipelined like the single-GPU path. */
#define B200VIS_COMM_ID_BYTES 128
B200VIS_API int32_t b200vis_comm_unique_id(uint8_t id[B200VIS_COMM_ID_BYTES]);
B200VIS_API int32_t b200vis_comm_init(b200vis_ctx *ctx, const uint8_t id[B200VIS_COMM_ID_BYTES]);
/* Peer-memory exchange (the default in bench.py): no collective call at all.  Every rank exports the CUDA IPC handle of its
 * gathered buffer, the host all-gathers the 64-byte handles (rank-major) by any means, every rank imports them; from then on
 * b200vis_run(B200VIS_STAGE_ALL) has the rank WRITE its slab into every rank's buffer with plain NVLink stores right after
 * CLUSTER_ASSIGN and publish a per-frame stamp (release, system scope); CLUSTER_LISTS spins on all ranks' stamps (acquire)
 * before reading.  world_size 2..8, all ranks on one node with peer access.  A rank that never arrives is reported as
 * cluster_index_overflow[v] == 2 after a few seconds instead of hanging the GPU. */
#define B200VIS_P2P_HANDLE_BYTES 64
B200VIS_API int32_t b200vis_p2p_export(b200vis_ctx *ctx, uint8_t handle[B200VIS_P2P_HANDLE_BYTES]);
B200VIS_API int32_t b200vis_p2p_import(b200vis_ctx *ctx, const uint8_t *handles /* [world_size][64], rank-major */);
/* One process, several GPUs (a Bevy App is one process): link the contexts of the process directly -- plain peer access, no
 * IPC handles, no collective library.  ctxs[r]: created with world_size = n, rank = r, one device each.  Then one host thread
 * calls b200vis_run(ctxs[r], B200VIS_STAGE_ALL) for every r per frame; the slab exchange happens on the devices. */
B200VIS_API int32_t b200vis_p2p_link(b200vis_ctx *const *ctxs, uint32_t n);
B200VIS_API int32_t b200vis_cluster_exchange_bytes(const b200vis_ctx *ctx, size_t *slab_bytes);
B200VIS_API int32_t b200vis_set_cluster_exchange_buffers(b200vis_ctx *ctx, void *send_device, void *recv_device);

/* ---- host-side mirror of the reference's per-view math (no GPU needed) --------------------------- */
/* PerspectiveProjection::get_clip_from_view (crates/bevy_camera/src/projection.rs:339-343) */
B200VIS_API void b200vis_host_perspective(float fov_y, float aspect, float near_z, float *clip_from_view16);
/* CameraProjection::compute_frustum (projection.rs:72-80): camera_gt[12] as in upload_global_transforms */
B200VIS_API void b200vis_host_compute_frustum(const float *clip_from_view16, const float *camera_gt12, float far_z,
                                  float half_spaces[6][4]);


/* The thresholds the device uses in place of view_z_to_z_slice (assign.rs:1046-1062): thresholds[k-1] is the smallest
 * u = -view_z whose slice index (computed with the HOST's libm, exactly the reference's float expression) is >= k;
 * slice(u) = number of thresholds <= u.  z_slices-1 values (NaN where the slice is never reached). */
B200VIS_API void b200vis_host_z_slice_thresholds(const float cluster_factors[2], uint32_t z_slices, uint32_t is_orthographic,
                                                 float *thresholds);
B200VIS_API void b200vis_host_default_cluster_config(b200vis_cluster_config *cfg, uint32_t screen_w, uint32_t screen_h);
/* The per-view prologue of assign_objects_to_clusters (assign.rs:324-485).  planes_scratch must hold
 * 3*4097*4 floats; out->x/y/z_planes point into it. */
B200VIS_API int32_t b200vis_host_cluster_view_setup(const b200vis_cluster_config *cfg, const float *camera_gt12,
                                        const float *clip_from_view16, const float frustum[6][4],
                                        uint64_t layer_mask, const b200vis_cluster_feedback *feedback,
                                        float *planes_scratch, b200vis_cluster_view *out);

#ifdef __cplusplus
}
#endif
#endif /* B200VIS_H */
