//! b200vis_plugin.rs — the Bevy-side shim for libb200vis (SOURCE ONLY: there is no Rust toolchain in the build image;
//! compile it in a crate that depends on bevy 0.20 and links `b200vis`).  `tests/host_shim.c` performs the same sequence
//! through the same C ABI in plain C and is run against the CPU oracle on the GPU box.
//!
//! The plugin removes four reference system sets from `PostUpdate` / `PostStartup` and adds replacements **with the same
//! query signatures, in the same sets**, that call the C ABI of `include/b200vis.h`:
//!   propagate  <- mark_dirty_trees / propagate_parent_transforms / sync_simple_transforms
//!                 (crates/bevy_transform/src/systems.rs:42, 111, 506; registered at plugins.rs:37-47)
//!   cull       <- check_visibility_cpu_culling (crates/bevy_camera/src/visibility/mod.rs:748) and check_visibility_ranges
//!                 (visibility/range.rs:230: the device evaluates the ranges itself from the tables' VisibilityRange columns)
//!   cluster    <- assign_objects_to_clusters   (crates/bevy_light/src/cluster/assign.rs:137; the only member of
//!                 SimulationLightSystems::AssignLightsToClusters, crates/bevy_light/src/lib.rs:187-191)
//!   light      <- check_point_light_mesh_visibility / check_dir_light_mesh_visibility (crates/bevy_light/src/lib.rs:342, 517;
//!                 SimulationLightSystems::CheckLightVisibility): the shadow lists come back as Entity lists through
//!                 `b200vis_set_shadow_entities_sink`, their set_visible() goes into the tables as a second write-back
//! The `VisibleEntityRanges` resource stays initialised and stays empty: nothing fills it once check_visibility_ranges is
//! gone, and neither the device's camera cull nor its shadow cull reads it (both test the ranges on the device).  Its
//! presence still switches range culling on, as in the reference (visibility/mod.rs:813-819).
//! `reset_view_visibility` and `mark_newly_hidden_entities_invisible` are private and share their sets with systems that
//! must stay, so in an UNFORKED Bevy they keep running on the CPU: the device applies `set_visible()` to the ViewVisibility
//! byte of every slot whose entity is visible in >= 1 view, straight in the archetype tables (`B200VIS_WB_SET_VISIBLE`),
//! reading the byte so that the light-visibility systems (they OR into the same byte) compose correctly (SURVEY.md 8b).
//! With a three-line patch that makes those two systems removable, the device's ViewVisibility bytes + change ticks are
//! written into the tables instead (`forked-bevy` feature below).
//!
//! Data flow (INTEGRATION.md section 2): Transform, other systems' GlobalTransforms, and the cull inputs Aabb, Sphere,
//! InheritedVisibility and VisibilityRange read by the device straight from the archetype tables by their change ticks
//! (`b200vis_set_tables_ex`, `b200vis_set_table_cull_inputs`, `b200vis_set_table_visibility_ranges`,
//! `b200vis_read_tables`), the range masks evaluated on the device; VisibilityClass and RenderLayers -> `upload_bounds`
//! on change (blocks 1..3, layers 64..255, with `upload_render_layers_ext`, `set_view_render_layers_ext` and
//! `set_light_render_layers_ext`; a layer past 255 is an error); results -> pinned host buffers the GPU writes itself (`b200vis_set_result_sink`,
//! and VisibleEntities as per-class Entity lists through `b200vis_set_visible_entities_sink`), read after one
//! `b200vis_synchronize` per system; GlobalTransform and ViewVisibility with their change ticks straight into the archetype
//! tables (`b200vis_writeback_tables`).
#![allow(non_camel_case_types, clippy::too_many_arguments, clippy::type_complexity)]
use bevy::camera::primitives::{Aabb, Frustum, Sphere};
use bevy::camera::visibility::*;
use bevy::camera::{RenderTarget, ShadowLodOrigin};
use bevy::ecs::component::Tick;
use bevy::ecs::entity::EntityHashMap;
use bevy::ecs::schedule::ScheduleCleanupPolicy::RemoveSystemsOnly;
use bevy::ecs::system::SystemChangeTick;
use bevy::camera::primitives::{CascadesFrusta, CubemapFrusta};
use bevy::light::{cluster::*, get_shadow_lod_origin, DirectionalLight, NotShadowCaster, PointLight, SimulationLightSystems, SpotLight};
use bevy::prelude::*;
use bevy::transform::{systems::*, TransformSystems};
use core::any::TypeId;
use core::ffi::c_char;
use core::mem::{offset_of, size_of};

// ---- FFI (mirrors include/b200vis.h, ABI version 2) -----------------------------------------------------------------------
#[repr(C)] pub struct b200vis_ctx { _p: [u8; 0] }
#[repr(C)] pub struct b200vis_config { device: i32, max_entities: u32, max_lights: u32, max_views: u32, max_cluster_indices: u32,
                                        world_size: u32, rank: u32, reserved: u32 }
#[repr(C)] #[derive(Clone, Copy)]
pub struct b200vis_view { half_spaces: [[f32; 4]; 6], layer_mask: u64, flags: u8, range_view_index: i8, pad: [u8; 6] }
#[repr(C)] #[derive(Default)]
pub struct b200vis_frame_stats { visible_count: [u32; 8], cluster_index_count: [u32; 8], cluster_farthest_z: [f32; 8],
                                 cluster_index_overflow: [u32; 8], gt_changed_count: u32, vv_changed_count: u32, frame: u32, pad: u32 }
#[repr(C)] pub struct b200vis_cluster_view { enabled: u32, dims: [u32; 3], tile_size: [u32; 2], is_orthographic: u32, near_z: f32,
    far_z: f32, cluster_factors: [f32; 2], view_from_world: [f32; 16], clip_from_view: [f32; 16], view_from_world_scale: [f32; 3],
    view_from_world_scale_max: f32, frustum: [[f32; 4]; 6], layer_mask: u64, x_planes: *const f32, y_planes: *const f32,
    z_planes: *const f32 }
#[repr(C)] pub struct b200vis_cluster_config { kind: u32, dims: [u32; 3], total: u32, z_slices: u32, first_slice_depth: f32,
    far_z_mode: u32, far_z_constant: f32, dynamic_resizing: u32, screen_w: u32, screen_h: u32, view_cluster_bindings_max_indices: u32 }
#[repr(C)] #[derive(Default, Clone, Copy)]
pub struct b200vis_cluster_feedback { has_farthest_z: u32, farthest_z: f32, has_index_count: u32, index_count: u32 }
#[repr(C)] pub struct b200vis_result_sink { stats: *mut b200vis_frame_stats, visible_rows: *mut u32, visible_capacity: u32,
    visible_classes: *mut u8, cluster_offsets: *mut u32, cluster_indices: *mut u32, cluster_capacity: u32 }
#[repr(C)] pub struct b200vis_visible_entities_sink { entities: *mut u64, capacity: u32, offsets: *mut [u32; 9] }
#[repr(C)] #[derive(Clone, Copy, PartialEq)]
pub struct b200vis_table { global_transforms: *mut GlobalTransform, gt_changed_ticks: *mut Tick, view_visibility: *mut ViewVisibility,
    vv_changed_ticks: *mut Tick, len: u32, capacity: u32 }
#[repr(C)] pub struct b200vis_transform_layout { stride: u32, translation: u32, rotation: u32, scale: u32 }
#[repr(C)] #[derive(Clone, Copy, PartialEq)]
pub struct b200vis_table_inputs { transforms: *const Transform, transform_changed_ticks: *const Tick }
#[repr(C)] pub struct b200vis_bounds_layout { aabb_stride: u32, aabb_center: u32, aabb_half_extents: u32, sphere_stride: u32,
                                             sphere_center: u32, sphere_radius: u32 }
#[repr(C)] #[derive(Clone, Copy, PartialEq)]
pub struct b200vis_table_cull_inputs { aabbs: *const Aabb, aabb_changed_ticks: *const Tick, spheres: *const Sphere,
    sphere_changed_ticks: *const Tick, inherited_visibility: *const InheritedVisibility, iv_changed_ticks: *const Tick, flags: u32 }
#[repr(C)] pub struct b200vis_visibility_range_layout { stride: u32, start: u32, end: u32, use_aabb: u32 }
#[repr(C)] #[derive(Clone, Copy, PartialEq)]
pub struct b200vis_table_visibility_ranges { ranges: *const VisibilityRange, changed_ticks: *const Tick }
#[repr(C)] pub struct b200vis_shadow_item { kind: u32, light_row: u32, range: f32, range_view_index: i32, layer_mask: u64,
                                           frusta: [[[f32; 4]; 6]; 6] }
#[repr(C)] pub struct b200vis_shadow_entities_sink { entities: *mut u64, capacity: u32, max_items: u32, offsets: *mut u32, active: *mut u8 }

#[link(name = "b200vis")]
extern "C" {
    fn b200vis_create(cfg: *const b200vis_config, out: *mut *mut b200vis_ctx) -> i32;
    fn b200vis_destroy(ctx: *mut b200vis_ctx);
    fn b200vis_last_error(ctx: *const b200vis_ctx) -> *const c_char;
    fn b200vis_synchronize(ctx: *mut b200vis_ctx) -> i32;
    fn b200vis_set_topology(ctx: *mut b200vis_ctx, n: u32, parent_row: *const u32, entity_bits: *const u64) -> i32;
    fn b200vis_plan_row_order(n: u32, parent_row: *const u32, new_to_old: *mut u32) -> i32;
    fn b200vis_upload_transforms(ctx: *mut b200vis_ctx, first: u32, count: u32, trs: *const f32) -> i32;
    fn b200vis_upload_global_transforms(ctx: *mut b200vis_ctx, first: u32, count: u32, gt: *const f32) -> i32;
    fn b200vis_upload_bounds(ctx: *mut b200vis_ctx, first: u32, count: u32, bounds: *const f32, flags: *const u8, class_mask: *const u8,
                             layer_mask: *const u64, range_mask: *const u32) -> i32;
    fn b200vis_upload_view_visibility(ctx: *mut b200vis_ctx, first: u32, count: u32, vv: *const u8) -> i32;
    fn b200vis_upload_render_layers_ext(ctx: *mut b200vis_ctx, first: u32, count: u32, blocks: *const [u64; 3]) -> i32;
    fn b200vis_set_view_render_layers_ext(ctx: *mut b200vis_ctx, view: u32, blocks: *const [u64; 3]) -> i32;
    fn b200vis_set_light_render_layers_ext(ctx: *mut b200vis_ctx, n: u32, blocks: *const [u64; 3]) -> i32;
    fn b200vis_set_static_transform_optimizations(ctx: *mut b200vis_ctx, enabled: i32) -> i32;
    fn b200vis_set_views(ctx: *mut b200vis_ctx, n: u32, views: *const b200vis_view) -> i32;
    fn b200vis_set_lights(ctx: *mut b200vis_ctx, n: u32, light_row: *const u32, range: *const f32, layers: *const u64) -> i32;
    fn b200vis_set_cluster_view(ctx: *mut b200vis_ctx, view: u32, p: *const b200vis_cluster_view) -> i32;
    fn b200vis_host_cluster_view_setup(cfg: *const b200vis_cluster_config, camera_gt12: *const f32, clip_from_view16: *const f32,
                                       frustum: *const [f32; 4], layer_mask: u64, feedback: *const b200vis_cluster_feedback,
                                       planes_scratch: *mut f32, out: *mut b200vis_cluster_view) -> i32;
    fn b200vis_run(ctx: *mut b200vis_ctx, stages: u32) -> i32;
    fn b200vis_set_result_sink(ctx: *mut b200vis_ctx, sink: *const b200vis_result_sink) -> i32;
    fn b200vis_set_view_stats_sink(ctx: *mut b200vis_ctx, per_view: *mut [u32; 4]) -> i32;
    fn b200vis_set_visible_entities_sink(ctx: *mut b200vis_ctx, sink: *const b200vis_visible_entities_sink) -> i32;
    fn b200vis_set_table_rows(ctx: *mut b200vis_ctx, table: u32, first_slot: u32, count: u32, rows: *const u32) -> i32;
    fn b200vis_writeback_tables(ctx: *mut b200vis_ctx, which: u32, gt_tick: u32, vv_tick: u32) -> i32;
    fn b200vis_set_tables_ex(ctx: *mut b200vis_ctx, n: u32, tables: *const b200vis_table, inputs: *const b200vis_table_inputs,
                             layout: *const b200vis_transform_layout) -> i32;
    fn b200vis_read_tables(ctx: *mut b200vis_ctx, which: u32, last_run: u32, this_run: u32) -> i32;
    fn b200vis_set_table_cull_inputs(ctx: *mut b200vis_ctx, n: u32, inputs: *const b200vis_table_cull_inputs,
                                     layout: *const b200vis_bounds_layout) -> i32;
    fn b200vis_set_table_visibility_ranges(ctx: *mut b200vis_ctx, n: u32, ranges: *const b200vis_table_visibility_ranges,
                                           layout: *const b200vis_visibility_range_layout) -> i32;
    fn b200vis_set_visibility_range_views(ctx: *mut b200vis_ctx, n: u32, positions: *const f32) -> i32;
    fn b200vis_set_table_shadow_casters(ctx: *mut b200vis_ctx, n: u32, is_caster: *const u8) -> i32;
    fn b200vis_set_shadow_items(ctx: *mut b200vis_ctx, n: u32, items: *const b200vis_shadow_item, list_capacity: u32) -> i32;
    fn b200vis_set_shadow_item_render_layers_ext(ctx: *mut b200vis_ctx, n: u32, blocks: *const [u64; 3]) -> i32;
    fn b200vis_run_shadow_culling(ctx: *mut b200vis_ctx) -> i32;
    fn b200vis_set_shadow_entities_sink(ctx: *mut b200vis_ctx, sink: *const b200vis_shadow_entities_sink) -> i32;
    fn b200vis_emit_shadow_entities(ctx: *mut b200vis_ctx) -> i32;
}
const NO_PARENT: u32 = 0xFFFF_FFFF; const DETACHED: u32 = 0xFFFF_FFFE;
const STAGE_PROPAGATE: u32 = 1; const STAGE_CULL: u32 = 2; const STAGE_CLUSTER: u32 = 12;
const WB_GLOBAL_TRANSFORM: u32 = 1; const WB_VIEW_VISIBILITY: u32 = 2; const WB_SET_VISIBLE: u32 = 4; const UNMAPPED: u32 = 0xFFFF_FFFF;
const RD_TRANSFORM: u32 = 1; const RD_GLOBAL_TRANSFORM: u32 = 2; const RD_CULL_INPUTS: u32 = 4;
const F_INHERITED: u8 = 0x01; const F_AABB: u8 = 0x02; const F_SPHERE: u8 = 0x04; const F_NO_FRUSTUM: u8 = 0x08;
const F_RANGE: u8 = 0x10; const F_NO_CPU_CULLING: u8 = 0x20; const F_SPHERE_FROM_GT: u8 = 0x40;
const VIEW_ACTIVE: u8 = 1; const VIEW_NO_CPU_CULLING: u8 = 2;
const SHADOW_POINT: u32 = 0; const SHADOW_SPOT: u32 = 1; const SHADOW_DIRECTIONAL_CASCADE: u32 = 2;
const ERR_HIERARCHY_CYCLE: i32 = 4;
const MAX_CAMERAS: usize = 32; const MAX_CLUSTERS: usize = 4096;

/// Device context, the entity <-> row map, and the pinned host buffers the GPU writes into.  `Send + Sync`: exactly one
/// system touches it at a time (`ResMut`).  The result buffers are allocated once at full capacity and never reallocated:
/// the library registers them with cudaHostRegister and the GPU keeps their addresses.
#[derive(Resource)]
pub struct B200Vis {
    ctx: *mut b200vis_ctx,
    max_entities: usize,
    n: usize,
    row_of: EntityHashMap<u32>,
    entity_of: Vec<Entity>,
    columns_epoch: u64,           // bumped when rows are renumbered: every mirrored column must be uploaded again
    bounds_epoch: u64,
    lights_epoch: u64,
    classes: Vec<TypeId>,         // VisibilityClass registry: bit k of the class mask = classes[k] (at most 8)
    view_entities: Vec<Entity>,   // view v of the device = this camera entity (query order of the cull system)
    light_entities: Vec<Entity>,  // light ordinal -> entity (query order of the cluster system)
    // sinks
    stats: Box<b200vis_frame_stats>,
    view_stats: Vec<[u32; 4]>,    // every view: visible_count, cluster_index_count, cluster_farthest_z bits, overflow
    max_views: usize,
    // VisibleEntities as Entity::to_bits(), every view's class lists back to back, and their offsets
    visible_entities: Vec<u64>, entity_offsets: Vec<[u32; 9]>, cluster_offsets: Vec<u32>, cluster_indices: Vec<u32>, cluster_cap: usize,
    planes_scratch: Vec<f32>,
    // the archetype tables registered with b200vis_set_tables_ex (one entry per table holding GlobalTransform, with its
    // Transform and ViewVisibility columns), their cull inputs, the entities each slot map
    // was built from, and the rows epoch of the maps
    tables: Vec<b200vis_table>, table_inputs: Vec<b200vis_table_inputs>, table_cull: Vec<b200vis_table_cull_inputs>,
    table_entities: Vec<Vec<Entity>>, maps_epoch: u64,
    // the tables' VisibilityRange columns, attached while the VisibleEntityRanges resource exists (None = detached)
    table_ranges: Option<Vec<b200vis_table_visibility_ranges>>,
    // some row has had a RenderLayers layer in 64..255: the rows' blocks 1..3 are uploaded with their block 0 from then on
    rows_ext: bool,
    // the table -> shadow-caster bytes attached with b200vis_set_table_shadow_casters (attached after every cull-input attach)
    table_casters: Vec<u8>,
    // the range views b200_check_visibility gave b200vis_set_visibility_range_views this frame (their bit = their position)
    range_views: Vec<Entity>,
    // the shadow entity sink: every shadow list of a run as Entity::to_bits(), its offsets and active flags.  It grows, up to
    // max_shadow_entries entries, when a run's lists do not fit; a replaced sink's buffers stay alive with the context,
    // because the library keeps their registration
    shadow_entities: Vec<u64>, shadow_offsets: Vec<u32>, shadow_active: Vec<u8>, shadow_max_items: usize,
    max_shadow_entries: usize, retired_shadow_sinks: Vec<(Vec<u64>, Vec<u32>, Vec<u8>)>,
}
unsafe impl Send for B200Vis {}
unsafe impl Sync for B200Vis {}
impl Drop for B200Vis { fn drop(&mut self) { unsafe { b200vis_destroy(self.ctx) } } }

impl B200Vis {
    fn check(&self, rc: i32) -> Result<(), BevyError> {
        if rc == 0 { return Ok(()); }
        let msg = unsafe { std::ffi::CStr::from_ptr(b200vis_last_error(self.ctx)) }.to_string_lossy().into_owned();
        // crates/bevy_transform/src/systems.rs:715 panics on a malformed hierarchy; keep that behaviour
        if rc == ERR_HIERARCHY_CYCLE { panic!("Malformed hierarchy: {msg}"); }
        Err(format!("b200vis error {rc}: {msg}").into())
    }
    /// Registers a shadow entity sink of `capacity` entries for `max_items` items in place of the current one.
    fn set_shadow_sink(&mut self, capacity: usize, max_items: usize) -> Result<(), BevyError> {
        let old = (core::mem::replace(&mut self.shadow_entities, vec![0; capacity.max(1)]),
                   core::mem::replace(&mut self.shadow_offsets, vec![0; max_items * 6 + 1]),
                   core::mem::replace(&mut self.shadow_active, vec![0; max_items.max(1)]));
        if !old.0.is_empty() { self.retired_shadow_sinks.push(old); }
        self.shadow_max_items = max_items;
        let s = b200vis_shadow_entities_sink { entities: self.shadow_entities.as_mut_ptr(), capacity: self.shadow_entities.len() as u32,
            max_items: max_items as u32, offsets: self.shadow_offsets.as_mut_ptr(), active: self.shadow_active.as_mut_ptr() };
        self.check(unsafe { b200vis_set_shadow_entities_sink(self.ctx, &s) })
    }
    fn class_bit(&mut self, id: TypeId) -> u8 {
        if let Some(k) = self.classes.iter().position(|c| *c == id) { return 1 << k; }
        assert!(self.classes.len() < 8, "libb200vis carries at most 8 VisibilityClass ids");
        self.classes.push(id);
        1 << (self.classes.len() - 1)
    }
}

/// `max_cameras`: the most cameras (views) the app renders at once, 1..=32; views past the eighth cost one extra cull pass
/// per eight views (DESIGN.md section 4), and the result buffers are sized by it.  The VisibleEntities sink holds
/// `max_entities` entries per view: a view whose visible entities are in more than `max_entities` class lists in all (an
/// entity counts once per VisibilityClass it carries) makes the cull system return an error, so an app whose entities
/// carry several classes sets `max_entities` to cover that total.
/// `max_shadow_entries`: the most entries all shadow lists of a frame may hold together (every point-light face, spot
/// light and directional cascade list, an entity counting once per list it is in).  The sink starts small and doubles
/// when a frame needs more; a frame that needs more than this makes the light-visibility system return an error.
pub struct B200VisibilityPlugin { pub max_entities: u32, pub max_lights: u32, pub max_cameras: u32, pub max_shadow_entries: u32 }

impl Plugin for B200VisibilityPlugin {
    fn build(&self, app: &mut App) {
        let max_views = (self.max_cameras as usize).clamp(1, MAX_CAMERAS);
        let cfg = b200vis_config { device: 0, max_entities: self.max_entities, max_lights: self.max_lights, max_views: max_views as u32,
                                   max_cluster_indices: 0, world_size: 1, rank: 0, reserved: 0 };
        let mut ctx = core::ptr::null_mut();
        let rc = unsafe { b200vis_create(&cfg, &mut ctx) };
        assert_eq!(rc, 0, "b200vis_create failed: there is no CPU fallback");
        let n = self.max_entities as usize;
        let cluster_cap = 1usize << 18;
        let mut vis = B200Vis {
            ctx, max_entities: n, n: 0, row_of: Default::default(), entity_of: Vec::new(), columns_epoch: 0, bounds_epoch: u64::MAX,
            lights_epoch: u64::MAX, classes: Vec::new(), view_entities: Vec::new(), light_entities: Vec::new(),
            stats: Box::default(), view_stats: vec![[0; 4]; max_views], max_views, visible_entities: vec![0; max_views * n],
            entity_offsets: vec![[0; 9]; max_views],
            cluster_offsets: vec![0; max_views * (MAX_CLUSTERS + 1)], cluster_indices: vec![0; max_views * cluster_cap], cluster_cap,
            planes_scratch: vec![0.0; 3 * 4097 * 4], tables: Vec::new(), table_inputs: Vec::new(), table_cull: Vec::new(), table_entities: Vec::new(),
            maps_epoch: u64::MAX, table_ranges: None, rows_ext: false, table_casters: Vec::new(), range_views: Vec::new(),
            shadow_entities: Vec::new(), shadow_offsets: Vec::new(), shadow_active: Vec::new(), shadow_max_items: 0,
            max_shadow_entries: self.max_shadow_entries as usize, retired_shadow_sinks: Vec::new(),
        };
        // the sorted row lists stay on the device: VisibleEntities arrives as Entity values through the entities sink, and
        // GlobalTransform and ViewVisibility go straight into the archetype tables (b200vis_set_tables)
        let rs = b200vis_result_sink { stats: &mut *vis.stats, visible_rows: core::ptr::null_mut(), visible_capacity: 0,
            visible_classes: core::ptr::null_mut(), cluster_offsets: vis.cluster_offsets.as_mut_ptr(),
            cluster_indices: vis.cluster_indices.as_mut_ptr(), cluster_capacity: cluster_cap as u32 };
        let es = b200vis_visible_entities_sink { entities: vis.visible_entities.as_mut_ptr(), capacity: n as u32,
                                                 offsets: vis.entity_offsets.as_mut_ptr() };
        unsafe {
            assert_eq!(b200vis_set_result_sink(ctx, &rs), 0); assert_eq!(b200vis_set_visible_entities_sink(ctx, &es), 0);
            assert_eq!(b200vis_set_view_stats_sink(ctx, vis.view_stats.as_mut_ptr()), 0);   // per-view stats of every view
        }
        vis.set_shadow_sink((1usize << 16).min(vis.max_shadow_entries.max(1)), 64).expect("b200vis_set_shadow_entities_sink");
        app.insert_resource(vis);
        // CPU clustering mode, so that `Clusters` holds `ClusterableObjects::Cpu`, which the cluster system fills (SURVEY.md 0)
        app.insert_resource(GlobalClusterSettings { gpu_clustering: None, supports_storage_buffers: true,
            clustered_decals_are_usable: false, max_uniform_buffer_clusterable_objects: 204, view_cluster_bindings_max_indices: 16384 });
    }
    fn finish(&self, app: &mut App) {
        for schedule in [PostStartup.intern(), PostUpdate.intern()] {
            app.remove_systems_in_set(schedule, mark_dirty_trees, RemoveSystemsOnly);
            app.remove_systems_in_set(schedule, propagate_parent_transforms, RemoveSystemsOnly);
            app.remove_systems_in_set(schedule, sync_simple_transforms, RemoveSystemsOnly);
            app.add_systems(schedule, (b200_sync_tables, b200_propagate).chain().in_set(TransformSystems::Propagate));
        }
        app.remove_systems_in_set(PostUpdate, check_visibility_cpu_culling, RemoveSystemsOnly);
        // the device evaluates the ranges from the tables' VisibilityRange columns for both culls, so nothing reads
        // what check_visibility_ranges would write
        app.remove_systems_in_set(PostUpdate, check_visibility_ranges, RemoveSystemsOnly);
        app.remove_systems_in_set(PostUpdate, SimulationLightSystems::AssignLightsToClusters, RemoveSystemsOnly);
        app.remove_systems_in_set(PostUpdate, SimulationLightSystems::CheckLightVisibility, RemoveSystemsOnly);
        app.add_systems(PostUpdate, (
            (b200_sync_tables, b200_check_visibility).chain().in_set(VisibilitySystems::CheckVisibility),
            b200_assign_lights_to_clusters.in_set(SimulationLightSystems::AssignLightsToClusters)
                .after(TransformSystems::Propagate).after(VisibilitySystems::CheckVisibility),
            // the reference's ordering of the light-visibility systems (bevy_light/src/lib.rs:217-230)
            (b200_sync_tables, b200_check_light_visibility).chain().in_set(SimulationLightSystems::CheckLightVisibility)
                .after(VisibilitySystems::CalculateBounds).after(TransformSystems::Propagate)
                .after(SimulationLightSystems::UpdateLightFrusta).after(VisibilitySystems::CheckVisibility)
                .before(VisibilitySystems::MarkNewlyHiddenEntitiesInvisible),
        ));
    }
}

/// Blocks 0..3 (layers 0..255) of an entity's RenderLayers (render_layers.rs:20-23; none = the default layer 0).  The device
/// holds four blocks: a set layer past 255 is an error that names the entity, not a silent truncation.
fn layer_blocks(entity: Entity, layers: Option<&RenderLayers>) -> Result<[u64; 4], BevyError> {
    let Some(l) = layers else { return Ok([1, 0, 0, 0]) };
    let bits = l.bits();
    if bits.iter().skip(4).any(|&w| w != 0) {
        return Err(format!("{entity}: {l:?} has a layer past 255; the device holds RenderLayers 0..=255").into());
    }
    let mut out = [0u64; 4];
    for (o, w) in out.iter_mut().zip(bits) { *o = *w; }
    Ok(out)
}
fn ext_of(b: &[u64; 4]) -> [u64; 3] { [b[1], b[2], b[3]] }

fn pack_trs(t: &Transform, out: &mut Vec<f32>) {
    out.extend_from_slice(&[t.translation.x, t.translation.y, t.translation.z, t.rotation.x, t.rotation.y, t.rotation.z, t.rotation.w,
                            t.scale.x, t.scale.y, t.scale.z]);
}
fn pack_gt12(g: &GlobalTransform, out: &mut Vec<f32>) {
    let a = g.affine();
    out.extend_from_slice(&[a.matrix3.x_axis.x, a.matrix3.x_axis.y, a.matrix3.x_axis.z, a.matrix3.y_axis.x, a.matrix3.y_axis.y,
                            a.matrix3.y_axis.z, a.matrix3.z_axis.x, a.matrix3.z_axis.y, a.matrix3.z_axis.z, a.translation.x,
                            a.translation.y, a.translation.z]);
}
/// propagate: the data propagate_parent_transforms' queries (systems.rs:506-520) and sync_simple_transforms'
/// (systems.rs:42-55) read and write, as one query.
fn b200_propagate(
    this_run: SystemChangeTick,
    mut vis: ResMut<B200Vis>,
    // write access to GlobalTransform: the GPU writes the tables' columns while this system runs
    q: Query<(Entity, Ref<Transform>, &mut GlobalTransform, Option<&Children>, Option<&ChildOf>)>,
    structure_changed: Query<(), Or<(Added<GlobalTransform>, Changed<ChildOf>)>>,
    mut orphaned: RemovedComponents<ChildOf>,
    mut despawned: RemovedComponents<GlobalTransform>,
    opts: Res<StaticTransformOptimizations>,
) -> Result<(), BevyError> {
    let vis = &mut *vis;
    let rebuild = vis.n != q.iter().len() || !structure_changed.is_empty() || orphaned.read().next().is_some()
        || despawned.read().next().is_some();
    if rebuild {
        // ---- rows are renumbered: tree-contiguous BFS order (the layout the tile kernel likes), then every column again ----
        let old: Vec<(Entity, Option<Entity>)> = q.iter().map(|(e, _, _, _, p)| (e, p.map(|p| p.parent()))).collect();
        let n = old.len();
        assert!(n <= vis.max_entities, "B200VisibilityPlugin::max_entities is too small");
        let old_row: EntityHashMap<u32> = old.iter().enumerate().map(|(i, (e, _))| (*e, i as u32)).collect();
        // ChildOf whose parent lacks Transform/GlobalTransform is outside NodeQuery (systems.rs:752-764): DETACHED
        let parent_old: Vec<u32> = old.iter().map(|(_, p)| match p { None => NO_PARENT, Some(p) => *old_row.get(p).unwrap_or(&DETACHED) }).collect();
        let mut new_to_old = vec![0u32; n];
        vis.check(unsafe { b200vis_plan_row_order(n as u32, parent_old.as_ptr(), new_to_old.as_mut_ptr()) })?;
        let mut new_of_old = vec![0u32; n];
        for (new, &o) in new_to_old.iter().enumerate() { new_of_old[o as usize] = new as u32; }
        vis.entity_of = new_to_old.iter().map(|&o| old[o as usize].0).collect();
        vis.row_of = vis.entity_of.iter().enumerate().map(|(r, e)| (*e, r as u32)).collect();
        let parent_new: Vec<u32> = new_to_old.iter().map(|&o| { let p = parent_old[o as usize]; if p < n as u32 { new_of_old[p as usize] } else { p } }).collect();
        let bits: Vec<u64> = vis.entity_of.iter().map(|e| e.to_bits()).collect();
        vis.check(unsafe { b200vis_set_topology(vis.ctx, n as u32, parent_new.as_ptr(), bits.as_ptr()) })?;
        let (mut trs, mut gt) = (Vec::with_capacity(n * 10), Vec::with_capacity(n * 12));
        for e in &vis.entity_of {
            let (_, t, g, _, _) = q.get(*e).unwrap();
            pack_trs(&t, &mut trs); pack_gt12(&g, &mut gt);
        }
        // upload_transforms marks every row Changed<Transform>: the first propagate visits everything, like Added<GlobalTransform>
        vis.check(unsafe { b200vis_upload_transforms(vis.ctx, 0, n as u32, trs.as_ptr()) })?;
        vis.check(unsafe { b200vis_upload_global_transforms(vis.ctx, 0, n as u32, gt.as_ptr()) })?;
        vis.n = n;
        vis.columns_epoch += 1;
    } else {
        // ---- steady state: the device finds Changed<Transform> and Changed<GlobalTransform> in the tables itself and
        // reads only those slots: no entity loop here.  Changed<GlobalTransform> as this system sees it (systems.rs:709-710)
        // is exactly the writes of other systems, because this system's own write-back of its last run is not newer than
        // its last_run (Tick::is_newer_than, the rule the device applies to every slot).
        vis.check(unsafe { b200vis_read_tables(vis.ctx, RD_TRANSFORM | RD_GLOBAL_TRANSFORM, this_run.last_run().get(),
                                               this_run.this_run().get()) })?;
    }
    // the registry b200_sync_tables left is current for this frame's tables; a rebuild above renumbered the rows and
    // b200vis_set_topology unmapped every slot, so the maps are sent again
    if rebuild { send_table_maps(vis, None)?; }
    unsafe {
        vis.check(b200vis_set_static_transform_optimizations(vis.ctx, opts.is_enabled() as i32))?;
        vis.check(b200vis_run(vis.ctx, STAGE_PROPAGATE))?;
        // the changed matrices into the tables, each stamped with this run's tick (set_if_neq semantics, systems.rs:719:
        // what assigning through `Mut` does, change_detection/params.rs:1093-1135)
        vis.check(b200vis_writeback_tables(vis.ctx, WB_GLOBAL_TRANSFORM, this_run.this_run().get(), 0))?;
        vis.check(b200vis_synchronize(vis.ctx))?;
    }
    Ok(())
}

/// The table registry (INTEGRATION.md section 2): one entry per archetype table that holds GlobalTransform -- that column and
/// its changed ticks, and the table's ViewVisibility column and ticks -- read from
/// `World::storages().tables` with `Table::entity_count` / `Table::capacity` (storage/table/mod.rs).  Exclusive and chained
/// right before each write-back system, so no table moves between the registration and the write-back that uses it.  The
/// registry is replaced when a table's pointers, len or capacity changed; a table's slot -> row map is sent again when its
/// entity list differs from the one the map was built from (an archetype move or swap_remove reorders slots without changing
/// len) or the rows were renumbered.  Bevy never removes a table, so a table keeps its index in the registry.
fn b200_sync_tables(world: &mut World) -> Result<(), BevyError> {
    let Some(gt_id) = world.component_id::<GlobalTransform>() else { return Ok(()) };
    let t_id = world.component_id::<Transform>();
    // Transform is repr(Rust): its layout is whatever this build of rustc chose
    let layout = b200vis_transform_layout { stride: size_of::<Transform>() as u32, translation: offset_of!(Transform, translation) as u32,
                                            rotation: offset_of!(Transform, rotation) as u32, scale: offset_of!(Transform, scale) as u32 };
    // Aabb and Sphere are repr(Rust) too
    let bounds_layout = b200vis_bounds_layout { aabb_stride: size_of::<Aabb>() as u32, aabb_center: offset_of!(Aabb, center) as u32,
        aabb_half_extents: offset_of!(Aabb, half_extents) as u32, sphere_stride: size_of::<Sphere>() as u32,
        sphere_center: offset_of!(Sphere, center) as u32, sphere_radius: offset_of!(Sphere, radius) as u32 };
    let (aabb_id, sphere_id) = (world.component_id::<Aabb>(), world.component_id::<Sphere>());
    let (iv_id, vis_vv_id) = (world.component_id::<InheritedVisibility>(), world.component_id::<ViewVisibility>());
    // per-archetype bits of check_visibility_cpu_culling's query (visibility/mod.rs:758-772), fixed for a whole table
    let markers = [(world.component_id::<NoFrustumCulling>(), F_NO_FRUSTUM), (world.component_id::<VisibilityRange>(), F_RANGE),
                   (world.component_id::<NoCpuCulling>(), F_NO_CPU_CULLING)];
    let light_id = world.component_id::<PointLight>();
    // the archetypes of the light systems' visible_entity_query (lib.rs:526-537): With<Mesh3d>, Without<NotShadowCaster>,
    // Without<DirectionalLight>
    let (mesh_id, not_caster_id, dir_id) = (world.component_id::<Mesh3d>(), world.component_id::<NotShadowCaster>(),
                                            world.component_id::<DirectionalLight>());
    // VisibilityRange is repr(Rust) too.  Without the VisibleEntityRanges resource the reference does not range-cull at
    // all (visibility/mod.rs:813-819), so nothing is attached then.
    let range_layout = b200vis_visibility_range_layout { stride: size_of::<VisibilityRange>() as u32,
        start: (offset_of!(VisibilityRange, start_margin) + offset_of!(core::ops::Range<f32>, start)) as u32,
        end: (offset_of!(VisibilityRange, end_margin) + offset_of!(core::ops::Range<f32>, end)) as u32,
        use_aabb: offset_of!(VisibilityRange, use_aabb) as u32 };
    let range_id = world.component_id::<VisibilityRange>();
    let use_ranges = world.contains_resource::<VisibleEntityRanges>();
    world.resource_scope(|world, mut vis: Mut<B200Vis>| {
        let vis = &mut *vis;
        let (mut descs, mut inputs, mut culls, mut entities, mut ranges) = (Vec::new(), Vec::new(), Vec::new(), Vec::new(), Vec::new());
        let mut casters = Vec::new();
        for table in world.storages().tables.iter() {
            if !table.has_column(gt_id) { continue; }
            // SAFETY: the columns hold GlobalTransform / ViewVisibility.  Only raw pointers are kept; the GPU writes through
            // them inside the write-back systems, which hold the only access to those columns while they run.
            let gt = unsafe { table.get_data_slice_for::<GlobalTransform>(gt_id) }.unwrap();
            let gt_ticks = table.get_changed_ticks_slice_for(gt_id).unwrap();
            let (vv, vv_ticks) = match vis_vv_id.filter(|id| table.has_column(*id)) {
                Some(id) => (unsafe { table.get_data_slice_for::<ViewVisibility>(id) }.unwrap().as_ptr() as *mut ViewVisibility,
                             table.get_changed_ticks_slice_for(id).unwrap().as_ptr() as *mut Tick),
                None => (core::ptr::null_mut(), core::ptr::null_mut()),
            };
            descs.push(b200vis_table { global_transforms: gt.as_ptr() as *mut GlobalTransform, gt_changed_ticks: gt_ticks.as_ptr() as *mut Tick,
                                       view_visibility: vv, vv_changed_ticks: vv_ticks, len: table.entity_count(),
                                       capacity: table.capacity() as u32 });
            // the Transform column and its ticks, which b200vis_read_tables reads (a table without Transform is not read)
            inputs.push(match t_id.filter(|id| table.has_column(*id)) {
                Some(id) => b200vis_table_inputs {
                    transforms: unsafe { table.get_data_slice_for::<Transform>(id) }.unwrap().as_ptr() as *const Transform,
                    transform_changed_ticks: table.get_changed_ticks_slice_for(id).unwrap().as_ptr() as *const Tick },
                None => b200vis_table_inputs { transforms: core::ptr::null(), transform_changed_ticks: core::ptr::null() },
            });
            // the cull inputs b200vis_read_tables(RD_CULL_INPUTS) reads: Aabb, Sphere and InheritedVisibility with their ticks,
            // and the bits the archetype fixes.  A table outside visible_aabb_query (NoCpuCulling, or no InheritedVisibility /
            // ViewVisibility) is NO_CPU_CULLING: the cull never looks at its rows.
            let has = |c: Option<bevy::ecs::component::ComponentId>| c.is_some_and(|c| table.has_column(c));
            let (aabb, aabb_t) = column::<Aabb>(table, aabb_id);
            let (sphere, sphere_t) = column::<Sphere>(table, sphere_id);
            let in_query = has(iv_id) && has(vis_vv_id) && !has(markers[2].0);
            let (iv, iv_t) = if in_query { column::<InheritedVisibility>(table, iv_id) } else { (core::ptr::null(), core::ptr::null()) };
            let mut flags = markers.iter().fold(0u8, |f, (c, bit)| if has(*c) { f | bit } else { f });
            if !in_query { flags |= F_NO_CPU_CULLING; }
            // a point light's Sphere is rebuilt from its GlobalTransform every frame (point_light.rs:195-209)
            if has(light_id) && aabb.is_null() && !sphere.is_null() { flags |= F_SPHERE_FROM_GT; }
            culls.push(b200vis_table_cull_inputs { aabbs: aabb, aabb_changed_ticks: aabb_t, spheres: sphere, sphere_changed_ticks: sphere_t,
                                                   inherited_visibility: iv, iv_changed_ticks: iv_t, flags: flags as u32 });
            casters.push((has(mesh_id) && !has(not_caster_id) && !has(dir_id)) as u8);
            // the VisibilityRange column goes with the table's F_RANGE bit, as the library requires
            let (range, range_t) = column::<VisibilityRange>(table, range_id);
            ranges.push(b200vis_table_visibility_ranges { ranges: range, changed_ticks: range_t });
            entities.push(table.entities());
        }
        let registry_changed = descs != vis.tables || inputs != vis.table_inputs;
        if registry_changed {
            vis.check(unsafe { b200vis_set_tables_ex(vis.ctx, descs.len() as u32, descs.as_ptr(), inputs.as_ptr(), &layout) })?;
            vis.tables = descs;
            vis.table_inputs = inputs;
            vis.table_ranges = None;                // ... and drops the cull inputs and the ranges
        }
        // b200vis_set_tables_ex drops the cull inputs: attach them again (a table whose entry is unchanged is not read in full)
        if registry_changed || culls != vis.table_cull {
            // the ranges leave first: the cull inputs may change which tables carry F_RANGE
            if vis.table_ranges.take().is_some() {
                vis.check(unsafe { b200vis_set_table_visibility_ranges(vis.ctx, 0, core::ptr::null(), core::ptr::null()) })?;
            }
            vis.check(unsafe { b200vis_set_table_cull_inputs(vis.ctx, culls.len() as u32, culls.as_ptr(), &bounds_layout) })?;
            vis.table_cull = culls;
            vis.table_casters.clear();              // attached again below, before the frame's cull read
        }
        // the shadow-caster byte of every table, read with the cull inputs.  The first attach also switches on the
        // visible-set bookkeeping the shadow stage reads, so it must precede the frame's CULL read.
        if !vis.tables.is_empty() && casters != vis.table_casters {
            vis.check(unsafe { b200vis_set_table_shadow_casters(vis.ctx, casters.len() as u32, casters.as_ptr()) })?;
            vis.table_casters = casters;
        }
        // the VisibilityRange columns the cull read takes the range parameters from (an attach after none reads every
        // ranged table in full)
        let want = if use_ranges && !vis.tables.is_empty() { Some(ranges) } else { None };
        if want != vis.table_ranges {
            match &want {
                Some(r) => vis.check(unsafe { b200vis_set_table_visibility_ranges(vis.ctx, r.len() as u32, r.as_ptr(), &range_layout) })?,
                None => vis.check(unsafe { b200vis_set_table_visibility_ranges(vis.ctx, 0, core::ptr::null(), core::ptr::null()) })?,
            }
            vis.table_ranges = want;
        }
        let renumbered = vis.maps_epoch != vis.columns_epoch;
        let stale: Vec<bool> = entities.iter().enumerate()
            .map(|(t, e)| renumbered || vis.table_entities.get(t).map_or(true, |old| old.as_slice() != *e)).collect();
        vis.table_entities = entities.iter().map(|e| e.to_vec()).collect();
        send_table_maps(vis, Some(&stale))
    })
}

/// A table's column of T and its changed ticks as raw pointers, or two NULLs when the table has no such column.
fn column<T: Component>(table: &bevy::ecs::storage::Table, id: Option<bevy::ecs::component::ComponentId>) -> (*const T, *const Tick) {
    match id.filter(|c| table.has_column(*c)) {
        // SAFETY: the column holds T.  Only raw pointers are kept; the GPU reads through them inside the systems that
        // call b200vis_read_tables, while no other system can write the column.
        Some(c) => (unsafe { table.get_data_slice_for::<T>(c) }.unwrap().as_ptr() as *const T,
                    table.get_changed_ticks_slice_for(c).unwrap().as_ptr() as *const Tick),
        None => (core::ptr::null(), core::ptr::null()),
    }
}

/// b200vis_set_table_rows for every table (`only` = None) or the tables marked in `only`: slot s -> the row of the entity
/// in it, B200VIS_UNMAPPED for an entity without a row (GlobalTransform without Transform).  The calls only queue the
/// changes; they reach the device with the next write-back.
fn send_table_maps(vis: &mut B200Vis, only: Option<&[bool]>) -> Result<(), BevyError> {
    for (t, entities) in vis.table_entities.iter().enumerate() {
        if only.is_some_and(|o| !o[t]) { continue; }
        let rows: Vec<u32> = entities.iter().map(|e| vis.row_of.get(e).copied().unwrap_or(UNMAPPED)).collect();
        vis.check(unsafe { b200vis_set_table_rows(vis.ctx, t as u32, 0, rows.len() as u32, rows.as_ptr()) })?;
    }
    vis.maps_epoch = vis.columns_epoch;
    Ok(())
}

/// cull: the parameter list of check_visibility_cpu_culling (visibility/mod.rs:748-774), plus the rows whose VisibilityClass
/// or RenderLayers changed, which the device cannot read from the tables.
fn b200_check_visibility(
    this_run: SystemChangeTick,
    mut vis: ResMut<B200Vis>,
    mut view_query: Query<(Entity, &mut VisibleEntities, &Frustum, Option<&RenderLayers>, &Camera, Has<NoCpuCulling>)>,
    visible_aabb_query: Query<(Entity, Ref<InheritedVisibility>, &mut ViewVisibility, Option<Ref<VisibilityClass>>, Option<Ref<RenderLayers>>,
                                   Option<Ref<Aabb>>, Option<Ref<Sphere>>, &GlobalTransform, Has<NoFrustumCulling>, Has<VisibilityRange>,
                                   Has<PointLight>), Without<NoCpuCulling>>,
    // check_visibility_ranges' view query and its cap of 32 (visibility/range.rs:236, 247)
    range_views: Query<(Entity, &GlobalTransform), Or<(With<Camera>, With<ShadowLodOrigin>)>>,
    dirty_query: Query<Entity, (Without<NoCpuCulling>, Or<(Changed<VisibilityClass>, Changed<RenderLayers>)>)>,
    mut removed_layers: RemovedComponents<RenderLayers>,
) -> Result<(), BevyError> {
    let vis = &mut *vis;
    // ---- the VisibilityRange views: the device evaluates check_visibility_ranges itself, from the tables' range columns
    // b200_sync_tables attached (only while the VisibleEntityRanges resource exists) and this frame's GlobalTransforms ----
    let ranged = vis.table_ranges.is_some();
    let (mut range_entities, mut range_pos) = (Vec::new(), Vec::new());
    if ranged {
        for (e, g) in range_views.iter().take(32) {
            let t = g.translation();
            range_entities.push(e); range_pos.extend_from_slice(&[t.x, t.y, t.z]);
        }
        vis.check(unsafe { b200vis_set_visibility_range_views(vis.ctx, range_entities.len() as u32, range_pos.as_ptr()) })?;
    }
    // the light-visibility system gives each shadow item the bit of its view among these
    vis.range_views.clone_from(&range_entities);
    // ---- views: half spaces copied verbatim from `Frustum` (bit-identical by construction) ----
    let (mut views, mut view_ext) = (Vec::new(), Vec::new());
    vis.view_entities.clear();
    for (entity, _, frustum, layers, camera, no_cpu_culling) in view_query.iter() {
        let blocks = layer_blocks(entity, layers)?;
        view_ext.push(ext_of(&blocks));
        let mut v = b200vis_view { half_spaces: [[0.0; 4]; 6], layer_mask: blocks[0],
                                   flags: (camera.is_active as u8 * VIEW_ACTIVE) | (no_cpu_culling as u8 * VIEW_NO_CPU_CULLING),
                                   range_view_index: -1, pad: [0; 6] };
        for (k, hs) in frustum.half_spaces.iter().enumerate() { v.half_spaces[k] = hs.normal_d().to_array(); }
        // the view's bit in the device's range masks; -1 = not among the range views: entity_is_in_range_of_view is
        // then false for every entity with a VisibilityRange (range.rs:218-220), so the view culls them all
        if ranged { v.range_view_index = range_entities.iter().position(|r| *r == entity).map_or(-1, |i| i as i8); }
        views.push(v); vis.view_entities.push(entity);
        if views.len() == vis.max_views { break; }
    }
    vis.check(unsafe { b200vis_set_views(vis.ctx, views.len() as u32, views.as_ptr()) })?;
    // blocks 1..3 of every view: its camera cull here, its cluster view in b200_assign_lights_to_clusters (same view index)
    for (v, ext) in view_ext.iter().enumerate() {
        vis.check(unsafe { b200vis_set_view_render_layers_ext(vis.ctx, v as u32, ext) })?;
    }
    // ---- VisibilityClass and RenderLayers (which the device cannot read from the tables): every row after a renumbering,
    // otherwise only the rows whose class or layers changed, as contiguous ranges.
    // upload_bounds also takes the rows' current bounds and flags; the table read below, enqueued after it, then brings
    // every row's Aabb / Sphere / InheritedVisibility up to date by their change ticks.  No loop over every entity. ----
    let all = vis.bounds_epoch != vis.columns_epoch;
    let n = vis.n;
    let mut dirty: Vec<u32> = if all { (0..n as u32).collect() } else {
        dirty_query.iter().chain(removed_layers.read()).filter_map(|e| vis.row_of.get(&e).copied()).collect()
    };
    dirty.sort_unstable();
    dirty.dedup();
    let k = dirty.len();
    let (mut bounds, mut flags, mut class, mut layer) = (vec![0f32; k * 6], vec![F_NO_CPU_CULLING; k], vec![0u8; k], vec![1u64; k]);
    let mut layer_ext = vec![[0u64; 3]; k];
    for (i, &r) in dirty.iter().enumerate() {
        let e = vis.entity_of[r as usize];
        // a row outside visible_aabb_query stays NO_CPU_CULLING, as its table's cull inputs say
        let Ok((_, inherited, _, vclass, layers, aabb, sphere, _, no_frustum, has_range, is_light)) = visible_aabb_query.get(e) else { continue };
        let mut f = if inherited.get() { F_INHERITED } else { 0 } | if no_frustum { F_NO_FRUSTUM } else { 0 } | if has_range { F_RANGE } else { 0 };
        if let Some(a) = &aabb { f |= F_AABB; bounds[i * 6..i * 6 + 6].copy_from_slice(&[a.center.x, a.center.y, a.center.z, a.half_extents.x, a.half_extents.y, a.half_extents.z]); }
        else if let Some(s) = &sphere {
            f |= F_SPHERE | if is_light { F_SPHERE_FROM_GT } else { 0 };
            bounds[i * 6..i * 6 + 4].copy_from_slice(&[s.center.x, s.center.y, s.center.z, s.radius]);
        }
        flags[i] = f;
        class[i] = vclass.as_ref().map_or(0, |c| c.iter().fold(0u8, |m, id| m | vis.class_bit(*id)));
        let blocks = layer_blocks(e, layers.as_deref())?;
        layer[i] = blocks[0]; layer_ext[i] = ext_of(&blocks);
    }
    // blocks 1..3 go to the device once some row uses them (the cull's block-0 path serves everyone else)
    vis.rows_ext |= layer_ext.iter().any(|b| b.iter().any(|&w| w != 0));
    let mut i = 0;
    while i < k {                                               // coalesce into [first, first + count) ranges
        let mut j = i + 1;
        while j < k && dirty[j] == dirty[j - 1] + 1 { j += 1; }
        vis.check(unsafe { b200vis_upload_bounds(vis.ctx, dirty[i], (j - i) as u32, bounds[i * 6..].as_ptr(), flags[i..].as_ptr(),
            class[i..].as_ptr(), layer[i..].as_ptr(), core::ptr::null()) })?;
        if vis.rows_ext {
            vis.check(unsafe { b200vis_upload_render_layers_ext(vis.ctx, dirty[i], (j - i) as u32, layer_ext[i..].as_ptr()) })?;
        }
        i = j;
    }
    // Aabb, Sphere, InheritedVisibility and VisibilityRange straight from the tables, by this system's own change ticks;
    // rows (re)mapped since the last read (archetype moves, a renumbering) are read in full, their per-archetype flags
    // with them
    if !vis.tables.is_empty() {
        vis.check(unsafe { b200vis_read_tables(vis.ctx, RD_CULL_INPUTS, this_run.last_run().get(), this_run.this_run().get()) })?;
    }
    if all {
        #[cfg(feature = "forked-bevy")]
        { let vv: Vec<u8> = vis.entity_of.iter().map(|e| visible_aabb_query.get(*e).map_or(0, |q| q.2.bits())).collect();
          vis.check(unsafe { b200vis_upload_view_visibility(vis.ctx, 0, n as u32, vv.as_ptr()) })?; }
        vis.bounds_epoch = vis.columns_epoch;
    }
    // ViewVisibility straight into the tables b200_sync_tables registered.  Unforked, the CPU's reset_view_visibility and
    // mark_newly_hidden_entities_invisible own the 2-bit state: the device applies set_visible() to the byte each visible
    // slot holds, with this run's tick where it goes from hidden to visible.  Forked, the device owns the state and writes
    // the bytes, with the tick where Changed<ViewVisibility> fires.
    unsafe {
        vis.check(b200vis_run(vis.ctx, STAGE_CULL))?;
        #[cfg(not(feature = "forked-bevy"))]
        vis.check(b200vis_writeback_tables(vis.ctx, WB_SET_VISIBLE, 0, this_run.this_run().get()))?;
        #[cfg(feature = "forked-bevy")]
        vis.check(b200vis_writeback_tables(vis.ctx, WB_VIEW_VISIBILITY, 0, this_run.this_run().get()))?;
        vis.check(b200vis_synchronize(vis.ctx))?;       // stats, Entity lists and the tables' ViewVisibility are written now
    }
    // ---- VisibleEntities: one sorted Vec per class (mod.rs:846-874), each filled with one slice of the device's Entity list:
    // the device wrote every class list already split, in Entity::to_bits() order, so the reference's sort_unstable has
    // nothing left to do.  No loop over entities. ----
    // Entity is repr(C, align(8)) and "equivalent to a u64" (bevy_ecs/src/entity/mod.rs:423-432): its memory is to_bits()
    const _: () = assert!(size_of::<Entity>() == size_of::<u64>() && core::mem::align_of::<Entity>() == core::mem::align_of::<u64>());
    for (v, view_entity) in vis.view_entities.iter().enumerate() {
        let Ok((_, mut visible_entities, _, _, camera, _)) = view_query.get_mut(*view_entity) else { continue };
        if !camera.is_active { continue; }                       // an inactive view keeps its lists (mod.rs:780-782)
        for list in visible_entities.entities.values_mut() { list.clear(); }
        let off = vis.entity_offsets[v];
        if off[8] as usize > vis.max_entities {
            return Err(format!("view {v}: {} VisibleEntities entries exceed the sink's {} per view (entities in several \
                                VisibilityClasses): raise max_entities", off[8], vis.max_entities).into());
        }
        let all = &vis.visible_entities[v * vis.max_entities..][..off[8] as usize];
        // SAFETY: every entry is the to_bits() of a live Entity, given to b200vis_set_topology; layout asserted above
        let all = unsafe { core::slice::from_raw_parts(all.as_ptr() as *const Entity, all.len()) };
        for (k, id) in vis.classes.iter().enumerate() {
            let list = &all[off[k] as usize..off[k + 1] as usize];
            if !list.is_empty() { visible_entities.get_mut(*id).extend_from_slice(list); }
        }
    }
    Ok(())
}

/// cluster: the queries of assign_objects_to_clusters for point lights (assign.rs:137-153).
fn b200_assign_lights_to_clusters(
    mut vis: ResMut<B200Vis>,
    mut views: Query<(Entity, &GlobalTransform, &Camera, &Frustum, Option<&ClusterConfig>, &mut Clusters, Option<&RenderLayers>)>,
    point_lights_query: Query<(Entity, &GlobalTransform, &ViewVisibility, Ref<PointLight>, Option<Ref<RenderLayers>>)>,
    mut removed_lights: RemovedComponents<PointLight>,
    settings: Res<GlobalClusterSettings>,
) -> Result<(), BevyError> {
    let vis = &mut *vis;
    // ---- lights: ordinal = query order; positions and ViewVisibility are read on the device from the lights' own rows ----
    let lights_changed = vis.lights_epoch != vis.columns_epoch || removed_lights.read().next().is_some()
        || point_lights_query.iter().any(|(_, _, _, l, r)| l.is_changed() || r.is_some_and(|r| r.is_changed()));
    if lights_changed {
        vis.light_entities.clear();
        let (mut rows, mut ranges, mut layers, mut ext) = (Vec::new(), Vec::new(), Vec::new(), Vec::new());
        for (e, _, _, light, layer) in point_lights_query.iter() {
            let Some(&r) = vis.row_of.get(&e) else { continue };
            let blocks = layer_blocks(e, layer.as_deref())?;
            vis.light_entities.push(e); rows.push(r); ranges.push(light.range); layers.push(blocks[0]); ext.push(ext_of(&blocks));
        }
        vis.check(unsafe { b200vis_set_lights(vis.ctx, rows.len() as u32, rows.as_ptr(), ranges.as_ptr(), layers.as_ptr()) })?;
        // set_lights emptied the lights' blocks 1..3: give them again where some light has a layer in 64..255
        if ext.iter().any(|b| b.iter().any(|&w| w != 0)) {
            vis.check(unsafe { b200vis_set_light_render_layers_ext(vis.ctx, ext.len() as u32, ext.as_ptr()) })?;
        }
        vis.lights_epoch = vis.columns_epoch;
    }
    // ---- per view: the prologue of assign_objects_to_clusters (assign.rs:324-485) through the library's host helper, which
    // restates it op for op (dims via ClusterConfig::dimensions_for_screen_size, Clusters::update, far_z / cluster_factors
    // from last frame's feedback, the x / y / z HalfSpace tables) ----
    let mut order = Vec::new();
    for (entity, camera_transform, camera, frustum, config, clusters, layers) in views.iter() {
        let Some(v) = vis.view_entities.iter().position(|e| *e == entity) else { continue };
        let size = camera.physical_viewport_size().unwrap_or(UVec2::ZERO);
        let config = config.copied().unwrap_or_default();
        let (kind, dims, total, z_slices, z_cfg, dyn_resize) = match config {        // cluster/mod.rs:107-139
            ClusterConfig::None => (0, [0; 3], 0, 0, ClusterZConfig::default(), false),
            ClusterConfig::Single => (1, [1; 3], 0, 0, ClusterZConfig::default(), false),
            ClusterConfig::XYZ { dimensions, z_config, dynamic_resizing } => (2, dimensions.to_array(), 0, 0, z_config, dynamic_resizing),
            ClusterConfig::FixedZ { total, z_slices, z_config, dynamic_resizing } => (3, [0; 3], total, z_slices, z_config, dynamic_resizing),
        };
        let (far_z_mode, far_z_constant) = match z_cfg.far_z_mode {
            ClusterFarZMode::MaxClusterableObjectRange => (0, 0.0), ClusterFarZMode::Constant(z) => (1, z) };
        let cfg = b200vis_cluster_config { kind, dims, total, z_slices, first_slice_depth: z_cfg.first_slice_depth, far_z_mode,
            far_z_constant, dynamic_resizing: dyn_resize as u32, screen_w: size.x, screen_h: size.y,
            view_cluster_bindings_max_indices: settings.view_cluster_bindings_max_indices as u32 };
        let fb = b200vis_cluster_feedback { has_farthest_z: clusters.last_frame_farthest_z.is_some() as u32,
            farthest_z: clusters.last_frame_farthest_z.unwrap_or(0.0),
            has_index_count: clusters.last_frame_total_cluster_index_count.is_some() as u32,
            index_count: clusters.last_frame_total_cluster_index_count.unwrap_or(0) as u32 };
        let mut gt12 = Vec::with_capacity(12); pack_gt12(camera_transform, &mut gt12);
        let cfv = camera.clip_from_view().to_cols_array();
        let hs: Vec<[f32; 4]> = frustum.half_spaces.iter().map(|h| h.normal_d().to_array()).collect();
        let mut cv = core::mem::MaybeUninit::<b200vis_cluster_view>::zeroed();
        unsafe {
            // block 0 here; blocks 1..3 are the view's, set by b200_check_visibility for the same view index
            vis.check(b200vis_host_cluster_view_setup(&cfg, gt12.as_ptr(), cfv.as_ptr(), hs.as_ptr(), layer_blocks(entity, layers)?[0], &fb,
                                                      vis.planes_scratch.as_mut_ptr(), cv.as_mut_ptr()))?;
            vis.check(b200vis_set_cluster_view(vis.ctx, v as u32, cv.as_ptr()))?;
            order.push((entity, v, cv.assume_init()));
        }
    }
    unsafe { vis.check(b200vis_run(vis.ctx, STAGE_CLUSTER))?; vis.check(b200vis_synchronize(vis.ctx))?; }
    // ---- results: Clusters::update / reset_for_new_frame restated (cluster/mod.rs:398-468), then one add_point_light per index ----
    for (entity, v, cv) in order {
        let Ok((_, _, _, _, _, mut clusters, _)) = views.get_mut(entity) else { continue };
        if cv.enabled == 0 {                                     // clusters.clear(): ClusterConfig::None or an empty viewport (assign.rs:334-340)
            clusters.tile_size = UVec2::ONE; clusters.dimensions = UVec3::ZERO; clusters.near = 0.0; clusters.far = 0.0;
            if let ClusterableObjects::Cpu(list) = &mut clusters.clusterable_objects { list.clear(); }
            continue;
        }
        clusters.tile_size = UVec2::new(cv.tile_size[0], cv.tile_size[1]);
        clusters.dimensions = UVec3::new(cv.dims[0], cv.dims[1], cv.dims[2]);
        clusters.near = cv.near_z; clusters.far = cv.far_z;
        let nc = (cv.dims[0] * cv.dims[1] * cv.dims[2]) as usize;
        let mut cells = vec![ObjectsInClusterCpu::default(); nc];
        let off = &vis.cluster_offsets[v * (MAX_CLUSTERS + 1)..][..nc + 1];
        let idx = &vis.cluster_indices[v * vis.cluster_cap..];
        for (c, cell) in cells.iter_mut().enumerate() {
            for i in off[c]..off[c + 1] { cell.add_point_light(vis.light_entities[idx[i as usize] as usize]); }   // ascending light order = push order (assign.rs:487)
        }
        clusters.clusterable_objects = ClusterableObjects::Cpu(cells);
        clusters.last_frame_total_cluster_index_count = Some(vis.view_stats[v][1] as usize);
        clusters.last_frame_farthest_z = Some(f32::from_bits(vis.view_stats[v][2]));     // assign.rs:810-811
    }
    Ok(())
}

/// Where a shadow item's lists go.
enum ShadowDest { Point(Entity), Spot(Entity), Cascade { light: Entity, view: Entity, cascade: usize } }

/// light: check_point_light_mesh_visibility and check_dir_light_mesh_visibility (bevy_light/src/lib.rs:342-749) as one
/// device pass.  The items come from the lights' own components (CubemapFrusta, Frustum, CascadesFrusta copied verbatim);
/// whether a point or spot light is in some view's VisibleEntities, the caster bytes and the shadow LOD origin's range
/// bit are decided on the device.  The lists come back sorted, as Entity values.
fn b200_check_light_visibility(
    this_run: SystemChangeTick,
    mut vis: ResMut<B200Vis>,
    mut point_lights: Query<(Entity, &PointLight, &CubemapFrusta, &mut CubemapVisibleEntities, Option<&RenderLayers>)>,
    mut spot_lights: Query<(Entity, &SpotLight, &Frustum, &mut VisibleMeshEntities, Option<&RenderLayers>)>,
    mut directional_lights: Query<(Entity, &DirectionalLight, &CascadesFrusta, &mut CascadesVisibleEntities, Option<&RenderLayers>),
                                  Without<SpotLight>>,
    // write access to every ViewVisibility column: the write-backs below set bytes and change ticks in the tables while
    // this system runs (the reference's check_point_light_mesh_visibility holds &mut ViewVisibility too, lib.rs:537).
    // The directional lights' own visibility is read through it.
    view_visibility: Query<&mut ViewVisibility>,
    // get_shadow_lod_origin's lenses, as check_point_light_mesh_visibility builds them (lib.rs:561-565)
    mut camera_query: Query<(Entity, &RenderTarget), With<Camera>>,
    mut shadow_lod_origin_query: Query<Entity, With<ShadowLodOrigin>>,
    mut point_and_spot_light_query: Query<Entity, Or<(With<PointLight>, With<SpotLight>)>>,
) -> Result<(), BevyError> {
    let vis = &mut *vis;
    // no table holds GlobalTransform yet: no light or mesh has a row, and the shadow stage has no caster column
    if vis.table_casters.is_empty() { return Ok(()); }
    let lod_origin = get_shadow_lod_origin(camera_query.transmute_lens_filtered(), shadow_lod_origin_query.transmute_lens_filtered(),
                                           point_and_spot_light_query.transmute_lens_filtered());
    // the bit of a view in the device's range masks: its position among this frame's range views, -1 = not among them
    let range_bit = |e: Option<Entity>, views: &[Entity]| e.and_then(|e| views.iter().position(|r| *r == e)).map_or(-1, |i| i as i32);
    let lod_bit = range_bit(lod_origin, &vis.range_views);
    let (mut items, mut ext, mut dest) = (Vec::new(), Vec::new(), Vec::new());
    let item = |kind, light_row, range, range_view_index, layer_mask| b200vis_shadow_item { kind, light_row, range, range_view_index,
                                                                                            layer_mask, frusta: [[[0.0; 4]; 6]; 6] };
    // ---- one point item per PointLight with shadow maps, one spot item per SpotLight with shadow maps ----
    for (e, light, frusta, _, layers) in point_lights.iter() {
        if !light.shadow_maps_enabled { continue; }
        let Some(&row) = vis.row_of.get(&e) else { continue };
        let blocks = layer_blocks(e, layers)?;
        let mut it = item(SHADOW_POINT, row, light.range, lod_bit, blocks[0]);
        for (f, face) in frusta.frusta.iter().enumerate() {
            for (k, hs) in face.half_spaces.iter().enumerate() { it.frusta[f][k] = hs.normal_d().to_array(); }
        }
        items.push(it); ext.push(ext_of(&blocks)); dest.push(ShadowDest::Point(e));
    }
    for (e, light, frustum, _, layers) in spot_lights.iter() {
        if !light.shadow_maps_enabled { continue; }
        let Some(&row) = vis.row_of.get(&e) else { continue };
        let blocks = layer_blocks(e, layers)?;
        let mut it = item(SHADOW_SPOT, row, light.range, lod_bit, blocks[0]);
        for (k, hs) in frustum.half_spaces.iter().enumerate() { it.frusta[0][k] = hs.normal_d().to_array(); }
        items.push(it); ext.push(ext_of(&blocks)); dest.push(ShadowDest::Spot(e));
    }
    // ---- one cascade item per (view, cascade) of a directional light with shadow maps that is visible (lib.rs:395-399) ----
    let light_visible = |e: Entity| view_visibility.get(e).is_ok_and(|v| v.get());
    for (e, light, frusta, _, layers) in directional_lights.iter() {
        if !light.shadow_maps_enabled || !light_visible(e) { continue; }
        let blocks = layer_blocks(e, layers)?;
        for (view, view_frusta) in &frusta.frusta {
            let view_bit = range_bit(Some(*view), &vis.range_views);
            for (c, frustum) in view_frusta.iter().enumerate() {
                let mut it = item(SHADOW_DIRECTIONAL_CASCADE, 0, 0.0, view_bit, blocks[0]);
                for (k, hs) in frustum.half_spaces.iter().enumerate() { it.frusta[0][k] = hs.normal_d().to_array(); }
                items.push(it); ext.push(ext_of(&blocks)); dest.push(ShadowDest::Cascade { light: e, view: *view, cascade: c });
            }
        }
    }
    let n = items.len();
    // a sink for fewer items than these would make b200vis_set_shadow_items refuse them: grow it first
    if n > vis.shadow_max_items {
        let cap = vis.shadow_entities.len();
        vis.set_shadow_sink(cap, n.max(2 * vis.shadow_max_items))?;
    }
    // list_capacity 1: the lists come from the entity sink, the row lists are never read
    unsafe {
        vis.check(b200vis_set_shadow_items(vis.ctx, n as u32, items.as_ptr(), 1))?;
        if ext.iter().any(|b| b.iter().any(|&w| w != 0)) {
            vis.check(b200vis_set_shadow_item_render_layers_ext(vis.ctx, n as u32, ext.as_ptr()))?;
        }
        vis.check(b200vis_run_shadow_culling(vis.ctx))?;
        // set_visible() of the rows only lights see, with this system's tick (the rows the cameras made visible hold
        // their bit already).  Forked, the device's bytes are written instead.
        #[cfg(not(feature = "forked-bevy"))]
        vis.check(b200vis_writeback_tables(vis.ctx, WB_SET_VISIBLE, 0, this_run.this_run().get()))?;
        #[cfg(feature = "forked-bevy")]
        vis.check(b200vis_writeback_tables(vis.ctx, WB_VIEW_VISIBILITY, 0, this_run.this_run().get()))?;
        vis.check(b200vis_synchronize(vis.ctx))?;
    }
    // ---- a sink too small for this frame: grow it and have the same lists written again (running the stage again would
    // not do: it would move the shadow diff forward) ----
    let total = vis.shadow_offsets[n * 6] as usize;
    if total > vis.shadow_entities.len() {
        if total > vis.max_shadow_entries {
            return Err(format!("the shadow lists of this frame hold {total} entries, more than B200VisibilityPlugin::max_shadow_entries \
                                ({}): raise it", vis.max_shadow_entries).into());
        }
        let cap = total.max(2 * vis.shadow_entities.len()).min(vis.max_shadow_entries);
        let max_items = vis.shadow_max_items;
        vis.set_shadow_sink(cap, max_items)?;
        unsafe { vis.check(b200vis_emit_shadow_entities(vis.ctx))?; vis.check(b200vis_synchronize(vis.ctx))?; }
    }
    // SAFETY: every entry is the to_bits() of a live Entity, given to b200vis_set_topology (layout asserted in
    // b200_check_visibility)
    let all = unsafe { core::slice::from_raw_parts(vis.shadow_entities.as_ptr() as *const Entity, total) };
    let off = &vis.shadow_offsets;
    let list = |l: usize| &all[off[l] as usize..off[l + 1] as usize];
    // ---- CubemapVisibleEntities faces and spot VisibleMeshEntities: only active items.  An inactive light is not in any
    // view's VisibleEntities: the reference `continue`s past it and its component keeps what it held ----
    for (i, d) in dest.iter().enumerate() {
        if vis.shadow_active[i] == 0 { continue; }
        match *d {
            ShadowDest::Point(e) => {
                let Ok((_, _, _, mut faces, _)) = point_lights.get_mut(e) else { continue };
                for (f, face) in faces.iter_mut().enumerate() { face.entities.clear(); face.entities.extend_from_slice(list(i * 6 + f)); }
            }
            ShadowDest::Spot(e) => {
                let Ok((_, _, _, mut visible, _)) = spot_lights.get_mut(e) else { continue };
                visible.entities.clear(); visible.entities.extend_from_slice(list(i * 6));
            }
            ShadowDest::Cascade { .. } => {}
        }
    }
    // ---- CascadesVisibleEntities, as check_dir_light_mesh_visibility keeps it (lib.rs:380-404): every view's vector sized
    // to its cascades, views that left CascadesFrusta dropped and new ones added, everything cleared for a light without
    // shadow maps or not visible; then each cascade's list replaced ----
    for (e, light, frusta, mut visible, _) in directional_lights.iter_mut() {
        let visible = &mut *visible;
        visible.entities.retain(|view, _| frusta.frusta.contains_key(view));
        for (view, view_frusta) in &frusta.frusta {
            visible.entities.entry(*view).or_default().resize(view_frusta.len(), Default::default());
        }
        if !light.shadow_maps_enabled || !light_visible(e) { visible.entities.clear(); }
    }
    for (i, d) in dest.iter().enumerate() {
        let ShadowDest::Cascade { light, view, cascade } = *d else { continue };
        let Ok((_, _, _, mut visible, _)) = directional_lights.get_mut(light) else { continue };
        let Some(lists) = visible.entities.get_mut(&view) else { continue };
        let dst = &mut lists[cascade].entities;
        dst.clear(); dst.extend_from_slice(list(i * 6));
    }
    Ok(())
}
