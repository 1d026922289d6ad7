"""Host-side mirror of the reference's three systems on top of the C ABI.

`VisibilityPipeline` plays the role of the `B200VisibilityPlugin` a Bevy app
would add (INTEGRATION.md): it owns one device context, mirrors a scene's
columns into it, recomputes the per-view constants each frame exactly where
the reference does (update_frusta, the per-view prologue of
assign_objects_to_clusters) and exposes the stages under the reference's names.
"""
import numpy as np

from . import abi


class WideFrameStats:
    """FrameStats of a context with more than abi.MAX_VIEWS views: the per-view fields are arrays over every view."""

    def __init__(self, stats, per_view):
        self.visible_count = per_view["visible_count"]
        self.cluster_index_count = per_view["cluster_index_count"]
        self.cluster_farthest_z = per_view["cluster_farthest_z"]
        self.cluster_index_overflow = per_view["cluster_index_overflow"]
        self.gt_changed_count, self.vv_changed_count, self.frame = stats.gt_changed_count, stats.vv_changed_count, stats.frame


class VisibilityPipeline:
    def __init__(self, scene, device=0, static_transform_optimizations=True, max_cluster_indices=0,
                 world_size=1, rank=0, cluster_config=None, max_lights=None, max_entities=None):
        """max_entities: row capacity of the context (default: the scene's rows), room for rows spawned by edit_topology."""
        self.scene = scene
        n, L, V = scene.n, len(scene.light_row), max(len(scene.cameras), 1)
        self.ctx = abi.Context(max(n, max_entities or 0), max_lights=max(L, 1) if max_lights is None else max(max_lights, L, 1), max_views=V, device=device,
                               max_cluster_indices=max_cluster_indices, world_size=world_size, rank=rank)
        c = self.ctx
        c.set_static_transform_optimizations(static_transform_optimizations)
        c.set_topology(scene.parent, scene.entity_bits)
        c.upload_transforms(0, scene.trs)
        identity = np.tile(np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], np.float32), (n, 1))
        c.upload_global_transforms(0, identity)                       # GlobalTransform::IDENTITY at spawn
        c.upload_bounds(0, scene.bounds, scene.flags, scene.class_mask, scene.layer_mask, scene.range_mask)
        c.upload_view_visibility(0, np.zeros(n, np.uint8))             # ViewVisibility::HIDDEN
        c.set_lights(scene.light_row, scene.light_range, scene.light_layers)
        self.cluster_config = cluster_config or abi.host_default_cluster_config(*scene.screen)
        self.feedback = [abi.ClusterFeedback() for _ in range(V)]
        self._scratch = [None] * V
        self.cluster_views = [None] * V
        self.update_views()

    # -- update_frusta (visibility/mod.rs:627-636) + the per-view prologue of assign_objects_to_clusters
    def update_views(self, clusters=True):
        views = []
        for v, cam in enumerate(self.scene.cameras):
            cfv = abi.host_perspective(cam.fov, cam.aspect, cam.near) if cam.clip_from_view is None \
                else np.ascontiguousarray(cam.clip_from_view, np.float32)
            frustum = abi.host_compute_frustum(cfv, cam.gt, cam.far)
            sc = self.scene
            layers = 1 if sc.view_layers is None else int(sc.view_layers[v])
            views.append(abi.View.make(frustum, layers,
                                       abi.VIEW_ACTIVE if sc.view_flags is None else int(sc.view_flags[v]),
                                       -1 if sc.view_range_index is None else int(sc.view_range_index[v])))
            if clusters and len(self.scene.light_row):
                cv, scratch = abi.host_cluster_view_setup(self.cluster_config, cam.gt, cfv, frustum, layers, self.feedback[v])
                self._scratch[v] = scratch
                self.cluster_views[v] = cv
                self.ctx.set_cluster_view(v, cv)
        self.ctx.set_views(views)
        self.views = views

    def update_views_fast(self):
        """Same as update_views through b200vis_update_camera: one C call per camera, no numpy on the way.  The camera
        descriptor has no projection field, so this path is perspective only."""
        sc = self.scene
        if any(cam.clip_from_view is not None for cam in sc.cameras):
            raise ValueError("update_views_fast builds perspective projections only: use update_views for a camera with clip_from_view")
        if not hasattr(self, "_cam_desc"):
            self._cam_desc = [abi.CameraDesc() for _ in sc.cameras]
            self.cluster_views = [abi.ClusterView() for _ in sc.cameras]
            self.ctx.set_view_count(len(sc.cameras))
        clusters = len(sc.light_row) > 0
        for v, cam in enumerate(sc.cameras):
            d = self._cam_desc[v]
            d.global_transform[:] = cam.gt.tolist()
            d.fov_y, d.aspect, d.near_z, d.far_z = cam.fov, cam.aspect, cam.near, cam.far
            d.layer_mask = 1 if sc.view_layers is None else int(sc.view_layers[v])
            d.flags = abi.VIEW_ACTIVE if sc.view_flags is None else int(sc.view_flags[v])
            d.range_view_index = -1 if sc.view_range_index is None else int(sc.view_range_index[v])
            self.ctx.update_camera(v, d, self.cluster_config if clusters else None, self.feedback[v], self.cluster_views[v])

    # -- the three systems, by the names BASELINE.json / the reference use -----------------------
    def propagate_transforms(self):
        """TransformSystems::Propagate: mark_dirty_trees + propagate_parent_transforms + sync_simple_transforms."""
        self.ctx.run(abi.STAGE_PROPAGATE)

    def check_visibility(self):
        """reset_view_visibility + check_visibility_cpu_culling + mark_newly_hidden_entities_invisible."""
        self.ctx.run(abi.STAGE_CULL)

    def assign_lights_to_clusters(self):
        """assign_objects_to_clusters (point lights)."""
        self.ctx.run(abi.STAGE_CLUSTER)

    def run_frame(self):
        """The fused per-frame path: one launch sequence for all three systems."""
        self.ctx.run(abi.STAGE_ALL if len(self.scene.light_row) else (abi.STAGE_PROPAGATE | abi.STAGE_CULL))

    def check_point_light_mesh_visibility(self, shadow_ordinals, shadow_map_near_z=0.1, lod_origin_range_index=-1):
        """SURVEY 8(f) N3 (bevy_light/src/lib.rs:517): call after run_frame().  The CubemapFrusta come from the lights'
        GlobalTransforms of this frame (update_point_light_frusta), as a shim would read them from the component."""
        sc = self.scene
        ords = np.asarray(shadow_ordinals, np.uint32)
        frusta = np.zeros((len(ords), 6, 6, 4), np.float32)
        for i, o in enumerate(ords):
            gt, _ = self.ctx.download_global_transforms(int(sc.light_row[o]), 1, want_changed=False)
            frusta[i] = abi.host_point_light_frusta(gt[0], float(sc.light_range[o]), shadow_map_near_z)
        layers = None if sc.light_layers is None else sc.light_layers[ords]
        self.ctx.set_shadow_lights(ords, frusta, layers, lod_origin_range_index)
        self.ctx.run_shadow_culling()

    def enable_visible_diff(self, enabled=True):
        """SURVEY 8(f) N1: have the CULL stage also produce each view's added / removed rows
        (RenderVisibleEntitiesClass::update_cpu_culled_entities, bevy_render/src/view/visibility/mod.rs:194-249)."""
        self.ctx.enable_visible_diff(enabled)
        self.visible_diff = bool(enabled)

    def read_feedback(self):
        """Clusters::last_frame_* (assign.rs:810-811): feeds next frame's far_z and dynamic resizing.  Returns the frame's
        FrameStats; a context with more than abi.MAX_VIEWS views gets a WideFrameStats with the same fields over every view."""
        s = self.ctx.download_frame_stats()
        if self.ctx.max_views > abi.MAX_VIEWS:
            s = WideFrameStats(s, self.ctx.download_view_stats())
        for v in range(len(self.scene.cameras)):
            cv = self.cluster_views[v]
            if cv is None or not cv.enabled:
                continue
            fb = self.feedback[v]
            fb.has_farthest_z = 1; fb.farthest_z = s.cluster_farthest_z[v]
            fb.has_index_count = 1; fb.index_count = s.cluster_index_count[v]
        return s

    def close(self):
        self.ctx.close()
