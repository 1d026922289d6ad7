"""Differential harness: the CUDA path (through the C ABI) against the CPU oracle on the same scene,
frame by frame.  Bit-exact for GlobalTransform bits, change flags, ViewVisibility bytes, visible lists
and cluster index lists (north_star: bit-exact bits/indices; 1e-5 abs on GlobalTransform floats -- we
hold the floats to bit equality too and report the max abs difference if that ever fails)."""
from dataclasses import dataclass

import numpy as np

import bevy_b200 as bb
from bevy_b200 import scenes
import oracle as orc

IDENTITY = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], np.float32)
CONFIG_KINDS = {"none": 0, "single": 1, "xyz": 2, "fixedz": 3}


@dataclass
class ClusterSpec:
    """One ClusterConfig (crates/bevy_light/src/cluster/mod.rs:107-139) + viewport + GlobalClusterSettings max indices, from
    which both sides are built: `abi_config()` for the device, `oracle_kwargs()` for orc.default_cluster_view_in."""
    kind: str = "fixedz"
    dims: tuple = (0, 0, 0)            # XYZ
    total: int = 4096                  # FixedZ
    z_slices: int = 24                 # FixedZ
    first_slice_depth: float = 5.0
    far_z_constant: float = None       # None => ClusterFarZMode::MaxClusterableObjectRange
    dynamic_resizing: bool = True
    screen: tuple = (1920, 1080)
    max_indices: int = 16384

    def abi_config(self):
        c = bb.ClusterConfig()
        c.kind = CONFIG_KINDS[self.kind]
        c.dims[:] = list(self.dims)
        c.total, c.z_slices, c.first_slice_depth = self.total, self.z_slices, self.first_slice_depth
        c.far_z_mode = 0 if self.far_z_constant is None else 1
        c.far_z_constant = 0.0 if self.far_z_constant is None else self.far_z_constant
        c.dynamic_resizing = int(self.dynamic_resizing)
        c.screen_w, c.screen_h = self.screen
        c.view_cluster_bindings_max_indices = self.max_indices
        return c

    def oracle_kwargs(self):
        return dict(screen=tuple(self.screen), config_kind=CONFIG_KINDS[self.kind], cfg_dims=tuple(self.dims), total=self.total,
                    z_slices=self.z_slices, first_slice_depth=self.first_slice_depth,
                    far_z_mode=0 if self.far_z_constant is None else 1,
                    far_z_constant=0.0 if self.far_z_constant is None else self.far_z_constant,
                    dynamic_resizing=self.dynamic_resizing, max_indices=self.max_indices)


def clip_from_view(cam):
    """The camera's projection on the oracle side: its explicit clip_from_view, else the oracle's perspective."""
    if cam.clip_from_view is not None:
        return np.ascontiguousarray(cam.clip_from_view, np.float32)
    return orc.perspective(cam.fov, cam.aspect, cam.near)


class OracleWorld:
    """The reference-side world state for one scene, advanced by the oracle."""

    def __init__(self, scene, static_opt=True, cluster_kwargs=None):
        self.scene = scene
        self.cluster_kwargs = cluster_kwargs or {}
        self.fb_used = None            # the Clusters feedback each view's last frame() started from
        n = scene.n
        self.gt = np.tile(IDENTITY, (n, 1))
        self.vv = np.zeros(n, np.uint8)
        self.tchanged = np.ones(n, np.uint8)     # Added<GlobalTransform> on the first frame
        self.static_opt = static_opt
        self.fb = [dict(far=None, cnt=None) for _ in scene.cameras]
        self.last_lists = [np.zeros(0, np.uint32) for _ in scene.cameras]

    def frame(self, views_planes, view_flags=None, cluster=True, mt=False):
        sc = self.scene
        rc, gt_changed = orc.propagate(sc.parent, sc.trs, self.gt, self.tchanged, self.static_opt, mt=mt)
        assert rc == 0
        self.tchanged[:] = 0
        if getattr(sc, "range_se", None) is not None:   # SURVEY 8(f) N4: check_visibility_ranges runs before the cull
            sc.range_mask = orc.check_visibility_ranges(self.gt, sc.bounds, sc.flags, sc.range_se, sc.range_use_aabb, sc.range_view_pos)
        shadow = getattr(sc, "shadow_lights", None) is not None
        orc.set_defer_mark_newly_hidden(shadow)   # the light-visibility systems run before mark_newly_hidden_entities_invisible
        try:
            vv_changed, lists = orc.cull(self.gt, sc.bounds, sc.flags, sc.class_mask, sc.entity_bits, self.vv,
                                         views_planes, view_layers=sc.view_layers,
                                         view_flags=view_flags if view_flags is not None else sc.view_flags,
                                         layer_mask=sc.layer_mask, range_mask=sc.range_mask,
                                         view_range_index=sc.view_range_index, mt=mt)
        finally:
            orc.set_defer_mark_newly_hidden(False)
        if shadow:   # SURVEY 8(f) N3: check_point_light_mesh_visibility for the shadow lights some view's VisibleEntities hold
            cur = [l if l is not None else self.last_lists[v] for v, l in enumerate(lists)]
            listed = np.unique(np.concatenate(cur)) if len(cur) else np.zeros(0, np.uint32)
            sel = [int(o) for o in sc.shadow_lights if sc.light_row[o] in set(listed.tolist())]
            rows = sc.light_row[sel]
            sphere = np.concatenate([self.gt[rows, 9:12], sc.light_range[sel, None]], 1).astype(np.float32).reshape(-1, 4)
            frusta = np.stack([orc.point_light_frusta(self.gt[r], sc.light_range[o], sc.shadow_near_z) for r, o in zip(rows, sel)]) \
                if len(sel) else np.zeros((0, 6, 6, 4), np.float32)
            ll = None if sc.light_layers is None else np.ascontiguousarray(sc.light_layers[sel], np.uint64)
            sh = orc.check_point_light_mesh_visibility(self.gt, sc.bounds, sc.flags, sc.shadow_caster, sc.entity_bits, self.vv,
                                                       vv_changed, sphere, frusta, layer_mask=sc.layer_mask,
                                                       range_mask=sc.range_mask, lod_origin_index=sc.shadow_lod_origin,
                                                       light_layers=ll)
            self.shadow_result = dict(zip(sel, sh))
            orc.mark_newly_hidden(sc.flags, self.vv, vv_changed)
        clusters = []
        if cluster and len(sc.light_row):
            vis = np.nonzero(self.vv[sc.light_row] & 1)[0]
            lights = np.concatenate([self.gt[sc.light_row[vis], 9:12], sc.light_range[vis, None]], 1).astype(np.float32)
            ll = None if sc.light_layers is None else np.ascontiguousarray(sc.light_layers[vis], np.uint64)
            self.fb_used = [dict(f) for f in self.fb]
            for v, cam in enumerate(sc.cameras):
                kw = dict(screen=sc.screen)
                kw.update(self.cluster_kwargs)
                vin = orc.default_cluster_view_in(cam.gt, clip_from_view(cam), views_planes[v],
                                                  view_layers=1 if sc.view_layers is None else int(sc.view_layers[v]),
                                                  last_farthest_z=self.fb[v]["far"], last_index_count=self.fb[v]["cnt"], **kw)
                out, offsets, idx, _ = orc.assign_lights_to_clusters(vin, lights, ll)
                self.fb[v]["far"] = out.farthest_z; self.fb[v]["cnt"] = out.total_index_count
                clusters.append((out, offsets, vis[idx].astype(np.uint32)))
        return gt_changed, vv_changed, lists, clusters


def compare_frame(pipe, world, frame_no, cluster=True, check_gt=True, run_device=True):
    sc = pipe.scene
    n = sc.n
    planes = np.stack([np.ctypeslib.as_array(v.half_spaces).reshape(6, 4).copy() for v in pipe.views])
    gt_changed, vv_changed, lists, clusters = world.frame(planes, cluster=cluster)
    if run_device:
        pipe.run_frame()
        if getattr(sc, "shadow_lights", None) is not None:
            pipe.check_point_light_mesh_visibility(sc.shadow_lights, sc.shadow_near_z, sc.shadow_lod_origin)
    tag = f"[{sc.name} frame {frame_no}]"
    if check_gt:
        gt, ch = pipe.ctx.download_global_transforms(0, n)
        same = gt.view(np.uint32) == world.gt.view(np.uint32)
        if not same.all():
            bad = np.nonzero(~same.all(1))[0]
            raise AssertionError(f"{tag} GlobalTransform bits differ on {len(bad)} rows (first {bad[:5]}), "
                                 f"max abs diff {np.nanmax(np.abs(gt - world.gt))}")
        assert (ch == gt_changed).all(), f"{tag} Changed<GlobalTransform> differs on {np.nonzero(ch != gt_changed)[0][:8]}"
    vv, vch = pipe.ctx.download_view_visibility(0, n)
    assert (vv == world.vv).all(), f"{tag} ViewVisibility differs on rows {np.nonzero(vv != world.vv)[0][:8]}"
    assert (vch == vv_changed).all(), f"{tag} Changed<ViewVisibility> differs on rows {np.nonzero(vch != vv_changed)[0][:8]}"
    for v in range(len(sc.cameras)):
        got = pipe.ctx.download_visible(v)
        want = lists[v]
        if want is None:                      # inactive view: VisibleEntities keep last frame's contents
            want = world.last_lists[v]
        assert len(got) == len(want) and (got == want).all(), f"{tag} view {v}: visible list differs ({len(got)} vs {len(want)})"
        if getattr(pipe, "visible_diff", False):   # SURVEY 8(f) N1: the render world's added / removed lists
            old = world.last_lists[v]
            bits = sc.entity_bits
            a_r, _, r_r, _ = orc.update_cpu_culled_entities(old, bits[old], want, bits[want])
            if lists[v] is None:
                assert len(a_r) == 0 and len(r_r) == 0
            g_a, g_r = pipe.ctx.download_visible_diff(v)
            assert len(g_a) == len(a_r) and (g_a == a_r).all(), f"{tag} view {v}: added rows differ ({len(g_a)} vs {len(a_r)})"
            assert len(g_r) == len(r_r) and (g_r == r_r).all(), f"{tag} view {v}: removed rows differ ({len(g_r)} vs {len(r_r)})"
    world.last_lists = [l if l is not None else world.last_lists[v] for v, l in enumerate(lists)]
    if getattr(sc, "shadow_lights", None) is not None:
        for i, o in enumerate(sc.shadow_lights):
            want6 = world.shadow_result.get(int(o))
            for face in range(6):
                got = pipe.ctx.download_shadow_visible(i, face)
                want = want6[face] if want6 is not None else np.zeros(0, np.uint32)   # light in no view's list: not processed
                assert len(got) == len(want) and (got == want).all(), \
                    f"{tag} shadow light {o} face {face}: CubemapVisibleEntities differ ({len(got)} vs {len(want)})"
    if getattr(sc, "range_se", None) is not None:
        got = pipe.ctx.download_visibility_ranges(0, n)
        assert (got == sc.range_mask).all(), f"{tag} VisibleEntityRanges masks differ on rows {np.nonzero(got != sc.range_mask)[0][:8]}"
    stats = pipe.read_feedback()
    if cluster and len(sc.light_row):
        for v in range(len(sc.cameras)):
            out, offsets, idx = clusters[v]
            cv = pipe.cluster_views[v]
            assert tuple(cv.dims) == tuple(out.dims), f"{tag} view {v}: cluster dims {tuple(cv.dims)} vs {tuple(out.dims)}"
            goff, gidx = pipe.ctx.download_clusters(v)
            nc = out.dims[0] * out.dims[1] * out.dims[2]
            assert (goff[:nc + 1] == offsets).all(), f"{tag} view {v}: cluster offsets differ"
            assert len(gidx) == len(idx) and (gidx == idx).all(), f"{tag} view {v}: cluster index lists differ"
            assert stats.cluster_index_count[v] == out.total_index_count
            assert np.float32(stats.cluster_farthest_z[v]).view(np.uint32) == np.float32(out.farthest_z).view(np.uint32), \
                f"{tag} view {v}: farthest_z {stats.cluster_farthest_z[v]} vs {out.farthest_z}"
    return stats


def run_parity(scene, frames=3, static_opt=True, animate=True, cluster=True, visible_diff=False, cluster_spec=None,
               before_frame=None, on_frame=None):
    """`cluster_spec` (ClusterSpec) sets the cluster config of both sides; `before_frame(pipe, world, f)` may edit the scene
    before frame f is set up, `on_frame(pipe, world, f)` runs after frame f matched."""
    pipe = bb.VisibilityPipeline(scene, static_transform_optimizations=static_opt,
                                 cluster_config=None if cluster_spec is None else cluster_spec.abi_config())
    world = OracleWorld(scene, static_opt, cluster_kwargs=None if cluster_spec is None else cluster_spec.oracle_kwargs())
    if visible_diff:
        pipe.enable_visible_diff()
    try:
        for f in range(frames):
            if f > 0 and animate:
                scenes.advance_cameras(scene)
                if scene.roots is not None and len(scene.roots):
                    rows, trs = scenes.mutate_roots(scene, f)
                    pipe.ctx.upload_transforms_scattered(rows, trs)
                    world.tchanged[rows] = 1
            if before_frame is not None:
                before_frame(pipe, world, f)
            pipe.update_views(clusters=cluster)
            compare_frame(pipe, world, f, cluster=cluster)
            if on_frame is not None:
                on_frame(pipe, world, f)
    finally:
        pipe.close()
