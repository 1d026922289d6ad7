"""Contexts with more than eight views: views past the eighth are culled by group passes of eight views (k_cull's MERGE
instantiation) behind the tile pass.  Everything is compared bit for bit against the oracle run once over all views."""
import copy
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import bevy_b200 as bb
from bevy_b200 import scenes
import oracle as orc

from parity import OracleWorld, compare_frame
from test_gpu_compaction import Twins, order_keeping_reparents
from test_gpu_edge_cases import _random_scene

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _check_vv_count(pipe):
    """The frame's Changed<ViewVisibility> count (merged by the group passes) equals the rows compare_frame matched."""
    _, vch = pipe.ctx.download_view_visibility(0, pipe.scene.n)
    assert pipe.ctx.download_frame_stats().vv_changed_count == int(vch.sum())


def _forest_ring(n_cameras=16, n_trees=120, levels=5):
    sc = scenes.many_cameras_lights(n_cameras, forest_kwargs=dict(n_trees=n_trees, levels=levels))
    sc.trs[sc.roots, 0:3] *= np.float32(0.03)              # the trees inside and around the camera ring
    return sc


def _shadows(sc, pipe):
    sc.shadow_lights = np.arange(len(sc.light_row), dtype=np.uint32)   # shadow_maps_enabled on all five
    sc.shadow_caster = np.ones(sc.n, np.uint8); sc.shadow_caster[sc.light_row] = 0
    sc.shadow_near_z = 0.1
    sc.shadow_lod_origin = -1
    pipe.ctx.upload_shadow_casters(0, sc.shadow_caster)


@pytest.mark.parametrize("with_forest", [False, True])
def test_many_cameras_lights_rotating_with_shadows(with_forest):
    sc = _forest_ring() if with_forest else scenes.many_cameras_lights()
    pipe = bb.VisibilityPipeline(sc)
    world = OracleWorld(sc, True)
    try:
        _shadows(sc, pipe)
        for f in range(4):
            if f:
                scenes.rotate_cameras(sc, 0.35)
                if sc.roots is not None:
                    rows, trs = scenes.mutate_roots(sc, f)
                    pipe.ctx.upload_transforms_scattered(rows, trs)
                    world.tchanged[rows] = 1
            pipe.update_views()
            stats = compare_frame(pipe, world, f)
            _check_vv_count(pipe)
            assert len(stats.visible_count) == 16 and int(np.sum(stats.visible_count)) > 0
    finally:
        pipe.close()


def _wide_random_scene(seed, V):
    """The feature-rich random scene (shuffled Entity bits: the rank map takes the atomics path) with V cameras: inactive
    and NoCpuCulling cameras past the eighth, RenderLayers per view, and a VisibilityRange bit past the eighth."""
    sc = _random_scene(seed, views=V)
    rng = np.random.default_rng(seed + 1000)
    sc.view_layers = [int(x) for x in rng.choice([1, 3, 2, 1], V)]
    flags = [bb.VIEW_ACTIVE] * V
    flags[8] = 0                                             # inactive past the eighth
    if V > 10:
        flags[10] = bb.VIEW_ACTIVE | bb.VIEW_NO_CPU_CULLING
    flags[1] = bb.VIEW_ACTIVE | bb.VIEW_NO_CPU_CULLING
    sc.view_flags = flags
    ri = [-1] * V
    ri[0], ri[2] = 0, 2
    ri[V - 1] = 9                                            # VisibleEntityRanges bit 9 belongs to the last view
    sc.view_range_index = ri
    ranged = rng.random(sc.n) < 0.5
    sc.range_mask[ranged] |= np.uint32(1 << 9)
    return sc


@pytest.mark.parametrize("V", [9, 16, 24, 32])
def test_view_counts_feature_rich_with_diff_and_layers_ext(V):
    sc = _wide_random_scene(V, V)
    n = sc.n
    rng = np.random.default_rng(V)
    ext = rng.integers(0, 4, (n, 3)).astype(np.uint64) << np.uint64(5)      # RenderLayers blocks 1..3
    view_ext = np.zeros((V, 3), np.uint64)
    view_ext[8:] = rng.integers(0, 4, (V - 8, 3)).astype(np.uint64) << np.uint64(5)
    orc.set_render_layers_ext(ext, view_ext)
    pipe = bb.VisibilityPipeline(sc)
    world = OracleWorld(sc, True)
    try:
        pipe.ctx.upload_render_layers_ext(0, ext)
        for v in range(V):
            pipe.ctx.set_view_render_layers_ext(v, view_ext[v])
        pipe.enable_visible_diff()
        for f in range(4):
            if f:
                scenes.advance_cameras(sc, 0.1)
                rows = np.unique(rng.integers(0, n, n // 20)).astype(np.uint32)
                sc.trs[rows, 0:3] += rng.uniform(-2, 2, (len(rows), 3)).astype(np.float32)
                pipe.ctx.upload_transforms_scattered(rows, sc.trs[rows])
                world.tchanged[rows] = 1
                sc.view_flags[8] = bb.VIEW_ACTIVE if f == 2 else 0
            pipe.update_views()
            compare_frame(pipe, world, f)
            _check_vv_count(pipe)
    finally:
        orc.set_render_layers_ext(None, None)
        pipe.close()


def test_rows_visible_only_past_the_eighth_view_toggle():
    """Views 0..7 render layer 1 only, view 8 the default layer: rows on layer 0 alone are visible in view 8 only.  They go
    0 -> 1, stay 1 (ViewVisibility bit 1 = last frame's), go 1 -> 0 with view 8 off, and come back; rows on both layers are
    seen by group 0 and left alone by the merge.  NoCpuCulling rows keep their uploaded ViewVisibility."""
    sc = _forest_ring(n_cameras=9, n_trees=80)
    rng = np.random.default_rng(5)
    n = sc.n
    sc.layer_mask = rng.choice([1, 1, 3], n).astype(np.uint64)
    sc.view_layers = [2] * 8 + [1]
    no_cull = rng.random(n) < 0.05
    sc.flags[no_cull] |= bb.F_NO_CPU_CULLING
    pipe = bb.VisibilityPipeline(sc)
    world = OracleWorld(sc, True)
    vv0 = np.where(no_cull & (rng.random(n) < 0.5), 1, 0).astype(np.uint8)
    pipe.ctx.upload_view_visibility(0, vv0); world.vv[:] = vv0
    seen = []
    try:
        for f, on in enumerate([1, 1, 0, 1, 1]):
            sc.view_flags = [bb.VIEW_ACTIVE] * 8 + [bb.VIEW_ACTIVE if on else 0]
            pipe.update_views()
            compare_frame(pipe, world, f)
            _check_vv_count(pipe)
            only8 = (sc.layer_mask == 1) & ~no_cull
            seen.append(int(((world.vv & 1) == 1)[only8].sum()))
            if f == 1:
                assert ((world.vv[only8] & 3) == 3).sum() > 20     # visible this frame and last
        assert seen[0] > 20 and seen[2] == 0 and seen[3] == seen[0]
    finally:
        pipe.close()


def test_light_seen_only_by_view_20_is_clustered_with_bindings():
    """A light above the camera ring that only view 20 (looking up) sees: its ViewVisibility comes from a group pass, so
    the cluster gather must run after the group passes; the ViewClusterBindings of views past the eighth are packed too."""
    sc = scenes.many_cameras_lights(21)
    r0 = sc.light_row[0]
    sc.trs[r0, 0:3] = (0.0, 60.0, 0.0)                       # above the ring: outside views 0..19
    cam = sc.cameras[20]
    q = scenes.look_at_quats(np.array([[0.0, 2.5, 0.0]]), target=(0.3, 60.0, 0.2))[0]
    cam.quat, cam.gt = q, scenes.quat_to_gt(q, (0.0, 2.5, 0.0))
    pipe = bb.VisibilityPipeline(sc)
    world = OracleWorld(sc, True)
    try:
        pipe.ctx.set_cluster_bindings(1)
        for f in range(3):
            pipe.update_views()
            compare_frame(pipe, world, f)
            assert world.vv[r0] & 1, "the light must be visible (in view 20 only)"
            # ... and no view of groups 0 and 1 sees it: a cull over views 0..19 alone neither lists it nor marks it visible
            planes = np.stack([np.ctypeslib.as_array(v.half_spaces).reshape(6, 4).copy() for v in pipe.views])
            vv = np.zeros(sc.n, np.uint8)
            _, lists = orc.cull(world.gt, sc.bounds, sc.flags, sc.class_mask, sc.entity_bits, vv, planes[:20])
            assert not vv[r0] & 1 and not any(r0 in l for l in lists)
            for v in range(21):
                offsets, idx = pipe.ctx.download_clusters(v)
                cv = pipe.cluster_views[v]
                nc = cv.dims[0] * cv.dims[1] * cv.dims[2]
                w_oc, w_il, w_no, w_ni = orc.cluster_bindings(offsets[:nc + 1], idx, None, storage=True)
                g_oc, g_il, g_no, g_ni = pipe.ctx.download_cluster_bindings(v)
                assert (g_no, g_ni) == (w_no, w_ni) and np.array_equal(g_oc, w_oc) and np.array_equal(g_il, w_il), v
            _, idx20 = pipe.ctx.download_clusters(20)
            assert (idx20 == 0).any(), "view 20 reaches the light: its clusters list it"
    finally:
        pipe.close()


def wide_frames(split, frames=4, n_cameras=16):
    """The forest ring with 16 cameras, every frame either fused (run_frame) or split into run(PROPAGATE), run(CULL) and
    run(CLUSTER) calls: the group passes follow the tile pass of a CULL-only run too."""
    sc = _forest_ring(n_cameras=n_cameras, n_trees=100)
    pipe = bb.VisibilityPipeline(sc)
    world = OracleWorld(sc, True)
    if split:
        pipe.run_frame = lambda: (pipe.ctx.run(bb.STAGE_PROPAGATE), pipe.ctx.run(bb.STAGE_CULL), pipe.ctx.run(bb.STAGE_CLUSTER))
    try:
        for f in range(frames):
            if f:
                scenes.rotate_cameras(sc, 0.3)
                rows, trs = scenes.mutate_roots(sc, f)
                pipe.ctx.upload_transforms_scattered(rows, trs)
                world.tchanged[rows] = 1
            pipe.update_views()
            compare_frame(pipe, world, f)
            _check_vv_count(pipe)
    finally:
        pipe.close()


def test_split_propagate_cull_cluster_runs():
    wide_frames(split=True)


def _run_case(code, env, timeout=600):
    e = {k: v for k, v in os.environ.items() if not k.startswith("B200VIS_")}
    e.update(env)
    prog = (f"import sys; sys.path.insert(0, {ROOT!r}); sys.path.insert(0, {os.path.join(ROOT, 'tests')!r})\n"
            "import test_gpu_many_views as t\n" + code)
    res = subprocess.run([sys.executable, "-c", prog], env=e, capture_output=True, text=True, timeout=timeout)
    assert res.returncode == 0, f"{env}\n{res.stdout[-2000:]}\n{res.stderr[-4000:]}"


@pytest.mark.parametrize("env", [{"B200VIS_PIPELINE": "0"}, {"B200VIS_TILE_KERNEL": "lean"}, {"B200VIS_SPLIT_DEEP_TILES": "1"}],
                         ids=["serial", "lean", "split_deep_tiles"])
def test_other_frame_paths_in_their_own_interpreter(env):
    _run_case("t.wide_frames(False)\nt.wide_frames(True, frames=3)", env)


def test_view_count_16_to_4_to_16():
    sc = _forest_ring(n_cameras=16, n_trees=80)
    all_cams = list(sc.cameras)
    pipe = bb.VisibilityPipeline(sc)
    world = OracleWorld(sc, True)
    try:
        for f, k in enumerate([16, 4, 4, 16, 16]):
            sc.cameras = all_cams[:k]
            if f:
                scenes.rotate_cameras(sc, 0.2)
            pipe.update_views()
            stats = compare_frame(pipe, world, f)
            _check_vv_count(pipe)
            assert len(stats.visible_count) == 16
    finally:
        pipe.close()


def test_four_views_on_a_wide_context_match_a_narrow_context_byte_for_byte():
    narrow_sc, wide_sc = (scenes.forest(n_trees=80, levels=6, n_lights=32) for _ in range(2))
    wide_sc.cameras = wide_sc.cameras * 4                     # the context is created for 16 views ...
    narrow, wide = bb.VisibilityPipeline(narrow_sc), bb.VisibilityPipeline(wide_sc)
    wide_sc.cameras = wide_sc.cameras[:4]                     # ... and runs 4
    assert (narrow.ctx.max_views, wide.ctx.max_views) == (4, 16)
    try:
        for f in range(3):
            for sc, p in ((narrow_sc, narrow), (wide_sc, wide)):
                if f:
                    scenes.advance_cameras(sc, 0.1)
                    rows, trs = scenes.mutate_roots(sc, f)
                    p.ctx.upload_transforms_scattered(rows, trs)
                p.update_views()
                p.run_frame()
            a, b = narrow.ctx, wide.ctx
            for x, y in zip(a.download_global_transforms(0, narrow_sc.n), b.download_global_transforms(0, wide_sc.n)):
                assert x.tobytes() == y.tobytes()
            for x, y in zip(a.download_view_visibility(0, narrow_sc.n), b.download_view_visibility(0, wide_sc.n)):
                assert x.tobytes() == y.tobytes()
            narrow.read_feedback(); wide.read_feedback()
            assert bytes(a.download_frame_stats()) == bytes(b.download_frame_stats())
            for v in range(4):
                assert a.download_visible(v).tobytes() == b.download_visible(v).tobytes()
                for x, y in zip(a.download_clusters(v), b.download_clusters(v)):
                    assert x.tobytes() == y.tobytes()
    finally:
        narrow.close(); wide.close()


def test_step_with_16_cameras_result_and_view_stats_sinks_and_column_write_back():
    """b200vis_step with 16 cameras: its Clusters feedback covers every view, the view-stats sink carries views 8..15 with
    the result sink's single synchronisation, and the host ViewVisibility column includes visibility only group passes find."""
    torch = pytest.importorskip("torch")
    sc = _forest_ring(n_cameras=16, n_trees=100)
    n, V = sc.n, 16
    pipe = bb.VisibilityPipeline(sc)
    world = OracleWorld(sc, True)
    st_t = torch.zeros(ctypes.sizeof(bb.FrameStats), dtype=torch.uint8).pin_memory()
    per_view = torch.zeros((V, 4), dtype=torch.int32).pin_memory().numpy().view(np.uint32)
    W = (n + 31) // 32
    gt_h = torch.zeros((n, 12), dtype=torch.float32).pin_memory().numpy()
    gbits = torch.zeros(W, dtype=torch.int32).pin_memory().numpy().view(np.uint32)
    vbits = torch.zeros(W, dtype=torch.int32).pin_memory().numpy().view(np.uint32)
    vv_h = torch.zeros(n, dtype=torch.uint8).pin_memory().numpy()
    try:
        pipe.ctx.set_result_sink(st_t.data_ptr(), None, None, None)
        pipe.ctx.set_view_stats_sink(per_view)
        pipe.ctx.set_column_sinks(gt_h, gbits, vv_h, vbits)
        group_only = 0
        for f in range(4):
            if f:
                scenes.rotate_cameras(sc, 0.25)
            rows, trs = scenes.mutate_roots(sc, f + 1)
            world.tchanged[rows] = 1
            r = np.ascontiguousarray(rows, np.uint32); t_ = np.ascontiguousarray(trs, np.float32)
            arr = (bb.CameraDesc * V)()
            for v, cam in enumerate(sc.cameras):
                arr[v].global_transform[:] = cam.gt.tolist()
                arr[v].fov_y, arr[v].aspect, arr[v].near_z, arr[v].far_z = cam.fov, cam.aspect, cam.near, cam.far
                arr[v].layer_mask, arr[v].flags, arr[v].range_view_index = 1, bb.VIEW_ACTIVE, -1
            pipe.ctx.step(len(r), r.ctypes.data, t_.ctypes.data, arr, V, pipe.cluster_config, wait=True, writeback=True)
            pipe.ctx.synchronize()
            planes = np.stack([bb.host_compute_frustum(bb.host_perspective(c.fov, c.aspect, c.near), c.gt, c.far) for c in sc.cameras])
            _, vv_changed, lists, clusters = world.frame(planes)
            assert (vv_h == world.vv).all(), f"frame {f}: host ViewVisibility column differs from the oracle"
            only_late = np.zeros(n, bool); early = np.zeros(n, bool)
            for v in range(V):
                (early if v < 8 else only_late)[lists[v]] = True
            group_only += int((only_late & ~early).sum())
            ref = pipe.ctx.download_view_stats()
            for v in range(V):
                out, _, idx = clusters[v]
                assert per_view[v, 0] == len(lists[v]) == ref["visible_count"][v], (f, v)
                assert per_view[v, 1] == out.total_index_count == ref["cluster_index_count"][v], (f, v)
                assert per_view[v, 2] == np.float32(out.farthest_z).view(np.uint32), (f, v)
                goff, gidx = pipe.ctx.download_clusters(v)
                assert np.array_equal(gidx, idx), (f, v)
        assert group_only > 0
    finally:
        pipe.ctx.set_column_sinks()
        pipe.ctx.set_view_stats_sink(None)
        pipe.ctx.set_result_sink(None, None, None, None)
        pipe.close()


def test_errors():
    for max_views, world_size in [(33, 1), (9, 2)]:
        with pytest.raises(bb.B200VisError) as e:
            bb.Context(64, max_views=max_views, world_size=world_size)
        assert e.value.code == 1
    ctx = bb.Context(64, max_lights=1, max_views=12)
    try:
        assert len(ctx.download_view_stats()["visible_count"]) == 12
        for first, count in [(12, 1), (0, 13), (11, 2)]:
            with pytest.raises(bb.B200VisError) as e:
                ctx.download_view_stats(first, count)
            assert e.value.code == 1
        with pytest.raises(bb.B200VisError):
            ctx.set_view_render_layers_ext(12, np.zeros(3, np.uint64))
        ctx.set_view_render_layers_ext(11, np.zeros(3, np.uint64))
    finally:
        ctx.close()
    narrow = bb.Context(64, max_lights=1, max_views=4)
    try:   # views 0..7 are accepted whatever max_views is, as they always were
        narrow.set_view_render_layers_ext(7, np.ones(3, np.uint64))
        with pytest.raises(bb.B200VisError):
            narrow.set_view_render_layers_ext(8, np.zeros(3, np.uint64))
    finally:
        narrow.close()


class WideTwins(Twins):
    """Twins (a compacting context and its twin) whose check covers every view of a wide context."""

    def check(self):
        ca, cb = self.a.pipe.ctx, self.b.pipe.ctx
        nb = self.b.sc.n
        live = np.nonzero(self.b.alive)[0]
        assert (self.m[live] != 0xFFFFFFFF).all()
        ma = self.m[live]
        ga, gcha = ca.download_global_transforms(0, self.a.sc.n)
        gb, gchb = cb.download_global_transforms(0, nb)
        assert (ga[ma].view(np.uint32) == gb[live].view(np.uint32)).all() and (gcha[ma] == gchb[live]).all()
        va, vcha = ca.download_view_visibility(0, self.a.sc.n)
        vb, vchb = cb.download_view_visibility(0, nb)
        assert (va[ma] == vb[live]).all() and (vcha[ma] == vchb[live]).all()
        sa, sb = ca.download_frame_stats(), cb.download_frame_stats()
        for f in ("frame", "gt_changed_count", "vv_changed_count"):
            assert getattr(sa, f) == getattr(sb, f), f
        wa, wb = ca.download_view_stats(), cb.download_view_stats()
        for k in wa:
            assert wa[k].tobytes() == wb[k].tobytes(), k
        for v in range(len(self.b.sc.cameras)):
            la, lb = ca.download_visible(v), cb.download_visible(v)
            assert (la == self.m[lb]).all(), f"view {v}: visible list"
            (aa, ra), (ab, rb) = ca.download_visible_diff(v), cb.download_visible_diff(v)
            assert (aa == self.m[ab]).all() and (ra == self.m[rb]).all(), f"view {v}: visible diff"
            oa, ia = ca.download_clusters(v)
            ob, ib = cb.download_clusters(v)
            assert (oa == ob).all() and (ia == ib).all()


def _late_only_leaves(ch, k):
    """Live leaves (no light, no root) that only views >= 8 list in the last frame's VisibleEntities."""
    sc, lists = ch.sc, ch.world.last_lists
    early = np.zeros(sc.n, bool); late = np.zeros(sc.n, bool)
    for v, l in enumerate(lists):
        (early if v < 8 else late)[l] = True
    ok = ch.alive & (ch.children() == 0) & late & ~early
    ok[sc.light_row] = False
    if sc.roots is not None:
        ok[sc.roots] = False
    rows = np.nonzero(ok)[0]
    return sorted(int(r) for r in ch.rng.choice(rows, size=min(k, len(rows)), replace=False)) if len(rows) else []


def _twin_despawn(t, despawn):
    """b despawns `despawn` (its row numbers) and spawns two flat rows; a does the same in its own numbers."""
    a, b = t.a, t.b
    spawn_parent = [0xFFFFFFFF] * 2
    trs = np.zeros((2, 10), np.float32); trs[:, 3:7] = (0, 0, 0, 1); trs[:, 7:10] = 1.0
    trs[:, 0:3] = b.rng.uniform(-20, 20, (2, 3))
    bits = b.new_bits(2)
    state = copy.deepcopy(b.rng.bit_generator.state)
    n_a = a.sc.n
    b.edit(despawn, [], [], spawn_parent, trs, bits)
    a.rng.bit_generator.state = state
    a.edit(t.map_rows(despawn), [], [], spawn_parent, trs, bits)
    t.m = np.concatenate([t.m, np.arange(n_a, n_a + 2)])


def test_edits_and_compaction_in_a_16_view_world():
    """A 16-view world with the visible diff on and shuffled entity bits, edited every frame.  Twice, rows that only views
    >= 8 list are despawned and the world is compacted right away, before any frame: the compaction keeps them as
    tombstones while those lists hold them, renumbers every view's lists and diff sets, and the next frame reports them
    removed.  Both contexts match the oracle frame by frame, and the compacting one matches its twin after every step."""
    t = WideTwins(lambda: _wide_random_scene(31, 16), 3000, seed=31)
    rng = np.random.default_rng(131)
    despawned = 0
    try:
        t.frame(0, animate=False)
        for f in range(1, 8):
            if f in (2, 5):
                late = _late_only_leaves(t.b, 6)
                despawned += len(late)
                _twin_despawn(t, late)
                t.compact(*order_keeping_reparents(t, 2, rng))
                t.check()                     # right after the compaction, before any run
            else:
                t.random_edit(n_despawn=4, n_flat=6, n_kids=2)
            t.frame(f)
            for ch in (t.a, t.b):
                _check_vv_count(ch.pipe)
        assert despawned > 0 and t.compactions == 2
    finally:
        t.close()
