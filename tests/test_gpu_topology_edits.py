"""b200vis_edit_topology on the device, bit-exact against the CPU oracle (tests/parity.py).

The oracle's arrays are edited the same way as the device world: spawned rows are appended, a despawned row becomes
B200VIS_DETACHED with flags NO_CPU_CULLING only, no class and ViewVisibility 0.  Every frame is then compared as usual:
GlobalTransform bits, both change columns, ViewVisibility, the sorted visible lists, the visible diff (against the
oracle's update_cpu_culled_entities, so a despawned visible row must be reported removed and nothing else may churn),
clusters with their feedback, and shadow lists where set up."""
import os
import subprocess
import sys

import numpy as np
import pytest

import bevy_b200 as bb
from bevy_b200 import abi, scenes
from parity import IDENTITY, OracleWorld, compare_frame

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
NO_PARENT, DETACHED = 0xFFFFFFFF, 0xFFFFFFFE
F_NO_CPU_CULL = 0x20
INVALID_ARG, CAPACITY, UNSUPPORTED = 1, 6, 8


class Churn:
    """Edits a scene, its oracle world and the device world in step.  Optional per-row columns (RenderLayers,
    VisibleEntityRanges masks, shadow casters) are followed when the scene has them."""

    def __init__(self, scene, headroom, static_opt=True, seed=0, visible_diff=True, cluster_config=None, cluster_kwargs=None):
        self.sc = scene
        self.pipe = bb.VisibilityPipeline(scene, static_transform_optimizations=static_opt, max_entities=scene.n + headroom,
                                          cluster_config=cluster_config)
        self.world = OracleWorld(scene, static_opt, cluster_kwargs=cluster_kwargs)
        if visible_diff:
            self.pipe.enable_visible_diff()
        if getattr(scene, "shadow_caster", None) is not None:
            self.pipe.ctx.upload_shadow_casters(0, scene.shadow_caster)
        self.rng = np.random.default_rng(seed)
        self.alive = np.ones(scene.n, bool)
        self.next_index = int((scene.entity_bits & np.uint64(0xFFFFFFFF)).max()) + 1
        self.gen = 8
        # new rows' optional columns: uploaded (True), or left at what the edit writes (False: layer 0, no range bits,
        # not a caster) -- which is what rows reused after a compaction must show
        self.upload_optional = True

    def children(self):
        n = self.sc.n
        kids = np.zeros(n, np.int64)
        p = self.sc.parent
        real = p < n
        np.add.at(kids, p[real], 1)
        return kids

    def new_bits(self, k):
        """Half reuse a dead row's index under a new generation (ranks after every older generation of it), half take
        fresh indices: over a few frames the keys interleave with the old ones."""
        out = []
        dead = np.nonzero(~self.alive)[0]
        for _ in range(k):
            if len(dead) and self.rng.random() < 0.5:
                idx = int(self.sc.entity_bits[int(self.rng.choice(dead))]) & 0xFFFFFFFF
                out.append(idx | (self.gen << 32)); self.gen += 1
            else:
                out.append(self.next_index); self.next_index += 1
        return np.asarray(out, np.uint64)

    def random_edit(self, n_despawn=4, n_flat=4, n_kids=2, n_reparent=2, kill_light=True):
        sc, rng = self.sc, self.rng
        kids = self.children()
        lights = np.zeros(sc.n, bool); lights[sc.light_row] = True
        roots = np.zeros(sc.n, bool)
        if sc.roots is not None:
            roots[sc.roots] = True
        leaves = np.nonzero(self.alive & (kids == 0) & ~roots & ~lights)[0]
        despawn = rng.choice(leaves, size=min(n_despawn, len(leaves)), replace=False).tolist()
        if kill_light and len(sc.light_row) > 2:           # a light that is not a shadow light
            sl = getattr(sc, "shadow_lights", None)
            shadow = set() if sl is None else set(int(sc.light_row[o]) for o in sl)
            cands = [int(r) for r in sc.light_row if int(r) not in shadow and kids[r] == 0]
            if cands:
                despawn.append(int(rng.choice(cands)))
        despawn = sorted(set(int(d) for d in despawn))
        gone = np.zeros(sc.n, bool); gone[despawn] = True
        cands = np.nonzero(self.alive & (kids == 0) & ~roots & ~lights & ~gone & (sc.parent < sc.n))[0]
        reparent, new_parent = [], []
        for r in rng.choice(cands, size=min(n_reparent, len(cands)), replace=False).tolist() if len(cands) else []:
            p = NO_PARENT
            if rng.random() >= 0.4:
                # a row that already has children: no tile gains a parent slot (a leaf becoming a parent could need a
                # 129th slot in a full tile, which the edit refuses with UNSUPPORTED)
                lo = max(0, r - 300)
                below = lo + np.nonzero(self.alive[lo:r] & (kids[lo:r] > 0) & ~gone[lo:r])[0]
                if len(below):
                    p = int(rng.choice(below))
            reparent.append(int(r)); new_parent.append(p)
        pool = np.nonzero(self.alive & ~gone & ~lights)[0]
        parents = [int(x) for x in rng.choice(pool, size=n_kids)]
        spawn_parent = [NO_PARENT] * n_flat + parents
        trs = np.zeros((len(spawn_parent), 10), np.float32)
        trs[:, 3:7] = (0, 0, 0, 1); trs[:, 7:10] = 1.0
        trs[:n_flat, 0:3] = rng.uniform(-40, 40, (n_flat, 3))          # near the cameras: many of them are visible
        trs[n_flat:, 0:3] = rng.uniform(-2, 2, (n_kids, 3))
        return self.edit(despawn, reparent, new_parent, spawn_parent, trs)

    def edit(self, despawn, reparent, new_parent, spawn_parent, trs, bits=None):
        sc, w, c = self.sc, self.world, self.pipe.ctx
        n0, k = sc.n, len(spawn_parent)
        bits = self.new_bits(k) if bits is None else np.asarray(bits, np.uint64)
        # a light leaves the light list before its row is despawned (the edit refuses a row that is still a light)
        if len(despawn) and np.isin(sc.light_row, despawn).any():
            keep = ~np.isin(sc.light_row, despawn)
            if getattr(sc, "shadow_lights", None) is not None:         # shadow lights are ordinals into the light list
                new_ord = np.cumsum(keep) - 1
                sc.shadow_lights = new_ord[sc.shadow_lights].astype(np.uint32)
            sc.light_row, sc.light_range = sc.light_row[keep], sc.light_range[keep]
            if sc.light_layers is not None:
                sc.light_layers = sc.light_layers[keep]
            c.set_lights(sc.light_row, sc.light_range, sc.light_layers)
        c.edit_topology(despawn, reparent, new_parent, spawn_parent, bits)
        # oracle side: tombstones, new parents, appended rows
        d = np.asarray(despawn, np.int64)
        sc.parent[d] = DETACHED; sc.flags[d] = F_NO_CPU_CULL; sc.class_mask[d] = 0
        w.vv[d] = 0; w.tchanged[d] = 0
        if getattr(sc, "shadow_caster", None) is not None:
            sc.shadow_caster[d] = 0
        self.alive[d] = False
        for r, p in zip(reparent, new_parent):
            sc.parent[r] = p; w.tchanged[r] = 1
        bounds = np.zeros((k, 6), np.float32); bounds[:, 3:6] = 0.5
        flags = np.full(k, scenes.F_INHERITED_VISIBLE | scenes.F_HAS_AABB, np.uint8)
        cls = np.full(k, scenes.CLASS_MESH, np.uint8)
        rng = self.rng
        layers = rng.choice(np.array([1, 2, 3], np.uint64), k) if self.upload_optional else np.ones(k, np.uint64)
        ranges = rng.integers(0, 8, k).astype(np.uint32) if self.upload_optional else np.zeros(k, np.uint32)
        casters = (rng.random(k) < 0.7).astype(np.uint8) if self.upload_optional else np.zeros(k, np.uint8)
        sc.parent = np.concatenate([sc.parent, np.asarray(spawn_parent, np.uint32)])
        sc.trs = np.concatenate([sc.trs, trs]); sc.bounds = np.concatenate([sc.bounds, bounds])
        sc.flags = np.concatenate([sc.flags, flags]); sc.class_mask = np.concatenate([sc.class_mask, cls])
        sc.entity_bits = np.concatenate([sc.entity_bits, bits])
        if sc.layer_mask is not None:
            sc.layer_mask = np.concatenate([sc.layer_mask, layers])
        if sc.range_mask is not None:
            sc.range_mask = np.concatenate([sc.range_mask, ranges])
        if getattr(sc, "shadow_caster", None) is not None:
            sc.shadow_caster = np.concatenate([sc.shadow_caster, casters])
        w.gt = np.concatenate([w.gt, np.tile(IDENTITY, (k, 1))]); w.vv = np.concatenate([w.vv, np.zeros(k, np.uint8)])
        w.tchanged = np.concatenate([w.tchanged, np.ones(k, np.uint8)])
        self.alive = np.concatenate([self.alive, np.ones(k, bool)])
        if sc.roots is not None and len(despawn):
            sc.roots = sc.roots[~np.isin(sc.roots, despawn)]
        # device side: the new rows' columns
        if k:
            c.upload_transforms(n0, trs)
            c.upload_global_transforms(n0, np.tile(IDENTITY, (k, 1)))
            opt = self.upload_optional
            c.upload_bounds(n0, bounds, flags, cls, layers if opt and sc.layer_mask is not None else None,
                            ranges if opt and sc.range_mask is not None else None)
            if opt and getattr(sc, "shadow_caster", None) is not None:
                c.upload_shadow_casters(n0, casters)
        return list(range(n0, n0 + k))

    def compact(self):
        """What the shim's fallback does: the live rows renumbered through set_topology, every column uploaded again."""
        sc, w, c = self.sc, self.world, self.pipe.ctx
        n = sc.n
        live = np.nonzero(self.alive)[0]
        remap = np.full(n, -1, np.int64); remap[live] = np.arange(len(live))
        p = sc.parent[live].astype(np.int64)
        real = p < n
        p[real] = remap[p[real]]
        sc.parent = p.astype(np.uint32)
        for name in ("trs", "bounds", "flags", "class_mask", "entity_bits", "layer_mask", "range_mask", "shadow_caster"):
            if getattr(sc, name, None) is not None:
                setattr(sc, name, getattr(sc, name)[live])
        sc.light_row = remap[sc.light_row].astype(np.uint32)
        if sc.roots is not None:
            sc.roots = remap[sc.roots].astype(np.uint32)
        w.gt, w.vv, w.tchanged = w.gt[live], w.vv[live], np.ones(len(live), np.uint8)
        w.last_lists = [np.zeros(0, np.uint32) for _ in sc.cameras]        # fresh frame state: every visible row is added
        self.alive = np.ones(len(live), bool)
        c.set_topology(sc.parent, sc.entity_bits)
        c.upload_transforms(0, sc.trs)
        c.upload_global_transforms(0, w.gt)
        c.upload_bounds(0, sc.bounds, sc.flags, sc.class_mask, sc.layer_mask, sc.range_mask)
        c.upload_view_visibility(0, w.vv)
        if getattr(sc, "shadow_caster", None) is not None:
            c.upload_shadow_casters(0, sc.shadow_caster)
        c.set_lights(sc.light_row, sc.light_range, sc.light_layers)
        assert c.topology_summary()[:2] == (len(live), len(live))

    def frame(self, f, animate=True):
        sc = self.sc
        if animate:
            scenes.advance_cameras(sc, 0.05)
            rows, trs = scenes.mutate_roots(sc, f)
            self.pipe.ctx.upload_transforms_scattered(rows, trs)
            self.world.tchanged[rows] = 1
        self.pipe.update_views()
        return compare_frame(self.pipe, self.world, f)

    def close(self):
        self.pipe.close()


def run_unchecked(ch):
    """One frame on both sides without comparing it (the next compared frame still checks the diff against it)."""
    pipe, world = ch.pipe, ch.world
    planes = np.stack([np.ctypeslib.as_array(v.half_spaces).reshape(6, 4).copy() for v in pipe.views])
    _, _, lists, _ = world.frame(planes)
    world.last_lists = [l if l is not None else world.last_lists[v] for v, l in enumerate(lists)]
    pipe.run_frame()


def churn(n_trees=60, n_lights=24, frames=12, static_opt=True, seed=1, headroom=4000, last_only=False, **edit_kw):
    """Random churn every frame on a forest; every frame (or only the last one) compared with the oracle."""
    ch = Churn(scenes.forest(n_trees, 8, n_lights, seed=seed), headroom, static_opt=static_opt, seed=seed)
    try:
        ch.frame(0, animate=False)
        for f in range(1, frames):
            ch.random_edit(**edit_kw)
            if last_only and f < frames - 1:
                scenes.advance_cameras(ch.sc, 0.05)
                rows, trs = scenes.mutate_roots(ch.sc, f)
                ch.pipe.ctx.upload_transforms_scattered(rows, trs)
                ch.world.tchanged[rows] = 1
                ch.pipe.update_views()
                run_unchecked(ch)
                ch.pipe.read_feedback()
            else:
                ch.frame(f)
        n, live, tiles, passes = ch.pipe.ctx.topology_summary()
        assert n == ch.sc.n and live == int(ch.alive.sum()) and passes >= 1
        return ch.pipe.ctx.topology_summary()
    finally:
        ch.close()


@pytest.mark.parametrize("static_opt", [True, False])
def test_random_churn_matches_the_oracle(static_opt):
    churn(static_opt=static_opt)


def test_spawning_visible_rows_reports_exactly_them_added():
    sc = scenes.forest(20, 6, 8, seed=3)
    sc.entity_bits = sc.entity_bits * np.uint64(2) + np.uint64(2)        # even keys from 2: room before and between them
    ch = Churn(sc, 100)
    try:
        for f in range(2):
            ch.frame(f, animate=False)
        trs = np.zeros((3, 10), np.float32); trs[:, 3:7] = (0, 0, 0, 1); trs[:, 7:10] = 1.0
        trs[:, 0:3] = [(0, 0, -10), (1, 0, -12), (-1, 1, -15)]          # in front of camera 0 (looks down -Z)
        new = ch.edit([], [], [], [NO_PARENT] * 3, trs, bits=[1, 1 << 40, 7])   # ranks before, after and between old keys
        ch.frame(2, animate=False)
        added, removed = ch.pipe.ctx.download_visible_diff(0)
        assert sorted(added.tolist()) == sorted(new) and len(removed) == 0
        for v in range(1, len(ch.sc.cameras)):
            a, r = ch.pipe.ctx.download_visible_diff(v)
            assert len(r) == 0 and set(a.tolist()) <= set(new)
        # despawning one of them: reported removed, nothing else
        ch.edit([new[1]], [], [], [], np.zeros((0, 10), np.float32))
        ch.frame(3, animate=False)
        added, removed = ch.pipe.ctx.download_visible_diff(0)
        assert len(added) == 0 and removed.tolist() == [new[1]]
    finally:
        ch.close()


def test_errors_change_nothing_and_compaction_continues():
    ch = Churn(scenes.forest(20, 6, 8, seed=4), 40)
    try:
        ch.frame(0, animate=False)
        ch.random_edit(n_flat=3, n_kids=2)
        ch.frame(1, animate=False)
        c, sc = ch.pipe.ctx, ch.sc
        n = sc.n
        kids = ch.children()
        with_kids = int(np.nonzero((kids > 0) & ch.alive)[0][0])
        dead = int(np.nonzero(~ch.alive)[0][0])
        leaf = int(np.nonzero((kids == 0) & ch.alive)[0][-1])
        before_leaf = int(np.nonzero(ch.alive[:leaf])[0][-1])
        cases = [
            (dict(spawn_parent=[NO_PARENT] * 41, spawn_entity_bits=np.arange(41) + (9 << 40)), CAPACITY),
            (dict(despawn=[n]), INVALID_ARG),
            (dict(despawn=[dead]), INVALID_ARG),
            (dict(despawn=[with_kids]), INVALID_ARG),
            (dict(spawn_parent=[NO_PARENT], spawn_entity_bits=[int(sc.entity_bits[dead])]), INVALID_ARG),   # dead rows keep their key
            (dict(spawn_parent=[NO_PARENT], spawn_entity_bits=[int(sc.entity_bits[0])]), INVALID_ARG),
            (dict(spawn_parent=[NO_PARENT, NO_PARENT], spawn_entity_bits=[3 << 40, 3 << 40]), INVALID_ARG),
            (dict(reparent=[before_leaf], new_parent=[leaf]), UNSUPPORTED),
        ]
        cases.append((dict(despawn=[int(sc.light_row[0])]), INVALID_ARG))      # still a light: set_lights first
        for kw, code in cases:
            with pytest.raises(bb.B200VisError) as e:
                c.edit_topology(**kw)
            assert e.value.code == code, kw
        with pytest.raises(bb.B200VisError) as e:
            c.set_lights(np.asarray([dead], np.uint32), np.ones(1, np.float32), None)
        assert e.value.code == INVALID_ARG
        assert c.topology_summary()[0] == n
        ch.frame(2, animate=False)
        ch.compact()
        ch.frame(3, animate=False)
        ch.random_edit()
        ch.frame(4)
    finally:
        ch.close()


def run_case(code, env, timeout=600):
    e = dict(os.environ)
    for k in [k for k in e if k.startswith("B200VIS_")]:
        del e[k]
    e.update(env)
    prog = f"import sys; sys.path.insert(0, {ROOT!r}); sys.path.insert(0, {HERE!r})\nimport test_gpu_topology_edits as t\n" + code
    res = subprocess.run([sys.executable, "-c", prog], env=e, capture_output=True, text=True, timeout=timeout)
    assert res.returncode == 0, f"{env}\n{res.stdout[-2000:]}\n{res.stderr[-4000:]}"
    return res.stdout


@pytest.mark.parametrize("variant", ["default", "lean", "warp"])
def test_bench_scale_churn(variant):
    # the bench world (config #3, ~1 M rows, 256 lights, 4 views): 16 projectiles despawned and spawned per frame plus
    # children under existing trees for 50 frames, the last one compared with the oracle; each tile kernel in its own
    # interpreter
    env = {"default": {}, "lean": {"B200VIS_TILE_KERNEL": "lean"}, "warp": {"B200VIS_TILE_KERNEL": "warp", "B200VIS_WARP_VARIANT": "2p"}}[variant]
    out = run_case("print(t.churn(n_trees=3922, n_lights=256, frames=50, headroom=20000, last_only=True, n_despawn=16, n_flat=16, n_kids=2))",
                   env, timeout=900)
    assert out.strip()


def test_a_failed_edit_after_the_descriptor_buffers_grew_changes_nothing():
    # enough spawned rows to outgrow the tile-descriptor buffers, and a despawn that makes the edit fail: the next
    # frame must still run the old plan
    ch = Churn(scenes.forest(20, 6, 8, seed=6), 1600)
    try:
        ch.frame(0, animate=False)
        n = ch.sc.n
        with pytest.raises(bb.B200VisError) as e:
            ch.pipe.ctx.edit_topology(despawn=[n], spawn_parent=[NO_PARENT] * 1500,
                                      spawn_entity_bits=np.arange(1500, dtype=np.uint64) + np.uint64(5 << 40))
        assert e.value.code == INVALID_ARG
        assert ch.pipe.ctx.topology_summary()[0] == n
        ch.frame(1)
        ch.random_edit()
        ch.frame(2)
        trs = np.zeros((1500, 10), np.float32); trs[:, 3:7] = (0, 0, 0, 1); trs[:, 7:10] = 1.0
        trs[:, 0:3] = ch.rng.uniform(-40, 40, (1500, 3))
        ch.edit([], [], [], [NO_PARENT] * 1500, trs)
        ch.frame(3)
    finally:
        ch.close()


@pytest.mark.parametrize("seed,static_opt", [(21, True), (22, False)])
def test_feature_rich_churn_with_shadows_layers_ranges_and_compaction(seed, static_opt):
    """The edge-case scene (RenderLayers, VisibleEntityRanges, NoCpuCulling, detached subtrees, shuffled entity bits so
    every spawn merges ranks) with point-light shadow culling, churned every frame.  After a compaction the spawned rows
    reuse row numbers that held other columns: they get no layer / range / caster upload, so the values the edit writes
    are what the oracle sees."""
    import test_gpu_edge_cases as ec
    sc = ec._random_scene(seed, n_roots=90, n_lights=20)
    rng = np.random.default_rng(seed)
    sc.shadow_lights = np.sort(rng.choice(len(sc.light_row), 6, replace=False)).astype(np.uint32)
    sc.shadow_caster = (rng.random(sc.n) < 0.8).astype(np.uint8)
    sc.shadow_caster[sc.light_row] = 0
    sc.shadow_near_z, sc.shadow_lod_origin = 0.1, 0
    ch = Churn(sc, 3000, static_opt=static_opt, seed=seed)
    try:
        ch.frame(0, animate=False)
        for f in range(1, 6):
            ch.random_edit(n_despawn=6, n_flat=6, n_kids=3)
            ch.frame(f)
        ch.compact()
        ch.frame(6, animate=False)
        ch.upload_optional = False
        for f in range(7, 11):
            ch.random_edit(n_despawn=6, n_flat=6, n_kids=3)
            ch.frame(f)
        assert sum(len(l) for six in ch.world.shadow_result.values() for l in six) > 0
    finally:
        ch.close()


def test_step_with_result_and_column_sinks_across_edits():
    """b200vis_step with a result sink and column sinks, edits between the steps: the host mirror updated only through
    the sinks stays identical to a full download (new rows' ViewVisibility is sent on their first write-back), and the
    sink's stats and visible rows equal the download calls."""
    torch = pytest.importorskip("torch")
    import ctypes
    sc = scenes.forest(70, 6, 12, seed=7)
    H = 400
    ch = Churn(sc, H, seed=7)
    N, V = sc.n + H, len(sc.cameras)
    W = (N + 31) // 32
    gt_h = torch.zeros((N, 16), dtype=torch.float32).pin_memory().numpy()
    gt_h[:] = np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0], np.float32)
    gbits = torch.zeros(W, dtype=torch.int32).pin_memory().numpy().view(np.uint32)
    vbits = torch.zeros(W, dtype=torch.int32).pin_memory().numpy().view(np.uint32)
    vv_h = torch.zeros(N, dtype=torch.uint8).pin_memory().numpy()
    vis = torch.zeros((V, N), dtype=torch.int32).pin_memory().numpy().view(np.uint32)
    off = torch.zeros((V, 4097), dtype=torch.int32).pin_memory().numpy().view(np.uint32)
    idx = torch.zeros((V, 1 << 16), dtype=torch.int32).pin_memory().numpy().view(np.uint32)
    st_t = torch.zeros(ctypes.sizeof(bb.FrameStats), dtype=torch.uint8).pin_memory()
    st = bb.FrameStats.from_address(st_t.data_ptr())
    c = ch.pipe.ctx

    def unpack(bits, n):
        return np.unpackbits(bits.view(np.uint8), bitorder="little")[:n]
    try:
        c.set_column_sinks(gt_h, gbits, vv_h, vbits)
        c.set_result_sink(st_t.data_ptr(), vis, off, idx)
        for f in range(7):
            if f:
                ch.random_edit(n_despawn=3, n_flat=6, n_kids=2)
            scenes.advance_cameras(sc, 0.05)
            rows, trs = scenes.mutate_roots(sc, f + 1)
            arr = (bb.CameraDesc * V)()
            for v, cam in enumerate(sc.cameras):
                arr[v].global_transform[:] = cam.gt.tolist()
                arr[v].fov_y, arr[v].aspect, arr[v].near_z, arr[v].far_z = cam.fov, cam.aspect, cam.near, cam.far
                arr[v].layer_mask, arr[v].flags, arr[v].range_view_index = 1, bb.VIEW_ACTIVE, -1
            r = np.ascontiguousarray(rows, np.uint32); t_ = np.ascontiguousarray(trs, np.float32)
            c.step(len(r), r.ctypes.data, t_.ctypes.data, arr, V, ch.pipe.cluster_config, wait=True, writeback=True)
            c.synchronize()
            n = sc.n
            gt, gch = c.download_global_transforms(0, n, stride=16)
            vv, vch = c.download_view_visibility(0, n)
            assert (unpack(gbits, n) == gch).all() and (unpack(vbits, n) == vch).all(), f
            assert (gt_h[:n].view(np.uint32) == gt.view(np.uint32)).all(), f"frame {f}: host GlobalTransform mirror differs"
            assert (vv_h[:n] == vv).all(), f"frame {f}: host ViewVisibility mirror differs"
            ref = c.download_frame_stats()
            assert (st.frame, st.gt_changed_count, st.vv_changed_count) == (ref.frame, ref.gt_changed_count, ref.vv_changed_count)
            for v in range(V):
                assert st.visible_count[v] == ref.visible_count[v]
                assert (vis[v, :st.visible_count[v]] == c.download_visible(v)).all()
        c.set_column_sinks()
        c.set_result_sink(None, None, None, None)
    finally:
        ch.close()


def test_back_to_back_pipelined_frames_with_edits_between():
    """run(STAGE_ALL) frames submitted without reading anything back, an edit before each: the edit joins the tail of the
    frame in flight (it reads the rank arrays and the visible sets).  Only the last frame is compared; the cluster config
    is feedback-free so no per-frame read-back is needed."""
    sc = scenes.forest(n_trees=300, levels=8, n_lights=48, seed=9)
    cfg = bb.host_default_cluster_config(*sc.screen)
    cfg.far_z_mode, cfg.far_z_constant, cfg.dynamic_resizing = 1, 90.0, 0
    kw = dict(far_z_mode=1, far_z_constant=90.0, dynamic_resizing=False)
    ch = Churn(sc, 3000, seed=9, cluster_config=cfg, cluster_kwargs=kw)
    try:
        frames = 8
        for f in range(frames):
            if f:
                ch.random_edit(n_despawn=8, n_flat=8, n_kids=3)
                scenes.advance_cameras(sc, 0.01)
                rows, trs = scenes.mutate_roots(sc, f)
                ch.pipe.ctx.upload_transforms_scattered(rows, trs)
                ch.world.tchanged[rows] = 1
            ch.pipe.update_views()
            if f < frames - 1:
                run_unchecked(ch)
            else:
                compare_frame(ch.pipe, ch.world, f)
    finally:
        ch.close()
