"""RenderLayers blocks 1..3 (layers 64..255) of lights and shadow items on the device, against the oracle restated over the
whole RenderLayers (tests/light_layers_reference.py):

1. Clusters: lights with the default layer, none(), block 0 only, blocks 1..3 only and both, views with and without a
   layer in block 0, over several frames of the Clusters feedback loop, with 4 and 12 views, under every cluster-kernel
   switch (one interpreter per switch: the switches are read once per process).
2. Moving every layer k to k + 64 j gives bit-identical cluster lists, index counts and farthest z on the device.
3. A context that never calls the new entry points and one that calls them with empty blocks and then NULL give
   bit-identical outputs.
4. Shadows: point, spot and cascade items with blocks 1..3 against rows with blocks 1..3: the lists, the ViewVisibility
   bytes and change flags, the entity sink and the diff sink, every frame.
5. Lifetime and errors: b200vis_set_lights and b200vis_set_shadow_items empty the blocks, an edit and a compaction keep
   them, a count mismatch is INVALID_ARG and changes nothing.  (world_size > 1 returns UNSUPPORTED; that needs two GPUs
   and is not exercised here.)"""
import copy
import os
import subprocess
import sys

import numpy as np
import pytest

import bevy_b200 as bb
import light_layers_reference as LR
import oracle as orc
from bevy_b200 import abi, scenes
from light_layers_reference import RenderLayers
from test_gpu_cull_outputs import pinned
from test_gpu_shadow_outputs import ShadowSink

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
U64 = np.uint64
INVALID_ARG = 1
IDENT9 = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1], np.float32)

LIGHT_KINDS = [[0], None, [3], [70], [5, 130], [201], [0, 140]]      # None = RenderLayers::none()
VIEW_KINDS = [[0], [70], [0, 140], [3, 201], [130], [5]]
ROW_KINDS = [[0], [70], [3, 140], [201], None, [0, 130], [5]]


def blocks_of(kinds, n, rng=None):
    pick = (np.arange(n) % len(kinds)) if rng is None else rng.integers(0, len(kinds), n)
    return np.stack([RenderLayers.from_layers(kinds[k] or []).blocks4() for k in pick]) if n else np.zeros((0, 4), U64)


def fold(kinds):
    return [None if x is None else sorted({k % 64 for k in x}) for x in kinds]


def layered_scene(n_cams, seed=0, n_lights=64, shift=0, low=False):
    """A compact forest (roots within +-50, among the lights), n_cams cameras, and RenderLayers everywhere.  A light's row
    has the light's own RenderLayers (one component per entity).  low: every layer taken modulo 64 (block 0 only);
    shift: then every layer k becomes k + 64 shift."""
    sc = scenes.forest(n_trees=48, levels=6, n_lights=n_lights, seed=seed)
    sc.trs[sc.roots, 0:3] *= np.float32(0.1)
    sc.cameras = [scenes._camera(2 * np.pi * k / n_cams + 0.1 * seed) for k in range(n_cams)]
    rng = np.random.default_rng(seed)
    rb = blocks_of(fold(ROW_KINDS) if low else ROW_KINDS, sc.n, rng)
    lb = blocks_of(fold(LIGHT_KINDS) if low else LIGHT_KINDS, n_lights)
    vb = blocks_of(fold(VIEW_KINDS) if low else VIEW_KINDS, n_cams)
    rb[sc.light_row] = lb
    rb, lb, vb = LR.shifted(rb, shift), LR.shifted(lb, shift), LR.shifted(vb, shift)
    sc.layer_mask = np.ascontiguousarray(rb[:, 0]); sc.light_layers = np.ascontiguousarray(lb[:, 0])
    sc.view_layers = [int(x) for x in vb[:, 0]]
    return sc, rb, vb, lb


class LayeredOracle:
    """The oracle side of a layered scene: propagate, the camera cull with the entity / view blocks, the clusters over
    the whole RenderLayers with each view's Clusters feedback."""

    def __init__(self, sc, rb, vb, lb):
        self.sc, self.rb, self.vb, self.lb = sc, rb, vb, lb
        self.gt = np.tile(orc.IDENTITY_GT, (sc.n, 1))
        self.vv = np.zeros(sc.n, np.uint8)
        self.tchanged = np.ones(sc.n, np.uint8)
        self.fb = [dict(far=None, cnt=None) for _ in sc.cameras]
        self.last_lists = [np.zeros(0, np.uint32) for _ in sc.cameras]

    def cull(self, planes, defer=False):
        sc = self.sc
        orc.propagate(sc.parent, sc.trs, self.gt, self.tchanged, True)
        self.tchanged[:] = 0
        orc.set_render_layers_ext(self.rb[:, 1:], self.vb[:, 1:])
        orc.set_defer_mark_newly_hidden(defer)
        try:
            vv_changed, lists = orc.cull(self.gt, sc.bounds, sc.flags, sc.class_mask, sc.entity_bits, self.vv, planes,
                                         view_layers=np.ascontiguousarray(self.vb[:, 0]), layer_mask=sc.layer_mask)
        finally:
            orc.set_render_layers_ext(None, None)
            orc.set_defer_mark_newly_hidden(False)
        self.last_lists = [l if l is not None else self.last_lists[v] for v, l in enumerate(lists)]
        return vv_changed

    def clusters(self, planes):
        sc = self.sc
        vis = np.nonzero(self.vv[sc.light_row] & 1)[0]
        lights = np.concatenate([self.gt[sc.light_row[vis], 9:12], sc.light_range[vis, None]], 1).astype(np.float32)
        out = []
        for v, cam in enumerate(sc.cameras):
            vin = orc.default_cluster_view_in(cam.gt, orc.perspective(cam.fov, cam.aspect, cam.near), planes[v], screen=sc.screen,
                                              last_farthest_z=self.fb[v]["far"], last_index_count=self.fb[v]["cnt"])
            o, off, idx, _ = LR.assign_lights_to_clusters(vin, lights, self.lb[vis], self.vb[v])
            self.fb[v] = dict(far=o.farthest_z, cnt=o.total_index_count)
            out.append((tuple(o.dims), off, vis[idx].astype(np.uint32), o.total_index_count, np.float32(o.farthest_z)))
        return out


def setup_device(sc, rb, vb, lb, ext=True):
    pipe = bb.VisibilityPipeline(sc)
    if ext:
        pipe.ctx.upload_render_layers_ext(0, rb[:, 1:])
        pipe.ctx.set_light_render_layers_ext(lb[:, 1:])
    return pipe


def device_frame(pipe, vb, ext=True):
    pipe.update_views()
    if ext:
        for v in range(len(vb)):
            pipe.ctx.set_view_render_layers_ext(v, vb[v, 1:])
    pipe.run_frame()
    return np.stack([np.ctypeslib.as_array(v.half_spaces).reshape(6, 4).copy() for v in pipe.views])


def device_clusters(pipe):
    st = pipe.read_feedback()
    out = []
    for v in range(len(pipe.scene.cameras)):
        off, idx = pipe.ctx.download_clusters(v)
        out.append((tuple(pipe.cluster_views[v].dims), off, idx, int(st.cluster_index_count[v]),
                    np.float32(st.cluster_farthest_z[v])))
    return out


def same_clusters(got, want, tag):
    for v, (g, w) in enumerate(zip(got, want)):
        assert g[0] == w[0], f"{tag} view {v}: dims {g[0]} vs {w[0]}"
        nc = int(np.prod(w[0]))
        assert (g[1][:nc + 1] == w[1][:nc + 1]).all(), f"{tag} view {v}: offsets differ"
        assert len(g[2]) == len(w[2]) and (g[2] == w[2]).all(), f"{tag} view {v}: indices differ ({len(g[2])} vs {len(w[2])})"
        assert g[3] == w[3], f"{tag} view {v}: index count {g[3]} vs {w[3]}"
        assert g[4].view(np.uint32) == w[4].view(np.uint32), f"{tag} view {v}: farthest_z {g[4]} vs {w[4]}"


# ---- 1 + 2: clusters -----------------------------------------------------------------------------------------------------
def case_clusters(n_cams, frames=4, shift=0, seed=0, low=False):
    """Device against the oracle every frame; returns the device's per-frame clusters."""
    sc, rb, vb, lb = layered_scene(n_cams, seed, shift=shift, low=low)
    pipe = setup_device(sc, rb, vb, lb)
    orw = LayeredOracle(sc, rb, vb, lb)
    frames_out, layered_hits = [], 0
    try:
        for f in range(frames):
            if f:
                scenes.advance_cameras(sc, 0.05)
            planes = device_frame(pipe, vb)
            orw.cull(planes)
            want = orw.clusters(planes)
            got = device_clusters(pipe)
            vv, _ = pipe.ctx.download_view_visibility(0, sc.n)
            assert (vv == orw.vv).all(), f"frame {f}: ViewVisibility differs on {np.nonzero(vv != orw.vv)[0][:8]}"
            same_clusters(got, want, f"[{n_cams} views, shift {shift}, frame {f}]")
            frames_out.append(got)
            # light ordinals reaching a view only through blocks 1..3
            ext_only = ~LR.intersects(lb[:, :1], vb[:, None, :1]) & LR.intersects(lb, vb[:, None])
            layered_hits += sum(int(np.isin(g[2], np.nonzero(ext_only[v])[0]).sum()) for v, g in enumerate(got))
        assert sum(g[3] for g in frames_out[-1]) > 0
        assert layered_hits > 0 or (low and not shift), "no light was clustered through blocks 1..3"
    finally:
        pipe.close()
    return frames_out


@pytest.mark.parametrize("n_cams", [4, 12])
def test_clusters_match_the_oracle(n_cams):
    case_clusters(n_cams)


def switch_cases():
    case_clusters(4)
    case_clusters(12, frames=3)


SWITCHES = {
    "default": {},
    "split": {"B200VIS_CLUSTER_KERNEL": "split"},
    "ctas_4": {"B200VIS_CLUSTER_CTAS": "4"},
    "ctas_16": {"B200VIS_CLUSTER_CTAS": "16"},
    "no_branch": {"B200VIS_CLUSTER_BRANCH": "0"},
    "serial": {"B200VIS_PIPELINE": "0"},
}


@pytest.mark.parametrize("switch", list(SWITCHES))
def test_cluster_kernel_switches(switch):
    e = {k: v for k, v in os.environ.items() if not k.startswith("B200VIS_") or k == "B200VIS_LIB"}
    e.update(SWITCHES[switch])
    prog = (f"import sys; sys.path.insert(0, {ROOT!r}); sys.path.insert(0, {HERE!r})\n"
            "import test_gpu_light_layers as t\nt.switch_cases()\n")
    res = subprocess.run([sys.executable, "-c", prog], env=e, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, f"{SWITCHES[switch]}\n{res.stdout[-2000:]}\n{res.stderr[-4000:]}"


def test_shifting_every_layer_by_whole_blocks_is_bit_identical_on_the_device():
    base = case_clusters(4, frames=4, shift=0, low=True)
    for j in (1, 2, 3):
        moved = case_clusters(4, frames=4, shift=j, low=True)
        for f, (a, b) in enumerate(zip(base, moved)):
            same_clusters(b, a, f"shift {j} frame {f}")


# ---- 3: no change when unused --------------------------------------------------------------------------------------------
def test_empty_blocks_and_null_change_nothing():
    """Twin contexts on a block-0 scene: one never calls the new entry points, the other gives empty blocks (frames 0-2),
    then NULL (frames 3-5).  Clusters, statistics, ViewVisibility, visible lists and shadow lists are bit-identical."""
    sc, rb, vb, lb = layered_scene(4, seed=2)
    rb[:, 1:] = 0; lb[:, 1:] = 0; vb[:, 1:] = 0
    sc2 = copy.deepcopy(sc)
    a, b = bb.VisibilityPipeline(sc), bb.VisibilityPipeline(sc2)
    caster = np.ones(sc.n, np.uint8); caster[sc.light_row] = 0
    try:
        for p in (a, b):
            p.ctx.upload_shadow_casters(0, caster)
        for f in range(6):
            if f:
                scenes.advance_cameras(sc, 0.05); scenes.advance_cameras(sc2, 0.05)
            items = [dict(kind=0, light_row=int(sc.light_row[o]), range=float(sc.light_range[o]) * 4, layer_mask=int(lb[o, 0]),
                          frusta=orc.point_light_frusta(np.concatenate([IDENT9, sc.trs[sc.light_row[o], 0:3]]).astype(np.float32),
                                                        float(sc.light_range[o]) * 4)) for o in range(0, 64, 5)]
            blocks = np.zeros((len(sc.light_row), 3), U64) if f < 3 else None
            b.ctx.set_light_render_layers_ext(blocks, n_lights=len(sc.light_row))
            device_frame(a, vb, ext=False)
            device_frame(b, vb, ext=False)
            for p in (a, b):
                p.ctx.set_shadow_items(items)
            b.ctx.set_shadow_item_render_layers_ext(np.zeros((len(items), 3), U64) if f < 3 else None, n_items=len(items))
            for p in (a, b):
                p.ctx.run_shadow_culling()
            same_clusters(device_clusters(b), device_clusters(a), f"frame {f}")
            va, ca = a.ctx.download_view_visibility(0, sc.n)
            vb_, cb_ = b.ctx.download_view_visibility(0, sc.n)
            assert (va == vb_).all() and (ca == cb_).all()
            for v in range(4):
                assert (a.ctx.download_visible(v) == b.ctx.download_visible(v)).all()
            for i in range(len(items)):
                for face in range(6):
                    assert (a.ctx.download_shadow_visible(i, face) == b.ctx.download_shadow_visible(i, face)).all()
    finally:
        a.close(); b.close()


# ---- 4: shadows ----------------------------------------------------------------------------------------------------------
def shadow_items(sc, orw, ib, n_point=8, n_spot=6, casc_views=2):
    """Point and spot items over lights, cascades around the first views' cameras; item blocks ib [items, 4]."""
    items, jobs = [], []
    for kind, ords in ((0, range(0, 8 * n_point, 8)), (1, range(3, 3 + 8 * n_spot, 8))):
        for o in ords:
            row = int(sc.light_row[o]); rg = float(sc.light_range[o]) * 3
            fr = orc.point_light_frusta(orw.gt[row], rg, 0.1)
            fr = fr[o % 6] if kind == 1 else fr
            i = len(items)
            items.append(dict(kind=kind, light_row=row, range=rg, range_view_index=0, layer_mask=int(ib[i, 0]), frusta=fr))
            jobs.append((kind, row, rg, fr, i))
    for v in range(casc_views):
        for c, r in enumerate((25.0, 70.0)):
            centre = np.asarray(sc.cameras[v].gt[9:12], np.float32) + np.float32(5.0 * c)
            fr = orc.point_light_frusta(np.concatenate([IDENT9, centre]).astype(np.float32), r, 0.1)[(v + c) % 6]
            i = len(items)
            items.append(dict(kind=2, range_view_index=-1, layer_mask=int(ib[i, 0]), frusta=fr))
            jobs.append((2, 0, 0.0, fr, i))
    return items, jobs


def oracle_shadows(sc, orw, caster, jobs, ib, vv_changed):
    listed = set(np.concatenate(orw.last_lists).tolist())
    want, active = {}, []
    args = (orw.gt, sc.bounds, sc.flags, caster, sc.entity_bits, orw.vv, vv_changed)
    for kind, row, rg, fr, i in jobs:
        if kind == 2:
            want[(i, 0)] = LR.check_dir_light_mesh_visibility(*args, [(fr[None], ib[i], -1)], orw.rb)[0][0]
            active.append(True)
            continue
        active.append(row in listed)
        if row not in listed:
            continue
        sphere = np.concatenate([orw.gt[row, 9:12], [rg]]).astype(np.float32)[None]
        if kind == 1:
            want[(i, 0)] = LR.check_spot_light_mesh_visibility(*args, sphere, fr[None], orw.rb, ib[i:i + 1], lod_origin_index=0)[0]
        else:
            r = LR.check_point_light_mesh_visibility(*args, sphere, fr[None], orw.rb, ib[i:i + 1], lod_origin_index=0)[0]
            for face in range(6):
                want[(i, face)] = r[face]
    return want, active


def run_shadow_frame(pipe, orw, sc, vb, caster, ib, diff_slots=None, set_ext=True):
    """set_ext=False: the items' blocks 1..3 are not given again after set_shadow_items, so the oracle takes them empty."""
    planes = device_frame(pipe, vb)
    vv_changed = orw.cull(planes, defer=True)
    items, jobs = shadow_items(sc, orw, ib)
    pipe.ctx.set_shadow_items(items, diff_slots=diff_slots)
    if set_ext:
        pipe.ctx.set_shadow_item_render_layers_ext(ib[:, 1:])
    pipe.ctx.run_shadow_culling()
    if not set_ext:
        ib = ib.copy(); ib[:, 1:] = 0
    want, active = oracle_shadows(sc, orw, caster, jobs, ib, vv_changed)
    orc.mark_newly_hidden(sc.flags, orw.vv, vv_changed)
    return want, active, vv_changed, len(items)


def check_shadow_lists(pipe, want, active, n_items, tag, o2n=None):
    total = 0
    for i in range(n_items):
        for face in range(6):
            got = pipe.ctx.download_shadow_visible(i, face)
            w = want.get((i, face), np.zeros(0, np.uint32)) if active[i] else np.zeros(0, np.uint32)
            assert len(got) == len(w) and (got == w).all(), f"{tag} item {i} face {face}: {len(got)} vs {len(w)} rows"
            total += len(w)
    return total


def test_shadows_match_the_oracle_with_sinks():
    sc, rb, vb, lb = layered_scene(4, seed=4)
    rng = np.random.default_rng(4)
    caster = (rng.random(sc.n) < 0.85).astype(np.uint8); caster[sc.light_row] = 0
    pipe = setup_device(sc, rb, vb, lb)
    orw = LayeredOracle(sc, rb, vb, lb)
    n_items = 8 + 6 + 4
    ib = blocks_of(LIGHT_KINDS, n_items, rng)
    ib[0] = RenderLayers.from_layers([70]).blocks4(); ib[8] = RenderLayers.from_layers([140]).blocks4()
    ib[14] = RenderLayers.from_layers([201]).blocks4()
    cap = sc.n * 8
    sink = ShadowSink(pipe.ctx, cap, n_items)
    added, removed = pinned((cap,), np.uint64, 0), pinned((cap,), np.uint64, 0)
    a_off, r_off = pinned((n_items * 6 + 1,), np.uint32, 0), pinned((n_items * 6 + 1,), np.uint32, 0)
    pipe.ctx.set_shadow_diff_sink(added, removed, a_off, r_off, max_slots=n_items)
    try:
        pipe.ctx.upload_shadow_casters(0, caster)
        prev = {}
        ext_rows = 0
        for f in range(5):
            if f:
                scenes.advance_cameras(sc, 0.05)
                if f == 3:                                    # change some item blocks between frames
                    ib[1:4] = blocks_of([[130], [0, 201], None], 3)
            want, active, _, n = run_shadow_frame(pipe, orw, sc, vb, caster, ib, diff_slots=np.arange(n_items, dtype=np.uint32))
            assert n == n_items
            tag = f"[frame {f}]"
            tot = check_shadow_lists(pipe, want, active, n_items, tag)
            pipe.ctx.synchronize()
            vv, ch = pipe.ctx.download_view_visibility(0, sc.n)
            assert (vv == orw.vv).all(), f"{tag} ViewVisibility differs on {np.nonzero(vv != orw.vv)[0][:8]}"
            sink.check(want, active, sc.entity_bits, tag)
            for i in range(n_items):                          # the diff sink: list \ prev, prev \ list per (slot, face)
                for face in range(6):
                    l = i * 6 + face
                    new = set(sc.entity_bits[want.get((i, face), [])].tolist()) if active[i] else set()
                    old = prev.get(l, set())
                    wa, wr = (sorted(new - old), sorted(old - new)) if active[i] else ([], [])
                    ga, gr = added[a_off[l]:a_off[l + 1]].tolist(), removed[r_off[l]:r_off[l + 1]].tolist()
                    assert ga == wa and gr == wr, f"{tag} item {i} face {face}: diff differs"
                    prev[l] = new
            # rows listed for an item only through blocks 1..3
            for (i, face), rows_ in want.items():
                if active[i]:
                    ext_rows += int((~LR.intersects(rb[rows_, :1], ib[i, :1]) & LR.intersects(rb[rows_], ib[i])).sum())
            assert tot > 0
        assert ext_rows > 0, "no row was shadow-listed through blocks 1..3"
    finally:
        pipe.close()


# ---- 5: lifetime and errors ----------------------------------------------------------------------------------------------
def test_resets_count_errors_and_compaction():
    sc, rb, vb, lb = layered_scene(4, seed=6)
    rng = np.random.default_rng(6)
    caster = np.ones(sc.n, np.uint8); caster[sc.light_row] = 0
    pipe = setup_device(sc, rb, vb, lb)
    orw = LayeredOracle(sc, rb, vb, lb)
    ib = blocks_of(LIGHT_KINDS, 18, rng)
    try:
        pipe.ctx.upload_shadow_casters(0, caster)
        want, active, _, n = run_shadow_frame(pipe, orw, sc, vb, caster, ib)
        check_shadow_lists(pipe, want, active, n, "[with blocks]")
        same_clusters(device_clusters(pipe), orw.clusters(np.stack([np.ctypeslib.as_array(v.half_spaces).reshape(6, 4)
                                                                      for v in pipe.views])), "[with blocks]")
        # count mismatches: INVALID_ARG, nothing changes
        for call in (lambda: pipe.ctx.set_light_render_layers_ext(np.zeros((len(sc.light_row) - 1, 3), U64)),
                     lambda: pipe.ctx.set_shadow_item_render_layers_ext(np.zeros((n + 1, 3), U64)),
                     lambda: pipe.ctx.set_shadow_item_render_layers_ext(None, n_items=n - 1)):
            with pytest.raises(bb.B200VisError) as e:
                call()
            assert e.value.code == INVALID_ARG
        scenes.advance_cameras(sc, 0.05)
        want, active, _, n = run_shadow_frame(pipe, orw, sc, vb, caster, ib, set_ext=False)   # set_shadow_items emptied them
        check_shadow_lists(pipe, want, active, n, "[after set_shadow_items]")
        vv, _ = pipe.ctx.download_view_visibility(0, sc.n)
        assert (vv == orw.vv).all()
        planes = np.stack([np.ctypeslib.as_array(v.half_spaces).reshape(6, 4) for v in pipe.views])
        same_clusters(device_clusters(pipe), orw.clusters(planes), "[mismatch changed nothing]")
        # set_lights empties the light blocks
        pipe.ctx.set_lights(sc.light_row, sc.light_range, sc.light_layers)
        lb_saved = orw.lb.copy()
        orw.lb = orw.lb.copy(); orw.lb[:, 1:] = 0
        scenes.advance_cameras(sc, 0.05)
        planes = device_frame(pipe, vb)
        orw.cull(planes)
        same_clusters(device_clusters(pipe), orw.clusters(planes), "[after set_lights]")
        orw.lb = lb_saved
        pipe.ctx.set_light_render_layers_ext(lb[:, 1:])
        # an edit (despawn leaves that are in no list) and a compaction keep the blocks
        # (rows in no visible list and in no shadow list of the last run, so that no held result keeps them)
        levels_leaf0 = (1 << 5) - 1                           # first leaf of a 6-level tree
        listed = set(np.concatenate(orw.last_lists).tolist())
        listed |= {int(r) for i in range(n) for face in range(6) for r in pipe.ctx.download_shadow_visible(i, face)}
        leaves = [t * 63 + levels_leaf0 + k for t in range(48) for k in range(0, 32, 7)]
        dead = np.array([r for r in leaves if r not in listed][:20], np.uint32)
        assert len(dead) >= 10
        pipe.ctx.edit_topology(despawn=dead)
        for r in dead:                                        # the oracle's view of a despawned row
            sc.flags[r] = abi.F_NO_CPU_CULLING; sc.class_mask[r] = 0; caster[r] = 0
        scenes.advance_cameras(sc, 0.05)
        run_shadow_frame(pipe, orw, sc, vb, caster, ib)
        o2n = pipe.ctx.compact_topology()
        assert (o2n[dead] == 0xFFFFFFFF).all()
        keep = np.nonzero(o2n != 0xFFFFFFFF)[0]
        new_of = o2n[keep]
        perm = np.empty(len(keep), np.int64); perm[new_of] = keep      # new row -> old row
        old_parent = sc.parent[perm]
        sc.parent = np.where(old_parent >= 0xFFFFFFFE, old_parent, o2n[np.minimum(old_parent, len(o2n) - 1)]).astype(np.uint32)
        for name in ("trs", "bounds", "flags", "class_mask", "entity_bits", "layer_mask"):
            setattr(sc, name, np.ascontiguousarray(getattr(sc, name)[perm]))
        sc.light_row = o2n[sc.light_row].astype(np.uint32)
        sc.roots = None
        caster = np.ascontiguousarray(caster[perm])
        orw.rb = np.ascontiguousarray(orw.rb[perm]); orw.gt = np.ascontiguousarray(orw.gt[perm])
        orw.vv = np.ascontiguousarray(orw.vv[perm]); orw.tchanged = np.ascontiguousarray(orw.tchanged[perm])
        orw.last_lists = [o2n[l].astype(np.uint32) for l in orw.last_lists]
        for f in range(2):
            scenes.advance_cameras(sc, 0.05)
            want, active, _, n = run_shadow_frame(pipe, orw, sc, vb, caster, ib)
            check_shadow_lists(pipe, want, active, n, f"[compacted {f}]")
            same_clusters(device_clusters(pipe), orw.clusters(np.stack([np.ctypeslib.as_array(v.half_spaces).reshape(6, 4)
                                                                          for v in pipe.views])), f"[compacted {f}]")
            vv, _ = pipe.ctx.download_view_visibility(0, len(sc.parent))
            assert (vv == orw.vv).all()
    finally:
        pipe.close()
