"""SURVEY.md 8(f) rows beside the path, on the device, at the inputs where a kernel can go wrong.

N4a  check_visibility_ranges inside every cull loop, on rows whose distance to a range view is exactly a threshold or one
     step either side of it (scenes from test_cpu_next_rows_edges, which proves each one detects the mutants).
N4b  visibility_propagate_system over the plan shapes that walk the T_EXT_PARENT branch, over edited and compacted worlds.
N2   ViewClusterBindings at MAX_INDICES, past the 9-bit count field, with indices past 8 bits and a map that is too short."""
import numpy as np
import pytest

import bevy_b200 as bb
from bevy_b200 import abi, scenes
import oracle as orc

from parity import OracleWorld, compare_frame
from test_cpu_next_rows_edges import RANGE_CASES, check_range_sensitivity, range_scene, range_views
from test_gpu_bench_scale import run_case
from test_gpu_compaction import NONE, Twins, order_keeping_reparents
from test_gpu_split_stages import deep_chain, same_bits
from test_gpu_topology_edits import NO_PARENT, Churn

pytestmark = pytest.mark.gpu

INH, HID, VIS, NOC = orc.VIS_INHERITED, orc.VIS_HIDDEN, orc.VIS_VISIBLE, orc.VIS_NO_COMPONENTS


# ---- N4a: VisibilityRange thresholds -------------------------------------------------------------------------------------------
def range_frames(seed, offset, path="fused"):
    """Three frames: the range views rotate between frames, the third is a Changed<Transform> frame that leaves every value
    as it was.  path: "fused" (run_frame), "split" (PROPAGATE, then CULL alone: k_cull<false>), or "ext" (frame 1 has
    pending write_global_transforms_scattered marks: the marked kernel 1b)."""
    sc, extra = range_scene(seed, offset)
    pipe = bb.VisibilityPipeline(sc)
    world = OracleWorld(sc)
    c = pipe.ctx
    try:
        c.upload_shadow_casters(0, sc.shadow_caster)
        c.upload_visibility_ranges(0, sc.range_se, sc.range_use_aabb)
        for f in range(3):
            sc.range_view_pos = range_views(sc, extra, f)
            c.set_visibility_range_views(sc.range_view_pos)
            if f == 2:
                rows = np.arange(0, sc.n, 3, dtype=np.uint32)
                c.upload_transforms_scattered(rows, sc.trs[rows])
                world.tchanged[rows] = 1
            ext = path == "ext" and f == 1
            if ext:                                    # another system writes the GlobalTransforms the rows already have
                rows = np.nonzero(sc.parent == NO_PARENT)[0].astype(np.uint32)
                c.write_global_transforms_scattered(rows, world.gt[rows])
            pipe.update_views()
            if path == "split":
                pipe.propagate_transforms()
                pipe.check_visibility()
                pipe.assign_lights_to_clusters()
            else:
                pipe.run_frame()
            pipe.check_point_light_mesh_visibility(sc.shadow_lights, sc.shadow_near_z, sc.shadow_lod_origin)
            compare_frame(pipe, world, f, check_gt=not ext, run_device=False)
            if ext:                                    # the values are unchanged; Changed<GlobalTransform> is the marks' business
                gt, _ = c.download_global_transforms(0, sc.n)
                assert same_bits(gt, world.gt).all()
            if f == 0:
                check_range_sensitivity(sc, world.gt)
            listed = np.concatenate([c.download_visible(v) for v in range(len(sc.cameras))])
            ranged = ((sc.flags & bb.F_HAS_VIS_RANGE) != 0) & ((sc.flags & bb.F_NO_CPU_CULLING) == 0)
            assert np.isin(np.nonzero(ranged)[0], listed).any()        # boundary rows reach the visible lists
            assert sum(len(c.download_shadow_visible(i, k)) for i in range(len(sc.shadow_lights)) for k in range(6)) > 0
    finally:
        pipe.close()


@pytest.mark.parametrize("seed,offset", RANGE_CASES)
@pytest.mark.parametrize("path", ["fused", "split", "ext"])
def test_visibility_range_thresholds(seed, offset, path):
    range_frames(seed, offset, path)


RANGE_VARIANTS = {"lean": {"B200VIS_TILE_KERNEL": "lean"},
                  "lean_sphere_reject": {"B200VIS_TILE_KERNEL": "lean", "B200VIS_LEAN_PROBE": "8"},
                  "warp": {"B200VIS_TILE_KERNEL": "warp", "B200VIS_WARP_VARIANT": "2p"}, "classic": {"B200VIS_TILE_KERNEL": "classic"},
                  "scout": {"B200VIS_TILE_KERNEL": "scout"}, "flow": {"B200VIS_TILE_KERNEL": "flow"}}


@pytest.mark.parametrize("variant", list(RANGE_VARIANTS))
def test_visibility_range_thresholds_in_every_tile_kernel(variant):
    """The general (non-SIMPLE) instantiation of each tile kernel: the range columns are resident."""
    run_case("from test_gpu_next_rows_edges import range_frames, RANGE_CASES\n"
             "for seed, offset in RANGE_CASES:\n"
             "    range_frames(seed, offset)", RANGE_VARIANTS[variant])


# ---- N4b: InheritedVisibility -------------------------------------------------------------------------------------------------
def fixpoint(parent, vis):
    """The state the change-driven system converges to, for rows with the components (parents precede children)."""
    n = len(parent)
    assert ((parent >= n) | (parent < np.arange(n))).all()
    out = np.zeros(n, np.uint8)
    for i in range(n):
        if vis[i] & NOC:
            continue
        k, p = vis[i] & 3, int(parent[i])
        out[i] = 1 if k == VIS else 0 if k == HID else (out[p] if p < n and not (vis[p] & NOC) else 1)
    return out


def propagate_and_check(ctx, parent, vis, inh, changed, removed=(), dead=None, tag=""):
    """One visibility_propagate_system run on both sides.  Tombstones (`dead`) are outside every query: the device reports
    them as not inherited-visible and never written, and they are left out of the comparison.  Returns the new column."""
    n = len(parent)
    want, want_ch = orc.visibility_propagate(parent, vis, inh, np.asarray(changed, np.uint32), np.asarray(removed, np.uint32))
    ctx.propagate_visibility()
    got, got_ch = ctx.download_inherited_visibility(0, n)
    live = np.ones(n, bool) if dead is None else ~dead
    bad = np.nonzero(live & ((got != want) | (got_ch != want_ch)))[0]
    assert not len(bad), f"{tag}: InheritedVisibility or its change byte differs on rows {bad[:8]}: {got[bad[:8]]} vs {want[bad[:8]]}"
    if dead is not None:
        assert not got[dead].any() and not got_ch[dead].any(), f"{tag}: a tombstone reports InheritedVisibility"
    fx = fixpoint(parent, vis)
    comp = live & ((vis & NOC) == 0)
    assert (want[comp] == fx[comp]).all(), f"{tag}: the change set given to the oracle misses rows"
    return want


def random_visibility(rng, n, noc=0.03):
    vis = rng.choice([INH] * 3 + [HID, VIS], n).astype(np.uint8)
    vis[rng.random(n) < noc] |= NOC
    return vis


def with_inherited(flags, inh, rows):
    out = flags.copy()
    out[rows] = (out[rows] & ~np.uint8(1)) | inh[rows]
    return out


@pytest.mark.parametrize("shape", ["config1", "chain_fanout"])
def test_inherited_visibility_over_multi_pass_plans(shape):
    """Config #1 (three passes) and the 700-deep chain beside a 3000-child fan-out: every Hidden / Visible / Inherited /
    no-components parent on every position of a tile, so each kind reaches the T_EXT_PARENT branch of a later pass."""
    sc = scenes.propagate_bench_scene() if shape == "config1" else deep_chain()
    n = sc.n
    rng = np.random.default_rng(3)
    pattern = np.array([INH, HID, INH, INH, VIS, NOC, INH, HID | NOC, INH, VIS | NOC, INH], np.uint8)   # length 11: every phase
    vis = pattern[np.arange(n) % len(pattern)]
    vis[sc.parent == NO_PARENT] = INH
    # a row without the components is in no query and keeps its flag at 0: a child must not read it (:655-659)
    sc.flags[(vis & NOC) != 0] &= np.uint8(0xFE)
    pipe = bb.VisibilityPipeline(sc)
    world = OracleWorld(sc)
    try:
        passes = pipe.ctx.topology_summary()[3]
        assert passes >= (3 if shape == "config1" else 5)
        inh = (sc.flags & 1).astype(np.uint8)
        changed = np.arange(n)
        for step in range(4):
            if step:
                changed = np.unique(rng.integers(0, n, 40))
                if shape == "chain_fanout":           # and the chain's top, which reaches every later tile
                    changed = np.unique(np.concatenate([changed, [0, 1]]))
                vis[changed] = (vis[changed] & NOC) | rng.choice([INH, HID, VIS], len(changed)).astype(np.uint8)
            pipe.ctx.upload_visibility(0, vis)
            inh = propagate_and_check(pipe.ctx, sc.parent, vis, inh, changed, tag=f"{shape} step {step}")
            assert inh.any() and (inh == 0).any()
            sc.flags = with_inherited(sc.flags, inh, np.arange(n))
            pipe.update_views()
            compare_frame(pipe, world, step, cluster=False)
    finally:
        pipe.close()


def test_inherited_visibility_through_topology_edits():
    """Despawns, order-keeping reparents and reparents to no parent, flat spawns and spawned children of existing trees
    (appended tiles with external parents), with Visibility uploaded over sub-ranges."""
    ch = Churn(scenes.forest(50, 6, 8, seed=4), 3000, seed=4)
    rng = np.random.default_rng(4)
    sc, c = ch.sc, ch.pipe.ctx
    try:
        n = sc.n
        vis = random_visibility(rng, n)
        c.upload_visibility(0, vis[:n // 3]); c.upload_visibility(n // 3, vis[n // 3:])
        inh = propagate_and_check(c, sc.parent, vis, (sc.flags & 1).astype(np.uint8), np.arange(n), tag="initial")
        sc.flags = with_inherited(sc.flags, inh, np.arange(n))
        ch.frame(0, animate=False)
        hidden_spawns = 0
        for f in range(1, 7):
            n0 = sc.n
            parent_before = sc.parent.copy()
            new_rows = ch.random_edit(n_despawn=5, n_flat=3, n_kids=4, n_reparent=4)
            # more spawned children, under rows that are alive after the edit and were not inherited-visible before it
            hidden_pool = np.nonzero(ch.alive[:n0] & (inh == 0) & ~np.isin(np.arange(n0), sc.light_row))[0]
            if len(hidden_pool):
                extra = [int(p) for p in rng.choice(hidden_pool, 3)]
                tr = np.zeros((3, 10), np.float32); tr[:, 3:7] = (0, 0, 0, 1); tr[:, 7:10] = 1.0
                new_rows += ch.edit([], [], [], extra, tr)
            n = sc.n
            dead = ~ch.alive
            vis = np.concatenate([vis, np.zeros(n - n0, np.uint8)])        # the edit leaves Visibility::Inherited
            vis[dead] = NOC
            inh = np.concatenate([inh, (sc.flags[n0:] & 1).astype(np.uint8)])
            inh[dead] = 0
            moved = np.nonzero((parent_before != sc.parent[:n0]) & ch.alive[:n0])[0]
            removed = moved[sc.parent[moved] == NO_PARENT]
            edited = np.unique(rng.integers(0, n0, 12))
            edited = edited[ch.alive[edited]]
            vis[edited] = (vis[edited] & NOC) | rng.choice([INH, HID, VIS], len(edited)).astype(np.uint8)
            for r in edited:                                              # partial uploads, one row at a time
                c.upload_visibility(int(r), vis[r:r + 1])
            changed = np.unique(np.concatenate([edited, moved[sc.parent[moved] != NO_PARENT], np.arange(n0, n)]))
            inh = propagate_and_check(c, sc.parent, vis, inh, changed, removed, dead, tag=f"edit frame {f}")
            hidden_spawns += int((inh[n0:] == 0).sum())
            sc.flags = with_inherited(sc.flags, inh, np.nonzero(ch.alive)[0])
            ch.frame(f)
        assert hidden_spawns > 0 and c.topology_summary()[3] >= 2
    finally:
        ch.close()


def test_inherited_visibility_across_compaction_and_regrowth():
    """A compacting context `a` beside its uncompacted twin `b`.  After the first upload, each Visibility column only
    receives the rows an edit changes, so the propagation after compact_topology reads the column the compaction
    permuted.  InheritedVisibility and its change bytes are compared through old_to_new right after the compaction (before
    any run) and after every propagation.  Then more rows are spawned than the compaction dropped: they start as
    Visibility::Inherited."""
    t = Twins(lambda: scenes.forest(40, 6, 8, seed=6), 3000, seed=6)
    rng = np.random.default_rng(6)
    ca, cb = t.a.pipe.ctx, t.b.pipe.ctx
    try:
        vb = random_visibility(rng, t.b.sc.n)
        inh_b = (t.b.sc.flags & 1).astype(np.uint8)
        ca.upload_visibility(0, vb); cb.upload_visibility(0, vb)          # the twins start with the same row numbers

        def same_through_m(tag):
            """a's InheritedVisibility and change bytes equal b's on every live row of b, renumbered."""
            ga, cha = ca.download_inherited_visibility(0, t.a.sc.n)
            gb, chb = cb.download_inherited_visibility(0, t.b.sc.n)
            live = np.nonzero(t.b.alive)[0]
            bad = live[(ga[t.m[live]] != gb[live]) | (cha[t.m[live]] != chb[live])]
            assert not len(bad), f"{tag}: the compacting context differs from its twin on b's rows {bad[:8]}"

        def propagate_both(changed_b, removed_b, tag):
            nonlocal inh_b
            inh_b = propagate_and_check(cb, t.b.sc.parent, vb, inh_b, changed_b, removed_b, ~t.b.alive, tag + " (twin)")
            ca.propagate_visibility()
            same_through_m(tag)
            for ch_ in (t.a, t.b):
                g, _ = ch_.pipe.ctx.download_inherited_visibility(0, ch_.sc.n)
                ch_.sc.flags = with_inherited(ch_.sc.flags, g, np.nonzero(ch_.alive)[0])

        propagate_both(np.arange(t.b.sc.n), [], "initial")
        t.frame(0, animate=False)
        compacted = False
        for f in range(1, 5):
            nb0 = t.b.sc.n
            parent_before = t.b.sc.parent.copy()
            t.random_edit(n_despawn=30 if f == 1 else 4, n_flat=2, n_kids=2, n_reparent=2)
            # the edit writes the column on both sides: NO_COMPONENTS for tombstones, Inherited for spawned rows
            vb = np.concatenate([vb, np.zeros(t.b.sc.n - nb0, np.uint8)]); vb[~t.b.alive] = NOC
            inh_b = np.concatenate([inh_b, (t.b.sc.flags[nb0:] & 1).astype(np.uint8)]); inh_b[~t.b.alive] = 0
            moved = np.nonzero((parent_before != t.b.sc.parent[:nb0]) & t.b.alive[:nb0])[0]
            changed = [moved[t.b.sc.parent[moved] != NO_PARENT], np.arange(nb0, t.b.sc.n)]
            removed = moved[t.b.sc.parent[moved] == NO_PARENT]
            if f != 3:                                # Changed<Visibility> on a few live rows, uploaded row by row on both
                edited = np.nonzero(t.b.alive)[0]
                edited = np.unique(rng.choice(edited, 8))
                vb[edited] = (vb[edited] & NOC) | rng.choice([INH, HID, VIS], len(edited)).astype(np.uint8)
                for r in edited:
                    cb.upload_visibility(int(r), vb[r:r + 1]); ca.upload_visibility(int(t.m[r]), vb[r:r + 1])
                changed.append(edited)
            propagate_both(np.unique(np.concatenate(changed)), removed, f"frame {f}")
            if f == 2:
                rp, npar = order_keeping_reparents(t, 3, rng)
                before = t.a.sc.n
                t.compact(rp, npar)
                assert t.a.sc.n < before
                moved_rows = np.nonzero(t.m[np.nonzero(t.b.alive)[0]] != np.nonzero(t.b.alive)[0])[0]
                assert len(moved_rows) > 100                                  # most rows changed places
                same_through_m(f"frame {f} right after compaction")          # the permuted change bytes and flags
                compacted = True
                # nothing uploaded: `a` reads the permuted Visibility column; the twin sees the reparents as
                # Changed<ChildOf> / RemovedComponents<ChildOf>
                propagate_both([r for r, p in zip(rp, npar) if p != NO_PARENT], [r for r, p in zip(rp, npar) if p == NO_PARENT],
                               f"frame {f} after compaction")
            t.frame(f)
        assert compacted
        # regrow past b's row count: `a`'s new rows land on slots past its compacted count
        na0, nb0 = t.a.sc.n, t.b.sc.n
        grow = nb0 - na0 + 40
        tr = np.zeros((grow, 10), np.float32); tr[:, 3:7] = (0, 0, 0, 1); tr[:, 7:10] = 1.0
        tr[:, 0:3] = rng.uniform(-30, 30, (grow, 3))
        bits = t.b.new_bits(grow)
        t.b.edit([], [], [], [NO_PARENT] * grow, tr, bits)
        t.a.edit([], [], [], [NO_PARENT] * grow, tr, bits)
        t.m = np.concatenate([t.m, np.arange(na0, na0 + grow)])
        assert t.a.sc.n > nb0
        vb = np.concatenate([vb, np.zeros(grow, np.uint8)])
        inh_b = np.concatenate([inh_b, (t.b.sc.flags[nb0:] & 1).astype(np.uint8)])
        ca.propagate_visibility()                                 # nothing uploaded for the new rows: Inherited, no parent
        ga, cha = ca.download_inherited_visibility(0, t.a.sc.n)
        assert ga[na0:].all() and not cha[na0:].any()
        propagate_both(np.arange(nb0, t.b.sc.n), [], "after regrowth")
    finally:
        t.close()


# ---- N2: ViewClusterBindings at the packing limits --------------------------------------------------------------------------------
def _bindings_scene(n_base, light_range, n_tiny, tiny_pos):
    """The forest of test_n2 with `n_base` lights of one range, plus `n_tiny` lights of range 0.01 at one point, each of
    which lands in exactly one cluster."""
    sc = scenes.forest(n_trees=30, levels=5, n_lights=n_base)
    sc.light_range[:] = light_range
    sc.bounds[sc.light_row, 3] = light_range
    if n_tiny:
        n0 = sc.n
        sc.parent = np.concatenate([sc.parent, np.full(n_tiny, NO_PARENT, np.uint32)])
        trs = np.zeros((n_tiny, 10), np.float32); trs[:, 0:3] = tiny_pos; trs[:, 3:7] = (0, 0, 0, 1); trs[:, 7:10] = 1.0
        sc.trs = np.concatenate([sc.trs, trs])
        b = np.zeros((n_tiny, 6), np.float32); b[:, 3] = 0.01
        sc.bounds = np.concatenate([sc.bounds, b])
        sc.flags = np.concatenate([sc.flags, np.full(n_tiny, scenes.F_INHERITED_VISIBLE | scenes.F_HAS_SPHERE | scenes.F_SPHERE_FROM_GT, np.uint8)])
        sc.class_mask = np.concatenate([sc.class_mask, np.full(n_tiny, scenes.CLASS_LIGHT, np.uint8)])
        sc.entity_bits = np.concatenate([sc.entity_bits, np.arange(n_tiny, dtype=np.uint64) + np.uint64(n0 + 1000)])
        sc.light_row = np.concatenate([sc.light_row, np.arange(n0, n0 + n_tiny, dtype=np.uint32)])
        sc.light_range = np.concatenate([sc.light_range, np.full(n_tiny, 0.01, np.float32)])
    return sc


def _oracle_csr(sc):
    """View 0's cluster CSR on frame 0, from the oracle (dynamic resizing off)."""
    world = OracleWorld(sc, cluster_kwargs=dict(dynamic_resizing=False))
    planes = np.stack([bb.host_compute_frustum(bb.host_perspective(c.fov, c.aspect, c.near), c.gt, c.far) for c in sc.cameras])
    _, _, _, clusters = world.frame(planes)
    out, offsets, _ = clusters[0]
    return np.asarray(offsets, np.int64)


TINY_POS = np.array([0.13, -0.07, -2.37], np.float32)     # in front of camera 0, well inside one cluster
N_TINY = (600, 900)                                          # tiny lights added: always more than 511 in one cluster


def tiny_lights_needed(off, limit):
    """How many tiny lights take view 0's CSR (offsets `off`, without them) to `limit`, or None.  They all land in one
    cluster near the camera, before every cluster that matters here, so each adds one to the total and to every later
    offset.  "total_N": N indices in all.  "offset_16384": a cluster that holds lights ends exactly at index 16384, two
    empty clusters follow it, and a later cluster holds lights again."""
    if limit.startswith("total_"):
        k = int(limit[6:]) - int(off[-1])
        return k if N_TINY[0] <= k <= N_TINY[1] else None
    for c in range(1, len(off) - 2):
        k = 16384 - int(off[c])
        if off[c] > off[c - 1] and off[c + 2] == off[c] and off[-1] > off[c] and N_TINY[0] <= k <= N_TINY[1]:
            return k
    return None


def tuned_bindings_scene(limit):
    """Scan the range of 200 base lights upwards until `tiny_lights_needed` finds a count, then add those tiny lights.
    Returns the scene and view 0's oracle CSR, checked to have moved exactly one cluster's count."""
    for r in np.arange(20.0, 35.0, 0.01):               # the view-0 total grows by tens of indices per step here
        off0 = _oracle_csr(_bindings_scene(200, r, 0, TINY_POS))
        k = tiny_lights_needed(off0, limit)
        if k is not None:
            break
    else:
        raise AssertionError(f"no base light range reaches {limit}")
    sc = _bindings_scene(200, r, k, TINY_POS)
    off = _oracle_csr(sc)
    grew = np.diff(off) - np.diff(off0)
    assert grew.max() == k and (grew != 0).sum() == 1, "the tiny lights span several clusters"
    return sc, off


def step_cameras(sc):
    arr = (bb.CameraDesc * len(sc.cameras))()
    for v, cam in enumerate(sc.cameras):
        arr[v].global_transform[:] = cam.gt.tolist()
        arr[v].fov_y, arr[v].aspect, arr[v].near_z, arr[v].far_z = cam.fov, cam.aspect, cam.near, cam.far
        arr[v].layer_mask, arr[v].flags, arr[v].range_view_index = 1, bb.VIEW_ACTIVE, -1
    return arr


@pytest.mark.parametrize("driver", ["run_frame", "step"])
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("limit", ["total_16383", "total_16384", "total_16385", "offset_16384"])
def test_cluster_bindings_at_the_packing_limits(limit, mode, driver):
    """Frames through pipelined run_frame (with ClusterConfig::None on the last view) or b200vis_step (every view
    clustered, the library's own feedback); every view's bindings against the oracle's packing of the device's CSR."""
    sc, off = tuned_bindings_scene(limit)
    counts = np.diff(off)
    if limit.startswith("total_"):
        assert off[-1] == int(limit[6:])
    else:
        c = int(np.nonzero(off[:-1] == 16384)[0][0])
        assert counts[c - 1] > 0 and counts[c] == 0 and counts[c + 1] == 0 and off[-1] > 16384
    assert counts.max() > 511 and len(sc.light_row) > 256
    cfg = abi.host_default_cluster_config(*sc.screen)
    cfg.dynamic_resizing = 0
    cfg.view_cluster_bindings_max_indices = 1 << 22
    L = len(sc.light_row)
    pipe = bb.VisibilityPipeline(sc, cluster_config=cfg, max_cluster_indices=1 << 20)
    rng = np.random.default_rng(9)
    # storage: GPU indices up to 2L, the last 40 ordinals unmapped; uniform: the first 300 ordinals mapped (8-bit slots OR-ed)
    gmap = rng.permutation(2 * L)[:L - 40].astype(np.uint32) if mode == 1 else rng.permutation(300).astype(np.uint32)
    none_view = 3 if driver == "run_frame" else None
    try:
        pipe.ctx.set_cluster_bindings(mode, gmap)
        for f in range(3):
            if driver == "step":
                pipe.ctx.step(0, 0, 0, step_cameras(sc), len(sc.cameras), cfg, wait=True)
            else:
                pipe.update_views()
                cv = pipe.cluster_views[none_view]
                cv.enabled = 0
                pipe.ctx.set_cluster_view(none_view, cv)
                pipe.run_frame()
                pipe.read_feedback()
            for v in range(len(sc.cameras)):
                offsets, idx = pipe.ctx.download_clusters(v)
                nc = 0 if v == none_view else pipe.ctx.cluster_dims(v)
                if v == 0 and f == 0:
                    assert (offsets[:nc + 1] == off).all(), "the device's CSR is not the one tuned on the oracle"
                w = orc.cluster_bindings(offsets[:nc + 1], idx[:offsets[nc]] if nc else idx[:0], gmap, storage=(mode == 1))
                g = pipe.ctx.download_cluster_bindings(v)
                assert g[2:] == w[2:], f"frame {f} view {v}: n_offsets / n_indices {g[2:]} vs {w[2:]}"
                assert np.array_equal(g[0], w[0]), f"frame {f} view {v}: offsets_and_counts differ"
                assert np.array_equal(g[1], w[1]), f"frame {f} view {v}: index lists differ"
                if v == none_view:
                    assert g[2:] == (0, 0)
            if f == 0 and mode == 1:
                assert (pipe.ctx.download_cluster_bindings(0)[1] == 0xFFFFFFFF).any()
    finally:
        pipe.close()


# ---- small related checks ------------------------------------------------------------------------------------------------------
def test_visible_diff_sink_below_the_list_length_keeps_the_first_rows_and_the_full_count():
    import torch
    sc = scenes.forest(n_trees=40, levels=6, n_lights=4)
    pipe = bb.VisibilityPipeline(sc)
    V, cap = pipe.ctx.max_views, 7
    rows = torch.zeros((2, V, cap), dtype=torch.int32).pin_memory()
    counts = torch.zeros((V, 2), dtype=torch.int32).pin_memory()
    try:
        pipe.enable_visible_diff()
        pipe.ctx.set_visible_diff_sink(rows.numpy().view(np.uint32), counts.numpy().view(np.uint32))
        seen = False
        for f in range(3):
            if f:
                scenes.advance_cameras(sc, 0.4)
            pipe.update_views()
            pipe.run_frame()
            pipe.ctx.synchronize()
            for v in range(len(sc.cameras)):
                a, r = pipe.ctx.download_visible_diff(v)
                assert counts[v, 0].item() == len(a) and counts[v, 1].item() == len(r)
                assert np.array_equal(rows[0, v, :min(cap, len(a))].numpy().view(np.uint32), a[:cap])
                assert np.array_equal(rows[1, v, :min(cap, len(r))].numpy().view(np.uint32), r[:cap])
                seen |= len(a) > cap
        assert seen
    finally:
        pipe.ctx.set_visible_diff_sink(None, None)
        pipe.close()


def test_shadow_item_list_capacity_truncates_and_keeps_the_count():
    sc = scenes.forest(n_trees=80, levels=5, n_lights=6)
    sc.trs[sc.roots, 0:3] *= np.float32(0.12)
    sc.light_range[:] = 45.0
    sc.bounds[sc.light_row, 3] = 45.0
    caster = np.ones(sc.n, np.uint8); caster[sc.light_row] = 0
    pipe = bb.VisibilityPipeline(sc)
    try:
        pipe.ctx.upload_shadow_casters(0, caster)
        pipe.update_views()
        pipe.ctx.run(bb.STAGE_ALL)
        gt, _ = pipe.ctx.download_global_transforms(0, sc.n)
        items = [dict(kind=0, light_row=int(r), range=45.0, range_view_index=-1, layer_mask=1,
                      frusta=abi.host_point_light_frusta(gt[r], 45.0, 0.1)) for r in sc.light_row]
        cap = 5                                      # the first call sizes the lists (a later, larger capacity grows them)
        pipe.ctx.set_shadow_items(items, list_capacity=cap)
        pipe.ctx.run_shadow_culling()
        counts, kept = [], []
        for i in range(len(items)):
            for k in range(6):
                cnt = abi.C.c_uint32(0)
                assert pipe.ctx._lib.b200vis_download_shadow_visible(pipe.ctx._h, i, k, None, 0, abi.C.byref(cnt)) == 0
                counts.append(cnt.value)
                if cnt.value > cap:           # a truncated list cannot be downloaded: the call refuses it, whatever the buffer
                    buf = np.zeros(cnt.value, np.uint32)
                    with pytest.raises(bb.B200VisError) as e:
                        pipe.ctx._check(pipe.ctx._lib.b200vis_download_shadow_visible(pipe.ctx._h, i, k, abi._ptr(buf), len(buf),
                                                                                       abi.C.byref(cnt)))
                    assert e.value.code == 6                             # B200VIS_ERR_CAPACITY
                    kept.append(None)
                else:
                    kept.append(pipe.ctx.download_shadow_visible(i, k))
        pipe.ctx.set_shadow_items(items)
        pipe.ctx.run_shadow_culling()
        full = [pipe.ctx.download_shadow_visible(i, k) for i in range(len(items)) for k in range(6)]
        assert counts == [len(l) for l in full]                  # the truncated lists still counted every row
        assert all(np.array_equal(a, b) for a, b in zip(kept, full) if a is not None)   # lists that fit are whole
        assert sum(len(l) > cap for l in full) > 0
    finally:
        pipe.close()
