"""b200vis_compact_topology on the device.

Two contexts run the same scene and the same churn; one of them compacts every few frames.  Each is compared bit for bit
with its own CPU oracle world (tests/parity.py), and after every frame -- and right after every compaction, before any
run -- every output of the compacting context must equal its twin's, renumbered through the accumulated old_to_new:
GlobalTransform bits, both change columns, ViewVisibility, visible lists and classes, the visible diff, shadow lists,
clusters and the frame statistics."""
import copy

import numpy as np
import pytest

import bevy_b200 as bb
from bevy_b200 import scenes
from parity import compare_frame
from test_gpu_topology_edits import Churn, DETACHED, INVALID_ARG, NO_PARENT, run_unchecked

pytestmark = pytest.mark.gpu

NONE = 0xFFFFFFFF
HIERARCHY_CYCLE = 4


def renumber(ch, o2n, reparent=(), new_parent=()):
    """The scene and oracle arrays of a Churn after its context compacted: rows moved through old_to_new."""
    sc, w = ch.sc, ch.world
    n = sc.n
    keep = np.nonzero(o2n != NONE)[0]
    n2 = len(keep)
    dst = o2n[keep].astype(np.int64)

    def move(a):
        out = np.zeros((n2,) + a.shape[1:], a.dtype)
        out[dst] = a[keep]
        return out
    p = sc.parent.astype(np.int64).copy()
    for r, q in zip(reparent, new_parent):
        p[r] = q
        w.tchanged[r] = 1
    real = p < n
    p[real] = o2n[p[real]]
    sc.parent = move(p.astype(np.uint32))
    for name in ("trs", "bounds", "flags", "class_mask", "entity_bits", "layer_mask", "range_mask", "shadow_caster",
                 "range_se", "range_use_aabb"):
        if getattr(sc, name, None) is not None:
            setattr(sc, name, move(getattr(sc, name)))
    sc.light_row = o2n[sc.light_row].astype(np.uint32)
    if sc.roots is not None:
        sc.roots = o2n[sc.roots].astype(np.uint32)
    w.gt, w.vv, w.tchanged = move(w.gt), move(w.vv), move(w.tchanged)
    w.last_lists = [o2n[l].astype(np.uint32) for l in w.last_lists]
    ch.alive = move(ch.alive)


class Twins:
    """A compacting Churn `a` and its twin `b`; m[r] = the row of b's row r in a (NONE once dropped)."""

    def __init__(self, make_scene, headroom, **kw):
        self.b = Churn(make_scene(), headroom, **kw)
        self.a = Churn(make_scene(), headroom, **kw)
        self.m = np.arange(self.b.sc.n, dtype=np.int64)
        self.compactions = 0

    def close(self):
        self.a.close(); self.b.close()

    def map_rows(self, rows):
        return [int(self.m[r]) for r in rows]

    def map_parents(self, ps):
        return [int(p) if p >= DETACHED else int(self.m[p]) for p in ps]

    def random_edit(self, **kw):
        """b's random edit, applied to both (a in its own row numbers, with the same entity bits and column values)."""
        a, b = self.a, self.b
        orig = b.edit

        def both(despawn, reparent, new_parent, spawn_parent, trs, bits=None):
            bits = b.new_bits(len(spawn_parent)) if bits is None else bits
            state = copy.deepcopy(b.rng.bit_generator.state)
            n_a = a.sc.n
            out = orig(despawn, reparent, new_parent, spawn_parent, trs, bits)
            a.rng.bit_generator.state = state
            a.edit(self.map_rows(despawn), self.map_rows(reparent), self.map_parents(new_parent), self.map_parents(spawn_parent), trs, bits)
            self.m = np.concatenate([self.m, np.arange(n_a, n_a + len(spawn_parent))])
            return out
        b.edit = both
        try:
            return b.random_edit(**kw)
        finally:
            b.edit = orig

    def compact(self, reparent=(), new_parent=()):
        """a compacts with these reparents (rows in b's numbers, order-keeping there), b applies them as an edit."""
        a, b = self.a, self.b
        if len(reparent):
            b.pipe.ctx.edit_topology(reparent=reparent, new_parent=new_parent)
            for r, p in zip(reparent, new_parent):
                b.sc.parent[r] = p; b.world.tchanged[r] = 1
        ra, pa = self.map_rows(reparent), self.map_parents(new_parent)
        before = a.pipe.ctx.topology_summary()
        o2n = a.pipe.ctx.compact_topology(ra, pa).astype(np.int64)
        assert len(o2n) == before[0]
        renumber(a, o2n, ra, pa)
        self.m = np.where(self.m != NONE, o2n[np.minimum(self.m, len(o2n) - 1)], NONE)
        self.compactions += 1
        return o2n

    def frame(self, f, animate=True):
        self.b.frame(f, animate)
        self.a.frame(f, animate)
        self.check()

    def check(self):
        """Every output of a equals b's, renumbered."""
        ca, cb = self.a.pipe.ctx, self.b.pipe.ctx
        nb = self.b.sc.n
        live = np.nonzero(self.b.alive)[0]
        assert (self.m[live] != NONE).all()
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
        for v in range(len(self.b.sc.cameras)):
            assert sa.visible_count[v] == sb.visible_count[v]
            assert sa.cluster_index_count[v] == sb.cluster_index_count[v]
            assert np.float32(sa.cluster_farthest_z[v]).view(np.uint32) == np.float32(sb.cluster_farthest_z[v]).view(np.uint32)
            la, lb = ca.download_visible(v), cb.download_visible(v)
            assert (la == self.m[lb]).all(), f"view {v}: visible list"
            ka, kb = ca.download_visible_by_class(v), cb.download_visible_by_class(v)
            assert sorted(ka) == sorted(kb) and all((ka[k] == self.m[kb[k]]).all() for k in kb), f"view {v}: class lists"
            if getattr(self.b.pipe, "visible_diff", False):
                (aa, ra), (ab, rb) = ca.download_visible_diff(v), cb.download_visible_diff(v)
                assert (aa == self.m[ab]).all() and (ra == self.m[rb]).all(), f"view {v}: visible diff"
            oa, ia = ca.download_clusters(v)
            ob, ib = cb.download_clusters(v)
            assert (oa == ob).all() and (ia == ib).all()
        if getattr(self.b.sc, "shadow_lights", None) is not None:
            for i in range(len(self.b.sc.shadow_lights)):
                for face in range(6):
                    assert (ca.download_shadow_visible(i, face) == self.m[cb.download_shadow_visible(i, face)]).all()


def order_keeping_reparents(t, k, rng):
    """k live leaves of b moved under an earlier live row with children (or to NO_PARENT)."""
    b = t.b
    kids = b.children()
    lights = set(b.sc.light_row.tolist())
    leaves = [int(r) for r in np.nonzero(b.alive & (kids == 0) & (b.sc.parent < b.sc.n))[0] if int(r) not in lights]
    reparent, new_parent = [], []
    for r in rng.choice(leaves, size=min(k, len(leaves)), replace=False).tolist():
        lo = max(0, r - 300)
        below = lo + np.nonzero(b.alive[lo:r] & (kids[lo:r] > 0))[0]
        reparent.append(int(r)); new_parent.append(int(rng.choice(below)) if len(below) and rng.random() < 0.7 else NO_PARENT)
    return reparent, new_parent


def run_twins(make_scene, headroom, frames, every, static_opt=True, seed=0, edit_kw=None, reparents=2):
    t = Twins(make_scene, headroom, static_opt=static_opt, seed=seed)
    rng = np.random.default_rng(seed + 100)
    try:
        t.frame(0, animate=False)
        for f in range(1, frames):
            t.random_edit(**(edit_kw or {}))
            if f % every == 0:
                t.compact(*order_keeping_reparents(t, reparents, rng))
                t.check()                     # downloads right after the compaction, before any run
            t.frame(f)
        n, live, _, _ = t.a.pipe.ctx.topology_summary()
        assert t.compactions and n - live < t.b.pipe.ctx.topology_summary()[0] - t.b.pipe.ctx.topology_summary()[1]
    finally:
        t.close()


@pytest.mark.parametrize("static_opt", [True, False])
def test_twins_on_a_churned_forest(static_opt):
    run_twins(lambda: scenes.forest(60, 8, 24, seed=1), 4000, frames=12, every=3, static_opt=static_opt, seed=1)


@pytest.mark.parametrize("seed,static_opt", [(21, True), (22, False)])
def test_twins_on_the_feature_rich_scene(seed, static_opt):
    """RenderLayers blocks 0-3, VisibleEntityRanges, NoCpuCulling, detached subtrees, shuffled entity bits (every spawn
    merges ranks, so the keys are resident on the device) and point-light shadows."""
    import test_gpu_edge_cases as ec

    def make():
        sc = ec._random_scene(seed, n_roots=90, n_lights=20)
        rng = np.random.default_rng(seed)
        sc.shadow_lights = np.sort(rng.choice(len(sc.light_row), 6, replace=False)).astype(np.uint32)
        sc.shadow_caster = (rng.random(sc.n) < 0.8).astype(np.uint8)
        sc.shadow_caster[sc.light_row] = 0
        sc.shadow_near_z, sc.shadow_lod_origin = 0.1, 0
        return sc
    run_twins(make, 3000, frames=10, every=2, static_opt=static_opt, seed=seed, edit_kw=dict(n_despawn=6, n_flat=6, n_kids=3))


def test_reparents_that_break_row_order_match_the_oracle():
    """Subtrees moved under later rows, one of them under a row of a full 256-row tile; frames before and after match the
    oracle, and the diff after the compaction reports only real changes."""
    from bevy_b200 import abi
    ch = Churn(scenes.forest(40, 8, 12, seed=5), 1000, seed=5)
    try:
        ch.frame(0, animate=False)
        c, sc = ch.pipe.ctx, ch.sc
        # 600 flat rows appended: the greedy tiler packs them into full tiles
        parent0, n0, k = sc.parent.copy(), sc.n, 600
        trs = np.zeros((k, 10), np.float32); trs[:, 3:7] = (0, 0, 0, 1); trs[:, 7:10] = 1.0
        trs[:, 0:3] = ch.rng.uniform(-40, 40, (k, 3))
        ch.edit([], [], [], [NO_PARENT] * k, trs)
        plan = abi.host_edit_plan(parent0, [([], [], [], [NO_PARENT] * k)])
        assert plan.rc == 0 and c.topology_summary()[2] == len(plan.desc)      # the context runs this plan
        full = [(int(b), int(nr)) for b, nr in plan.desc[:, :2] if nr == 256 and b >= n0]
        assert full, "no full tile among the appended rows"
        target = full[0][0] + 17
        ch.frame(1, animate=False)
        kids = ch.children()
        tree_roots = [int(r) for r in sc.roots]
        # the second level of tree 0 under the last tree's root; a whole subtree of tree 1 under a flat row of the full
        # tile; a leaf under the last row that has children
        mid = [int(r) for r in np.nonzero(sc.parent == tree_roots[0])[0]][:1]
        sub = [int(r) for r in np.nonzero(sc.parent == tree_roots[1])[0]][:1]
        leaf = int(next(r for r in np.nonzero((sc.parent < sc.n) & (kids == 0))[0] if r > 600 and r not in sc.light_row))
        last = int(np.nonzero(kids > 0)[0][-1])
        assert target > sub[0] and last > leaf
        reparent, new_parent = mid + sub + [leaf], [tree_roots[-1], target, last]
        o2n = c.compact_topology(reparent, new_parent).astype(np.int64)
        renumber(ch, o2n, reparent, new_parent)
        assert ch.sc.parent[o2n[sub[0]]] == o2n[target]
        ch.frame(2, animate=False)          # compare_frame checks the diff against the oracle's: only real changes
        for v in range(len(sc.cameras)):
            added, removed = c.download_visible_diff(v)
            assert len(added) + len(removed) < max(1, len(c.download_visible(v)))
        ch.random_edit()
        ch.frame(3)
    finally:
        ch.close()


def test_a_row_despawned_while_visible_is_reported_removed_after_a_compaction():
    ch = Churn(scenes.forest(30, 6, 8, seed=7), 200, seed=7)
    try:
        for f in range(2):
            ch.frame(f, animate=False)
        c = ch.pipe.ctx
        vis = c.download_visible(0)
        kids = ch.children()
        victim = int(next(r for r in vis if kids[r] == 0 and r not in ch.sc.light_row))
        bits = int(ch.sc.entity_bits[victim])
        ch.edit([victim], [], [], [], np.zeros((0, 10), np.float32))
        o2n = c.compact_topology().astype(np.int64)
        assert o2n[victim] != NONE                                 # held: last frame's visible sets name it
        n, live, _, _ = c.topology_summary()
        assert n == live + 1
        renumber(ch, o2n)
        ch.frame(2, animate=False)
        _, removed = c.download_visible_diff(0)
        assert int(o2n[victim]) in removed.tolist()
        o2n2 = c.compact_topology().astype(np.int64)           # the removed list still names it
        renumber(ch, o2n2)
        ch.frame(3, animate=False)
        o2n3 = c.compact_topology().astype(np.int64)            # now nothing does
        assert (o2n3 == NONE).sum() == 1 and ch.sc.entity_bits[np.nonzero(o2n3 == NONE)[0][0]] == bits
        renumber(ch, o2n3)
        n, live, _, _ = c.topology_summary()
        assert n == live
        ch.random_edit()
        ch.frame(4)
    finally:
        ch.close()


def test_an_inactive_view_keeps_a_despawned_row_until_it_lets_go():
    ch = Churn(scenes.forest(30, 6, 8, seed=8), 200, seed=8)
    try:
        ch.frame(0, animate=False)
        c, sc = ch.pipe.ctx, ch.sc
        kept = c.download_visible(1)
        kids = ch.children()
        victim = int(next(r for r in kept if kids[r] == 0 and r not in sc.light_row))
        sc.view_flags = [bb.VIEW_ACTIVE if v != 1 else 0 for v in range(len(sc.cameras))]     # view 1 keeps its list
        ch.edit([victim], [], [], [], np.zeros((0, 10), np.float32))
        for f in range(1, 3):
            o2n = c.compact_topology().astype(np.int64)
            assert o2n[victim] != NONE, "the inactive view's kept list names the row"
            victim = int(o2n[victim])
            renumber(ch, o2n)
            assert victim in c.download_visible(1).tolist()
            ch.frame(f, animate=False)
    finally:
        ch.close()


def test_shrink_then_grow_back_past_chunk_boundaries():
    """A world of more than two 32768-row chunks, mostly despawned, compacted, then grown back: every mask word and chunk
    counter past the shrunken end must have been zero."""
    sc = scenes.forest(300, 8, 16, seed=11)            # 76 800 rows
    ch = Churn(sc, 40000, seed=11)
    try:
        ch.frame(0, animate=False)
        ch.frame(1)
        kids = ch.children()
        lights = set(sc.light_row.tolist())
        trees = np.split(np.arange(sc.n), np.nonzero(sc.parent == NO_PARENT)[0][1:])
        doomed = [t for t in trees[1:] if not (set(t.tolist()) & lights)][:220]
        despawn = np.concatenate(doomed).tolist()
        ch.edit(despawn, [], [], [], np.zeros((0, 10), np.float32))
        ch.frame(2)
        o2n = ch.pipe.ctx.compact_topology().astype(np.int64)
        renumber(ch, o2n)
        assert ch.sc.n < 32768
        ch.frame(3)
        for f in range(4, 7):              # spawn back past the old chunk boundaries, visible rows among them
            k = 16000
            trs = np.zeros((k, 10), np.float32); trs[:, 3:7] = (0, 0, 0, 1); trs[:, 7:10] = 1.0
            trs[:, 0:3] = ch.rng.uniform(-40, 40, (k, 3))
            ch.edit([], [], [], [NO_PARENT] * k, trs)
            ch.frame(f)
        assert ch.sc.n > 2 * 32768
    finally:
        ch.close()


def test_compaction_restores_the_pass_count_of_a_fresh_plan():
    sc = scenes.forest(200, 8, 16, seed=12)
    ch = Churn(sc, 2000, seed=12)
    try:
        ch.frame(0, animate=False)
        assert ch.pipe.ctx.topology_summary()[3] == 1
        for f in range(1, 4):
            ch.random_edit(n_kids=6)
            ch.frame(f)
        assert ch.pipe.ctx.topology_summary()[3] >= 2
        o2n = ch.pipe.ctx.compact_topology().astype(np.int64)
        renumber(ch, o2n)
        summary = ch.pipe.ctx.topology_summary()
        fresh = bb.Context(ch.sc.n + 10)
        try:
            fresh.set_topology(ch.sc.parent, ch.sc.entity_bits)
            assert summary[2:] == fresh.topology_summary()[2:]
        finally:
            fresh.close()
        assert summary[3] == 1
        ch.frame(4)
    finally:
        ch.close()


def test_errors_change_nothing():
    t = Twins(lambda: scenes.forest(20, 6, 8, seed=4), 100, seed=4)
    try:
        t.frame(0, animate=False)
        t.random_edit()
        t.frame(1)
        a = t.a
        c, sc = a.pipe.ctx, a.sc
        n = sc.n
        kids = a.children()
        dead = int(np.nonzero(~a.alive)[0][0])
        parent_row = int(np.nonzero((kids > 0) & a.alive)[0][0])
        child = int(np.nonzero(sc.parent == parent_row)[0][0])
        cases = [
            (dict(reparent=[parent_row], new_parent=[child]), HIERARCHY_CYCLE),
            (dict(reparent=[child], new_parent=[child]), HIERARCHY_CYCLE),
            (dict(reparent=[dead], new_parent=[NO_PARENT]), INVALID_ARG),
            (dict(reparent=[n], new_parent=[NO_PARENT]), INVALID_ARG),
            (dict(reparent=[child], new_parent=[dead]), INVALID_ARG),
            (dict(reparent=[child], new_parent=[n + 5]), INVALID_ARG),
            (dict(reparent=[child, child], new_parent=[NO_PARENT, DETACHED]), INVALID_ARG),
        ]
        before = c.topology_summary()
        for kw, code in cases:
            with pytest.raises(bb.B200VisError) as e:
                c.compact_topology(**kw)
            assert e.value.code == code, kw
            assert c.topology_summary() == before
        t.check()
        t.frame(2)
        t.compact()
        t.frame(3)
    finally:
        t.close()


def test_back_to_back_pipelined_frames_around_a_compaction():
    """run(STAGE_ALL) frames submitted without reading back, an edit and a compaction between them; the last frame is
    compared with the oracle (a pipelined context joins the frame in flight before it renumbers anything)."""
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
                if f % 3 == 0:
                    renumber(ch, ch.pipe.ctx.compact_topology().astype(np.int64))
                scenes.advance_cameras(sc, 0.01)
                rows, trs = scenes.mutate_roots(ch.sc, f)
                ch.pipe.ctx.upload_transforms_scattered(rows, trs)
                ch.world.tchanged[rows] = 1
            ch.pipe.update_views()
            if f < frames - 1:
                run_unchecked(ch)
            else:
                compare_frame(ch.pipe, ch.world, f)
    finally:
        ch.close()


def test_step_with_result_and_column_sinks_across_compactions():
    """b200vis_step with a result sink and column sinks; edits every step and compactions between some steps.  The host
    mirror is renumbered by the caller through old_to_new and otherwise fed only by the sinks: it stays equal to a full
    download, and the sink's stats and visible rows equal the download calls."""
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
        for f in range(9):
            if f:
                ch.random_edit(n_despawn=3, n_flat=6, n_kids=2)
            if f in (3, 4, 7):
                o2n = c.compact_topology().astype(np.int64)
                keep = np.nonzero(o2n != NONE)[0]
                for arr in (gt_h, vv_h):          # the caller's host columns, renumbered
                    moved = arr[keep].copy()
                    arr[o2n[keep]] = moved
                renumber(ch, o2n)
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


@pytest.mark.parametrize("trees,levels,lights,headroom", [(1, 2, 1, 10), (1, 3, 3, 10), (3, 3, 2, 12), (2, 3, 2, 24)])
def test_twins_in_contexts_of_a_few_dozen_rows(trees, levels, lights, headroom):
    """Contexts of 14 to 40 rows with RenderLayers blocks 1-3 resident: below about 30 rows the compaction's maps and its
    widest column do not fit the 64 B/row staging buffer, above it they do.  Tombstones, held rows, spawns and a
    compaction every frame; the compacting context still equals its twin and the oracle."""
    t = Twins(lambda: scenes.forest(trees, levels, lights, seed=3), headroom, seed=3)
    try:
        rng = np.random.default_rng(5)
        ext = rng.integers(0, 1 << 62, (t.b.sc.n, 3), dtype=np.uint64)     # the views hold no layer of blocks 1-3
        for ch in (t.a, t.b):
            ch.pipe.ctx.upload_render_layers_ext(0, ext)
        t.frame(0, animate=False)
        for f in range(1, 6):
            t.random_edit(n_despawn=2, n_flat=1, n_kids=1, n_reparent=1)
            t.compact()
            t.check()
            t.frame(f)
        assert t.a.pipe.ctx.topology_summary()[0] < t.b.pipe.ctx.topology_summary()[0]
    finally:
        t.close()


def test_the_shadow_stage_reads_the_renumbered_visible_sets_while_the_diff_is_off():
    """The shadow stage reads last frame's visible sets even after the visible diff was switched off (they then stay as
    the last diffed frame left them): a compaction in that state renumbers them like the rest."""
    import test_gpu_edge_cases as ec

    def make():
        sc = ec._random_scene(31, n_roots=90, n_lights=20)
        rng = np.random.default_rng(31)
        sc.shadow_lights = np.sort(rng.choice(len(sc.light_row), 6, replace=False)).astype(np.uint32)
        sc.shadow_caster = (rng.random(sc.n) < 0.8).astype(np.uint8)
        sc.shadow_caster[sc.light_row] = 0
        sc.shadow_near_z, sc.shadow_lod_origin = 0.1, 0
        return sc
    t = Twins(make, 1000, seed=31)
    try:
        t.frame(0, animate=False)
        t.random_edit(n_despawn=6, n_flat=6, n_kids=3)
        t.frame(1)
        for ch in (t.a, t.b):
            ch.pipe.ctx.enable_visible_diff(False)
        t.compact()
        for ch in (t.b, t.a):
            ch.pipe.update_views()
            ch.pipe.run_frame()
            ch.pipe.ctx.run_shadow_culling()                 # the shadow items of frame 1, rows renumbered in `a`
        ca, cb = t.a.pipe.ctx, t.b.pipe.ctx
        listed = 0
        for i in range(len(t.b.sc.shadow_lights)):
            for face in range(6):
                lb = cb.download_shadow_visible(i, face)
                listed += len(lb)
                assert (ca.download_shadow_visible(i, face) == t.m[lb]).all(), (i, face)
        assert listed > 0
        for v in range(len(t.b.sc.cameras)):
            assert (ca.download_visible(v) == t.m[cb.download_visible(v)]).all()
    finally:
        t.close()
