"""b200vis_write_global_transforms_scattered on the device, bit for bit against orc.propagate's gt_ext_changed input.

Another system writes GlobalTransforms between frames (physics writing global poses, TransformHelper computing a parent
ahead of propagation).  The written value is what CULL sees, and the next propagate pass treats the rows as
p_global_transform.is_changed() (systems.rs:706-724): a visited marked row re-propagates its children even when set_if_neq
keeps its bits.  Writes here mix values equal to the propagated ones (with a child written off its propagated value, which
only a re-propagation repairs) and values off them, in dirty and clean trees, in one-pass and several-pass plans.
Checked: GlobalTransform bits, both change columns, ViewVisibility, visible lists and classes, the visible diff, clusters."""
import contextlib
import ctypes

import numpy as np
import pytest

import bevy_b200 as bb
from bevy_b200 import scenes
from bevy_b200.scenes import Scene
import oracle as orc
from parity import compare_frame
from test_gpu_bench_scale import run_case
from test_gpu_compaction import renumber
from test_gpu_split_stages import HostColumns, deep_chain, same_bits
from test_gpu_topology_edits import Churn

pytestmark = pytest.mark.gpu

NO_PARENT = 0xFFFFFFFF
INVALID_ARG, NOT_READY, UNSUPPORTED = 1, 7, 8


@contextlib.contextmanager
def oracle_marks(world, propagate=True):
    """orc.propagate as the frame's propagate system sees the world's pending writes (consumed), or -- for a frame
    without PROPAGATE -- not run at all."""
    real = orc.propagate

    def with_marks(parent, trs, gt, tchanged, static_opt=True, gt_ext_changed=None, mt=False):
        ext = world.ext.copy()
        world.ext[:] = 0
        return real(parent, trs, gt, tchanged, static_opt, gt_ext_changed=ext, mt=mt)

    def skipped(parent, trs, gt, tchanged, static_opt=True, gt_ext_changed=None, mt=False):
        return 0, np.zeros(len(parent), np.uint8)
    orc.propagate = with_marks if propagate else skipped
    try:
        yield
    finally:
        orc.propagate = real


def attach(ch):
    ch.world.ext = np.zeros(ch.sc.n, np.uint8)
    return ch


def write(ch, rows, vals, cols=None):
    """The outside system's write: the oracle's column and marks (and the host column it writes into, when the test
    keeps one), then the device call."""
    rows = np.asarray(rows, np.int64)
    vals = np.asarray(vals, np.float32).reshape(-1, 12)
    for r, v in zip(rows, vals):                 # in order: a row listed twice keeps its last value
        ch.world.gt[r] = v
        if cols is not None:
            cols.gt[r] = v
    ch.world.ext[rows] = 1
    ch.pipe.ctx.write_global_transforms_scattered(rows.astype(np.uint32), vals)


def children(sc):
    kids = [[] for _ in range(sc.n)]
    for r, p in enumerate(sc.parent):
        if p < sc.n:
            kids[p].append(r)
    return kids


def random_writes(ch, rng, k, dup=False, cols=None):
    """k rows, half written with their current (propagated) value and half off it; most of the former also get one child
    written off its value."""
    sc, gt = ch.sc, ch.world.gt
    kids = children(sc)
    live = np.nonzero(ch.alive)[0]
    rows, vals = [], []
    for r in rng.choice(live, size=min(k, len(live)), replace=False):
        r = int(r)
        off = rng.random() < 0.5
        rows.append(r); vals.append(gt[r] + (rng.uniform(-0.5, 0.5, 12).astype(np.float32) if off else 0))
        if not off and kids[r] and rng.random() < 0.8:
            c = int(rng.choice(kids[r]))
            rows.append(c); vals.append(gt[c] + rng.uniform(-0.5, 0.5, 12).astype(np.float32))
    if dup and rows:
        rows.append(rows[0]); vals.append(gt[rows[0]] + np.float32(0.25))
    write(ch, rows, vals, cols)


def touch_deep(ch, rng, k):
    """New Transforms for k non-root rows: their ancestors are dirty, but are visited without changing."""
    sc = ch.sc
    cand = np.nonzero(ch.alive & (sc.parent < sc.n))[0]
    rows = np.unique(rng.choice(cand, size=min(k, len(cand)), replace=False))
    sc.trs[rows, 0:3] += rng.uniform(-0.1, 0.1, (len(rows), 3)).astype(np.float32)
    ch.pipe.ctx.upload_transforms_scattered(rows.astype(np.uint32), sc.trs[rows])
    ch.world.tchanged[rows] = 1


def fused(ch, f):
    with oracle_marks(ch.world):
        return ch.frame(f, animate=False)


def split(ch, f, cols=None):
    """PROPAGATE, then CULL, then CLUSTER, each its own run (the plugin's frame)."""
    sc, w, pipe = ch.sc, ch.world, ch.pipe
    pipe.propagate_transforms()
    if cols is not None:
        pipe.ctx.writeback_columns(1)
    ext = w.ext.copy(); w.ext[:] = 0
    rc, want = orc.propagate(sc.parent, sc.trs, w.gt, w.tchanged, w.static_opt, gt_ext_changed=ext)
    assert rc == 0
    w.tchanged[:] = 0
    gt, chg = pipe.ctx.download_global_transforms(0, sc.n)
    bad = ~same_bits(gt, w.gt).all(1)
    assert not bad.any(), f"[{sc.name} split frame {f}] GlobalTransform bits differ on rows {np.nonzero(bad)[0][:8]}"
    assert (chg == want).all(), f"[{sc.name} split frame {f}] Changed<GlobalTransform> differs on {np.nonzero(chg != want)[0][:8]}"
    if cols is not None:
        cols.check_gt(f"split frame {f}")
    pipe.update_views()
    pipe.check_visibility()
    if len(sc.light_row):
        pipe.assign_lights_to_clusters()
    compare_frame(pipe, w, f, check_gt=False, run_device=False)     # the oracle's second propagate has nothing to do


def cull_only(ch, f):
    """run(CULL) while writes are pending: the written values are culled, and the marks survive for the next propagate."""
    sc, w, pipe = ch.sc, ch.world, ch.pipe
    tch = w.tchanged.copy()
    pipe.update_views()
    pipe.check_visibility()
    if len(sc.light_row):
        pipe.assign_lights_to_clusters()
    with oracle_marks(w, propagate=False):
        compare_frame(pipe, w, f, check_gt=False, run_device=False)
    w.tchanged[:] = tch
    gt, _ = pipe.ctx.download_global_transforms(0, sc.n)
    assert same_bits(gt, w.gt).all(), f"[{sc.name} frame {f}] CULL changed the written GlobalTransforms"


def fan_scene():
    """R -> P -> 700 children (three tiles besides P's) and a 40-deep branch under P: touching the branch dirties P,
    which is visited but keeps its bits; its other children are only re-propagated when P hands them a mark."""
    parent = [NO_PARENT, 0] + [1] * 700
    b = len(parent)
    parent += [1] + list(range(b, b + 39))
    parent += [NO_PARENT] + [len(parent)] * 300            # a second tree
    n = len(parent)
    rng = np.random.default_rng(9)
    trs = np.zeros((n, 10), np.float32)
    trs[:, 0:3] = rng.uniform(-0.5, 0.5, (n, 3)); trs[:, 3:7] = scenes.random_unit_quats(rng, n); trs[:, 7:10] = 1.0
    trs[2:702, 0:3] = rng.uniform(-30, 30, (700, 3))
    bounds = np.zeros((n, 6), np.float32); bounds[:, 3:6] = 0.5
    return Scene("fan", np.array(parent, np.uint32), trs, bounds,
                 np.full(n, scenes.F_INHERITED_VISIBLE | scenes.F_HAS_AABB, np.uint8), np.ones(n, np.uint8),
                 np.arange(n, dtype=np.uint64), cameras=[scenes._camera(0.3)], roots=np.array([0, 742], np.uint32))


def run_marked(ch, frames, seed, k=40, kinds=("fused",)):
    rng = np.random.default_rng(seed)
    fused(ch, 0)
    for f in range(1, frames):
        kind = kinds[f % len(kinds)]
        if f % 3 == 1:
            scenes.advance_cameras(ch.sc, 0.05)
            before = ch.sc.trs.copy()
            rows, trs = scenes.mutate_roots(ch.sc, f)
            rows, trs = rows[:2], trs[:2]                   # two trees move; the rest stay put
            ch.sc.trs[:] = before
            ch.sc.trs[rows] = trs
            ch.pipe.ctx.upload_transforms_scattered(rows, trs)
            ch.world.tchanged[rows] = 1
        touch_deep(ch, rng, 6)
        random_writes(ch, rng, k, dup=f % 2 == 0)
        if kind == "cull_first":
            cull_only(ch, f)
            random_writes(ch, rng, k // 4)                  # more writes after the CULL, before the propagate
            split(ch, f)
        elif kind == "split":
            split(ch, f)
        else:
            ch.pipe.update_views()
            fused(ch, f)


@pytest.mark.parametrize("static_opt", [True, False])
def test_random_forest_marks_fused_and_split(static_opt):
    ch = attach(Churn(scenes.forest(n_trees=120, levels=7, n_lights=16), 0, static_opt=static_opt, seed=1))
    try:
        run_marked(ch, 10, seed=2, kinds=("fused", "split", "cull_first"))
    finally:
        ch.close()


@pytest.mark.parametrize("static_opt", [True, False])
def test_several_pass_plans(static_opt):
    """Config #1 (trees across tiles, k_mark_dirty_global), the 700-deep chain and a fan-out over four tiles: marks
    handed over inside tiles and across tiles and passes."""
    for make, k in ((scenes.propagate_bench_scene, 200), (deep_chain, 60), (fan_scene, 60)):
        ch = attach(Churn(make(), 0, static_opt=static_opt, seed=3))
        try:
            assert ch.pipe.ctx.topology_summary()[3] > 1 or make is fan_scene
            run_marked(ch, 7, seed=4, k=k, kinds=("split", "fused", "cull_first"))
        finally:
            ch.close()


def test_fan_out_children_across_tiles_follow_a_marked_parent():
    """P (row 1) is written with the bits propagation gives it; its 700 children, written off theirs, must all be
    re-propagated -- in P's tile and in the three tiles after it."""
    ch = attach(Churn(fan_scene(), 0, seed=5))
    try:
        fused(ch, 0)
        kids = np.arange(2, 702)
        rng = np.random.default_rng(6)
        for f in range(1, 4):
            ch.sc.trs[730, 0:3] += np.float32(0.01)         # deep in P's branch: R and P are visited, P keeps its bits
            ch.pipe.ctx.upload_transforms_scattered(np.array([730], np.uint32), ch.sc.trs[730:731])
            ch.world.tchanged[730] = 1
            vals = np.concatenate([ch.world.gt[1:2], ch.world.gt[kids] + rng.uniform(-1, 1, (700, 12)).astype(np.float32)])
            write(ch, np.concatenate([[1], kids]), vals)
            ch.pipe.update_views()
            stats = fused(ch, f)
            _, chg = ch.pipe.ctx.download_global_transforms(0, ch.sc.n)
            assert chg[1] == 0 and chg[kids].all() and stats.gt_changed_count == int(chg.sum())
    finally:
        ch.close()


def test_a_propagate_consumes_the_marks():
    """P's mark is handed down once: the next frame, children written off their values with P unwritten keep them."""
    ch = attach(Churn(fan_scene(), 0, seed=15))
    kids = np.arange(2, 702, 7)
    rng = np.random.default_rng(16)
    try:
        fused(ch, 0)
        for f in range(1, 5):
            ch.sc.trs[730, 0:3] += np.float32(0.01)         # R and P visited every frame, P keeps its bits
            ch.pipe.ctx.upload_transforms_scattered(np.array([730], np.uint32), ch.sc.trs[730:731])
            ch.world.tchanged[730] = 1
            if f % 2:
                write(ch, [1], ch.world.gt[1:2])
            else:
                vals = ch.world.gt[kids] + rng.uniform(-1, 1, (len(kids), 12)).astype(np.float32)
                write(ch, kids, vals)
            ch.pipe.update_views()
            fused(ch, f)
            if not f % 2:
                gt, chg = ch.pipe.ctx.download_global_transforms(0, ch.sc.n)
                assert same_bits(gt[kids], vals).all() and not chg[kids].any()
    finally:
        ch.close()


def test_pipelined_back_to_back_frames():
    ch = attach(Churn(scenes.forest(n_trees=100, levels=7, n_lights=24), 0, seed=7))
    rng = np.random.default_rng(8)
    try:
        ch.pipe.enable_visible_diff()
        fused(ch, 0)
        for f in range(1, 7):
            touch_deep(ch, rng, 8)
            random_writes(ch, rng, 30)
            scenes.advance_cameras(ch.sc, 0.05)
            ch.pipe.update_views()
            if f % 3:                                     # enqueued behind the previous frame's tail, not compared
                planes = np.stack([np.ctypeslib.as_array(v.half_spaces).reshape(6, 4).copy() for v in ch.pipe.views])
                with oracle_marks(ch.world):
                    _, _, lists, _ = ch.world.frame(planes)
                ch.world.last_lists = [l if l is not None else ch.world.last_lists[v] for v, l in enumerate(lists)]
                ch.pipe.run_frame()
                ch.pipe.read_feedback()
            else:
                fused(ch, f)
    finally:
        ch.close()


def test_step_with_sinks():
    """b200vis_step (PROPAGATE|CULL, then CLUSTER) with the column sinks written back behind the tile pass."""
    torch = pytest.importorskip("torch")
    ch = attach(Churn(scenes.forest(n_trees=80, levels=7, n_lights=24), 0, seed=9))
    sc, pipe = ch.sc, ch.pipe
    rng = np.random.default_rng(10)
    V = len(sc.cameras)
    st_t = torch.zeros(ctypes.sizeof(bb.FrameStats), dtype=torch.uint8).pin_memory()
    try:
        cols = HostColumns(pipe)
        pipe.ctx.set_result_sink(st_t.data_ptr(), None, None, None)
        fused(ch, 0)
        pipe.ctx.writeback_columns(3)
        for f in range(1, 6):
            scenes.advance_cameras(sc, 0.05)
            touch_deep(ch, rng, 5)
            random_writes(ch, rng, 30, dup=True, cols=cols)
            arr = (bb.CameraDesc * V)()
            for v, cam in enumerate(sc.cameras):
                arr[v].global_transform[:] = cam.gt.tolist()
                arr[v].fov_y, arr[v].aspect, arr[v].near_z, arr[v].far_z = cam.fov, cam.aspect, cam.near, cam.far
                arr[v].layer_mask, arr[v].flags, arr[v].range_view_index = 1, bb.VIEW_ACTIVE, -1
            pipe.ctx.step(0, 0, 0, arr, V, pipe.cluster_config, wait=True, writeback=True)
            pipe.update_views(clusters=False)             # the same frustums, for the oracle side
            with oracle_marks(ch.world):
                compare_frame(pipe, ch.world, f, cluster=False, run_device=False)
            cols.check_gt(f"step {f}"); cols.check_vv(f"step {f}")
        pipe.ctx.set_result_sink(None, None, None, None)
        pipe.ctx.set_column_sinks()
    finally:
        ch.close()


def test_marks_across_edit_and_compaction():
    """A despawned marked row loses its mark; the marks of the others follow old_to_new through a compaction."""
    ch = attach(Churn(scenes.forest(n_trees=80, levels=7, n_lights=24), 2000, seed=11))
    rng = np.random.default_rng(12)
    try:
        ch.pipe.enable_visible_diff()
        fused(ch, 0)
        for f in range(1, 7):
            touch_deep(ch, rng, 6)
            random_writes(ch, rng, 30)
            kids = ch.children()
            marked_leaves = np.nonzero((ch.world.ext == 1) & (kids == 0) & ch.alive & (ch.sc.parent < ch.sc.n))[0]
            marked_leaves = marked_leaves[~np.isin(marked_leaves, ch.sc.light_row)]
            n0 = ch.sc.n
            ch.edit(marked_leaves[:3].tolist(), [], [], [NO_PARENT, 5], np.tile(
                np.array([0, 0, 0, 0, 0, 0, 1, 1, 1, 1], np.float32), (2, 1)))
            ch.world.ext = np.concatenate([ch.world.ext, np.zeros(ch.sc.n - n0, np.uint8)])
            ch.world.ext[marked_leaves[:3]] = 0
            if f % 2 == 0:
                o2n = ch.pipe.ctx.compact_topology().astype(np.int64)
                keep = np.nonzero(o2n != 0xFFFFFFFF)[0]
                ext = np.zeros(len(keep), np.uint8); ext[o2n[keep]] = ch.world.ext[keep]
                renumber(ch, o2n)
                ch.world.ext = ext
                random_writes(ch, rng, 10)                  # and writes after the compaction, in the new numbers
            ch.pipe.update_views()
            fused(ch, f)
    finally:
        ch.close()


def test_errors_leave_marks_pending():
    lib = bb.load_library()
    sc = scenes.forest(n_trees=30, levels=5, n_lights=4)
    c = bb.Context(sc.n, max_lights=4, max_views=1)
    try:
        rows = np.array([3], np.uint32); g = np.ones((1, 12), np.float32)
        with pytest.raises(bb.B200VisError) as e:
            c.write_global_transforms_scattered(rows, g)
        assert e.value.code == NOT_READY
    finally:
        c.close()
    ch = attach(Churn(sc, 10, seed=13))
    c = ch.pipe.ctx
    try:
        fused(ch, 0)
        h = c._h
        gt = np.ones((2, 12), np.float32)
        r = np.array([1, 2], np.uint32)
        assert lib.b200vis_write_global_transforms_scattered(h, 2, None, gt.ctypes.data) == INVALID_ARG
        assert lib.b200vis_write_global_transforms_scattered(h, 2, r.ctypes.data, None) == INVALID_ARG
        assert lib.b200vis_write_global_transforms_scattered(h, 0, None, None) == 0
        for bad in ([1, sc.n], [sc.n + 5]):
            with pytest.raises(bb.B200VisError) as e:
                c.write_global_transforms_scattered(bad, np.ones((len(bad), 12), np.float32))
            assert e.value.code == INVALID_ARG
        leaf = int(np.nonzero((ch.children() == 0) & (sc.parent < sc.n))[0][-1])
        ch.edit([leaf], [], [], [], np.zeros((0, 10), np.float32))
        ch.world.ext = np.zeros(sc.n, np.uint8)
        with pytest.raises(bb.B200VisError) as e:
            c.write_global_transforms_scattered([leaf], np.ones((1, 12), np.float32))
        assert e.value.code == INVALID_ARG
        # nothing above wrote anything: the device still matches the oracle (a failing run is the switch test below)
        fused(ch, 1)
        rng = np.random.default_rng(14)
        touch_deep(ch, rng, 4)
        random_writes(ch, rng, 12)
        ch.pipe.update_views()
        fused(ch, 2)
    finally:
        ch.close()


def test_experiment_tile_kernel_is_unsupported_with_marks():
    """B200VIS_TILE_KERNEL=lean (own interpreter: the switch is read once per process): a run that includes PROPAGATE
    while marks are pending fails with UNSUPPORTED, names the switch and consumes nothing; CULL alone still runs."""
    run_case("import numpy as np, bevy_b200 as bb\n"
             "sc = scenes.forest(n_trees=20, levels=5, n_lights=4)\n"
             "p = bb.VisibilityPipeline(sc)\n"
             "p.run_frame()\n"
             "g, _ = p.ctx.download_global_transforms(0, sc.n)\n"
             "w = g[7:8] + np.float32(1)\n"
             "p.ctx.write_global_transforms_scattered([7], w)\n"
             "for stages in (bb.STAGE_PROPAGATE, bb.STAGE_ALL):\n"
             "    try:\n"
             "        p.ctx.run(stages); raise SystemExit('run with pending marks succeeded')\n"
             "    except bb.B200VisError as e:\n"
             "        assert e.code == 8 and 'B200VIS_TILE_KERNEL=lean' in str(e), str(e)\n"
             "p.ctx.run(bb.STAGE_CULL)\n"
             "g2, _ = p.ctx.download_global_transforms(0, sc.n)\n"
             "assert (g2[7] == w[0]).all()\n"
             "try:\n"
             "    p.ctx.run(bb.STAGE_PROPAGATE); raise SystemExit('marks were consumed')\n"
             "except bb.B200VisError as e:\n"
             "    assert e.code == 8\n"
             "p.ctx.set_topology(sc.parent, sc.entity_bits)\n"
             "p.ctx.run(bb.STAGE_PROPAGATE)\n"
             "p.close()\n", {"B200VIS_TILE_KERNEL": "lean"})
