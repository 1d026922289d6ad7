"""Full-world sweeps alternate their direction: every kernel 1b launch over a pass and every k_cull launch walks the
rows opposite to the context's previous sweep.  The order must not change a result, so every case runs at least four
consecutive frames (both directions, both changes of direction) and checks each frame bit for bit against the oracle:
GlobalTransform bits, both change columns, ViewVisibility, the sorted visible lists and their diff, the cluster lists and
their feedback (which read the tile pass's light snapshot), and the frame's change counts.  A twin run of the bench forest
with B200VIS_SWEEP_ORDER=fixed (every sweep ascending) must give byte-identical outputs."""
import os
import subprocess
import sys

import numpy as np
import pytest

import bevy_b200 as bb
from bevy_b200 import scenes
import oracle as orc
from parity import OracleWorld, compare_frame
from test_gpu_compaction import renumber
from test_gpu_cull_outputs import shuffled_bits
from test_gpu_external_gt import attach, run_marked
from test_gpu_topology_edits import Churn

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))


def check_counts(pipe):
    """The frame's change counts (atomic sums over the CTAs) equal the change columns compare_frame matched."""
    n = pipe.scene.n
    _, gch = pipe.ctx.download_global_transforms(0, n)
    _, vch = pipe.ctx.download_view_visibility(0, n)
    st = pipe.ctx.download_frame_stats()
    assert st.vv_changed_count == int(vch.sum())
    assert st.gt_changed_count == int(gch.sum())


def run_frames(sc, frames=5, cluster=True, before_frame=None, **kw):
    pipe = bb.VisibilityPipeline(sc, **kw)
    world = OracleWorld(sc, True)
    pipe.enable_visible_diff()
    try:
        for f in range(frames):
            if f:
                scenes.advance_cameras(sc, 0.05)
                rows, trs = scenes.mutate_roots(sc, f)
                pipe.ctx.upload_transforms_scattered(rows, trs)
                world.tchanged[rows] = 1
            if before_frame is not None:
                before_frame(pipe, world, f)
            pipe.update_views(clusters=cluster)
            compare_frame(pipe, world, f, cluster=cluster)
            check_counts(pipe)
    finally:
        pipe.close()


def test_bench_forest_scaled_down():
    run_frames(scenes.forest(n_trees=300, levels=8, n_lights=16), frames=6)


def test_multi_pass_plan():
    """Config #1's 1077-node trees: passes keep their order, the tiles inside each pass are walked both ways."""
    sc = scenes.propagate_bench_scene()

    def passes(pipe, world, f):
        if f == 0:
            assert pipe.ctx.topology_summary()[3] > 1
    run_frames(sc, frames=5, cluster=False, before_frame=passes)


def test_non_identity_rank_map():
    """Entity keys out of row order: the tile pass and k_cull set the visible masks by atomicOr."""
    sc = scenes.forest(n_trees=200, levels=7, n_lights=16)
    shuffled_bits(sc, np.random.default_rng(3))
    run_frames(sc, frames=5)


def test_pending_external_global_transforms():
    """The marked instantiation of kernel 1b (every frame has writes pending)."""
    ch = attach(Churn(scenes.forest(n_trees=120, levels=7, n_lights=16), 0, seed=5))
    try:
        run_marked(ch, 6, seed=6)
    finally:
        ch.close()


def test_twelve_cameras_group_pass():
    """Views 8..11 in a k_cull group pass behind the tile pass: a tile pass and a group pass per frame, so each frame's
    tile pass runs the same direction and its group pass the other."""
    sc = scenes.many_cameras_lights(12, forest_kwargs=dict(n_trees=120, levels=5))
    sc.trs[sc.roots, 0:3] *= np.float32(0.03)
    pipe = bb.VisibilityPipeline(sc)
    world = OracleWorld(sc, True)
    try:
        for f in range(5):
            if f:
                scenes.rotate_cameras(sc, 0.35)
                rows, trs = scenes.mutate_roots(sc, f)
                pipe.ctx.upload_transforms_scattered(rows, trs)
                world.tchanged[rows] = 1
            pipe.update_views()
            compare_frame(pipe, world, f)
            check_counts(pipe)
    finally:
        pipe.close()


def test_propagate_only_run_between_full_frames():
    """A PROPAGATE-only run flips the direction like any other sweep; a CULL-only run (k_cull) does too."""
    sc = scenes.forest(n_trees=200, levels=7, n_lights=16)
    pipe = bb.VisibilityPipeline(sc)
    world = OracleWorld(sc, True)
    try:
        for f in range(7):
            if f:
                scenes.advance_cameras(sc, 0.05)
            if f and f != 3:            # frame 3 does not propagate: no Transform moves
                rows, trs = scenes.mutate_roots(sc, f)
                pipe.ctx.upload_transforms_scattered(rows, trs)
                world.tchanged[rows] = 1
            if f in (2, 5):
                pipe.propagate_transforms()
                rc, want = orc.propagate(sc.parent, sc.trs, world.gt, world.tchanged, world.static_opt)
                assert rc == 0
                world.tchanged[:] = 0
                gt, chg = pipe.ctx.download_global_transforms(0, sc.n)
                assert (gt.view(np.uint32) == world.gt.view(np.uint32)).all(), f"frame {f}: PROPAGATE-only GlobalTransforms"
                assert (chg == want).all(), f"frame {f}: PROPAGATE-only Changed<GlobalTransform>"
            if f == 3:      # CULL alone (k_cull), then CLUSTER
                pipe.update_views()
                pipe.check_visibility()
                pipe.assign_lights_to_clusters()
                compare_frame(pipe, world, f, check_gt=False, run_device=False)
                continue
            pipe.update_views()
            compare_frame(pipe, world, f)
            if f not in (2, 5):     # the PROPAGATE-only run's changes count into the same frame's stats
                check_counts(pipe)
    finally:
        pipe.close()


def test_edits_and_compaction_between_frames():
    ch = Churn(scenes.forest(n_trees=120, levels=7, n_lights=24), 3000, seed=8)
    try:
        ch.frame(0, animate=False)
        for f in range(1, 7):
            ch.random_edit()
            if f % 2 == 0:
                renumber(ch, ch.pipe.ctx.compact_topology().astype(np.int64))
            ch.frame(f)
            check_counts(ch.pipe)
    finally:
        ch.close()


TWIN = r"""
import sys
import numpy as np
from bevy_b200 import scenes
import bevy_b200 as bb
sc = scenes.forest(3922, 8, 256)
pipe = bb.VisibilityPipeline(sc)
pipe.enable_visible_diff()
out = {}
for f in range(5):
    if f:
        scenes.advance_cameras(sc, 0.05)
        rows, trs = scenes.mutate_roots(sc, f)
        pipe.ctx.upload_transforms_scattered(rows, trs)
    pipe.update_views()
    pipe.run_frame()
    st = pipe.read_feedback()
    gt, gch = pipe.ctx.download_global_transforms(0, sc.n)
    vv, vch = pipe.ctx.download_view_visibility(0, sc.n)
    out[f"gt{f}"] = gt.view(np.uint32); out[f"gch{f}"] = gch; out[f"vv{f}"] = vv; out[f"vch{f}"] = vch
    out[f"counts{f}"] = np.array([st.gt_changed_count, st.vv_changed_count] + list(st.visible_count) + list(st.cluster_index_count),
                                 np.uint32)
    out[f"far{f}"] = np.array(list(st.cluster_farthest_z), np.float32).view(np.uint32)
    for v in range(len(sc.cameras)):
        out[f"vis{f}_{v}"] = pipe.ctx.download_visible(v)
        a, r = pipe.ctx.download_visible_diff(v)
        out[f"add{f}_{v}"] = a; out[f"rem{f}_{v}"] = r
        off, idx = pipe.ctx.download_clusters(v)
        out[f"coff{f}_{v}"] = off; out[f"cidx{f}_{v}"] = idx
pipe.close()
np.savez(sys.argv[1], **out)
"""


def test_fixed_order_twin_is_byte_identical(tmp_path):
    res = {}
    for arm, env in (("alternating", {}), ("fixed", {"B200VIS_SWEEP_ORDER": "fixed"})):
        e = {k: v for k, v in os.environ.items() if not k.startswith("B200VIS_")}
        e.update(env)
        path = str(tmp_path / f"{arm}.npz")
        prog = f"import sys; sys.path.insert(0, {ROOT!r}); sys.path.insert(0, {HERE!r})\n" + TWIN
        r = subprocess.run([sys.executable, "-c", prog, path], env=e, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, f"{arm}\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"
        res[arm] = np.load(path)
    a, b = res["alternating"], res["fixed"]
    assert sorted(a.files) == sorted(b.files)
    for k in a.files:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), k
