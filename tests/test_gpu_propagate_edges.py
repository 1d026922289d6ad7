"""Transform propagation at signed zeros, NaN, subnormals and overflow, on the device, in every tile kernel.

The edge scene (tests/propagate_reference.py) puts probe chains on every parent -> child hand-over of the tile kernels
(cross-pass parents, the register-walked top levels, __syncwarp and named-barrier levels, tiles of more than 8 levels,
warp-kernel slots, scout levels).  Its frames: a first write; Transforms whose only change is the sign of a zero (set_if_neq
keeps the stored bits, and children are computed from them); NaN rows visited again (NaN != NaN: changed every visit) and
not; a static frame; another system writing -0 or NaN bits into probe parents (the marked kernel 1b); a static frame.  Each
frame is compared with the oracle (GlobalTransform bits with any NaN matching any NaN, Changed<GlobalTransform>,
ViewVisibility, visible lists, clusters) and held to the float64 bound on the device's own output; through the fused
run_frame, the split PROPAGATE + CULL frame with the host columns written back, and b200vis_step.

Sparse deep edits: one non-root row at depth >= 3 changes in a third of the trees, the rest stay clean, with the static
optimisations on: exactly the dirty trees' roots report Changed<GlobalTransform>, on one-pass and several-pass plans."""
import numpy as np
import pytest

import bevy_b200 as bb
from bevy_b200 import scenes
import oracle as orc

import propagate_reference as ref
from parity import OracleWorld, compare_frame
from test_gpu_bench_scale import run_case
from test_gpu_split_stages import HostColumns, same_bits

pytestmark = pytest.mark.gpu


def check_propagate(pipe, world, tag):
    """The oracle's propagate for this frame (with the pending marks), against the device: bits and change flags.  This is
    the comparison point of GlobalTransform.  compare_frame, called after it with check_gt=False, runs the oracle's
    propagate once more inside world.frame: with tchanged cleared that call leaves every bit as it is (it only revisits
    rows when the static optimisations are off), and its change flags are not compared."""
    sc = pipe.scene
    ext = world.ext.copy(); world.ext[:] = 0
    rc, want = orc.propagate(sc.parent, sc.trs, world.gt, world.tchanged, world.static_opt, gt_ext_changed=ext)
    assert rc == 0
    world.tchanged[:] = 0
    gt, ch = pipe.ctx.download_global_transforms(0, sc.n)
    bad = ~same_bits(gt, world.gt).all(1)
    assert not bad.any(), f"{tag}: GlobalTransform bits differ on rows {np.nonzero(bad)[0][:8]}"
    assert (ch == want).all(), f"{tag}: Changed<GlobalTransform> differs on rows {np.nonzero(ch != want)[0][:8]}"
    return gt, want


def cameras(sc):
    arr = (bb.CameraDesc * len(sc.cameras))()
    for v, cam in enumerate(sc.cameras):
        arr[v].global_transform[:] = cam.gt.tolist()
        arr[v].fov_y, arr[v].aspect, arr[v].near_z, arr[v].far_z = cam.fov, cam.aspect, cam.near, cam.far
        arr[v].layer_mask, arr[v].flags, arr[v].range_view_index = 1, bb.VIEW_ACTIVE, -1
    return arr


def edge_frames(static_opt=True, shape="fused", marks=True, seed=0):
    """The edge scene's frames; shape: 'fused' (run_frame), 'split' (PROPAGATE, CULL, CLUSTER runs with the host columns
    written back) or 'step' (b200vis_step with the column sinks).  marks=False leaves out the written GlobalTransforms
    (tile kernels other than 1b refuse them)."""
    es = ref.EdgeScene(seed)
    sc = es.scene
    pipe = bb.VisibilityPipeline(sc, static_transform_optimizations=static_opt)
    world = OracleWorld(sc, static_opt)
    world.ext = np.zeros(sc.n, np.uint8)
    try:
        cols = HostColumns(pipe) if shape in ("split", "step") else None
        for f, kind in enumerate(es.FRAMES):
            tag = f"[{sc.name} {shape} static_opt={static_opt} frame {f} {kind}]"
            rows, trs = es.uploads(f)
            world.tchanged[rows] = 1
            if shape != "step" and len(rows):
                pipe.ctx.upload_transforms_scattered(rows, trs)
            if marks:
                mrows, mvals = es.marks(f, world.gt)
                if len(mrows):
                    world.gt[mrows] = mvals; world.ext[mrows] = 1
                    if cols is not None:
                        cols.gt[mrows] = mvals
                    pipe.ctx.write_global_transforms_scattered(mrows, mvals)
            if shape == "fused":
                pipe.update_views()
                pipe.run_frame()
                gt, ch = check_propagate(pipe, world, tag)
                compare_frame(pipe, world, f, check_gt=False, run_device=False)
            elif shape == "split":
                pipe.propagate_transforms()
                pipe.ctx.writeback_columns(1)
                gt, ch = check_propagate(pipe, world, tag)
                cols.check_gt(tag)
                pipe.update_views()
                pipe.check_visibility()
                pipe.ctx.writeback_columns(2)
                cols.check_vv(tag)
                pipe.assign_lights_to_clusters()
                compare_frame(pipe, world, f, check_gt=False, run_device=False)
            else:
                rows = np.ascontiguousarray(rows, np.uint32); trs = np.ascontiguousarray(trs, np.float32)
                arr = cameras(sc)
                pipe.ctx.step(len(rows), rows.ctypes.data, trs.ctypes.data, arr, len(sc.cameras), pipe.cluster_config,
                              wait=True, writeback=True)
                gt, ch = check_propagate(pipe, world, tag)
                pipe.update_views(clusters=False)
                compare_frame(pipe, world, f, cluster=False, check_gt=False, run_device=False)
                cols.check_gt(tag); cols.check_vv(tag)
            if kind != "marks":
                r, checked = ref.bound_violation(gt, sc.parent, sc.trs)
                assert checked > 100000 and r <= 1.0, f"{tag}: the device's GlobalTransform exceeds the float64 bound by {r:.3g}x"
            if kind == "first":
                with np.errstate(invalid="ignore"):
                    assert np.isnan(gt).any() and np.isinf(gt).any() and ((gt != 0) & (np.abs(gt) < ref.TINY)).any()
            if kind == "zero_signs":
                flipped = np.array(sorted(es.flip), np.int64)
                assert (~ch[flipped]).sum() >= 5                   # visited, equal, kept
            if kind == "nan_revisit":
                again = np.array([r for r, a in es.nan_rows if a], np.int64)
                assert ch[again].all()
                if static_opt:
                    assert not ch[[r for r, a in es.nan_rows if not a]].any()
            if kind == "static" and static_opt:
                assert not ch.any()
        if cols is not None:
            pipe.ctx.set_column_sinks()
    finally:
        pipe.close()


def tree_of(parent):
    """(root row, depth) of every row."""
    n = len(parent)
    root = np.arange(n, dtype=np.int64)
    depth = np.zeros(n, np.int64)
    real = parent < n
    while True:
        step = real[root]
        if not step.any():
            break
        depth += step
        root = np.where(step, np.where(real, parent, 0).astype(np.int64)[root], root)
    return root, depth


def sparse_deep_frames(make, frames=4, seed=1, min_passes=1):
    """Static optimisations on; per frame one non-root row at depth >= 3 in a third of the trees gets a new Transform."""
    sc = make()
    rng = np.random.default_rng(seed)
    root, depth = tree_of(sc.parent)
    trees = np.unique(root[depth >= 3])
    pipe = bb.VisibilityPipeline(sc, static_transform_optimizations=True)
    world = OracleWorld(sc, True)
    world.ext = np.zeros(sc.n, np.uint8)
    try:
        assert pipe.ctx.topology_summary()[3] >= min_passes
        for f in range(frames):
            dirty_trees = np.zeros(0, np.int64)
            if f:
                dirty_trees = rng.choice(trees, size=len(trees) // 3, replace=False)
                rows = np.array([rng.choice(np.nonzero((root == t) & (depth >= 3))[0]) for t in dirty_trees], np.uint32)
                sc.trs[rows, 0:3] += rng.uniform(-0.3, 0.3, (len(rows), 3)).astype(np.float32)
                pipe.ctx.upload_transforms_scattered(rows, sc.trs[rows])
                world.tchanged[rows] = 1
            pipe.update_views()
            pipe.run_frame()
            _, ch = check_propagate(pipe, world, f"[{sc.name} sparse deep frame {f}]")
            compare_frame(pipe, world, f, check_gt=False, run_device=False)
            if f:
                want = np.isin(trees, dirty_trees)
                assert (ch[trees] == want).all(), \
                    f"frame {f}: roots reporting Changed<GlobalTransform> {np.nonzero(ch[trees] != want)[0][:8]} are not the dirty trees'"
    finally:
        pipe.close()


def forest_trees():
    return scenes.forest(n_trees=120, levels=8, n_lights=8, seed=3)


@pytest.mark.parametrize("static_opt", [True, False])
def test_edge_frames_fused(static_opt):
    edge_frames(static_opt, "fused")


@pytest.mark.parametrize("static_opt", [True, False])
def test_edge_frames_split_with_host_columns(static_opt):
    """The host GlobalTransform column, fed only by the dense write-back, holds the kept bits."""
    edge_frames(static_opt, "split")


def test_edge_frames_scatter_write_back():
    """B200VIS_WRITEBACK_DENSE=0: the column write-back takes the scatter kernel (own interpreter)."""
    run_case("from test_gpu_propagate_edges import edge_frames\n"
             "edge_frames(True, 'split')\nedge_frames(False, 'split')", {"B200VIS_WRITEBACK_DENSE": "0"})


def test_edge_frames_step():
    edge_frames(True, "step")


def test_sparse_deep_edits():
    """A one-pass plan (255-node trees, in-tile mark_dirty_trees) and config #1 (k_mark_dirty_global, several passes)."""
    sparse_deep_frames(forest_trees)
    sparse_deep_frames(scenes.propagate_bench_scene, min_passes=2)


KERNELS = {
    "default": ({}, True), "lean": ({"B200VIS_TILE_KERNEL": "lean"}, False),
    "lean_top_through_loop": ({"B200VIS_TILE_KERNEL": "lean", "B200VIS_LEAN_PROBE": "4"}, False),
    "lean_pipe": ({"B200VIS_TILE_KERNEL": "lean", "B200VIS_LEAN_PIPE": "1"}, False),
    "tma_2_tiles": ({"B200VIS_TILE_KERNEL": "tma", "B200VIS_TILES_PER_CTA": "2"}, True),
    "scout": ({"B200VIS_TILE_KERNEL": "scout"}, False), "flow": ({"B200VIS_TILE_KERNEL": "flow"}, False),
    "flow_cta_levels": ({"B200VIS_TILE_KERNEL": "flow", "B200VIS_LEVEL_SYNC": "cta"}, False),
    "warp": ({"B200VIS_TILE_KERNEL": "warp", "B200VIS_WARP_VARIANT": "2p"}, False),
    "warp_dynamic": ({"B200VIS_TILE_KERNEL": "warp", "B200VIS_WARP_DYNAMIC": "1", "B200VIS_WARP_VARIANT": "4n"}, False),
    "classic": ({"B200VIS_TILE_KERNEL": "classic"}, False),
    "split_deep_tiles": ({"B200VIS_SPLIT_DEEP_TILES": "1"}, True),
    "serial": ({"B200VIS_PIPELINE": "0"}, True),
}


@pytest.mark.parametrize("kernel", list(KERNELS))
def test_every_tile_kernel(kernel):
    """Each tile kernel in its own interpreter (the switches are read once per process): the edge frames with the
    static optimisations on and off (with written GlobalTransforms where the kernel reads them), and the sparse deep edits
    on a one-pass and a several-pass plan."""
    env, marks = KERNELS[kernel]
    run_case("from test_gpu_propagate_edges import edge_frames, sparse_deep_frames, forest_trees\n"
             f"edge_frames(True, 'fused', marks={marks})\nedge_frames(False, 'fused', marks={marks})\n"
             "sparse_deep_frames(forest_trees)\nsparse_deep_frames(scenes.propagate_bench_scene, min_passes=2)", env, timeout=600)
