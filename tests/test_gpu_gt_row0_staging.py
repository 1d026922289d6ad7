"""Kernel 1b stages old GlobalTransform row 0 alone in tiles whose rows row 0 proved changed on their last run, and reads
old rows 1-2 from HBM for any row row 0 does not prove changed.  Either staging must give the same bits, so every case runs
with row-0 staging (the default) and with B200VIS_GT_STAGE=full, and checks every frame bit for bit against the oracle:
GlobalTransform bits, both change columns, ViewVisibility, the visible lists, the clusters and the frame's change counts.

The worlds make the per-tile hint flip both ways and make the fall-back path carry whole frames: roots that only rotate
about x and move in y/z keep every row 0 of their trees, rows whose row 0 differs only by the sign of a zero, NaN in row 0,
static frames between moving ones, a multi-pass plan, edits, compactions and set_topology between frames.  A twin run of
the bench forest must give byte-identical outputs with both stagings."""
import os
import subprocess
import sys

import numpy as np
import pytest

import bevy_b200 as bb
from bevy_b200 import scenes
from parity import OracleWorld, compare_frame
from test_gpu_propagate_edges import edge_frames
from test_gpu_compaction import renumber
from test_gpu_sweep_order import TWIN, check_counts
from test_gpu_topology_edits import Churn

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
STAGINGS = ("row0", "full")


@pytest.fixture(params=STAGINGS)
def staging(request, monkeypatch):
    """The switch is read when a context is created."""
    if request.param == "full":
        monkeypatch.setenv("B200VIS_GT_STAGE", "full")
    else:
        monkeypatch.delenv("B200VIS_GT_STAGE", raising=False)
    return request.param


def quat_x(a):
    a = np.asarray(a, np.float64)
    return np.stack([np.sin(a / 2), np.zeros_like(a), np.zeros_like(a), np.cos(a / 2)], axis=-1)


def upload(pipe, world, sc, rows):
    rows = np.asarray(rows, np.int64)
    pipe.ctx.upload_transforms_scattered(rows, sc.trs[rows])
    world.tchanged[rows] = 1


def run(sc, frames, move, diff=True, before_frame=None, **kw):
    """move(f) -> rows whose Transform changed in frame f (already written into sc.trs), or None for a static frame."""
    pipe = bb.VisibilityPipeline(sc, **kw)
    world = OracleWorld(sc, kw.get("static_transform_optimizations", True))
    if diff:
        pipe.enable_visible_diff()
    try:
        for f in range(frames):
            if f:
                scenes.advance_cameras(sc, 0.05)
                rows = move(f)
                if rows is not None:
                    upload(pipe, world, sc, rows)
            if before_frame is not None:
                before_frame(pipe, world, f)
            pipe.update_views()
            compare_frame(pipe, world, f)
            check_counts(pipe)
    finally:
        pipe.close()


def bench_motion(sc):
    def move(f):
        rows, _ = scenes.mutate_roots(sc, f)
        return rows
    return move


def test_bench_forest_scaled_down(staging):
    sc = scenes.forest(n_trees=300, levels=8, n_lights=16)
    run(sc, 6, bench_motion(sc))


def test_static_frames_between_moving_ones(staging):
    """Moving tiles go to row-0 staging, a static frame sends them back to full staging, the next moving frame (static
    tiles in full staging, every row changed) to row-0 again."""
    sc = scenes.forest(n_trees=300, levels=8, n_lights=16)
    mv = bench_motion(sc)
    run(sc, 9, lambda f: None if f in (3, 4, 7) else mv(f))


def test_static_frames_without_static_optimizations(staging):
    """Every row is visited and compares equal: the fall-back compares rows 1-2 and keeps the old bits."""
    sc = scenes.forest(n_trees=200, levels=7, n_lights=16)
    mv = bench_motion(sc)
    run(sc, 7, lambda f: None if f in (3, 4) else mv(f), static_transform_optimizations=False)


def test_roots_rotating_about_x_keep_every_row_0(staging):
    """Rotation about x and translation in y/z: a root's row 0 stays (s.x, 0, 0, t.x) and a child's row 0 is that row
    times its local matrix, so no row 0 ever changes while every row does: every row falls back to rows 1-2."""
    sc = scenes.forest(n_trees=200, levels=7, n_lights=16)
    roots = sc.roots
    ang = np.arange(len(roots)) * 0.37
    sc.trs[roots, 3:7] = quat_x(ang).astype(np.float32)

    def move(f):
        sc.trs[roots, 3:7] = quat_x(ang + 0.01 * f).astype(np.float32)
        sc.trs[roots, 1] += np.float32(0.01)
        sc.trs[roots, 2] -= np.float32(0.02)
        return roots
    run(sc, 6, move)


def test_row_0_differing_by_signed_zero(staging):
    """Roots with an identity rotation whose T.x flips between +0 and -0, with children at local translation (-0, -0, -0):
    the children's row 0 differs from the old one by the sign of T.x alone (IEEE-equal), so rows 1-2 decide.  On some frames
    only the sign flips (rows 1-2 equal: the old bits, old sign included, are kept), on others t.y moves too.  The other
    roots move as on the bench, so their tiles run row-0 staging."""
    sc = scenes.forest(n_trees=120, levels=6, n_lights=16)
    roots = sc.roots
    zr, other = roots[:40], roots[40:]
    mv = bench_motion(sc)
    kids = np.nonzero(np.isin(sc.parent, zr))[0]
    sc.trs[zr, 0] = np.float32(0.0)
    sc.trs[zr, 3:7] = (0, 0, 0, 1)
    sc.trs[zr, 7:10] = 1.0
    sc.trs[kids, 0:3] = np.float32(-0.0)
    sc.trs[kids, 3:7] = (0, 0, 0, 1)
    sc.roots = other

    def move(f):
        sc.trs[zr, 0] = np.float32(-0.0) if f % 2 else np.float32(0.0)
        if f % 3 == 0:
            sc.trs[zr, 1] += np.float32(0.5)
        return np.concatenate([zr, kids, mv(f)])
    try:
        run(sc, 7, move)
    finally:
        sc.roots = roots


def test_signed_zeros_nan_subnormals_and_overflow(staging):
    """The propagate edge scene (probe chains on every hand-over, zero-sign-only changes, NaN rows visited again and not,
    static frames, written GlobalTransforms) under either staging."""
    edge_frames()


def test_multi_pass_plan(staging):
    sc = scenes.propagate_bench_scene()

    def passes(pipe, world, f):
        if f == 0:
            assert pipe.ctx.topology_summary()[3] > 1
    run(sc, 5, bench_motion(sc), diff=False, before_frame=passes)


def test_edits_and_compaction_between_frames(staging):
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


def test_set_topology_between_frames(staging):
    """A new plan starts every tile at full staging; the rows' state is kept."""
    sc = scenes.forest(n_trees=200, levels=7, n_lights=16)

    def again(pipe, world, f):
        if f in (3, 5):
            pipe.ctx.set_topology(sc.parent, sc.entity_bits)
    run(sc, 7, bench_motion(sc), diff=False, before_frame=again)


def test_both_stagings_are_byte_identical(tmp_path):
    res = {}
    for arm, env in (("row0", {}), ("full", {"B200VIS_GT_STAGE": "full"})):
        e = {k: v for k, v in os.environ.items() if not k.startswith("B200VIS_")}
        e.update(env)
        path = str(tmp_path / f"{arm}.npz")
        prog = f"import sys; sys.path.insert(0, {ROOT!r}); sys.path.insert(0, {HERE!r})\n" + TWIN
        r = subprocess.run([sys.executable, "-c", prog, path], env=e, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, f"{arm}\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"
        res[arm] = np.load(path)
    a, b = res["row0"], res["full"]
    assert sorted(a.files) == sorted(b.files)
    for k in a.files:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), k
