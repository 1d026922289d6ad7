"""The frame a Bevy app runs (rust/b200vis_plugin.rs): three systems, each its own b200vis_run call --
PROPAGATE + write-back of the GlobalTransform column, CULL + write-back of the ViewVisibility column, CLUSTER -- with the
propagate system in both PostStartup and PostUpdate, so the first frame propagates twice before it culls.  CULL without
PROPAGATE is the streaming kernel 1c (k_cull<SIMPLE> when rows are in Entity order, k_cull<false> otherwise), and PROPAGATE
alone is the PROP-only instantiation of the tile kernels.  The frame counter, statistics slots and constant slots advance
on CULL only, so split frames use them differently from the fused run_frame(); frames of both kinds are mixed here.
Everything is compared bit for bit with the oracle, and host columns fed only by the write-back must equal full downloads."""
import numpy as np
import pytest

import bevy_b200 as bb
from bevy_b200 import scenes
from bevy_b200.scenes import Scene
import oracle as orc

from parity import OracleWorld, compare_frame
from test_gpu_edge_cases import _random_scene as random_scene
from test_gpu_bench_scale import VARIANTS, run_case

pytestmark = pytest.mark.gpu


def same_bits(a, b):
    """Bit equality, except that any NaN matches any NaN (the NaN payload is not part of the contract)."""
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


class HostColumns:
    """The plugin's host columns (GlobalTransform, ViewVisibility + their change bit sets), registered as column sinks."""

    def __init__(self, pipe):
        import torch
        n = pipe.scene.n
        self.n, self.ctx = n, pipe.ctx
        W = (n + 31) // 32
        self.gt = torch.zeros((n, 12), dtype=torch.float32).pin_memory().numpy()
        self.gt[:] = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], np.float32)
        self.gbits = torch.zeros(W, dtype=torch.int32).pin_memory().numpy().view(np.uint32)
        self.vv = torch.zeros(n, dtype=torch.uint8).pin_memory().numpy()
        self.vbits = torch.zeros(W, dtype=torch.int32).pin_memory().numpy().view(np.uint32)
        pipe.ctx.set_column_sinks(self.gt, self.gbits, self.vv, self.vbits)

    def unpack(self, bits):
        return np.unpackbits(bits.view(np.uint8), bitorder="little")[:self.n]

    def check_gt(self, tag):
        self.ctx.synchronize()
        gt, ch = self.ctx.download_global_transforms(0, self.n)
        assert same_bits(self.gt, gt).all(), f"{tag}: host GlobalTransform column differs from the device"
        assert (self.unpack(self.gbits) == ch).all(), f"{tag}: host Changed<GlobalTransform> bits differ"

    def check_vv(self, tag):
        self.ctx.synchronize()
        vv, vch = self.ctx.download_view_visibility(0, self.n)
        assert (self.vv == vv).all(), f"{tag}: host ViewVisibility column differs from the device"
        assert (self.unpack(self.vbits) == vch).all(), f"{tag}: host Changed<ViewVisibility> bits differ"


def propagate_and_check(pipe, world, tag, cols):
    """run(PROPAGATE) [+ write-back of the GlobalTransform column], checked against orc.propagate.  Returns the changed count."""
    sc = pipe.scene
    pipe.propagate_transforms()
    if cols is not None:
        pipe.ctx.writeback_columns(1)
    rc, want = orc.propagate(sc.parent, sc.trs, world.gt, world.tchanged, world.static_opt)
    assert rc == 0
    world.tchanged[:] = 0
    gt, ch = pipe.ctx.download_global_transforms(0, sc.n)
    bad = ~same_bits(gt, world.gt).all(1)
    assert not bad.any(), f"{tag}: GlobalTransform bits differ on rows {np.nonzero(bad)[0][:8]}"
    assert (ch == want).all(), f"{tag}: Changed<GlobalTransform> differs on rows {np.nonzero(ch != want)[0][:8]}"
    if cols is not None:
        cols.check_gt(tag)
    return int(want.sum())


def split_frame(pipe, world, f, cols=None, propagate_twice=False):
    """One frame as the plugin runs it; the caller has uploaded this frame's Transforms."""
    sc = pipe.scene
    tag = f"[{sc.name} split frame {f}]"
    n_changed = propagate_and_check(pipe, world, tag, cols)
    if propagate_twice:                          # PostStartup + PostUpdate
        n_changed += propagate_and_check(pipe, world, tag + " (second propagate)", cols)
    pipe.update_views()
    pipe.check_visibility()
    if cols is not None:
        pipe.ctx.writeback_columns(2)
        cols.check_vv(tag)
    if len(sc.light_row):
        pipe.assign_lights_to_clusters()
    _, vch = pipe.ctx.download_view_visibility(0, sc.n)
    stats = compare_frame(pipe, world, f, check_gt=False, run_device=False)
    assert stats.gt_changed_count == n_changed, f"{tag}: frame stats count {stats.gt_changed_count} GlobalTransform changes, not {n_changed}"
    assert stats.vv_changed_count == int(vch.sum()), f"{tag}: frame stats count {stats.vv_changed_count} ViewVisibility changes"
    return stats


def fused_frame(pipe, world, f, cols=None):
    pipe.update_views()
    stats = compare_frame(pipe, world, f)
    if cols is not None:
        pipe.ctx.writeback_columns(3)
        cols.check_gt(f"[{pipe.scene.name} fused frame {f}]")
        cols.check_vv(f"[{pipe.scene.name} fused frame {f}]")
    return stats


def move(pipe, world, kind, f):
    """Upload this frame's changed Transforms: 'dense' moves every root (whole trees change), 'sparse' three roots,
    'static' nothing (and the cameras stay put)."""
    sc = pipe.scene
    if kind == "static":
        return
    scenes.advance_cameras(sc, 0.05)
    before = sc.trs[sc.roots].copy()
    rows, trs = scenes.mutate_roots(sc, f)
    if kind == "sparse":                         # only three roots change: the others keep their Transform
        sc.trs[rows[3:]] = before[3:]
        rows, trs = rows[:3], trs[:3]
    pipe.ctx.upload_transforms_scattered(rows, trs)
    world.tchanged[rows] = 1


DEFAULT_SEQUENCE = (("split", "dense"), ("split", "dense"), ("split", "sparse"), ("fused", "sparse"), ("split", "static"),
                    ("fused", "dense"), ("split", "dense"), ("split", "sparse"), ("fused", "static"), ("split", "sparse"))


def plugin_frames(sc, static_opt=True, sinks=True, sequence=DEFAULT_SEQUENCE):
    """Frame 0 is the plugin's first frame (PROPAGATE twice); then `sequence` of (split | fused, dense | sparse | static)."""
    pipe = bb.VisibilityPipeline(sc, static_transform_optimizations=static_opt)
    world = OracleWorld(sc, static_opt)
    try:
        cols = HostColumns(pipe) if sinks else None
        split_frame(pipe, world, 0, cols, propagate_twice=True)
        for f, (path, kind) in enumerate(sequence, start=1):
            move(pipe, world, kind, f)
            s = split_frame(pipe, world, f, cols) if path == "split" else fused_frame(pipe, world, f, cols)
            if kind == "static" and static_opt:     # without the static optimisations roots are rewritten (and flagged) every frame
                assert s.gt_changed_count == 0
        if sinks:
            pipe.ctx.set_column_sinks()
    finally:
        pipe.close()


def deep_chain():
    """A 700-deep chain next to a root with 3000 children: many tiles, many passes."""
    chain = 700
    parent = [scenes.NO_PARENT] + list(range(chain - 1))
    root = len(parent)
    parent += [scenes.NO_PARENT] + [root] * 3000
    n = len(parent)
    rng = np.random.default_rng(5)
    trs = np.zeros((n, 10), np.float32)
    trs[:, 0:3] = rng.uniform(-0.2, 0.2, (n, 3)); trs[:, 3:7] = scenes.random_unit_quats(rng, n); trs[:, 7:10] = 1.0
    bounds = np.zeros((n, 6), np.float32); bounds[:, 3:6] = 0.5
    return Scene("chain_fanout", np.array(parent, np.uint32), trs, bounds,
                 np.full(n, scenes.F_INHERITED_VISIBLE | scenes.F_HAS_AABB, np.uint8), np.ones(n, np.uint8),
                 np.arange(n, dtype=np.uint64), cameras=[scenes._camera(0.3)], roots=np.array([0, root], np.uint32))


@pytest.mark.parametrize("static_opt", [True, False])
def test_forest_in_entity_order_simple_cull(static_opt):
    """Rows in Entity order: CULL alone runs k_cull<SIMPLE> (stored ballots)."""
    plugin_frames(scenes.forest(n_trees=200, levels=7, n_lights=24), static_opt=static_opt)


@pytest.mark.parametrize("seed,static_opt", [(21, True), (22, False)])
def test_random_scene_general_cull(seed, static_opt):
    """Layers, range masks, shuffled entity bits, NoCpuCulling rows and views, detached rows: k_cull<false>; then a frame
    with an inactive view, whose VisibleEntities must survive the split CULL untouched."""
    sc = random_scene(seed)
    seq = DEFAULT_SEQUENCE[:5] + (("split", "sparse"),)
    plugin_frames(sc, static_opt=static_opt, sequence=seq)
    sc = random_scene(seed)
    sc.view_flags = [bb.VIEW_ACTIVE, 0, bb.VIEW_ACTIVE]
    plugin_frames(sc, static_opt=static_opt, sequence=(("split", "sparse"), ("fused", "sparse"), ("split", "dense")))


@pytest.mark.parametrize("static_opt", [True, False])
def test_multi_pass_plans(static_opt):
    """Config #1 (1077-node trees: parents in other tiles, k_mark_dirty_global) and a 700-deep chain."""
    seq = (("split", "sparse"), ("split", "dense"), ("fused", "sparse"), ("split", "static"), ("split", "sparse"))
    plugin_frames(scenes.propagate_bench_scene(), static_opt=static_opt, sequence=seq)
    plugin_frames(deep_chain(), static_opt=static_opt, sequence=seq)


def test_split_frames_without_column_sinks():
    plugin_frames(scenes.forest(n_trees=60, levels=6, n_lights=8), sinks=False)


def test_scatter_write_back_only():
    """B200VIS_WRITEBACK_DENSE=0: every write-back takes the scatter kernel, dense frames included (own interpreter: the
    switch is read once per process)."""
    run_case("from test_gpu_split_stages import plugin_frames\n"
             "plugin_frames(scenes.forest(n_trees=200, levels=7, n_lights=24))", {"B200VIS_WRITEBACK_DENSE": "0"})


@pytest.mark.parametrize("variant", ["default", "lean", "warp", "classic", "scout", "flow", "lean_pipe", "tma_2_tiles"])
def test_propagate_only_tile_pass_of_every_kernel(variant):
    """The PROP-only instantiation of each tile kernel, each in its own interpreter: the forest (one pass), config #1
    (several passes) and the random scene."""
    run_case("from test_gpu_split_stages import plugin_frames, random_scene\n"
             "seq = (('split', 'dense'), ('split', 'sparse'), ('fused', 'dense'), ('split', 'static'), ('split', 'dense'))\n"
             "plugin_frames(scenes.forest(n_trees=300, levels=8, n_lights=32), sequence=seq)\n"
             "plugin_frames(scenes.propagate_bench_scene(), sequence=seq)\n"
             "plugin_frames(random_scene(23), sequence=seq)", VARIANTS[variant])
