"""b200vis_emit_shadow_entities: after a run into a shadow entity sink that was too small, a larger sink and an emit give
the offsets, active flags and Entity lists a sink of that size would have had from the start, and nothing else moves:
not the ViewVisibility bits or change flags, not the frame statistics, not the row lists, not the shadow diff (its
outputs now, and what the next run reports).  Each check compares against a twin context that never emits."""
import copy
import ctypes
import os

import numpy as np
import pytest

import bevy_b200 as bb
from bevy_b200 import abi, scenes
from test_gpu_bench_scale import run_case
from test_gpu_shadow_diff import DiffSink
from test_gpu_shadow_outputs import ENT_SENTINEL, ShadowSink

pytestmark = pytest.mark.gpu

CAPACITY, NOT_READY = 6, 7
N_POINT_SPOT, N_CASCADES = 8, 2
N_ITEMS = N_POINT_SPOT + N_CASCADES
SMALL = 16


def emit_scene(seed):
    """60 trees pulled inside the lights' reach (range 45), 80% of the meshes shadow casters."""
    sc = scenes.forest(n_trees=60, levels=6, n_lights=12, seed=seed)
    sc.trs[sc.roots, 0:3] *= np.float32(0.12)
    sc.light_range[:] = 45.0
    sc.bounds[sc.light_row, 3] = 45.0
    caster = (np.random.default_rng(seed).random(sc.n) < 0.8).astype(np.uint8)
    caster[sc.light_row] = 0
    return sc, caster


def items_of(ctx, sc, f):
    """Point (even) and spot (odd) items from the device's light GlobalTransforms, and two cascades that move per frame."""
    items = []
    for k in range(N_POINT_SPOT):
        row = int(sc.light_row[k])
        gt, _ = ctx.download_global_transforms(row, 1, want_changed=False)
        fr = abi.host_point_light_frusta(gt[0], float(sc.light_range[k]))
        items.append(dict(kind=k % 2, light_row=row, range=float(sc.light_range[k]), frusta=fr if k % 2 == 0 else fr[k % 6]))
    for c in range(N_CASCADES):
        gt = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 2.0 * f, 0, 0], np.float32)
        items.append(dict(kind=2, frusta=abi.host_point_light_frusta(gt, 30.0 + 20.0 * c)[(c + f) % 6]))
    return items


def frame(pipes, f, rng, list_capacity=1, slots=None):
    """The same frame on every pipeline: move the cameras and some rows, cull, install the items."""
    sc0 = pipes[0].scene
    rows = np.unique(rng.integers(0, sc0.n, sc0.n // 20)).astype(np.uint32)
    delta = rng.uniform(-1, 1, (len(rows), 3)).astype(np.float32)
    for p in pipes:
        if f:
            scenes.advance_cameras(p.scene, 0.2)
            p.scene.trs[rows, 0:3] += delta
            p.ctx.upload_transforms_scattered(rows, p.scene.trs[rows])
        p.update_views()
        p.ctx.run(bb.STAGE_ALL)
        p.ctx.set_shadow_items(items_of(p.ctx, p.scene, f), list_capacity, diff_slots=slots)


def twins(seed):
    sc, caster = emit_scene(seed)
    pipes = (bb.VisibilityPipeline(sc), bb.VisibilityPipeline(copy.deepcopy(sc)))
    for p in pipes:
        p.ctx.upload_shadow_casters(0, caster)
    return pipes


def same_sink(got, want, tag):
    """got and want hold the same run's lists; got's capacity is at least the total."""
    n = N_ITEMS * 6 + 1
    total = int(want.off_buf[n - 1])
    assert (got.off_buf[:n] == want.off_buf[:n]).all(), f"{tag}: offsets differ"
    assert (got.act_buf[:N_ITEMS] == want.act_buf[:N_ITEMS]).all(), f"{tag}: active flags differ"
    assert got.ent_buf[:total].tobytes() == want.ent_buf[:total].tobytes(), f"{tag}: entities differ"
    assert (got.ent_buf[total:] == ENT_SENTINEL).all(), f"{tag}: written past the total"
    assert (got.off_buf[n:] == want.off_buf[n:]).all() and (got.act_buf[N_ITEMS:] == want.act_buf[N_ITEMS:]).all(), \
        f"{tag}: written past n_items"


def diff_bytes(d):
    return tuple(x.tobytes() for x in (d.added, d.removed, d.aoff, d.roff))


# ---- 1: grow and emit = a large sink from the start ------------------------------------------------------------------


def case_grown_sink_equals_a_large_sink_from_the_start(with_diff):
    """Every frame context a runs into a 16-entry sink, then registers a sink of exactly the run's total and emits;
    twin b has had a large sink all along.  with_diff: both also have a shadow diff sink with slots, and their diffs
    stay equal, so the emit neither wrote nor consumed anything the next run's diff reads."""
    a, b = twins(7)
    rng = np.random.default_rng(7)
    try:
        big_b = ShadowSink(b.ctx, 6 * b.scene.n, N_ITEMS)
        diffs = [DiffSink(p.ctx, 6 * p.scene.n, N_ITEMS, N_ITEMS) for p in (a, b)] if with_diff else None
        slots = np.arange(N_ITEMS) if with_diff else None
        grown = 0
        for f in range(5):
            small = ShadowSink(a.ctx, SMALL, N_ITEMS)
            big_b.reset()
            if diffs:
                for d in diffs:
                    d.reset()
            frame((a, b), f, rng, slots=slots)
            for p in (a, b):
                p.ctx.run_shadow_culling()
                p.ctx.synchronize()
            total = int(small.off_buf[N_ITEMS * 6])
            assert total == int(big_b.off_buf[N_ITEMS * 6])
            assert total > SMALL, f"frame {f}: the scene no longer overflows the small sink ({total})"
            grown_a = ShadowSink(a.ctx, total, N_ITEMS)
            a.ctx.emit_shadow_entities()
            a.ctx.synchronize()
            same_sink(grown_a, big_b, f"frame {f}")
            grown += 1
            if diffs:
                assert diff_bytes(diffs[0]) == diff_bytes(diffs[1]), f"frame {f}: the shadow diffs differ"
            for p in (a, b):
                p.read_feedback()
        assert grown == 5 and big_b.act_buf[:N_ITEMS].any()
    finally:
        a.close(); b.close()


# ---- 2: the emit changes nothing else ----------------------------------------------------------------------------------


def snapshot(p, diff):
    c = p.ctx
    vv, ch = c.download_view_visibility(0, p.scene.n)
    rows = [c.download_shadow_visible(i, face).tobytes() for i in range(N_ITEMS) for face in range(6)]
    return dict(vv=vv.tobytes(), changed=ch.tobytes(), stats=bytes(c.download_frame_stats()), rows=rows, diff=diff_bytes(diff))


def case_emit_changes_nothing_else():
    """Context a emits twice into a larger sink after every run (the second emit gives the same bytes); twin b never
    emits.  Around the emits a's ViewVisibility bits and change flags, frame statistics, row lists and diff outputs do
    not move, and every frame's diff (which reads the slots the emits must leave alone) equals b's."""
    a, b = twins(11)
    rng = np.random.default_rng(11)
    try:
        diffs = [DiffSink(p.ctx, 6 * p.scene.n, N_ITEMS, N_ITEMS) for p in (a, b)]
        for f in range(4):
            for d in diffs:
                d.reset()
            sinks = [ShadowSink(p.ctx, SMALL, N_ITEMS) for p in (a, b)]
            frame((a, b), f, rng, list_capacity=0, slots=np.arange(N_ITEMS))
            for p in (a, b):
                p.ctx.run_shadow_culling()
                p.ctx.synchronize()
            assert diff_bytes(diffs[0]) == diff_bytes(diffs[1]), f"frame {f}: the diff differs from the twin's"
            before = snapshot(a, diffs[0])
            total = int(sinks[0].off_buf[N_ITEMS * 6])
            assert total > SMALL
            grown = ShadowSink(a.ctx, total + 8, N_ITEMS)
            a.ctx.emit_shadow_entities()
            a.ctx.synchronize()
            first = (grown.ent_buf.tobytes(), grown.off_buf.tobytes(), grown.act_buf.tobytes())
            grown.reset()
            a.ctx.emit_shadow_entities()
            a.ctx.synchronize()
            assert (grown.ent_buf.tobytes(), grown.off_buf.tobytes(), grown.act_buf.tobytes()) == first, f"frame {f}: a second emit differs"
            assert int(grown.off_buf[N_ITEMS * 6]) == total
            after = snapshot(a, diffs[0])
            for k in before:
                assert before[k] == after[k], f"frame {f}: the emit changed {k}"
            assert snapshot(b, diffs[1])["vv"] == after["vv"]
            for p in (a, b):
                p.read_feedback()
    finally:
        a.close(); b.close()


# ---- 3: errors -------------------------------------------------------------------------------------------------------


def case_errors():
    sc, caster = emit_scene(13)
    p = bb.VisibilityPipeline(sc)
    c, lib = p.ctx, abi.load_library()
    emit = lambda: lib.b200vis_emit_shadow_entities(c._h)
    rng = np.random.default_rng(13)
    try:
        c.upload_shadow_casters(0, caster)
        frame((p,), 0, rng)
        assert emit() == NOT_READY                                 # no sink
        sink = ShadowSink(c, SMALL, N_ITEMS)
        assert emit() == NOT_READY                                 # items set, no run since
        c.run_shadow_culling()
        c.synchronize()
        want = (sink.ent_buf.copy(), sink.off_buf.copy(), sink.act_buf.copy())
        sink.reset()
        assert emit() == 0
        c.synchronize()
        assert (sink.ent_buf.tobytes(), sink.off_buf.tobytes(), sink.act_buf.tobytes()) == tuple(x.tobytes() for x in want)
        # a sink for fewer items than are installed is refused when it is registered (so the emit's own CAPACITY check
        # is a safeguard no caller reaches): the emit keeps writing into the sink that stays registered
        ent, off = np.zeros(64, np.uint64), np.zeros(N_ITEMS * 6, np.uint32)
        act = np.zeros(N_ITEMS, np.uint8)
        bad = abi.ShadowEntitiesSink(ent.ctypes.data, 64, N_ITEMS - 1, off.ctypes.data, act.ctypes.data)
        assert lib.b200vis_set_shadow_entities_sink(c._h, ctypes.byref(bad)) == CAPACITY
        sink.reset()
        assert emit() == 0
        c.synchronize()
        assert sink.off_buf[:N_ITEMS * 6 + 1].tobytes() == want[1][:N_ITEMS * 6 + 1].tobytes()
        c.set_shadow_entities_sink(None, None, None)
        assert emit() == NOT_READY                                 # no sink
        sink = ShadowSink(c, 6 * sc.n, N_ITEMS)
        assert emit() == 0                                         # a sink registered after the run is filled
        c.synchronize()
        assert int(sink.off_buf[N_ITEMS * 6]) == int(want[1][N_ITEMS * 6])
        c.set_shadow_items(items_of(c, sc, 0), 1)
        assert emit() == NOT_READY                                 # new items
        c.run_shadow_culling()
        assert emit() == 0
        c.set_shadow_lights([0, 1], np.zeros((2, 6, 6, 4), np.float32), list_capacity=1)
        assert emit() == NOT_READY                                 # new items through the point-light form
        c.run_shadow_culling()
        assert emit() == 0
        c.set_shadow_entities_sink(None, None, None)               # a run without a sink kept nothing to emit from
        c.run_shadow_culling()
        sink = ShadowSink(c, 6 * sc.n, N_ITEMS)
        assert emit() == NOT_READY
        c.set_shadow_items([])                                     # no items: the one offset is 0
        c.run_shadow_culling()
        sink.off_buf[0] = 99
        assert emit() == 0
        c.synchronize()
        assert sink.off_buf[0] == 0
        c.set_shadow_items(items_of(c, sc, 0), 1)
        c.run_shadow_culling()
        assert emit() == 0
        c.edit_topology()
        assert emit() == NOT_READY                                 # rows and rank order may have changed
        c.run_shadow_culling()
        assert emit() == 0
        c.compact_topology()
        assert emit() == NOT_READY
        c.run_shadow_culling()
        assert emit() == 0
        c.set_topology(sc.parent, sc.entity_bits)
        assert emit() == NOT_READY
    finally:
        p.close()


# ---- every case runs in a fresh interpreter (as in test_gpu_shadow_outputs) --------------------------------------------

def _fresh(call):
    run_case(f"import test_gpu_shadow_emit as m\nm.{call}", {k: os.environ[k] for k in ("B200VIS_LIB",) if k in os.environ},
             timeout=600)


@pytest.mark.parametrize("with_diff", [False, True])
def test_grown_sink_equals_a_large_sink_from_the_start(with_diff):
    _fresh(f"case_grown_sink_equals_a_large_sink_from_the_start({with_diff!r})")


def test_emit_changes_nothing_else():
    _fresh("case_emit_changes_nothing_else()")


def test_errors():
    _fresh("case_errors()")
