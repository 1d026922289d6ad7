"""b200vis_set_view_diff_sink: the added / removed Entity lists of every (camera, VisibilityClass), as
collect_visible_cpu_culled_entities runs update_cpu_culled_entities for the cameras, written by the device straight into
the caller's memory.  The expected lists come from the oracle's cull, split by visible_entities_by_class and mapped
through the entity bits, then update_cpu_culled_entities per (slot, class) under the slot rules of the render world
(render camera.rs:549-605, view/visibility/mod.rs:389-431): an active view's slot takes its lists, an inactive view's
slot reports nothing and is emptied, a slot no view names is emptied, a view without a slot reports nothing."""
import copy
import ctypes
import os

import numpy as np
import pytest

import bevy_b200 as bb
import oracle as orc
from bevy_b200 import abi, scenes
from parity import OracleWorld
from test_gpu_bench_scale import run_case
from test_gpu_cull_outputs import ENT_SENTINEL, OFF_SENTINEL, EntitySink, mixed_classes, pinned, shuffled_bits

pytestmark = pytest.mark.gpu

INVALID_ARG, NOT_READY, UNSUPPORTED = 1, 7, 8
NO_SLOT = abi.VIEW_NO_SLOT
EMPTY = np.zeros(0, np.uint64)


class ViewDiffSink:
    """A sentinel-filled view diff sink with guards past both capacities and past both offset arrays."""

    def __init__(self, ctx, capacity, max_slots, guard=64):
        self.cap = capacity
        n_off = ctx.max_views * 8 + 1
        self.added = pinned((capacity + guard,), np.uint64, ENT_SENTINEL)
        self.removed = pinned((capacity + guard,), np.uint64, ENT_SENTINEL)
        self.aoff = pinned((n_off + guard,), np.uint32, OFF_SENTINEL)
        self.roff = pinned((n_off + guard,), np.uint32, OFF_SENTINEL)
        ctx.set_view_diff_sink(self.added, self.removed, self.aoff, self.roff, max_slots, added_capacity=capacity,
                               removed_capacity=capacity)

    def reset(self):
        for a in (self.added, self.removed):
            a[:] = ENT_SENTINEL
        for a in (self.aoff, self.roff):
            a[:] = OFF_SENTINEL

    def check(self, want_added, want_removed, tag):
        """want_*[l] for l = view * 8 + class: the expected sorted Entity bits.  Returns the two true totals."""
        n_lists = len(want_added)
        totals = []
        for name, buf, off, want in (("added", self.added, self.aoff, want_added), ("removed", self.removed, self.roff, want_removed)):
            assert (buf[self.cap:] == ENT_SENTINEL).all(), f"{tag}: {name} written past capacity"
            assert (off[n_lists + 1:] == OFF_SENTINEL).all(), f"{tag}: {name} offsets written past n_views * 8"
            tot = np.concatenate([[0], np.cumsum([len(l) for l in want])]).astype(np.uint32)
            assert (off[:n_lists + 1] == tot).all(), f"{tag}: {name} offsets {off[:n_lists + 1]} vs {tot}"
            flat = np.concatenate(want) if want else EMPTY
            k = min(len(flat), self.cap)
            assert (buf[:k] == flat[:k]).all(), f"{tag}: {name} entities differ"
            assert (buf[k:self.cap] == ENT_SENTINEL).all(), f"{tag}: {name} entries past the true total"
            totals.append(int(tot[-1]))
        return totals


class SlotModel:
    """The render world's RenderVisibleEntities per camera, by slot: prev[slot] = the eight class lists last reported."""

    def __init__(self):
        self.prev = {}

    def step(self, slots, active, lists, n_views):
        """slots[v] for the views of the run (missing = no slot); lists[(view, class)] = this run's sorted Entity bits."""
        added, removed, prev = [], [], {}
        for v in range(n_views):
            s = slots[v] if v < len(slots) else NO_SLOT
            for k in range(8):
                if s == NO_SLOT or not active[v]:
                    added.append(EMPTY); removed.append(EMPTY)
                    continue
                old, new = self.prev.get(s, [EMPTY] * 8)[k], lists.get((v, k), EMPTY)
                _, a_m, _, r_m = orc.update_cpu_culled_entities(old, old, new, new)
                added.append(a_m); removed.append(r_m)
            if s != NO_SLOT and active[v]:
                prev[s] = [lists.get((v, k), EMPTY) for k in range(8)]
        self.prev = prev                        # inactive views' slots and slots no view names: emptied
        return added, removed


def class_lists(sc, rows_of_view, active):
    """{(view, class): sorted Entity bits} of the active views (visible_entities_by_class of each view's list)."""
    out = {}
    for v, rows in enumerate(rows_of_view):
        if not active[v] or rows is None:
            continue
        for k, r in orc.visible_entities_by_class(rows, sc.class_mask, sc.entity_bits).items():
            out[(v, k)] = np.sort(sc.entity_bits[r])
    return out


def per_view(sc, op):
    """Applies op to the scene's camera list and every per-view array it has."""
    sc.cameras = op(list(sc.cameras))
    for name in ("view_flags", "view_layers", "view_range_index"):
        a = getattr(sc, name)
        if a is not None:
            setattr(sc, name, np.asarray(op(list(a)), np.asarray(a).dtype))


def active_of(sc):
    return [bool(f & abi.VIEW_ACTIVE) for f in sc.view_flags]


def planes_of(pipe):
    return np.stack([np.ctypeslib.as_array(v.half_spaces).reshape(6, 4).copy() for v in pipe.views])


def camera_descs(sc):
    arr = (bb.CameraDesc * len(sc.cameras))()
    for v, cam in enumerate(sc.cameras):
        arr[v].global_transform[:] = cam.gt.tolist()
        arr[v].fov_y, arr[v].aspect, arr[v].near_z, arr[v].far_z = cam.fov, cam.aspect, cam.near, cam.far
        arr[v].layer_mask, arr[v].flags, arr[v].range_view_index = 1, int(sc.view_flags[v]), -1
    return arr


def make_scene(seed, n_cameras):
    if n_cameras == 4:
        sc = scenes.forest(60, 8, 24, seed=seed)
    else:
        sc = scenes.many_cameras_lights(n_cameras=n_cameras, forest_kwargs=dict(n_trees=40, levels=6, n_lights=16, seed=seed))
    rng = np.random.default_rng(seed)
    mixed_classes(sc, rng)
    shuffled_bits(sc, rng)
    sc.view_flags = np.full(len(sc.cameras), abi.VIEW_ACTIVE, np.uint8)
    return sc


# ---- 1: every frame against the model ----------------------------------------------------------------------------------


def case_diff_matches_the_model_every_frame(seed, n_cameras, twin_outputs, step, capacity=None):
    """Entities in several classes; rows moving and cameras advancing; at frame 2 visible single-class entities change
    class (removed from one class, added to the other); at 3 the view order is permuted with the slots following the
    cameras; the first view with a slot inactive at 4 and active again at 5 (everything added); at 6 a camera is dropped from the views
    (its slot is emptied) and at 7 another camera, new to the views, takes that slot (everything added, nothing
    removed); one camera never has a slot.  step: the frames run through b200vis_step.  twin_outputs: both contexts
    also have the VisibleEntities sink and the row diff, and a twin without the view diff sink writes the same bytes
    and rows.  capacity: both regions that small (truncated, with true totals)."""
    rng = np.random.default_rng(seed)
    sc = make_scene(seed, n_cameras)
    V = len(sc.cameras)
    tw_sc = copy.deepcopy(sc) if twin_outputs else None
    pipe = bb.VisibilityPipeline(sc)
    twin = bb.VisibilityPipeline(tw_sc) if twin_outputs else None
    world = OracleWorld(sc, True)
    try:
        pairs = ((sc, pipe),) + (((tw_sc, twin),) if twin else ())
        if twin:
            for _, p in pairs:
                p.enable_visible_diff()
            ent, tw_ent = EntitySink(pipe.ctx, sc.n), EntitySink(twin.ctx, sc.n)
        max_slots = V + 3
        diff = ViewDiffSink(pipe.ctx, capacity or 2 * sc.n, max_slots)
        cams = list(range(V))                                    # the camera identity at each view position
        slot_of = {c: int(s) for c, s in zip(range(V), rng.permutation(max_slots)[:V])}
        del slot_of[V - 1]                                       # this camera never has a slot
        model = SlotModel()
        seen = dict(added=0, removed=0, class_moves=0, reported_back=0)
        moved = {}
        dropped = off = None
        for f in range(8):
            if f:
                rows, trs = scenes.mutate_roots(sc, f)
                for s, p in pairs:
                    scenes.advance_cameras(s, 0.05)
                    s.trs[rows] = trs
                    p.ctx.upload_transforms_scattered(rows, trs)
                world.tchanged[rows] = 1
            if f == 2:                                            # single-class entities visible in view 0 change class
                vis = pipe.ctx.download_visible(0)
                single = vis[np.isin(sc.class_mask[vis], [1 << k for k in range(8)])][:40]
                for r in single:
                    old = int(sc.class_mask[r])
                    new = np.uint8(1 << ((old.bit_length() - 1 + 3) % 8))
                    moved[int(sc.entity_bits[r])] = (old.bit_length() - 1, int(new).bit_length() - 1)
                    for s, p in pairs:
                        s.class_mask[r] = new
                        one = lambda a: None if a is None else a[r:r + 1]
                        p.ctx.upload_bounds(int(r), one(s.bounds), one(s.flags), one(s.class_mask), one(s.layer_mask), one(s.range_mask))
            if f == 3:                                            # the view query's order changes; slots follow the cameras
                perm = rng.permutation(V)
                cams = [cams[i] for i in perm]
                for s, _ in pairs:
                    per_view(s, lambda l: [l[i] for i in perm])
            if f == 4:
                off = next(i for i, c in enumerate(cams) if c in slot_of)
            if f in (4, 5):
                for s, _ in pairs:
                    s.view_flags[off] = 0 if f == 4 else abi.VIEW_ACTIVE
            if f == 6:                                            # a camera leaves the views: its slot is named by nobody
                i = next(i for i, c in enumerate(cams) if c in slot_of)
                dropped = (cams[i], [(s.cameras[i], [getattr(s, n)[i] if getattr(s, n) is not None else None
                                                     for n in ("view_flags", "view_layers", "view_range_index")]) for s, _ in pairs])
                cams.pop(i)
                for s, _ in pairs:
                    per_view(s, lambda l: l[:i] + l[i + 1:])
            if f == 7:                                            # a camera new to the views takes the freed slot
                slot_of[100] = slot_of.pop(dropped[0])
                cams.append(100)
                for (s, _), (cam, vals) in zip(pairs, dropped[1]):
                    s.cameras.append(cam)
                    for n, x in zip(("view_flags", "view_layers", "view_range_index"), vals):
                        if x is not None:
                            setattr(s, n, np.append(getattr(s, n), x))
            slots = [slot_of.get(c, NO_SLOT) for c in cams]
            pipe.ctx.set_view_diff_slots(slots)
            diff.reset()
            for _, p in pairs:
                p.update_views()
            _, _, lists, _ = world.frame(planes_of(pipe), cluster=False)
            active = active_of(sc)
            for s, p in pairs:
                if step:
                    p.ctx.step(0, None, None, camera_descs(s), len(s.cameras), p.cluster_config, wait=True)
                else:
                    p.run_frame()
                p.ctx.synchronize()
            for v in range(len(cams)):                            # the device culled what the oracle culled
                if active[v]:
                    assert (pipe.ctx.download_visible(v) == lists[v]).all(), f"frame {f} view {v}: visible list"
            want = class_lists(sc, lists, active)
            want_a, want_r = model.step(slots, active, want, len(cams))
            got = diff.check(want_a, want_r, f"frame {f}")
            seen["added"] += got[0]; seen["removed"] += got[1]
            if f == 2:
                for v in range(len(cams)):
                    for e, (ko, kn) in moved.items():
                        if len(want_r[v * 8 + ko]) and e in set(want_r[v * 8 + ko].tolist()) and e in set(want_a[v * 8 + kn].tolist()):
                            seen["class_moves"] += 1
            if f in (5, 7):                                       # back in view, new to the slot: the whole lists added
                v = off if f == 5 else len(cams) - 1
                if slots[v] != NO_SLOT:
                    assert all(len(want_r[v * 8 + k]) == 0 for k in range(8))
                    assert sum(len(want_a[v * 8 + k]) for k in range(8)) == sum(len(want.get((v, k), EMPTY)) for k in range(8)) > 0
                    seen["reported_back"] += 1
            if twin:
                assert ent.buf.tobytes() == tw_ent.buf.tobytes() and ent.off.tobytes() == tw_ent.off.tobytes(), \
                    f"frame {f}: the VisibleEntities sink differs with the view diff sink registered"
                for v in range(len(cams)):
                    (a0, r0), (a1, r1) = pipe.ctx.download_visible_diff(v), twin.ctx.download_visible_diff(v)
                    assert (a0 == a1).all() and (r0 == r1).all(), f"frame {f} view {v}: the row diff differs"
            for _, p in pairs:
                p.read_feedback()
        assert seen["added"] > 100 and seen["removed"] > 0 and seen["class_moves"] > 0 and seen["reported_back"] == 2, seen
    finally:
        pipe.close()
        if twin:
            twin.close()


# ---- 2: errors and removal ---------------------------------------------------------------------------------------------


def case_errors_and_removal():
    sc = make_scene(41, 4)
    pipe = bb.VisibilityPipeline(sc)
    c, lib = pipe.ctx, abi.load_library()
    V = c.max_views
    try:
        four = np.arange(4, dtype=np.uint32)
        assert lib.b200vis_set_view_diff_slots(c._h, 4, four.ctypes.data) == NOT_READY      # no sink yet
        a, r = pinned((4 * sc.n,), np.uint64, 0), pinned((4 * sc.n,), np.uint64, 0)
        ao, ro = pinned((V * 8 + 1,), np.uint32, 0), pinned((V * 8 + 1,), np.uint32, 0)
        S, M = abi.ViewDiffSink, 4
        n = 4 * sc.n
        bad = [S(None, n, r.ctypes.data, n, ao.ctypes.data, ro.ctypes.data, M),
               S(a.ctypes.data, n, None, n, ao.ctypes.data, ro.ctypes.data, M),
               S(a.ctypes.data, n, r.ctypes.data, n, None, ro.ctypes.data, M),
               S(a.ctypes.data, n, r.ctypes.data, n, ao.ctypes.data, None, M),
               S(a.ctypes.data, 0, r.ctypes.data, n, ao.ctypes.data, ro.ctypes.data, M),
               S(a.ctypes.data, n, r.ctypes.data, 0, ao.ctypes.data, ro.ctypes.data, M),
               S(a.ctypes.data + 4, n - 1, r.ctypes.data, n, ao.ctypes.data, ro.ctypes.data, M),
               S(a.ctypes.data, n, r.ctypes.data + 4, n - 1, ao.ctypes.data, ro.ctypes.data, M)]
        for b in bad:
            assert lib.b200vis_set_view_diff_sink(c._h, ctypes.byref(b)) == INVALID_ARG
        assert lib.b200vis_set_view_diff_slots(c._h, 4, four.ctypes.data) == NOT_READY      # the refusals registered nothing
        c.set_view_diff_sink(a, r, ao, ro, M)
        c.set_view_diff_slots([2, 0, 3, 1])
        pipe.run_frame(); c.synchronize()
        total = sum(len(c.download_visible(v)) > 0 for v in range(4))
        assert total > 0 and ao[V * 8] > 0 and ro[V * 8] == 0     # the first run: everything added
        for s in ([M, 0, 1, 2], [0, 0, 1, 2]):                    # a slot >= max_slots, a slot twice
            assert lib.b200vis_set_view_diff_slots(c._h, 4, np.asarray(s, np.uint32).ctypes.data) == INVALID_ARG
        assert lib.b200vis_set_view_diff_slots(c._h, V + 1, np.full(V + 1, NO_SLOT, np.uint32).ctypes.data) == INVALID_ARG
        assert lib.b200vis_set_view_diff_slots(c._h, 2, None) == INVALID_ARG
        ao[:] = 7; ro[:] = 7
        pipe.run_frame(); c.synchronize()                         # refusals changed nothing: same slots, nothing moved
        assert (ao[:V * 8 + 1] == 0).all() and (ro[:V * 8 + 1] == 0).all()
        c.set_view_diff_slots([])                                 # no slots: empty lists, every slot emptied
        pipe.run_frame(); c.synchronize()
        assert (ao[:V * 8 + 1] == 0).all() and (ro[:V * 8 + 1] == 0).all()
        c.set_view_diff_slots([1, 3, 0, 2])                       # named again: everything added
        pipe.run_frame(); c.synchronize()
        first = ao[V * 8]
        assert first > 0 and ro[V * 8] == 0
        c.set_view_diff_sink(None, None, None, None)              # removal: nothing written, slots refused
        ao[:] = 7
        pipe.run_frame(); c.synchronize()
        assert (ao == 7).all()
        assert lib.b200vis_set_view_diff_slots(c._h, 4, four.ctypes.data) == NOT_READY
    finally:
        pipe.close()
    try:
        multi = abi.Context(64, max_lights=1, max_views=1, world_size=2, rank=0)
    except abi.B200VisError:
        return                                                    # no two-rank context on this machine
    try:
        x, y = pinned((8,), np.uint64, 0), pinned((9,), np.uint32, 0)
        s = abi.ViewDiffSink(x.ctypes.data, 8, x.ctypes.data, 8, y.ctypes.data, y.ctypes.data, 1)
        assert abi.load_library().b200vis_set_view_diff_sink(multi._h, ctypes.byref(s)) == UNSUPPORTED
    finally:
        multi.close()


# ---- 3: topology edits, compactions and set_topology -------------------------------------------------------------------


def case_diff_across_spawns_despawns_and_a_compacting_twin():
    """Edits that despawn and spawn and device compactions, against a twin that never compacts: both diffs equal the
    model byte for byte.  A despawned visible entity is reported removed with its own entity bits; spawned visible
    entities are reported added."""
    from test_gpu_compaction import Twins, order_keeping_reparents

    def make():
        sc = scenes.forest(60, 8, 24, seed=7)
        mixed_classes(sc, np.random.default_rng(7))
        return sc
    rng = np.random.default_rng(7)
    t = Twins(make, 3000, seed=7)
    slots = [3, 0, 5, 1]
    try:
        cap = 2 * (t.b.sc.n + 3000)
        da, db = (ViewDiffSink(x.pipe.ctx, cap, 6) for x in (t.a, t.b))
        for x in (t.a, t.b):
            x.pipe.ctx.set_view_diff_slots(slots)
        model = SlotModel()
        despawned_removed = spawned_added = 0
        for f in range(9):
            dead_bits, new_bits = EMPTY, EMPTY
            if f:
                n0, alive0 = t.b.sc.n, t.b.alive.copy()
                t.random_edit(n_despawn=12, n_flat=8, n_kids=6)
                dead_bits = t.b.sc.entity_bits[np.nonzero(alive0 & ~t.b.alive[:n0])[0]]
                new_bits = t.b.sc.entity_bits[n0:]
                if f % 3 == 0:
                    t.compact(*order_keeping_reparents(t, 2, rng))
            da.reset(); db.reset()
            t.frame(f, animate=f > 0)                             # both twins against the oracle, and against each other
            for x in (t.a, t.b):
                x.pipe.ctx.synchronize()
            sc = t.b.sc
            active = [True] * len(sc.cameras)
            lists = [t.b.pipe.ctx.download_visible(v) for v in range(len(sc.cameras))]
            want_a, want_r = model.step(slots, active, class_lists(sc, lists, active), len(sc.cameras))
            db.check(want_a, want_r, f"b frame {f}")
            da.check(want_a, want_r, f"a frame {f}")
            for x, y in ((da.added, db.added), (da.removed, db.removed), (da.aoff, db.aoff), (da.roff, db.roff)):
                assert x.tobytes() == y.tobytes(), f"frame {f}: the compacting twin's diff differs"
            removed, added = np.concatenate(want_r), np.concatenate(want_a)
            despawned_removed += int(np.isin(dead_bits, removed).sum())
            spawned_added += int(np.isin(new_bits, added).sum())
        assert t.compactions and despawned_removed > 0 and spawned_added > 0, (despawned_removed, spawned_added)
    finally:
        t.close()


def case_set_topology_reports_every_list_added():
    """b200vis_set_topology (the re-topology fallback of a churned world) empties every slot: the next run reports each
    list in full as added and nothing removed."""
    from test_gpu_topology_edits import Churn
    sc = scenes.forest(60, 6, 12, seed=12)
    mixed_classes(sc, np.random.default_rng(12))
    ch = Churn(sc, 400, seed=12)
    slots = [2, 0, 3, 1]
    try:
        diff = ViewDiffSink(ch.pipe.ctx, 2 * (ch.sc.n + 400), 4)
        ch.pipe.ctx.set_view_diff_slots(slots)
        model = SlotModel()
        for f in range(5):
            if f:
                ch.random_edit(n_despawn=4, n_flat=4, n_kids=2)
                if f == 3:
                    ch.compact()                                  # set_topology with the sink registered
                    model = SlotModel()
            diff.reset()
            ch.frame(f, animate=f > 0)
            ch.pipe.ctx.synchronize()
            active = [True] * len(ch.sc.cameras)
            lists = [ch.pipe.ctx.download_visible(v) for v in range(len(ch.sc.cameras))]
            want = class_lists(ch.sc, lists, active)
            totals = diff.check(*model.step(slots, active, want, len(ch.sc.cameras)), f"frame {f}")
            if f == 3:
                assert totals[0] == sum(len(x) for x in want.values()) > 0 and totals[1] == 0
    finally:
        ch.close()


# ---- 4: the full-size world -----------------------------------------------------------------------------------------


def case_config3_full_size():
    """The bench world (1,000,366 rows, 4 views), its class masks split into meshes and lights with some rows in both,
    with the VisibleEntities sink: the first frame's added lists are the sink's class lists, nothing removed; a second
    frame with nothing moved reports empty diffs."""
    sc = scenes.forest()
    assert sc.n == 1_000_366 and len(sc.cameras) == 4
    sc.class_mask = np.where(np.arange(sc.n) % 7 == 0, 3, 1).astype(np.uint8)
    sc.class_mask[sc.light_row] = 2
    pipe = bb.VisibilityPipeline(sc)
    try:
        ent = EntitySink(pipe.ctx, sc.n)
        diff = ViewDiffSink(pipe.ctx, 2 * sc.n, 4)
        pipe.ctx.set_view_diff_slots([0, 1, 2, 3])
        for f in range(2):
            diff.reset()
            pipe.update_views()
            pipe.run_frame()
            pipe.ctx.synchronize()
            if f == 0:
                want = [ent.ent[v, ent.off[v, k]:ent.off[v, k + 1]] for v in range(4) for k in range(8)]
                diff.check(want, [EMPTY] * 32, "first frame")
                assert ent.off[:, 8].sum() > 0 and (ent.off[:, 2] > ent.off[:, 1]).any()
            else:
                diff.check([EMPTY] * 32, [EMPTY] * 32, "steady frame")
            pipe.read_feedback()
    finally:
        pipe.close()


# ---- every case runs in a fresh interpreter (as in test_gpu_shadow_diff) -----------------------------------------------

def _fresh(call, **env):
    run_case(f"import test_gpu_view_diff as m\nm.{call}", dict(env, **{k: os.environ[k] for k in ("B200VIS_LIB",) if k in os.environ}),
             timeout=600)


@pytest.mark.parametrize("seed,n_cameras,twin_outputs,step,pipeline,capacity", [
    (21, 4, False, False, "1", None), (22, 4, True, False, "1", None), (23, 4, True, False, "0", None),
    (24, 4, False, True, "1", None), (25, 12, True, False, "1", None), (26, 4, False, False, "1", 50)])
def test_diff_matches_the_model_every_frame(seed, n_cameras, twin_outputs, step, pipeline, capacity):
    _fresh(f"case_diff_matches_the_model_every_frame({seed!r}, {n_cameras!r}, {twin_outputs!r}, {step!r}, {capacity!r})",
           B200VIS_PIPELINE=pipeline)


def test_errors_and_removal():
    _fresh("case_errors_and_removal()")


def test_diff_across_spawns_despawns_and_a_compacting_twin():
    _fresh("case_diff_across_spawns_despawns_and_a_compacting_twin()")


def test_set_topology_reports_every_list_added():
    _fresh("case_set_topology_reports_every_list_added()")


def test_config3_full_size():
    _fresh("case_config3_full_size()")
