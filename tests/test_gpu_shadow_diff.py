"""b200vis_set_shadow_diff_sink: the added / removed Entity lists of every light subview (update_cpu_culled_entities per
(slot, face), as collect_visible_cpu_culled_entities runs it for the shadow views), written by the device straight into
the caller's memory.  The expected lists come from the oracle's update_cpu_culled_entities applied per (slot, face) to
the lists the oracle (or the context's own row lists, across topology edits) gives, mapped through the entity bits, with
the three slot rules: an active item's slot takes its lists, an inactive item's slot reports nothing and is emptied, a
slot no item names is emptied."""
import copy
import os
import types

import numpy as np
import pytest

import bevy_b200 as bb
import oracle as orc
from bevy_b200 import abi, scenes
from parity import OracleWorld
from test_gpu_bench_scale import run_case
from test_gpu_cull_outputs import pinned
from test_gpu_shadow_outputs import ENT_SENTINEL, OFF_SENTINEL, ShadowSink, light_items, move_rows, oracle_frame, shadow_scene

pytestmark = pytest.mark.gpu

INVALID_ARG, CAPACITY, NOT_READY = 1, 6, 7
NO_SLOT = abi.SHADOW_NO_SLOT
EMPTY = np.zeros(0, np.uint64)


class DiffSink:
    """A sentinel-filled shadow diff sink with guards past both capacities and past both offset arrays."""

    def __init__(self, ctx, capacity, max_items, max_slots, guard=64):
        self.cap, self.max_items = capacity, max_items
        self.added = pinned((capacity + guard,), np.uint64, ENT_SENTINEL)
        self.removed = pinned((capacity + guard,), np.uint64, ENT_SENTINEL)
        self.aoff = pinned((max_items * 6 + 1 + guard,), np.uint32, OFF_SENTINEL)
        self.roff = pinned((max_items * 6 + 1 + guard,), np.uint32, OFF_SENTINEL)
        ctx.set_shadow_diff_sink(self.added, self.removed, self.aoff, self.roff, max_slots, added_capacity=capacity,
                                 removed_capacity=capacity, max_items=max_items)

    def reset(self):
        for a in (self.added, self.removed):
            a[:] = ENT_SENTINEL
        for a in (self.aoff, self.roff):
            a[:] = OFF_SENTINEL

    def check(self, want_added, want_removed, tag):
        """want_*[l] for l = item * 6 + face: the expected sorted Entity bits.  Returns the two true totals."""
        n_lists = len(want_added)
        totals = []
        for name, buf, off, want in (("added", self.added, self.aoff, want_added), ("removed", self.removed, self.roff, want_removed)):
            assert (buf[self.cap:] == ENT_SENTINEL).all(), f"{tag}: {name} written past capacity"
            assert (off[n_lists + 1:] == OFF_SENTINEL).all(), f"{tag}: {name} offsets written past n_items"
            tot = np.concatenate([[0], np.cumsum([len(l) for l in want])]).astype(np.uint32)
            assert (off[:n_lists + 1] == tot).all(), f"{tag}: {name} offsets {off[:n_lists + 1]} vs {tot}"
            flat = np.concatenate(want) if want else EMPTY
            k = min(len(flat), self.cap)
            assert (buf[:k] == flat[:k]).all(), f"{tag}: {name} entities differ"
            assert (buf[k:self.cap] == ENT_SENTINEL).all(), f"{tag}: {name} entries past the true total"
            totals.append(int(tot[-1]))
        return totals

    def lists(self, which, l):
        buf, off = (self.added, self.aoff) if which == "added" else (self.removed, self.roff)
        return buf[off[l]:off[l + 1]]


class SlotModel:
    """collect_visible_cpu_culled_entities over slots: prev[slot] = the six lists last reported for it."""

    def __init__(self):
        self.prev = {}

    def step(self, slots, active, lists):
        """lists[(item, face)] = this run's sorted Entity bits of an active item's list (missing = empty)."""
        added, removed, prev = [], [], {}
        for i, s in enumerate(slots):
            for f in range(6):
                if s == NO_SLOT or not active[i]:
                    added.append(EMPTY); removed.append(EMPTY)
                    continue
                old, new = self.prev.get(s, [EMPTY] * 6)[f], lists.get((i, f), EMPTY)
                _, a_m, _, r_m = orc.update_cpu_culled_entities(old, old, new, new)
                added.append(a_m); removed.append(r_m)
            if s != NO_SLOT and active[i]:
                prev[s] = [lists.get((i, f), EMPTY) for f in range(6)]
        self.prev = prev                        # inactive items' slots and slots no item names: emptied
        return added, removed


def with_slots(ctx, holder):
    """oracle_frame installs its items through ctx.set_shadow_items: give them holder["slots"]."""
    plain = ctx.set_shadow_items
    ctx.set_shadow_items = lambda items, list_capacity=0: plain(items, list_capacity, diff_slots=holder["slots"])


def oracle_lists(want, active, bits):
    return {k: np.sort(bits[v]) for k, v in want.items() if active[k[0]]}


# ---- 1 / 2: every frame against the model, with and without the entity sink ------------------------------------------


def case_diff_matches_the_model_every_frame(seed, shuffle, entity_sink):
    """Point, spot and cascade items mixed; casters moving, cameras advancing; items reordered every frame with their
    slots kept; a point light hidden from every view for two frames (its item inactive, then everything added); a point
    light left out for one frame (its slot emptied, then everything added); some items without a slot.  list_capacity
    = 1.  entity_sink: the context also has the entity sink, and a twin with only the entity sink writes the same bytes."""
    sc, rng, caster, spot_ords, point_ords = shadow_scene(seed, shuffle)
    tw_sc = copy.deepcopy(sc)
    pipe = bb.VisibilityPipeline(sc)
    twin = bb.VisibilityPipeline(tw_sc) if entity_sink else None
    world = OracleWorld(sc, True)
    n_casc_views = min(len(sc.cameras), 2)
    n_items = len(spot_ords) + len(point_ords) + 2 * n_casc_views
    slot_of = {("s", int(o)): k for k, o in enumerate(spot_ords)}
    slot_of.update({("p", int(o)): len(spot_ords) + k for k, o in enumerate(point_ords)})
    unslotted = int(spot_ords[-1])                            # this spot light's item never has a slot
    hidden = int(point_ords[0])
    hidden_row = int(sc.light_row[hidden])
    left_out = int(point_ords[-1])
    holder = {}
    with_slots(pipe.ctx, holder)
    try:
        ctxs = (pipe.ctx,) + ((twin.ctx,) if twin else ())
        for c in ctxs:
            c.upload_shadow_casters(0, caster)
        diff = DiffSink(pipe.ctx, sc.n * 4, n_items + 2, n_items + 5)
        if twin:
            ent, tw_ent = ShadowSink(pipe.ctx, sc.n * 4, n_items + 2), ShadowSink(twin.ctx, sc.n * 4, n_items + 2)
        model = SlotModel()
        seen = [0, 0]
        inactive_seen = False
        for f in range(8):
            if f:
                for s in (sc, tw_sc):
                    scenes.advance_cameras(s, 0.2)
                rows = np.unique(rng.integers(0, sc.n, sc.n // 20))
                delta = rng.uniform(-2, 2, (len(rows), 3)).astype(np.float32)
                move_rows(pipe, world, sc, rng, rows, delta)
                if twin:
                    twin.ctx.upload_transforms_scattered(rows.astype(np.uint32), sc.trs[rows.astype(np.uint32)])
                    tw_sc.trs[:] = sc.trs
            if f in (2, 4):                                       # hidden from every view at frame 2, back at frame 4
                for s, p in ((sc, pipe),) + (((tw_sc, twin),) if twin else ()):
                    if f == 2:
                        s.flags[hidden_row] &= np.uint8(0xFF ^ abi.F_INHERITED_VISIBLE)
                    else:
                        s.flags[hidden_row] |= np.uint8(abi.F_INHERITED_VISIBLE)
                    one = lambda a: None if a is None else a[hidden_row:hidden_row + 1]
                    p.ctx.upload_bounds(hidden_row, one(s.bounds), one(s.flags), one(s.class_mask), one(s.layer_mask), one(s.range_mask))
            sp, pt = rng.permutation(spot_ords), rng.permutation(point_ords)     # the items' order changes every frame
            if f == 5:
                pt = pt[pt != left_out]
            slots = [NO_SLOT if int(o) == unslotted else slot_of[("s", int(o))] for o in sp]
            slots += [slot_of[("p", int(o))] for o in pt]
            slots += [len(slot_of) + k for k in range(2 * n_casc_views)]
            holder["slots"] = slots
            diff.reset()
            if twin:
                ent.reset(); tw_ent.reset()
            want, active, _ = oracle_frame(pipe, world, sc, caster, sp, pt, n_casc_views, list_capacity=1)
            assert len(active) == len(slots)
            if twin:
                twin.update_views()
                items, _, _ = light_items(sc, world, sp, pt, n_casc_views)
                twin.ctx.run(bb.STAGE_ALL)
                twin.ctx.set_shadow_items(items, 1)
                twin.ctx.run_shadow_culling()
                twin.ctx.synchronize()
            pipe.ctx.synchronize()
            want_a, want_r = model.step(slots, active, oracle_lists(want, active, sc.entity_bits))
            got = diff.check(want_a, want_r, f"frame {f}")
            seen[0] += got[0]; seen[1] += got[1]
            if f in (0, 4, 6):                                    # first frame, back in view, back in the items: all added
                i = list(pt).index(hidden) if f == 4 else (list(pt).index(left_out) if f == 6 else 0)
                i += len(sp)
                for face in range(6):
                    assert (diff.lists("added", i * 6 + face) == np.sort(sc.entity_bits[want.get((i, face), [])])).all()
            inactive_seen |= not all(active)
            if twin:
                assert ent.ent_buf.tobytes() == tw_ent.ent_buf.tobytes() and ent.off_buf.tobytes() == tw_ent.off_buf.tobytes(), \
                    f"frame {f}: the entity sink differs with the diff sink registered"
                assert ent.act_buf.tobytes() == tw_ent.act_buf.tobytes(), f"frame {f}: active flags differ"
                twin.read_feedback()
            pipe.read_feedback()
        assert inactive_seen and seen[0] > 200 and seen[1] > 0, seen
    finally:
        pipe.close()
        if twin:
            twin.close()


# ---- 3 / 4: truncation, errors and removal ----------------------------------------------------------------------------


def case_truncation_and_launch_counts():
    """Capacities smaller than the run's lists: true totals in the offsets, no entry at or past either capacity, nothing
    past n_items.  Without the diff sink the shadow stage launches what it always did; the sink adds two launches."""
    sc, rng, caster, spot_ords, point_ords = shadow_scene(31, True)
    pipe = bb.VisibilityPipeline(sc)
    world = OracleWorld(sc, True)
    holder = {}
    try:
        pipe.ctx.upload_shadow_casters(0, caster)
        want, active, _ = oracle_frame(pipe, world, sc, caster, spot_ords, point_ords, 1)
        n_items = len(active)
        pipe.ctx.synchronize()
        n0 = abi.kernel_launch_count()
        pipe.ctx.run_shadow_culling(); pipe.ctx.synchronize()
        assert abi.kernel_launch_count() - n0 == 3                # select, cull, expand
        pipe.read_feedback()
        diff = DiffSink(pipe.ctx, 11, n_items, n_items)
        with_slots(pipe.ctx, holder)
        holder["slots"] = list(range(n_items))
        model = SlotModel()
        for f, radii in enumerate(((25.0, 80.0), (5.0, 10.0))):  # the cascades shrink: many removed entries
            diff.reset()
            want, active, _ = oracle_frame(pipe, world, sc, caster, spot_ords, point_ords, 1, list_capacity=1, radii=radii)
            pipe.ctx.synchronize()
            totals = diff.check(*model.step(holder["slots"], active, oracle_lists(want, active, sc.entity_bits)), f"frame {f}")
            assert totals[f] > 11, totals
            pipe.read_feedback()
        n0 = abi.kernel_launch_count()
        pipe.ctx.run_shadow_culling(); pipe.ctx.synchronize()
        assert abi.kernel_launch_count() - n0 == 5                # + the offsets scan and the emit
    finally:
        pipe.close()


def case_errors_and_removal():
    sc, rng, caster, spot_ords, point_ords = shadow_scene(41, False)
    pipe = bb.VisibilityPipeline(sc)
    world = OracleWorld(sc, True)
    c, lib = pipe.ctx, abi.load_library()
    import ctypes
    try:
        c.upload_shadow_casters(0, caster)
        want, active, _ = oracle_frame(pipe, world, sc, caster, spot_ords, point_ords, 1)
        n_items = len(active)
        items, _, _ = light_items(sc, world, spot_ords, point_ords, 1)
        slots = list(range(n_items))
        with pytest.raises(abi.B200VisError):                     # slots while no diff sink is registered
            c.set_shadow_items(items, diff_slots=slots)
        arr = (abi.ShadowItem * (n_items + 1))()
        sl = np.arange(n_items + 1, dtype=np.uint32)
        assert lib.b200vis_set_shadow_items_ex(c._h, n_items, arr, 0, sl.ctypes.data) == NOT_READY
        a, r = pinned((64,), np.uint64, 0), pinned((64,), np.uint64, 0)
        ao, ro = pinned((n_items * 6 + 1,), np.uint32, 0), pinned((n_items * 6 + 1,), np.uint32, 0)
        S, M = abi.ShadowDiffSink, n_items
        bad = [S(None, 64, r.ctypes.data, 64, ao.ctypes.data, ro.ctypes.data, n_items, M),
               S(a.ctypes.data, 64, None, 64, ao.ctypes.data, ro.ctypes.data, n_items, M),
               S(a.ctypes.data, 64, r.ctypes.data, 64, None, ro.ctypes.data, n_items, M),
               S(a.ctypes.data, 64, r.ctypes.data, 64, ao.ctypes.data, None, n_items, M),
               S(a.ctypes.data, 0, r.ctypes.data, 64, ao.ctypes.data, ro.ctypes.data, n_items, M),
               S(a.ctypes.data, 64, r.ctypes.data, 0, ao.ctypes.data, ro.ctypes.data, n_items, M),
               S(a.ctypes.data + 4, 32, r.ctypes.data, 64, ao.ctypes.data, ro.ctypes.data, n_items, M),
               S(a.ctypes.data, 64, r.ctypes.data + 4, 32, ao.ctypes.data, ro.ctypes.data, n_items, M)]
        for b in bad:
            assert lib.b200vis_set_shadow_diff_sink(c._h, ctypes.byref(b)) == INVALID_ARG
        small = S(a.ctypes.data, 64, r.ctypes.data, 64, ao.ctypes.data, ro.ctypes.data, n_items - 1, M)
        assert lib.b200vis_set_shadow_diff_sink(c._h, ctypes.byref(small)) == CAPACITY
        c.set_shadow_diff_sink(a, r, ao, ro, M)
        c.set_shadow_items(items, diff_slots=slots)
        c.run_shadow_culling(); c.synchronize()
        total = sum(len(want[k]) for k in want if active[k[0]])
        assert ao[n_items * 6] == total and ro[n_items * 6] == 0  # the first run: everything added
        # refusals change nothing: the installed items keep their slots
        for s in ([M] + slots[1:], [0, 0] + slots[2:]):           # a slot >= max_slots, a slot twice
            assert lib.b200vis_set_shadow_items_ex(c._h, n_items, arr, 0, np.asarray(s, np.uint32).ctypes.data) == INVALID_ARG
        no_slots = np.full(n_items + 1, NO_SLOT, np.uint32)
        assert lib.b200vis_set_shadow_items_ex(c._h, n_items + 1, arr, 0, no_slots.ctypes.data) == CAPACITY
        assert lib.b200vis_set_shadow_items(c._h, n_items + 1, arr, 0) == CAPACITY
        assert lib.b200vis_set_shadow_lights(c._h, n_items + 1, np.zeros(n_items + 1, np.uint32).ctypes.data,
                                             np.zeros((n_items + 1) * 144, np.float32).ctypes.data, None, -1, 0) == CAPACITY
        ao[:] = 7; ro[:] = 7
        c.run_shadow_culling(); c.synchronize()
        assert (ao == 0).all() and (ro == 0).all()                # the same lists under the same slots: no change
        c.set_shadow_items(items)                                 # no slots: no diff, every slot emptied
        c.run_shadow_culling(); c.synchronize()
        assert (ao == 0).all() and (ro == 0).all()
        c.set_shadow_items(items, diff_slots=slots[::-1])         # named again (other slots): everything added
        c.run_shadow_culling(); c.synchronize()
        assert ao[n_items * 6] == total and ro[n_items * 6] == 0
        c.set_shadow_items([])                                    # no items: the one offset is 0
        ao[0] = ro[0] = 99
        c.run_shadow_culling(); c.synchronize()
        assert ao[0] == 0 and ro[0] == 0
        c.set_shadow_diff_sink(None, None, None, None)            # removal: nothing written, slots refused
        ao[:] = 7
        c.set_shadow_items(items)
        c.run_shadow_culling(); c.synchronize()
        assert (ao == 7).all()
        assert lib.b200vis_set_shadow_items_ex(c._h, n_items, arr, 0, sl.ctypes.data) == NOT_READY
        assert lib.b200vis_set_shadow_items_ex(c._h, 0, None, 0, None) == 0     # NULL slots: set_shadow_items
    finally:
        pipe.close()


# ---- 5: topology edits, compactions and set_topology -------------------------------------------------------------------


def point_items(ctx, sc, ords):
    """Point (even position) and spot (odd) items of these light ordinals, from the device's light GlobalTransforms."""
    items = []
    for k, o in enumerate(ords):
        row = int(sc.light_row[o])
        gt, _ = ctx.download_global_transforms(row, 1, want_changed=False)
        fr = abi.host_point_light_frusta(gt[0], float(sc.light_range[o]))
        items.append(dict(kind=k % 2, light_row=row, range=float(sc.light_range[o]), frusta=fr if k % 2 == 0 else fr[k % 6]))
    return items


def run_slotted(ctx, sc, ords, slots, ent, world):
    """The shadow stage with slotted items; returns the context's own lists as sorted Entity bits and the active flags
    the entity sink ent reports (the row lists of an inactive item are empty).  The stage's set_visible() is taken
    into the oracle world's ViewVisibility (the oracle does not run these items; test_gpu_shadow_outputs checks it)."""
    items = point_items(ctx, sc, ords)
    ent.reset()
    ctx.set_shadow_items(items, diff_slots=slots)
    ctx.run_shadow_culling()
    ctx.synchronize()
    active = [bool(x) for x in ent.act_buf[:len(ords)]]
    world.vv[:], _ = ctx.download_view_visibility(0, sc.n)
    lists = {}
    for i, it in enumerate(items):
        for f in range(6 if it["kind"] == 0 else 1):
            lists[(i, f)] = np.sort(sc.entity_bits[ctx.download_shadow_visible(i, f)])
    return lists, active


def topo_scene(seed):
    sc = scenes.forest(n_trees=60, levels=6, n_lights=12, seed=seed)
    sc.trs[sc.roots, 0:3] *= np.float32(0.12)                   # the trees inside the lights' reach
    sc.light_range[:] = 45.0
    sc.bounds[sc.light_row, 3] = 45.0
    sc.shadow_caster = (np.random.default_rng(seed).random(sc.n) < 0.8).astype(np.uint8)
    sc.shadow_caster[sc.light_row] = 0
    return sc


def case_diff_across_spawns_despawns_and_a_compacting_twin():
    """Edits that despawn and spawn (new keys merging into the ranks) and device compactions, against a twin that never
    compacts: both diffs equal the model byte for byte.  A despawned caster in a slot's set is reported removed with its
    own entity bits; spawned casters are reported added."""
    from test_gpu_compaction import Twins, order_keeping_reparents
    rng = np.random.default_rng(5)
    t = Twins(lambda: topo_scene(5), 3000, seed=5)
    ords = [0, 1, 2, 3, 4, 5]
    slots = [3, 7, 0, 5, 1, 2]
    try:
        cap = 6 * (t.b.sc.n + 3000)
        da, db = (DiffSink(x.pipe.ctx, cap, len(ords), 8) for x in (t.a, t.b))
        ea, eb = (ShadowSink(x.pipe.ctx, cap, len(ords)) for x in (t.a, t.b))
        model = SlotModel()
        despawned_removed = spawned_added = 0
        seen = 0
        for f in range(9):
            dead_bits, new_bits = EMPTY, EMPTY
            if f:
                n0, alive0 = t.b.sc.n, t.b.alive.copy()
                t.random_edit(n_despawn=12, n_flat=8, n_kids=6, kill_light=False)
                dead_bits = t.b.sc.entity_bits[np.nonzero(alive0 & ~t.b.alive[:n0])[0]]
                new_bits = t.b.sc.entity_bits[n0:]
                if f % 3 == 0:
                    t.compact(*order_keeping_reparents(t, 2, rng))
            da.reset(); db.reset()
            t.frame(f, animate=f > 0)
            lists, active = run_slotted(t.b.pipe.ctx, t.b.sc, ords, slots, eb, t.b.world)
            lists_a, active_a = run_slotted(t.a.pipe.ctx, t.a.sc, ords, slots, ea, t.a.world)
            assert active == active_a and all(np.array_equal(lists[k], lists_a[k]) for k in lists), f"frame {f}: twins' lists differ"
            want_a, want_r = model.step(slots, active, lists)
            seen += sum(db.check(want_a, want_r, f"b frame {f}"))
            da.check(want_a, want_r, f"a frame {f}")
            for x, y in ((da.added, db.added), (da.removed, db.removed), (da.aoff, db.aoff), (da.roff, db.roff)):
                assert x.tobytes() == y.tobytes(), f"frame {f}: the compacting twin's diff differs"
            removed = np.concatenate(want_r) if want_r else EMPTY
            added = np.concatenate(want_a) if want_a else EMPTY
            despawned_removed += int(np.isin(dead_bits, removed).sum())
            spawned_added += int(np.isin(new_bits, added).sum())
            for x in (t.a, t.b):
                x.pipe.read_feedback()
        assert t.compactions and seen > 100 and despawned_removed > 0 and spawned_added > 0, (seen, despawned_removed, spawned_added)
    finally:
        t.close()


def case_set_topology_reports_every_list_added():
    """b200vis_set_topology (the re-topology fallback of a churned world) empties every slot: the next run reports each
    list in full as added and nothing removed."""
    from test_gpu_topology_edits import Churn
    ch = Churn(topo_scene(12), 400, seed=12)
    ords, slots = [0, 1, 2, 3], [2, 0, 3, 1]
    try:
        diff = DiffSink(ch.pipe.ctx, 6 * (ch.sc.n + 400), len(ords), 4)
        ent = ShadowSink(ch.pipe.ctx, 6 * (ch.sc.n + 400), len(ords))
        model = SlotModel()
        for f in range(5):
            if f:
                ch.random_edit(n_despawn=4, n_flat=4, n_kids=2, kill_light=False)
                if f == 3:
                    ch.compact()                                  # set_topology with the sink registered
                    model = SlotModel()
            diff.reset()
            ch.frame(f, animate=f > 0)
            lists, active = run_slotted(ch.pipe.ctx, ch.sc, ords, slots, ent, ch.world)
            totals = diff.check(*model.step(slots, active, lists), f"frame {f}")
            if f == 3:
                assert totals[0] == sum(len(v) for (i, _), v in lists.items() if active[i]) > 0 and totals[1] == 0
            ch.pipe.read_feedback()
    finally:
        ch.close()


# ---- 6: the full-size world -----------------------------------------------------------------------------------------


def case_config3_full_size():
    """The bench world (1,000,366 rows, 4 views) with 16 point lights, 8 spot lights and one directional light x 4 views x
    4 cascades, both sinks: the first run's added lists are the entity sink's lists, nothing removed; a second frame with
    nothing moved reports empty diffs."""
    sc = scenes.forest()
    assert sc.n == 1_000_366 and len(sc.cameras) == 4
    caster = np.ones(sc.n, np.uint8); caster[sc.light_row] = 0
    pipe = bb.VisibilityPipeline(sc)
    try:
        pipe.ctx.upload_shadow_casters(0, caster)
        n_items = 8 + 16 + 4 * 4
        ent = ShadowSink(pipe.ctx, 4 * sc.n, n_items)
        diff = DiffSink(pipe.ctx, 4 * sc.n, n_items, n_items)
        for f in range(2):
            ent.reset(); diff.reset()
            pipe.update_views()
            pipe.ctx.run(bb.STAGE_ALL)
            gt, _ = pipe.ctx.download_global_transforms(0, sc.n, want_changed=False)
            items, _, _ = light_items(sc, types.SimpleNamespace(gt=gt), np.arange(8), np.arange(8, 24), 4,
                                      radii=(10.0, 30.0, 90.0, 270.0))
            pipe.ctx.set_shadow_items(items, 1, diff_slots=np.arange(n_items))
            pipe.ctx.run_shadow_culling()
            pipe.ctx.synchronize()
            total = int(ent.off_buf[n_items * 6])
            if f == 0:
                assert total > 0 and sum(ent.act_buf[:24]) > 0
                assert (diff.aoff[:n_items * 6 + 1] == ent.off_buf[:n_items * 6 + 1]).all()
                assert diff.added[:total].tobytes() == ent.ent_buf[:total].tobytes()
                assert (diff.roff[:n_items * 6 + 1] == 0).all()
            else:
                assert (diff.aoff[:n_items * 6 + 1] == 0).all() and (diff.roff[:n_items * 6 + 1] == 0).all()
                assert (diff.added[:16] == ENT_SENTINEL).all() and (diff.removed[:16] == ENT_SENTINEL).all()
            pipe.read_feedback()
    finally:
        pipe.close()


# ---- every case runs in a fresh interpreter (as in test_gpu_shadow_outputs) --------------------------------------------

def _fresh(call, **env):
    run_case(f"import test_gpu_shadow_diff as m\nm.{call}", dict(env, **{k: os.environ[k] for k in ("B200VIS_LIB",) if k in os.environ}),
             timeout=600)


@pytest.mark.parametrize("seed,shuffle,entity_sink,pipeline", [(21, True, False, "1"), (22, False, True, "1"), (23, True, True, "0"),
                                                               (24, False, False, "0")])
def test_diff_matches_the_model_every_frame(seed, shuffle, entity_sink, pipeline):
    _fresh(f"case_diff_matches_the_model_every_frame({seed!r}, {shuffle!r}, {entity_sink!r})", B200VIS_PIPELINE=pipeline)


def test_truncation_and_launch_counts():
    _fresh("case_truncation_and_launch_counts()")


def test_errors_and_removal():
    _fresh("case_errors_and_removal()")


def test_diff_across_spawns_despawns_and_a_compacting_twin():
    _fresh("case_diff_across_spawns_despawns_and_a_compacting_twin()")


def test_set_topology_reports_every_list_added():
    _fresh("case_set_topology_reports_every_list_added()")


def test_config3_full_size():
    _fresh("case_config3_full_size()")
