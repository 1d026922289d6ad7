"""The light-visibility systems' outputs written by the device straight into the caller's memory:

A. b200vis_set_shadow_entities_sink: every shadow list of a run (point-light cubemap faces, spot lights, directional
   cascades) as sorted Entity values, checked every frame against the oracle's check_*_light_mesh_visibility lists
   mapped through the entity bits, with the active flags, the offsets, truncation and the errors.
B. b200vis_set_table_shadow_casters: the shadow-caster byte read from shuffled archetype tables, checked every frame
   against a twin context fed the same bytes by b200vis_upload_shadow_casters, through archetype moves, a change of a
   table's caster bit, detach / re-attach and a set_tables that drops the attachment.
C. set_visible() of the light pass in the tables: a second B200VIS_WB_SET_VISIBLE after b200vis_run_shadow_culling
   stamps its own tick on the rows only lights see, checked against tests/set_visible_model.py composed over the two
   systems and against a forked twin's B200VIS_WB_VIEW_VISIBILITY bytes."""
import copy
import ctypes
import os

import numpy as np
import pytest

import bevy_b200 as bb
import oracle as orc
import set_visible_model as svm
import table_cull_model as CM
from bevy_b200 import abi, scenes
from parity import OracleWorld
from test_gpu_bench_scale import run_case
from test_gpu_cull_outputs import pinned
from test_gpu_edge_cases import _random_scene
from test_gpu_table_writeback import NONE, Tables

pytestmark = pytest.mark.gpu

INVALID_ARG, CAPACITY, NOT_READY = 1, 6, 7
ENT_SENTINEL, OFF_SENTINEL, ACT_SENTINEL = np.uint64(0xA5A5A5A5A5A5A5A5), np.uint32(0xC3C3C3C3), np.uint8(0x5A)
IDENT9 = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1], np.float32)


class ShadowSink:
    """A sentinel-filled shadow entity sink with guards past capacity, past the offsets and past the active flags."""

    def __init__(self, ctx, capacity, max_items, guard=64):
        self.cap, self.max_items = capacity, max_items
        self.ent_buf = pinned((capacity + guard,), np.uint64, ENT_SENTINEL)
        self.off_buf = pinned((max_items * 6 + 1 + guard,), np.uint32, OFF_SENTINEL)
        self.act_buf = np.frombuffer(pinned((max_items + guard + 7) // 8, np.uint64, 0x5A5A5A5A5A5A5A5A).data, np.uint8)
        self.act_buf = self.act_buf[:max_items + guard]
        ctx.set_shadow_entities_sink(self.ent_buf, self.off_buf, self.act_buf, capacity=capacity, max_items=max_items)

    def reset(self):
        self.ent_buf[:] = ENT_SENTINEL; self.off_buf[:] = OFF_SENTINEL; self.act_buf[:] = ACT_SENTINEL

    def check(self, want, active, entity_bits, tag):
        """want[(item, face)] = oracle rows of every list of the run; active[item] = whether the item was culled."""
        n = len(active)
        assert (self.ent_buf[self.cap:] == ENT_SENTINEL).all(), f"{tag}: written past capacity"
        assert (self.off_buf[n * 6 + 1:] == OFF_SENTINEL).all(), f"{tag}: offsets written past n_items"
        assert (self.act_buf[n:] == ACT_SENTINEL).all(), f"{tag}: active written past n_items"
        assert (self.act_buf[:n] == np.asarray(active, np.uint8)).all(), f"{tag}: active {self.act_buf[:n]} vs {active}"
        lists = [np.sort(entity_bits[want[(i, f)]]) if active[i] and (i, f) in want else np.zeros(0, np.uint64)
                 for i in range(n) for f in range(6)]
        tot = np.concatenate([[0], np.cumsum([len(l) for l in lists])]).astype(np.uint32)
        assert (self.off_buf[:n * 6 + 1] == tot).all(), f"{tag}: offsets {self.off_buf[:n * 6 + 1]} vs {tot}"
        flat = np.concatenate(lists) if lists else np.zeros(0, np.uint64)
        k = min(len(flat), self.cap)
        assert (self.ent_buf[:k] == flat[:k]).all(), f"{tag}: entities differ"
        assert (self.ent_buf[k:self.cap] == ENT_SENTINEL).all(), f"{tag}: entries written past the true total"
        return int(tot[-1])


def light_items(sc, world, spot_ords, point_ords, n_casc_views, radii=(25.0, 80.0)):
    """Spot, point and cascade items from this frame's light GlobalTransforms (the oracle world's), with the oracle jobs."""
    items, jobs, casc = [], [], []
    for kind, ords in ((1, spot_ords), (0, point_ords)):
        for o in ords:
            row = int(sc.light_row[o])
            fr = orc.point_light_frusta(world.gt[row], sc.light_range[o], 0.1)
            fr = fr[int(o) % 6] if kind == 1 else fr
            ll = 1 if sc.light_layers is None else int(sc.light_layers[o])
            items.append(dict(kind=kind, light_row=row, range=float(sc.light_range[o]), range_view_index=0, layer_mask=ll, frusta=fr))
            jobs.append((kind, row, o, fr, ll))
    for v in range(n_casc_views):
        for c, rr in enumerate(radii):
            centre = np.asarray(sc.cameras[v].gt[9:12], np.float32) + np.float32(5.0 * c)
            fr = orc.point_light_frusta(np.concatenate([IDENT9, centre]).astype(np.float32), rr, 0.1)[(v + c) % 6]
            vri = -1 if sc.view_range_index is None else int(sc.view_range_index[v])
            items.append(dict(kind=2, range_view_index=vri, layer_mask=3, frusta=fr))
            casc.append((v, fr, vri))
    return items, jobs, casc


def oracle_frame(pipe, world, sc, caster, spot_ords, point_ords, n_casc_views, list_capacity=0, radii=(25.0, 80.0),
                 between=None):
    """One frame on the device (CULL, the shadow items, run_shadow_culling) and in the oracle (cull with
    mark_newly_hidden deferred, the light passes in the reference's order, then mark_newly_hidden).  Returns the oracle
    lists want[(item, face)] and the items' active flags.  between() runs after the CULL stage, before the shadow stage."""
    pipe.update_views()
    planes = np.stack([np.ctypeslib.as_array(v.half_spaces).reshape(6, 4).copy() for v in pipe.views])
    orc.propagate(sc.parent, sc.trs, world.gt, world.tchanged, True)
    world.tchanged[:] = 0
    orc.set_defer_mark_newly_hidden(True)
    try:
        vv_changed, lists = orc.cull(world.gt, sc.bounds, sc.flags, sc.class_mask, sc.entity_bits, world.vv, planes,
                                     view_layers=sc.view_layers, view_flags=sc.view_flags, layer_mask=sc.layer_mask,
                                     range_mask=sc.range_mask, view_range_index=sc.view_range_index)
    finally:
        orc.set_defer_mark_newly_hidden(False)
    lists = [l if l is not None else world.last_lists[v] for v, l in enumerate(lists)]
    world.last_lists = lists
    listed = set(np.concatenate(lists).tolist())
    items, jobs, casc = light_items(sc, world, spot_ords, point_ords, n_casc_views, radii)
    pipe.ctx.run(bb.STAGE_ALL if len(sc.light_row) else (bb.STAGE_PROPAGATE | bb.STAGE_CULL))
    if between is not None:
        between()
    pipe.ctx.set_shadow_items(items, list_capacity)
    pipe.ctx.run_shadow_culling()
    want, active = {}, []
    kw = dict(layer_mask=sc.layer_mask, range_mask=sc.range_mask)
    dir_items = []
    for v in range(n_casc_views):
        frs = np.stack([fr for (w, fr, _) in casc if w == v])
        dir_items.append((frs, 3, [c[2] for c in casc if c[0] == v][0]))
    got_dir = orc.check_dir_light_mesh_visibility(world.gt, sc.bounds, sc.flags, caster, sc.entity_bits, world.vv, vv_changed,
                                                  dir_items, **kw) if dir_items else []
    for i, (kind, row, o, fr, ll) in enumerate(jobs):
        active.append(row in listed)
        if row not in listed:                       # in no view's VisibleEntities: not processed (lib.rs:561-563)
            continue
        sphere = np.concatenate([world.gt[row, 9:12], [sc.light_range[o]]]).astype(np.float32)[None]
        fn = orc.check_spot_light_mesh_visibility if kind == 1 else orc.check_point_light_mesh_visibility
        r = fn(world.gt, sc.bounds, sc.flags, caster, sc.entity_bits, world.vv, vv_changed, sphere, fr[None],
               lod_origin_index=0, light_layers=np.array([ll], np.uint64), **kw)
        if kind == 1:
            want[(i, 0)] = r[0]
        else:
            for face in range(6):
                want[(i, face)] = r[0][face]
    k = len(jobs)
    for lists_of_item in got_dir:
        for rows_ in lists_of_item:
            want[(k, 0)] = rows_; active.append(True); k += 1
    orc.mark_newly_hidden(sc.flags, world.vv, vv_changed)
    return want, active, vv_changed


def shadow_scene(seed, shuffle):
    sc = _random_scene(seed, n_roots=90, n_lights=20, shuffle_entities=shuffle)
    rng = np.random.default_rng(seed)
    caster = (rng.random(sc.n) < 0.8).astype(np.uint8)
    caster[sc.light_row] = 0
    lights = rng.permutation(len(sc.light_row))
    return sc, rng, caster, np.sort(lights[:5]), np.sort(lights[5:9])


def move_rows(pipe, world, sc, rng, rows, delta):
    rows = np.asarray(rows, np.uint32)
    sc.trs[rows, 0:3] += np.asarray(delta, np.float32)
    pipe.ctx.upload_transforms_scattered(rows, sc.trs[rows])
    world.tchanged[rows] = 1


# ---- A: the sink ---------------------------------------------------------------------------------------------------


def case_sink_matches_the_oracle_every_frame(seed, shuffle, pipeline):
    """Point, spot and cascade items mixed, moving cameras and transforms, a light that leaves every view (its item
    inactive, its region empty), shuffled or identity entity bits, pipelined or serial frames.  A twin context without
    the sink downloads the same lists row by row, and they map to the same entities."""
    sc, rng, caster, spot_ords, point_ords = shadow_scene(seed, shuffle)
    tw_sc = copy.deepcopy(sc)
    pipe, twin = bb.VisibilityPipeline(sc), bb.VisibilityPipeline(tw_sc)
    world = OracleWorld(sc, True)
    n_casc_views = min(len(sc.cameras), 2)
    n_items = len(spot_ords) + len(point_ords) + 2 * n_casc_views
    gone = int(sc.light_row[point_ords[0]])
    try:
        for c in (pipe.ctx, twin.ctx):
            c.upload_shadow_casters(0, caster)
        sink = ShadowSink(pipe.ctx, sc.n * 4, n_items + 3)
        seen, inactive_seen = 0, False
        for f in range(6):
            if f:
                for s in (sc, tw_sc):
                    scenes.advance_cameras(s, 0.2)
                rows = np.unique(rng.integers(0, sc.n, sc.n // 20))
                delta = rng.uniform(-2, 2, (len(rows), 3)).astype(np.float32)
                move_rows(pipe, world, sc, rng, rows, delta)
                twin.ctx.upload_transforms_scattered(rows.astype(np.uint32), sc.trs[rows.astype(np.uint32)])
                tw_sc.trs[:] = sc.trs
            if f == 3:                                            # one point light leaves every view: hidden
                for s, p in ((sc, pipe), (tw_sc, twin)):
                    s.flags[gone] &= np.uint8(0xFF ^ abi.F_INHERITED_VISIBLE)
                    one = lambda a: None if a is None else a[gone:gone + 1]
                    p.ctx.upload_bounds(gone, one(s.bounds), one(s.flags), one(s.class_mask), one(s.layer_mask), one(s.range_mask))
            sink.reset()
            want, active, _ = oracle_frame(pipe, world, sc, caster, spot_ords, point_ords, n_casc_views, list_capacity=1)
            assert len(active) == n_items
            twin.update_views()
            items, _, _ = light_items(sc, world, spot_ords, point_ords, n_casc_views)
            twin.ctx.run(bb.STAGE_ALL)
            twin.ctx.set_shadow_items(items)
            twin.ctx.run_shadow_culling()
            pipe.ctx.synchronize()
            seen += sink.check(want, active, sc.entity_bits, f"frame {f}")
            inactive_seen |= not all(active)
            for i in range(n_items):
                for face in range(6):
                    lo, hi = sink.off_buf[i * 6 + face], sink.off_buf[i * 6 + face + 1]
                    rows_ = twin.ctx.download_shadow_visible(i, face)
                    assert (sc.entity_bits[rows_] == sink.ent_buf[lo:hi]).all(), f"frame {f} item {i} face {face}: twin differs"
            vv, _ = pipe.ctx.download_view_visibility(0, sc.n)
            assert (vv == world.vv).all(), f"frame {f}: ViewVisibility differs"
            pipe.read_feedback(); twin.read_feedback()
        assert seen > 200 and inactive_seen and not active[len(spot_ords)]
    finally:
        pipe.close(); twin.close()


def case_truncation_list_capacity_one_and_launch_counts():
    """A sink smaller than the run's lists: true offsets, no entry at or past capacity, nothing past n_items.  The row
    lists kept at one entry still download truncated.  A context without the sink launches what it always did; the sink
    adds one launch."""
    sc, rng, caster, spot_ords, point_ords = shadow_scene(31, True)
    pipe = bb.VisibilityPipeline(sc)
    world = OracleWorld(sc, True)
    try:
        pipe.ctx.upload_shadow_casters(0, caster)
        want, active, _ = oracle_frame(pipe, world, sc, caster, spot_ords, point_ords, 1)
        n_items = len(active)
        pipe.ctx.synchronize()
        n0 = abi.kernel_launch_count()
        pipe.ctx.run_shadow_culling()
        pipe.ctx.synchronize()
        assert abi.kernel_launch_count() - n0 == 3                # select, cull, expand: as before
        sink = ShadowSink(pipe.ctx, 11, n_items)
        pipe.read_feedback()
        want, active, _ = oracle_frame(pipe, world, sc, caster, spot_ords, point_ords, 1, list_capacity=1)
        pipe.ctx.synchronize()
        total = sink.check(want, active, sc.entity_bits, "truncated")
        assert total > 11
        n0 = abi.kernel_launch_count()
        pipe.ctx.run_shadow_culling()
        pipe.ctx.synchronize()
        assert abi.kernel_launch_count() - n0 == 4                # + the offsets scan
        for (i, face), rows_ in want.items():
            if active[i] and len(rows_):
                got = pipe.ctx._lib.b200vis_download_shadow_visible
                cnt = ctypes.c_uint32(0)
                one = np.zeros(1, np.uint32)
                assert got(pipe.ctx._h, i, face, None, 0, ctypes.byref(cnt)) == 0 and cnt.value == len(rows_)
                if len(rows_) > 1:
                    assert got(pipe.ctx._h, i, face, one.ctypes.data, 1, ctypes.byref(cnt)) == CAPACITY
                break
    finally:
        pipe.close()


def case_sink_errors_and_removal():
    sc, rng, caster, spot_ords, point_ords = shadow_scene(41, False)
    pipe = bb.VisibilityPipeline(sc)
    world = OracleWorld(sc, True)
    c, lib = pipe.ctx, abi.load_library()
    try:
        c.upload_shadow_casters(0, caster)
        want, active, _ = oracle_frame(pipe, world, sc, caster, spot_ords, point_ords, 1)
        n_items = len(active)
        ent, off = pinned((64,), np.uint64, 0), pinned((n_items * 6 + 1,), np.uint32, 0)
        act = np.frombuffer(pinned((n_items + 7) // 8 + 1, np.uint64, 0).data, np.uint8)
        S = abi.ShadowEntitiesSink
        for bad in (S(ent.ctypes.data, 0, n_items, off.ctypes.data, act.ctypes.data),
                    S(None, 64, n_items, off.ctypes.data, act.ctypes.data),
                    S(ent.ctypes.data, 64, n_items, None, act.ctypes.data),
                    S(ent.ctypes.data, 64, n_items, off.ctypes.data, None),
                    S(ent.ctypes.data + 4, 32, n_items, off.ctypes.data, act.ctypes.data)):
            assert lib.b200vis_set_shadow_entities_sink(c._h, ctypes.byref(bad)) == INVALID_ARG
        small = S(ent.ctypes.data, 64, n_items - 1, off.ctypes.data, act.ctypes.data)
        assert lib.b200vis_set_shadow_entities_sink(c._h, ctypes.byref(small)) == CAPACITY
        c.set_shadow_entities_sink(ent, off, act, max_items=n_items)
        items, _, _ = light_items(sc, world, spot_ords, point_ords, 1)
        arr = (abi.ShadowItem * (n_items + 1))()
        assert lib.b200vis_set_shadow_items(c._h, n_items + 1, arr, 0) == CAPACITY
        assert lib.b200vis_set_shadow_lights(c._h, n_items + 1, np.zeros(n_items + 1, np.uint32).ctypes.data,
                                             np.zeros((n_items + 1) * 144, np.float32).ctypes.data, None, -1, 0) == CAPACITY
        c.run_shadow_culling(); c.synchronize()                   # the items installed before the refusals still run
        assert off[n_items * 6] == sum(len(want[k]) for k in want if active[k[0]])
        c.set_shadow_entities_sink(None, None, None)
        off[:] = 0
        c.run_shadow_culling(); c.synchronize()
        assert (off == 0).all()
        c.set_shadow_items([])                                    # no items: the one offset is 0
        c.set_shadow_entities_sink(ent, off, act, max_items=n_items)
        off[0] = 99
        c.run_shadow_culling(); c.synchronize()
        assert off[0] == 0
    finally:
        pipe.close()


# ---- B: the caster byte from the tables ----------------------------------------------------------------------------

CASTER, NOT_CASTER, NOCPU, LIGHTS, OUTSIDE = range(5)      # NOCPU: a caster archetype the cull skips
TABLE_FLAGS = {CASTER: 0, NOT_CASTER: 0, NOCPU: abi.F_NO_CPU_CULLING}


class CasterTwins:
    """Context A reads its cull inputs and caster bytes from shuffled archetype tables; context B is fed the bytes the
    tables imply through b200vis_upload_shadow_casters.  Mesh rows get archetype-consistent flags (Aabb, the table's
    bits, their InheritedVisibility), so a full read gives A the device state B was uploaded."""

    def __init__(self, seed):
        sc = scenes.forest(n_trees=40, levels=6, n_lights=16, seed=seed)
        sc.trs[sc.roots, 0:3] *= np.float32(0.12)              # the trees inside the lights' reach
        sc.light_range[:] = 45.0
        sc.bounds[sc.light_row, 3] = 45.0
        self.rng = rng = np.random.default_rng(seed)
        lights = set(int(r) for r in sc.light_row)
        meshes = np.array([r for r in range(sc.n) if r not in lights], np.int64)
        pick = rng.integers(0, 10, len(meshes))
        table_of = np.full(sc.n, LIGHTS, np.int64)
        table_of[meshes] = np.where(pick < 5, CASTER, np.where(pick < 7, NOT_CASTER, np.where(pick < 8, NOCPU, OUTSIDE)))
        for t, bits in TABLE_FLAGS.items():
            r = np.nonzero(table_of == t)[0]
            sc.flags[r] = (sc.flags[r] & abi.F_INHERITED_VISIBLE) | abi.F_HAS_AABB | bits
        self.is_caster = np.array([1, 0, 0, 0, 1], np.uint8)     # OUTSIDE is never read: its byte must not matter
        self.upload = (rng.random(sc.n) < 0.5).astype(np.uint8)  # what upload_shadow_casters gave A's rows at the start
        self.upload[sc.light_row] = 0
        self.sc, self.table_of = sc, table_of
        self.a, self.b = bb.VisibilityPipeline(sc), bb.VisibilityPipeline(copy.deepcopy(sc))
        self.a.ctx.upload_shadow_casters(0, self.upload)
        self.model = self.upload.copy()
        groups = [np.nonzero(table_of == t)[0] for t in range(5)]
        caps = [len(g) + 64 for g in groups]
        self.tabs, self.tbuf = abi.host_tables(caps)             # len = capacity: the unmapped tail is skipped
        self.n = [len(g) for g in groups]
        self.maps = [np.full(c, NONE, np.uint32) for c in caps]
        self.culls, self.cbuf = abi.host_table_cull_inputs(caps)
        for t, c in enumerate(self.culls):
            c.has, c.flags = (("aabb", "iv"), TABLE_FLAGS[t]) if t in TABLE_FLAGS else ((), 0)
        self.a.ctx.set_tables(self.tabs)
        for t, g in enumerate(groups):
            self.maps[t][:len(g)] = rng.permutation(g).astype(np.uint32)
            self.a.ctx.set_table_rows(t, 0, self.maps[t][:len(g)])
            self.fill(t, np.arange(len(g)))
        self.attach_cull()
        self.attached = False
        self.items = None

    def fill(self, t, slots):
        """The cull columns of the slots hold their rows' true values, ticks 0 (never newer)."""
        c, sc = self.culls[t], self.sc
        slots = np.asarray(slots, np.int64)
        rows = self.maps[t][slots].astype(np.int64)
        b = sc.bounds[rows]
        CM.put(c.aabb, slots, ((abi.BEVY_BOUNDS_LAYOUT[1], b[:, 0:3]), (abi.BEVY_BOUNDS_LAYOUT[2], b[:, 3:6])))
        c.iv[slots] = sc.flags[rows] & abi.F_INHERITED_VISIBLE
        c.aabb_ticks[slots] = 0; c.iv_ticks[slots] = 0

    def realloc(self, t, capacity):
        """Table::reserve of table t: its output and cull columns move to new allocations (the contents below the old
        capacity copied), and the registry is sent again, which drops the cull inputs and the caster attachment."""
        old_tab, old_cull = self.tabs[t], self.culls[t]
        (new_tab,), tbuf = abi.host_tables([capacity])
        (new_cull,), cbuf = abi.host_table_cull_inputs([capacity])
        k = old_tab.capacity
        for name in ("aabb", "aabb_ticks", "sphere", "sphere_ticks", "iv", "iv_ticks"):
            getattr(new_cull, name)[:k] = getattr(old_cull, name)
        new_cull.has, new_cull.flags = old_cull.has, old_cull.flags
        self.tabs[t], self.culls[t] = new_tab, new_cull
        self.maps[t] = np.concatenate([self.maps[t], np.full(capacity - k, NONE, np.uint32)])
        self.a.ctx.set_tables(self.tabs)
        self.keep = getattr(self, "keep", []) + [tbuf, cbuf]    # the old buffers stay alive: the registry moved first
        assert new_tab.vv.ctypes.data != old_tab.vv.ctypes.data and new_cull.aabb.ctypes.data != old_cull.aabb.ctypes.data
        self.attached = False
        self.attach_cull()

    def attach_cull(self):
        self.a.ctx.set_table_cull_inputs([c if c.has else None for c in self.culls])

    def attach_casters(self, on=True):
        self.a.ctx.set_table_shadow_casters(self.is_caster if on else None)
        self.attached = on

    def move(self, src, s, dst):
        """An archetype move with swap_remove: the row of (src, s) to the end of dst, src's last row into s.  The
        remapped slots are read in full by the next cull read."""
        maps = self.maps
        row, last, d = int(maps[src][s]), self.n[src] - 1, self.n[dst]
        moved = int(maps[src][last])
        self.a.ctx.set_table_rows(dst, d, [row])
        if s != last:
            self.a.ctx.set_table_rows(src, s, [moved])
        self.a.ctx.set_table_rows(src, last, [NONE])
        maps[dst][d] = row
        maps[src][s] = moved if s != last else NONE
        maps[src][last] = NONE
        self.n[dst] += 1; self.n[src] -= 1
        self.fill(dst, [d])
        if s != last:
            self.fill(src, [s])
        self.table_of[row] = dst

    def frame(self, f):
        a, b, sc = self.a.ctx, self.b.ctx, self.sc
        a.read_tables(abi.RD_CULL_INPUTS, 0, 1)
        if self.attached:                                         # every mapped slot below len of a read table
            for t, tab in enumerate(self.tabs):
                if t in TABLE_FLAGS:
                    rows = self.maps[t]
                    self.model[rows[rows != NONE].astype(np.int64)] = self.is_caster[t]
        b.upload_shadow_casters(0, self.model)
        for p in (self.a, self.b):
            scenes.advance_cameras(p.scene, 0.1)
            p.update_views()
            p.run_frame()
        items = []
        for o in range(6):
            row = int(sc.light_row[o])
            gt, _ = a.download_global_transforms(row, 1, want_changed=False)
            fr = abi.host_point_light_frusta(gt[0], float(sc.light_range[o]))
            items.append(dict(kind=o % 2, light_row=row, range=float(sc.light_range[o]), frusta=fr if o % 2 == 0 else fr[o]))
        for c in (a, b):
            c.set_shadow_items(items)
            c.run_shadow_culling()
        n = 0
        for i in range(len(items)):
            for face in range(6 if i % 2 == 0 else 1):
                la, lb = a.download_shadow_visible(i, face), b.download_shadow_visible(i, face)
                assert len(la) == len(lb) and (la == lb).all(), f"frame {f}: item {i} face {face} differs"
                n += len(la)
        va, _ = a.download_view_visibility(0, sc.n)
        vb, _ = b.download_view_visibility(0, sc.n)
        assert (va == vb).all(), f"frame {f}: ViewVisibility differs"
        self.a.read_feedback(); self.b.read_feedback()
        return n

    def close(self):
        self.a.close(); self.b.close()


def case_table_casters_match_uploaded_bytes_through_moves_reattach_and_set_tables():
    tw = CasterTwins(7)
    c = tw.a.ctx
    try:
        lib = abi.load_library()
        assert lib.b200vis_set_table_shadow_casters(c._h, 4, tw.is_caster.ctypes.data) == INVALID_ARG
        assert lib.b200vis_set_table_shadow_casters(c._h, 5, None) == INVALID_ARG
        tw.attach_casters()
        seen = tw.frame(0)
        for f in range(1, 10):
            if f in (1, 2, 6):                                    # archetype moves into and out of the caster table
                for _ in range(12):
                    src, dst = (CASTER, NOT_CASTER) if tw.rng.random() < 0.5 else (NOT_CASTER, CASTER)
                    if tw.n[src] and tw.n[dst] < tw.tabs[dst].capacity:
                        tw.move(src, int(tw.rng.integers(0, tw.n[src])), dst)
            if f == 3:                                            # a table's caster bit changes: read in full
                tw.is_caster[NOT_CASTER] = 1
                tw.attach_casters()
            if f == 4:                                            # detached: moved rows keep their bytes
                tw.is_caster[NOT_CASTER] = 0
                tw.attach_casters(False)
                for _ in range(6):
                    tw.move(CASTER, int(tw.rng.integers(0, tw.n[CASTER])), NOT_CASTER)
            if f == 5:                                            # re-attached: every table read in full
                tw.attach_casters()
            if f == 7:                                            # a reallocation: set_tables drops the attachment
                tw.realloc(CASTER, tw.tabs[CASTER].capacity * 2)
                for _ in range(4):
                    tw.move(NOT_CASTER, int(tw.rng.integers(0, tw.n[NOT_CASTER])), CASTER)
            if f == 8:
                tw.attach_casters()
            seen += tw.frame(f)
        assert seen > 100
        # the bytes the tables gave differ from the initial upload somewhere that mattered
        assert (tw.model != tw.upload).any()
    finally:
        tw.close()


# ---- C: set_visible() of the light pass in the tables ------------------------------------------------------------


def case_light_set_visible_stamps_its_own_tick_in_the_tables():
    """Camera WB_SET_VISIBLE with tick a, the shadow stage, WB_SET_VISIBLE with tick b.  The rows the cameras list and
    the rows visible after the light passes come from the oracle (whose ViewVisibility the device's must equal).  Slots
    only lights see get bit 0 and tick b where bit 1 was clear; the forked twin's WB_VIEW_VISIBILITY bytes agree."""
    sc = scenes.forest(n_trees=80, levels=5, n_lights=6)
    sc.trs[sc.roots, 0:3] *= np.float32(0.12)                  # the trees inside the lights' reach
    sc.light_range[:] = 45.0
    sc.bounds[sc.light_row, 3] = 45.0
    sc.cameras = sc.cameras[:1]                                # most meshes outside the one camera's frustum
    caster = np.ones(sc.n, np.uint8); caster[sc.light_row] = 0
    groups = [np.arange(sc.n)[sc.n // 3:], np.arange(sc.n)[:sc.n // 3]]
    tw_sc = copy.deepcopy(sc)
    a, b = bb.VisibilityPipeline(sc), bb.VisibilityPipeline(tw_sc)
    world = OracleWorld(sc, True)
    try:
        for p in (a, b):
            p.ctx.upload_shadow_casters(0, caster)             # before the first CULL stage: the visible sets are kept
        T = Tables(a.ctx, groups, np.random.default_rng(3))
        U = Tables(b.ctx, groups, np.random.default_rng(3))
        for t in T.tabs + U.tabs:
            t.vv[:] = 0; t.vv_ticks[:] = 0
        for m in T.model + U.model:
            m["vv"][:] = 0; m["vv_ticks"][:] = 0
        light_only = 0
        points = np.arange(6)
        for f in range(5):
            ta, tb_, tm = 100 + 10 * f, 101 + 10 * f, 102 + 10 * f
            for t, tab in enumerate(T.tabs):                   # reset_view_visibility (CPU)
                svm.reset(tab.vv); svm.reset(T.model[t]["vv"])
            if f:
                scenes.advance_cameras(sc, 0.3); scenes.advance_cameras(tw_sc, 0.3)
            want, active, _ = oracle_frame(a, world, sc, caster, [], points, 0,
                                           between=lambda: a.ctx.writeback_tables(abi.WB_SET_VISIBLE, 0, ta))
            cams = set(np.concatenate(world.last_lists).tolist())
            b.update_views()
            items, _, _ = light_items(sc, world, [], points, 0)
            b.ctx.run(bb.STAGE_ALL)
            b.ctx.set_shadow_items(items)
            b.ctx.run_shadow_culling()
            a.ctx.writeback_tables(abi.WB_SET_VISIBLE, 0, tb_)
            b.ctx.writeback_tables(abi.WB_VIEW_VISIBILITY, 0, tm)
            a.ctx.synchronize(); b.ctx.synchronize()
            dev_vv, _ = a.ctx.download_view_visibility(0, sc.n)
            assert (dev_vv == world.vv).all(), f"frame {f}: device ViewVisibility differs from the oracle's"
            assert any(active)
            for t, tab in enumerate(T.tabs):
                rows = T.map[t][:tab.len].astype(np.int64)
                m = T.model[t]
                cam_slots = [s for s, r in enumerate(rows) if r in cams]
                svm.set_visible(m["vv"], m["vv_ticks"], cam_slots, ta)
                lit = [s for s, r in enumerate(rows) if world.vv[r] & 1]
                before = m["vv"].copy()
                svm.set_visible(m["vv"], m["vv_ticks"], lit, tb_)
                light_only += int(((before[lit] & 1) == 0).sum())
                assert (tab.vv == m["vv"]).all(), f"frame {f} table {t}: ViewVisibility bytes differ from the model"
                assert (tab.vv_ticks == m["vv_ticks"]).all(), f"frame {f} table {t}: ticks differ from the model"
                svm.mark_hidden(tab.vv, tab.vv_ticks, tm); svm.mark_hidden(m["vv"], m["vv_ticks"], tm)
                # the forked twin owns the 2-bit state: its bytes are what the CPU-owned ones end the frame as
                rows_u = U.map[t][:U.tabs[t].len].astype(np.int64)
                by_row = np.zeros(sc.n, np.int64); by_row[rows_u] = U.tabs[t].vv[:len(rows_u)]
                assert (by_row[rows] == tab.vv[:len(rows)]).all(), f"frame {f} table {t}: forked twin's bytes differ"
            a.read_feedback(); b.read_feedback()
        assert light_only > 0
    finally:
        a.close(); b.close()


# ---- A (continued): the sink across edits, compactions, re-topologies, many views and the full-size world ------------


def point_shadows(sc, rng, k=6):
    """k point lights with shadow maps (the scene's own shadow stage runs them through b200vis_set_shadow_lights)."""
    sc.shadow_lights = np.sort(rng.choice(len(sc.light_row), k, replace=False)).astype(np.uint32)
    sc.shadow_caster = (rng.random(sc.n) < 0.8).astype(np.uint8)
    sc.shadow_caster[sc.light_row] = 0
    sc.shadow_near_z, sc.shadow_lod_origin = 0.1, 0


def check_vs_rows(sink, ctx, n_items, bits, tag):
    """The sink after a synchronised frame against the context's own row lists (which the frame's compare_frame checked
    against the oracle) mapped through the entity bits; an inactive item's lists are empty."""
    ent, off, act, cap = sink.ent_buf, sink.off_buf, sink.act_buf, sink.cap
    assert (off[n_items * 6 + 1:] == OFF_SENTINEL).all() and (act[n_items:] == ACT_SENTINEL).all(), f"{tag}: past n_items"
    assert (ent[cap:] == ENT_SENTINEL).all(), f"{tag}: written past capacity"
    pos = 0
    for i in range(n_items):
        for face in range(6):
            rows = ctx.download_shadow_visible(i, face)
            assert off[i * 6 + face] == pos, f"{tag}: item {i} face {face} offset"
            assert act[i] in (0, 1) and (act[i] or not len(rows)), f"{tag}: item {i} inactive with entries"
            want = bits[rows]
            hi = min(pos + len(want), cap)
            assert (ent[min(pos, cap):hi] == want[:max(hi - pos, 0)]).all(), f"{tag}: item {i} face {face} entities"
            pos += len(rows)
    assert off[n_items * 6] == pos, f"{tag}: total"
    assert (ent[min(pos, cap):cap] == ENT_SENTINEL).all(), f"{tag}: entries past the true total"
    return pos


def case_sink_across_spawns_despawns_and_a_compacting_twin():
    """Edits that despawn and spawn (new keys merging into the ranks), device compactions that swap the key buffers, and
    a twin that never compacts: both sinks hold the same Entity values byte for byte, every frame."""
    from test_gpu_compaction import Twins, order_keeping_reparents

    def make():
        sc = _random_scene(21, n_roots=90, n_lights=20)
        point_shadows(sc, np.random.default_rng(21))
        return sc
    rng = np.random.default_rng(21)
    t = Twins(make, 3000, seed=21)
    try:
        n_items = len(t.b.sc.shadow_lights)
        sa, sb = (ShadowSink(x.pipe.ctx, 6 * (x.sc.n + 3000), n_items) for x in (t.a, t.b))
        seen = 0
        for f in range(9):
            if f:
                t.random_edit(n_despawn=6, n_flat=6, n_kids=3)
                if f % 3 == 0:
                    t.compact(*order_keeping_reparents(t, 2, rng))
            sa.reset(); sb.reset()
            t.frame(f, animate=f > 0)
            for x in (t.a, t.b):
                x.pipe.ctx.synchronize()
            seen += check_vs_rows(sa, t.a.pipe.ctx, n_items, t.a.sc.entity_bits, f"a frame {f}")
            check_vs_rows(sb, t.b.pipe.ctx, n_items, t.b.sc.entity_bits, f"b frame {f}")
            assert sa.ent_buf.tobytes() == sb.ent_buf.tobytes() and sa.off_buf.tobytes() == sb.off_buf.tobytes(), f"frame {f}"
            assert sa.act_buf.tobytes() == sb.act_buf.tobytes(), f"frame {f}"
        assert t.compactions and seen > 100
    finally:
        t.close()


def case_a_shadow_sink_registered_before_set_topology_reads_the_new_keys():
    """The sink first, then b200vis_set_topology (the re-topology fallback of a churned world, shuffled entity bits):
    the new world's keys are uploaded because the sink is set."""
    from test_gpu_topology_edits import Churn
    sc = _random_scene(12, n_roots=70, n_lights=16)
    point_shadows(sc, np.random.default_rng(12))
    ch = Churn(sc, 400, seed=12)
    try:
        n_items = len(sc.shadow_lights)
        sink = ShadowSink(ch.pipe.ctx, 6 * (sc.n + 400), n_items)
        seen = 0
        for f in range(6):
            if f:
                ch.random_edit(n_despawn=4, n_flat=4, n_kids=2)
                if f % 2 == 0:
                    ch.compact()                                  # set_topology with the sink registered
            sink.reset()
            ch.frame(f, animate=f > 0)
            ch.pipe.ctx.synchronize()
            seen += check_vs_rows(sink, ch.pipe.ctx, n_items, ch.sc.entity_bits, f"frame {f}")
        assert seen > 100
    finally:
        ch.close()


def case_sink_with_group_passes(n_views):
    """More than eight views (group passes decide which lights are in some view's VisibleEntities), and a truncated
    sink beside a full one on a twin."""
    from test_gpu_topology_edits import Churn
    sc = scenes.many_cameras_lights(n_cameras=n_views, forest_kwargs=dict(n_trees=40, levels=6, n_lights=16, seed=3))
    point_shadows(sc, np.random.default_rng(n_views), k=min(8, len(sc.light_row)))
    ch = Churn(sc, 200, seed=3)
    try:
        n_items = len(sc.shadow_lights)
        sink = ShadowSink(ch.pipe.ctx, 6 * sc.n, n_items)
        seen = 0
        for f in range(3):
            sink.reset()
            ch.frame(f, animate=f > 0)
            ch.pipe.ctx.synchronize()
            seen += check_vs_rows(sink, ch.pipe.ctx, n_items, sc.entity_bits, f"frame {f}")
        small = ShadowSink(ch.pipe.ctx, 9, n_items)              # replaces the sink: truncated, true offsets
        small.reset()
        ch.frame(3)
        ch.pipe.ctx.synchronize()
        assert check_vs_rows(small, ch.pipe.ctx, n_items, sc.entity_bits, "truncated") > 9
        assert seen > 0
    finally:
        ch.close()


def case_config3_full_size_one_frame():
    """The bench world (1,000,366 rows, 4 views) with 16 point lights, 8 spot lights and one directional light x 4 views
    x 4 cascades, one frame against the oracle."""
    sc = scenes.forest()
    assert sc.n == 1_000_366 and len(sc.cameras) == 4
    caster = np.ones(sc.n, np.uint8); caster[sc.light_row] = 0
    pipe = bb.VisibilityPipeline(sc)
    world = OracleWorld(sc, True)
    try:
        pipe.ctx.upload_shadow_casters(0, caster)
        n_items = 8 + 16 + 4 * 4
        sink = ShadowSink(pipe.ctx, 16 * sc.n, n_items)
        sink.reset()
        want, active, _ = oracle_frame(pipe, world, sc, caster, np.arange(8), np.arange(8, 24), 4, list_capacity=1,
                                       radii=(10.0, 30.0, 90.0, 270.0))
        assert len(active) == n_items
        pipe.ctx.synchronize()
        total = sink.check(want, active, sc.entity_bits, "config #3")
        assert total > 0 and sum(active[:24]) > 0
        vv, _ = pipe.ctx.download_view_visibility(0, sc.n)
        assert (vv == world.vv).all(), "ViewVisibility differs"
    finally:
        pipe.close()


# ---- every case runs in a fresh interpreter: the cases register and release many host buffers, and what they leave on
# the heap would decide whether a later test file's pageable arrays share a page with that file's registrations ----

def _fresh(call, **env):
    run_case(f"import test_gpu_shadow_outputs as m\nm.{call}", dict(env, **{k: os.environ[k] for k in ("B200VIS_LIB",) if k in os.environ}),
             timeout=600)


@pytest.mark.parametrize("seed,shuffle,pipeline", [(21, True, "1"), (22, False, "1"), (23, True, "0")])
def test_sink_matches_the_oracle_every_frame(seed, shuffle, pipeline):
    _fresh(f"case_sink_matches_the_oracle_every_frame({seed!r}, {shuffle!r}, {pipeline!r})", B200VIS_PIPELINE=pipeline)


def test_truncation_list_capacity_one_and_launch_counts():
    _fresh(f"case_truncation_list_capacity_one_and_launch_counts()")


def test_sink_errors_and_removal():
    _fresh(f"case_sink_errors_and_removal()")


def test_table_casters_match_uploaded_bytes_through_moves_reattach_and_set_tables():
    _fresh(f"case_table_casters_match_uploaded_bytes_through_moves_reattach_and_set_tables()")


def test_light_set_visible_stamps_its_own_tick_in_the_tables():
    _fresh(f"case_light_set_visible_stamps_its_own_tick_in_the_tables()")


def test_sink_across_spawns_despawns_and_a_compacting_twin():
    _fresh(f"case_sink_across_spawns_despawns_and_a_compacting_twin()")


def test_a_shadow_sink_registered_before_set_topology_reads_the_new_keys():
    _fresh(f"case_a_shadow_sink_registered_before_set_topology_reads_the_new_keys()")


@pytest.mark.parametrize("n_views", [9, 32])
def test_sink_with_group_passes(n_views):
    _fresh(f"case_sink_with_group_passes({n_views!r})")


def test_config3_full_size_one_frame():
    _fresh(f"case_config3_full_size_one_frame()")
