"""The cull system's outputs written by the device straight into the caller's memory:

A. b200vis_set_visible_entities_sink: VisibleEntities as one sorted Entity list per VisibilityClass, checked every frame
   against the oracle's split of the view's visible list (orc_visible_entities_by_class) mapped through the entity bits,
   over edits, compactions, many views, truncation and every frame path.
B. B200VIS_WB_SET_VISIBLE: set_visible() into shuffled archetype tables over plain numpy memory, between a numpy
   reset_view_visibility and mark_newly_hidden_entities_invisible (tests/set_visible_model.py), checked against that
   model, the oracle's ViewVisibility and a twin context that writes the device-owned bytes with WB_VIEW_VISIBILITY."""
import copy
import ctypes

import numpy as np
import pytest

import bevy_b200 as bb
import oracle as orc
import set_visible_model as svm
from bevy_b200 import abi, scenes
from test_gpu_compaction import Twins, order_keeping_reparents, renumber
from test_gpu_table_writeback import NONE, Tables, follow_archetypes, split
from test_gpu_topology_edits import Churn

pytestmark = pytest.mark.gpu

INVALID_ARG = 1
ENT_SENTINEL, OFF_SENTINEL = np.uint64(0xA5A5A5A5A5A5A5A5), np.uint32(0xC3C3C3C3)


def pinned(shape, dtype, fill):
    """A numpy array over pinned host memory (torch's allocator), which the library uses through its device alias."""
    torch = pytest.importorskip("torch")
    tdt = {np.dtype(np.uint64): torch.int64, np.dtype(np.uint32): torch.int32}[np.dtype(dtype)]
    a = torch.zeros(shape, dtype=tdt).pin_memory().numpy().view(dtype)
    a[...] = fill
    return a


class EntitySink:
    """A sentinel-filled entity sink of `capacity` entries per view, with a guard past the last view's region."""

    def __init__(self, ctx, capacity, guard=64):
        V = ctx.max_views
        self.ctx, self.cap, self.V = ctx, capacity, V
        self.buf = pinned((V * capacity + guard,), np.uint64, ENT_SENTINEL)
        self.ent = self.buf[:V * capacity].reshape(V, capacity)
        self.off = pinned((V, 9), np.uint32, OFF_SENTINEL)
        ctx.set_visible_entities_sink(self.ent, self.off)

    def snapshot(self):
        return self.ent.copy(), self.off.copy()

    def check(self, sc, active, before, tag):
        """The sink after a synchronised frame; `before` = the snapshot taken before it (inactive views must keep it)."""
        assert (self.buf[self.V * self.cap:] == ENT_SENTINEL).all(), f"{tag}: written past the last view's region"
        for v in range(self.V):
            if v >= len(active) or not active[v]:
                assert (self.ent[v] == before[0][v]).all() and (self.off[v] == before[1][v]).all(), f"{tag}: view {v} touched"
                continue
            rows = self.ctx.download_visible(v)
            by = orc.visible_entities_by_class(rows, sc.class_mask, sc.entity_bits)
            want = [sc.entity_bits[by[k]] if k in by else np.zeros(0, np.uint64) for k in range(8)]
            tot = np.concatenate([[0], np.cumsum([len(w) for w in want])]).astype(np.uint32)
            assert (self.off[v] == tot).all(), f"{tag}: view {v} offsets {self.off[v]} vs {tot}"
            flat = np.concatenate(want)
            n = min(len(flat), self.cap)
            assert (self.ent[v, :n] == flat[:n]).all(), f"{tag}: view {v} entities differ"
            for k in range(8):
                seg = self.ent[v, min(tot[k], self.cap):min(tot[k + 1], self.cap)]
                assert (seg[1:] > seg[:-1]).all(), f"{tag}: view {v} class {k} not strictly ascending"


def mixed_classes(sc, rng):
    """Classless rows, single-class rows and rows in several of the eight classes."""
    pick = rng.integers(0, 4, sc.n)
    cls = np.where(pick == 0, 0, np.where(pick == 1, 1 << rng.integers(0, 8, sc.n), rng.integers(1, 256, sc.n)))
    sc.class_mask = cls.astype(np.uint8)


def shuffled_bits(sc, rng):
    """Odd entity bits in an order unrelated to the rows (non-identity ranks); spawns take even bits below them."""
    sc.entity_bits = (rng.permutation(sc.n).astype(np.uint64) * np.uint64(2) + np.uint64(1001))


def even_bits(ch):
    state = {"next": 2}

    def new_bits(k):
        out = np.arange(state["next"], state["next"] + 2 * k, 2, dtype=np.uint64)
        state["next"] += 2 * k
        return out
    ch.new_bits = new_bits


def active_of(sc):
    return [True] * len(sc.cameras) if sc.view_flags is None else [bool(f & abi.VIEW_ACTIVE) for f in sc.view_flags]


def test_entity_lists_over_edits_with_rank_merges_and_an_inactive_view():
    rng = np.random.default_rng(5)
    sc = scenes.forest(60, 8, 24, seed=5)
    mixed_classes(sc, rng)
    shuffled_bits(sc, rng)
    sc.view_flags = np.full(len(sc.cameras), abi.VIEW_ACTIVE, np.uint8)
    ch = Churn(sc, 4000, seed=5)
    even_bits(ch)
    try:
        ch.frame(0, animate=False)
        sink = EntitySink(ch.pipe.ctx, sc.n + 4000)             # registered after a frame: the keys are uploaded now
        for f in range(1, 10):
            ch.random_edit(n_despawn=6, n_flat=6, n_kids=3)      # despawns of visible rows, spawns ranking first
            if f == 4:
                sc.view_flags[1] = 0
            if f == 7:
                sc.view_flags[1] = abi.VIEW_ACTIVE
            before = sink.snapshot()
            ch.frame(f)
            sink.check(sc, active_of(sc), before, f"frame {f}")
    finally:
        ch.close()


def test_a_compacting_twin_writes_byte_identical_entity_sinks():
    rng = np.random.default_rng(9)

    def make():
        sc = scenes.forest(60, 8, 24, seed=9)
        mixed_classes(sc, np.random.default_rng(9))
        return sc
    t = Twins(make, 4000, seed=9)
    try:
        sa, sb = EntitySink(t.a.pipe.ctx, t.a.sc.n + 4000), EntitySink(t.b.pipe.ctx, t.b.sc.n + 4000)
        t.frame(0, animate=False)
        for f in range(1, 9):
            t.random_edit()
            if f % 3 == 0:
                t.compact(*order_keeping_reparents(t, 2, rng))
            before = sa.snapshot()
            t.frame(f)
            sa.check(t.a.sc, active_of(t.a.sc), before, f"a frame {f}")
            assert sa.ent.tobytes() == sb.ent.tobytes() and sa.off.tobytes() == sb.off.tobytes(), f"frame {f}"
        assert t.compactions
    finally:
        t.close()


@pytest.mark.parametrize("n_views", [9, 32])
def test_group_passes_and_a_capacity_below_the_total(n_views):
    rng = np.random.default_rng(n_views)
    sc = scenes.many_cameras_lights(n_cameras=n_views, forest_kwargs=dict(n_trees=40, levels=6, n_lights=16, seed=3))
    mixed_classes(sc, rng)
    sc.view_flags = np.full(n_views, abi.VIEW_ACTIVE, np.uint8)
    sc.view_flags[n_views - 2] = 0
    ch = Churn(sc, 200, seed=3)
    try:
        sink = EntitySink(ch.pipe.ctx, 7)                         # truncated: true offsets, nothing past 7 entries
        for f in range(3):
            before = sink.snapshot()
            ch.frame(f, animate=f > 0)
            sink.check(sc, active_of(sc), before, f"frame {f}")
            assert (sink.off[:, 8][np.array(active_of(sc))] > 7).any()
    finally:
        ch.close()


def test_pipelining_off_and_step(monkeypatch):
    monkeypatch.setenv("B200VIS_PIPELINE", "0")
    rng = np.random.default_rng(2)
    sc = scenes.forest(50, 6, 12, seed=2)
    mixed_classes(sc, rng)
    shuffled_bits(sc, rng)
    ch = Churn(sc, 100, seed=2)
    try:
        sink = EntitySink(ch.pipe.ctx, sc.n + 100)
        for f in range(3):
            before = sink.snapshot()
            ch.frame(f, animate=f > 0)
            sink.check(sc, active_of(sc), before, f"serial frame {f}")
        c, V = ch.pipe.ctx, len(sc.cameras)
        for f in range(3, 6):                                     # b200vis_step, which waits for its frame
            scenes.advance_cameras(sc, 0.05)
            rows, trs = scenes.mutate_roots(sc, f)
            arr = (bb.CameraDesc * V)()
            for v, cam in enumerate(sc.cameras):
                arr[v].global_transform[:] = cam.gt.tolist()
                arr[v].fov_y, arr[v].aspect, arr[v].near_z, arr[v].far_z = cam.fov, cam.aspect, cam.near, cam.far
                arr[v].layer_mask, arr[v].flags, arr[v].range_view_index = 1, bb.VIEW_ACTIVE, -1
            r, t_ = np.ascontiguousarray(rows, np.uint32), np.ascontiguousarray(trs, np.float32)
            before = sink.snapshot()
            c.step(len(r), r.ctypes.data, t_.ctypes.data, arr, V, ch.pipe.cluster_config, wait=True)
            sink.check(sc, active_of(sc), before, f"step {f}")
    finally:
        ch.close()


def test_config3_full_size_one_frame():
    sc = scenes.forest()                                          # 1,000,366 rows, 4 views
    assert sc.n == 1_000_366 and len(sc.cameras) == 4
    ch = Churn(sc, 0, seed=0, visible_diff=False)
    try:
        sink = EntitySink(ch.pipe.ctx, sc.n)
        before = sink.snapshot()
        ch.frame(0, animate=False)
        sink.check(sc, active_of(sc), before, "config #3")
        assert sink.off[:, 8].sum() > 0
    finally:
        ch.close()


def test_entity_sink_errors_and_removal():
    sc = scenes.forest(10, 4, 2, seed=1)
    pipe = bb.VisibilityPipeline(sc)
    c = pipe.ctx
    try:
        V = c.max_views
        ent, off = pinned((V, 16), np.uint64, 0), pinned((V, 9), np.uint32, 0)
        lib = abi.load_library()
        for bad in (abi.VisibleEntitiesSink(ent.ctypes.data, 0, off.ctypes.data),
                    abi.VisibleEntitiesSink(None, 16, off.ctypes.data),
                    abi.VisibleEntitiesSink(ent.ctypes.data, 16, None),
                    abi.VisibleEntitiesSink(ent.ctypes.data + 4, 16, off.ctypes.data)):
            assert lib.b200vis_set_visible_entities_sink(c._h, ctypes.byref(bad)) == INVALID_ARG
        c.set_visible_entities_sink(ent, off)
        c.set_visible_entities_sink(None, None)                   # removed: the next frame writes nothing
        pipe.run_frame(); c.synchronize()
        assert (ent == 0).all() and (off == 0).all()
    finally:
        pipe.close()


# ---- B: set_visible into the tables --------------------------------------------------------------------------------


def cpu_side(T, sc, fn, *args):
    """A CPU system over every mapped slot below len (rows Without<NoCpuCulling>), on the tables and on their model."""
    for t, tab in enumerate(T.tabs):
        rows = T.map[t][:tab.len]
        s = np.nonzero(rows != NONE)[0]
        s = s[(sc.flags[rows[s].astype(np.int64)] & abi.F_NO_CPU_CULLING) == 0]
        for vv, ticks in ((tab.vv, tab.vv_ticks), (T.model[t]["vv"], T.model[t]["vv_ticks"])):
            sub_vv, sub_t = vv[s], ticks[s]
            fn(sub_vv, sub_t, *args)
            vv[s], ticks[s] = sub_vv, sub_t


def test_set_visible_matches_the_model_the_oracle_and_the_forked_twin():
    seed = 13
    sc = scenes.forest(60, 6, 24, seed=seed)
    ch = Churn(sc, 600, seed=seed, visible_diff=False)            # unforked: the CPU owns the 2-bit state
    tw = Churn(copy.deepcopy(sc), 600, seed=seed, visible_diff=False)   # forked: WB_VIEW_VISIBILITY
    T = Tables(ch.pipe.ctx, split(sc), np.random.default_rng(seed))
    U = Tables(tw.pipe.ctx, split(tw.sc), np.random.default_rng(seed))
    rng = np.random.default_rng(seed + 1)
    c = ch.pipe.ctx
    pre_stamped = 0
    try:
        for f in range(10):
            if f in (3, 6):                                       # an edit: the tables follow the archetypes
                t_state = copy.deepcopy(ch.rng.bit_generator.state)
                ch.random_edit(n_despawn=4, n_flat=4, n_kids=2)
                tw.rng.bit_generator.state = t_state
                tw.random_edit(n_despawn=4, n_flat=4, n_kids=2)
                follow_archetypes(ch, T); follow_archetypes(tw, U)
            if f == 4:                                            # a reallocated table
                T.realloc(1, 2 * T.tabs[1].capacity); U.realloc(1, 2 * U.tabs[1].capacity)
            if f == 8:                                            # a compaction: the library renumbers its maps itself
                for churn, tabs in ((ch, T), (tw, U)):
                    o2n = churn.pipe.ctx.compact_topology([], []).astype(np.int64)
                    renumber(churn, o2n)
                    for m in tabs.map:
                        live = m != NONE
                        m[live] = o2n[m[live]]
            tick = 1000 + 10 * f
            cpu_side(T, ch.sc, lambda vv, t: svm.reset(vv))
            ch.frame(f, animate=f > 0)
            tw.frame(f, animate=f > 0)
            vis = ch.world.vv & 1                                 # the device's bit 0 (== the oracle's)
            # another CheckVisibility system (an earlier this_run) marks some visible rows first: the device must read
            # their bit 0 and neither write them again nor stamp its own tick over the other system's
            pre = []
            for t, tab in enumerate(T.tabs):
                rows = T.map[t][:tab.len]
                s = np.nonzero((rows != NONE) & (vis[np.minimum(rows, len(vis) - 1).astype(np.int64)] == 1))[0]
                pre.append(s[rng.random(len(s)) < 0.3])
            stamped = []
            for t, s in enumerate(pre):
                stamped.append(s[(T.tabs[t].vv[s] & 3) == 0])     # hidden last frame: the other system stamps tick - 1
                for vv, ticks in ((T.tabs[t].vv, T.tabs[t].vv_ticks), (T.model[t]["vv"], T.model[t]["vv_ticks"])):
                    svm.set_visible(vv, ticks, s, tick - 1)
            pre_stamped += sum(len(s) for s in stamped)
            if f == 2:                                            # refused, nothing written
                snap = [tab.vv.copy() for tab in T.tabs]
                with pytest.raises(abi.B200VisError):
                    c.writeback_tables(abi.WB_SET_VISIBLE | abi.WB_VIEW_VISIBILITY, 0, tick)
                c.synchronize()
                assert all((a == tab.vv).all() for a, tab in zip(snap, T.tabs))
            c.writeback_tables(abi.WB_SET_VISIBLE, 0, tick)
            for t, tab in enumerate(T.tabs):                      # the model of the device step
                rows = T.map[t][:tab.len]
                s = np.nonzero(rows != NONE)[0]
                s = s[vis[rows[s].astype(np.int64)] == 1]
                svm.set_visible(T.model[t]["vv"], T.model[t]["vv_ticks"], s, tick)
            c.synchronize()
            cpu_side(T, ch.sc, svm.mark_hidden, tick)
            T.check(f"frame {f}")
            for t, s in enumerate(stamped):
                assert (T.tabs[t].vv_ticks[s] == tick - 1).all(), f"frame {f} table {t}: a slot set by another system was ticked again"
            U.ctx.writeback_tables(abi.WB_VIEW_VISIBILITY, 0, tick)
            U.ctx.synchronize()
            for t, (a, b) in enumerate(zip(T.tabs, U.tabs)):
                rows = T.map[t][:a.len]
                s = np.nonzero(rows != NONE)[0]
                bad = s[a.vv[s] != ch.world.vv[rows[s].astype(np.int64)]]
                assert len(bad) == 0, (f"frame {f} table {t}: oracle bytes differ at slots {bad[:6]} rows {rows[bad[:6]]}: "
                                       f"{a.vv[bad[:6]]} vs {ch.world.vv[rows[bad[:6]].astype(np.int64)]}, len {a.len}, "
                                       f"flags {ch.sc.flags[rows[bad[:6]].astype(np.int64)]}, n {ch.sc.n}")
                assert (a.vv[:a.len] == b.vv[:b.len]).all(), f"frame {f} table {t}: bytes differ from the forked twin"
                # the same ticks, except where the other system stamped first (one tick earlier than the twin's)
                d = a.vv_ticks[:a.len] != b.vv_ticks[:b.len]
                assert (a.vv_ticks[:a.len][d] == b.vv_ticks[:b.len][d] - 1).all(), f"frame {f} table {t}: ticks differ from the forked twin"
        assert pre_stamped > 0
        # WB_VIEW_VISIBILITY after WB_SET_VISIBLE sends every byte again.  A first WB_VIEW_VISIBILITY makes the shadow hold
        # the device bytes; only the WB_SET_VISIBLE in between can make the last call rewrite the bytes overwritten here
        def device_bytes_in_tables(tag):
            for t, tab in enumerate(T.tabs):
                rows = T.map[t][:tab.len]
                s = np.nonzero(rows != NONE)[0]
                assert (tab.vv[s] == ch.world.vv[rows[s].astype(np.int64)]).all(), f"table {t}: {tag}"
        c.writeback_tables(abi.WB_VIEW_VISIBILITY, 0, 5)
        c.synchronize()
        device_bytes_in_tables("bytes after the first WB_VIEW_VISIBILITY")
        c.writeback_tables(abi.WB_SET_VISIBLE, 0, 6)
        c.synchronize()
        for tab in T.tabs:
            tab.vv[:tab.len] = 0x7E
        c.writeback_tables(abi.WB_VIEW_VISIBILITY, 0, 7)
        c.synchronize()
        device_bytes_in_tables("bytes after WB_SET_VISIBLE then WB_VIEW_VISIBILITY")
    finally:
        ch.close(); tw.close()


def test_set_visible_with_null_columns_and_slots_past_len():
    sc = scenes.forest(40, 6, 8, seed=4)
    ch = Churn(sc, 100, seed=4, visible_diff=False)
    try:
        c = ch.pipe.ctx
        groups = split(sc)
        tabs, buf = abi.host_tables([len(g) + 16 for g in groups], [len(g) for g in groups], vv_fill=0, tick_fill=7)
        descs = [t.desc() for t in tabs]
        descs[0] = tabs[0].desc(("gt", "gt_ticks", "vv"))         # no ViewVisibility tick column
        descs[1] = tabs[1].desc(("gt", "gt_ticks", "vv_ticks"))   # no ViewVisibility column: skipped
        rng = np.random.default_rng(4)
        maps = []
        for t, g in enumerate(groups):
            m = np.full(tabs[t].capacity, NONE, np.uint32)
            m[:len(g)] = rng.permutation(np.asarray(g, np.uint32))
            maps.append(m)
        maps[2][[3, 40]] = NONE                                   # unmapped slots in the middle of a table: never written
        arr = (abi.Table * len(descs))(*descs)
        assert abi.load_library().b200vis_set_tables(c._h, len(descs), arr) == 0
        for t, g in enumerate(groups):
            c.set_table_rows(t, 0, maps[t][:len(g)])
        # two slots past len are mapped (the rows moved there stay mapped but are never written)
        last = tabs[2].len
        tabs[2].len -= 2
        arr[2] = tabs[2].desc()
        assert abi.load_library().b200vis_set_tables(c._h, len(descs), arr) == 0
        before = [(t.vv.copy(), t.vv_ticks.copy()) for t in tabs]
        ch.frame(0, animate=False)
        c.writeback_tables(abi.WB_SET_VISIBLE, 0, 99)
        c.synchronize()
        vis = ch.world.vv & 1
        for t, tab in enumerate(tabs):
            vv0, tk0 = before[t]
            want_vv, want_tk = vv0.copy(), tk0.copy()
            if t != 1:
                rows = maps[t][:tab.len]
                s = np.nonzero(rows != NONE)[0]
                s = s[vis[rows[s].astype(np.int64)] == 1]
                svm.set_visible(want_vv, None if t == 0 else want_tk, s, 99)
            assert (tab.vv == want_vv).all() and (tab.vv_ticks == want_tk).all(), f"table {t}"
            assert np.isnan(tab.gt).all() and (tab.gt_ticks == 7).all(), f"table {t}: GlobalTransform touched"
        assert (tabs[2].vv[tabs[2].len:last] == 0).all()
        assert vis.any()
        del buf
    finally:
        ch.close()


@pytest.mark.parametrize("offset", [1, 7, 15])
def test_set_visible_on_view_visibility_columns_at_a_byte_offset(offset):
    """A u8 column may start anywhere: each chunk's bytes are staged from the 16-byte boundary below it (up to nine
    pieces), and only the chunk's own slots are written."""
    sc = scenes.forest(40, 6, 8, seed=6)
    ch = Churn(sc, 100, seed=6, visible_diff=False)
    try:
        c = ch.pipe.ctx
        groups = [g for g in split(sc) if len(g)]
        tabs, buf = abi.host_tables([len(g) + 16 for g in groups], [len(g) for g in groups], vv_fill=0, tick_fill=7)
        rng = np.random.default_rng(offset)
        vvs, descs, maps = [], [], []
        for t, g in enumerate(groups):
            tab = tabs[t]
            vv = tab.vv[offset:offset + len(g)]                   # the column starts `offset` bytes into the buffer
            vv[:] = rng.integers(0, 4, len(g)) << 1               # what reset_view_visibility left: bit 1 only
            tab.vv[:offset] = 0xA0                                # guards before and after the column
            tab.vv[offset + len(g):] = 0xA0
            vvs.append(vv)
            descs.append(abi.Table(tab.gt.ctypes.data, tab.gt_ticks.ctypes.data, vv.ctypes.data, tab.vv_ticks.ctypes.data,
                                   len(g), len(g)))
            maps.append(rng.permutation(np.asarray(g, np.uint32)))
        arr = (abi.Table * len(descs))(*descs)
        assert abi.load_library().b200vis_set_tables(c._h, len(descs), arr) == 0
        for t, m in enumerate(maps):
            c.set_table_rows(t, 0, m)
        before = [(t.vv.copy(), t.vv_ticks.copy()) for t in tabs]
        ch.frame(0, animate=False)
        c.writeback_tables(abi.WB_SET_VISIBLE, 0, 99)
        c.synchronize()
        vis = ch.world.vv & 1
        assert vis.any() and max(len(g) for g in groups) > 128
        for t, tab in enumerate(tabs):
            want_vv, want_tk = before[t][0].copy(), before[t][1].copy()
            s = np.nonzero(vis[maps[t].astype(np.int64)] == 1)[0]
            col = want_vv[offset:offset + len(groups[t])]
            svm.set_visible(col, want_tk, s, 99)
            assert (tab.vv == want_vv).all() and (tab.vv_ticks == want_tk).all(), f"table {t}, offset {offset}"
        del buf
    finally:
        ch.close()


def test_a_sink_registered_before_set_topology_reads_the_new_keys():
    """The shim's order: the sink first, then b200vis_set_topology (here the re-topology fallback of a churned world),
    which uploads the new world's keys because the sink is set."""
    rng = np.random.default_rng(12)
    sc = scenes.forest(50, 6, 12, seed=12)
    mixed_classes(sc, rng)
    shuffled_bits(sc, rng)
    ch = Churn(sc, 400, seed=12)
    even_bits(ch)
    try:
        sink = EntitySink(ch.pipe.ctx, sc.n + 400)
        ch.frame(0, animate=False)
        sink.check(sc, active_of(sc), sink.snapshot(), "frame 0")
        for f in range(1, 5):
            ch.random_edit(n_despawn=4, n_flat=4, n_kids=2)
            if f % 2 == 0:
                ch.compact()                                      # set_topology with the sink registered
            before = sink.snapshot()
            ch.frame(f)
            sink.check(sc, active_of(sc), before, f"frame {f}")
    finally:
        ch.close()
