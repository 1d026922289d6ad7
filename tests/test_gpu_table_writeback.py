"""b200vis_set_tables / b200vis_set_table_rows / b200vis_writeback_tables: the GPU writes GlobalTransform, ViewVisibility
and both change ticks straight into archetype tables in their own slot order, checked against the CPU oracle every frame
and read back only through the tables.

A forest plus lights is split into Bevy's archetypes (roots, inner nodes, leaves, lights, and flat rows spawned later),
each table in a shuffled slot order, over plain numpy memory that is not pinned, the small tables sharing pages.  A model
of every column -- sentinel-filled at the start -- says what each slot must hold after each write-back: the row's
GlobalTransform and tick where the oracle's Changed flag is set, the row's ViewVisibility, its tick where
Changed<ViewVisibility> fires, and the old bytes everywhere else (unmapped slots and slots at or past len included).
Archetype moves are Bevy's: the component bytes travel with the row, the table swap_removes the hole."""
import numpy as np
import pytest

from bevy_b200 import abi, scenes
from test_gpu_compaction import renumber
from test_gpu_topology_edits import Churn

pytestmark = pytest.mark.gpu

NONE = abi.UNMAPPED
INVALID_ARG, CAPACITY, NOT_READY, UNSUPPORTED = 1, 6, 7, 8
TICK_SENTINEL, VV_SENTINEL = 0xDEAD0001, 0xEE
ROOTS, INNER, LEAVES, LIGHTS, FLAT = range(5)
IDENTITY12 = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], np.float32)


def affine3a(gt12):
    """[n, 12] x_axis, y_axis, z_axis, translation -> [n, 16] glam Affine3A (Vec3A lanes, padding 0)."""
    gt12 = np.asarray(gt12, np.float32).reshape(-1, 12)
    out = np.zeros((len(gt12), 16), np.float32)
    for k in range(4):
        out[:, 4 * k:4 * k + 3] = gt12[:, 3 * k:3 * k + 3]
    return out


COLUMNS = ("gt", "gt_ticks", "vv", "vv_ticks")


def raw(tab, name):
    a = getattr(tab, name)
    return a.view(np.uint32) if name == "gt" else a


class Tables:
    """The caller's archetype tables, their slot -> row maps and a model of every column."""

    def __init__(self, ctx, groups, rng, headroom=8):
        self.ctx, self.rng = ctx, rng
        caps = [len(g) + headroom for g in groups]
        self.tabs, buf = abi.host_tables(caps, [len(g) for g in groups], tick_fill=TICK_SENTINEL, vv_fill=VV_SENTINEL)
        self.bufs = {None: buf}
        self.map = [np.full(c, NONE, np.uint32) for c in caps]
        self.model = [{k: raw(t, k).copy() for k in COLUMNS} for t in self.tabs]
        ctx.set_tables(self.tabs)
        for t, g in enumerate(groups):
            self.map[t][:len(g)] = rng.permutation(np.asarray(g, np.uint32))     # slot order shuffled against rows
            ctx.set_table_rows(t, 0, self.map[t][:len(g)])

    def locate(self, r):
        for t, tab in enumerate(self.tabs):
            s = np.nonzero(self.map[t][:tab.len] == r)[0]
            if len(s):
                return t, int(s[0])
        return None

    def copy_slot(self, ta, sa, tb, sb):
        for k in COLUMNS:
            raw(self.tabs[tb], k)[sb] = raw(self.tabs[ta], k)[sa]
            self.model[tb][k][sb] = self.model[ta][k][sa]

    def realloc(self, t, capacity):
        """Table::reserve: the columns move to a new allocation (old contents copied, the rest uninitialised)."""
        old = self.tabs[t]
        (new,), buf = abi.host_tables([capacity], [old.len], tick_fill=TICK_SENTINEL, vv_fill=VV_SENTINEL)
        for k in COLUMNS:
            raw(new, k)[:old.capacity] = raw(old, k)
            fresh = raw(new, k).copy()
            fresh[:old.capacity] = self.model[t][k]
            self.model[t][k] = fresh
        self.map[t] = np.concatenate([self.map[t], np.full(capacity - old.capacity, NONE, np.uint32)])
        self.tabs[t] = new
        self.ctx.set_tables(self.tabs)
        self.bufs[t] = buf                                 # the old allocation is released after the registry moved
        assert new.gt.ctypes.data != old.gt.ctypes.data

    def swap_remove(self, t, s):
        tab = self.tabs[t]
        last = tab.len - 1
        if s != last:
            self.copy_slot(t, last, t, s)
            self.map[t][s] = self.map[t][last]
            self.ctx.set_table_rows(t, s, [self.map[t][s]])   # the last row moves into the hole
        self.map[t][last] = NONE
        tab.len -= 1

    def append(self, r, t, src=None):
        tab = self.tabs[t]
        if tab.len == tab.capacity:
            self.realloc(t, 2 * tab.capacity)
            tab = self.tabs[t]
        d = tab.len
        if src is None:                                    # a spawn: GlobalTransform::IDENTITY, ViewVisibility::HIDDEN, tick 0
            for k, v in (("gt", affine3a(IDENTITY12)[0].view(np.uint32)), ("gt_ticks", 0), ("vv", 0), ("vv_ticks", 0)):
                raw(tab, k)[d] = v
                self.model[t][k][d] = v
        else:
            self.copy_slot(src[0], src[1], t, d)
        self.map[t][d] = r
        tab.len += 1
        self.ctx.set_table_rows(t, d, [r])                 # also removes r's old mapping

    def move(self, r, t):
        """An archetype move: r's bytes go to the end of table t, its old table swap_removes the hole."""
        a, s = self.locate(r)
        self.append(r, t, src=(a, s))
        self.swap_remove(a, s)

    def sync(self):
        self.ctx.set_tables(self.tabs)                     # the lens changed

    def expect(self, gt12, gch, vv, vch, which, gt_tick, vv_tick):
        for t, tab in enumerate(self.tabs):
            m = self.model[t]
            rows = self.map[t][:tab.len]
            s = np.nonzero(rows != NONE)[0]
            r = rows[s].astype(np.int64)
            if which & abi.WB_GLOBAL_TRANSFORM:
                c = gch[r] != 0
                m["gt"][s[c]] = affine3a(gt12[r[c]]).view(np.uint32)
                m["gt_ticks"][s[c]] = gt_tick
            if which & abi.WB_VIEW_VISIBILITY:
                m["vv"][s] = vv[r]
                m["vv_ticks"][s[vch[r] != 0]] = vv_tick

    def check(self, tag):
        for t, tab in enumerate(self.tabs):
            for k in COLUMNS:
                got, want = raw(tab, k), self.model[t][k]
                bad = np.nonzero((got != want).reshape(len(got), -1).any(1))[0]
                assert len(bad) == 0, (f"{tag}: table {t} column {k} differs at slots {bad[:6]} (len {tab.len}, rows "
                                       f"{self.map[t][bad[:6]]})")


def archetype(sc, r, kids):
    if r in set(sc.light_row.tolist()):
        return LIGHTS
    has_parent = sc.parent[r] < sc.n
    return (INNER if has_parent else ROOTS) if kids[r] else (LEAVES if has_parent else FLAT)


def children(sc, alive):
    kids = np.zeros(sc.n, np.int64)
    real = (sc.parent < sc.n) & alive
    np.add.at(kids, sc.parent[real].astype(np.int64), 1)
    return kids


def split(sc):
    kids = children(sc, np.ones(sc.n, bool))
    groups = [[] for _ in range(5)]
    for r in range(sc.n):
        groups[archetype(sc, r, kids)].append(r)
    return groups


def follow_archetypes(ch, T):
    """After an edit: despawned rows leave their tables, spawned rows join, rows whose archetype changed move."""
    sc = ch.sc
    kids = children(sc, ch.alive)
    lights = set(sc.light_row.tolist())
    for r in range(sc.n):
        at = T.locate(r)
        if not ch.alive[r]:
            if at is not None:
                T.swap_remove(*at)                         # the library unmapped the row when it was despawned
            continue
        want = LIGHTS if r in lights else archetype(sc, r, kids)
        if at is None:
            T.append(r, want)
        elif at[0] != want:
            T.move(r, want)
    T.sync()


def run_frame(ch, T, f, pattern, writebacks=((3, None, None),), cols=None):
    """One frame: `pattern` picks the Transform changes (dense: every root, sparse: 8 roots, static: none), then the
    write-backs (which, gt_tick, vv_tick) -- ticks default to distinct per-frame values."""
    sc, c, w = ch.sc, ch.pipe.ctx, ch.world
    if pattern == "dense":
        scenes.advance_cameras(sc, 0.05)
        rows, trs = scenes.mutate_roots(sc, f)
    elif pattern == "sparse":
        scenes.advance_cameras(sc, 0.05)
        rows = np.sort(T.rng.choice(sc.roots, size=8, replace=False)).astype(np.uint32)
        trs = sc.trs[rows].copy()
        trs[:, 0:3] += T.rng.uniform(-0.5, 0.5, (8, 3)).astype(np.float32)
        sc.trs[rows] = trs
    else:
        rows, trs = np.zeros(0, np.uint32), np.zeros((0, 10), np.float32)
    if len(rows):
        c.upload_transforms_scattered(rows, trs)
        w.tchanged[rows] = 1
    ch.pipe.update_views()
    planes = np.stack([np.ctypeslib.as_array(v.half_spaces).reshape(6, 4).copy() for v in ch.pipe.views])
    gch, vch, _, _ = w.frame(planes, cluster=False)
    ch.pipe.run_frame()
    for i, (which, gtt, vvt) in enumerate(writebacks):
        gtt = 100 * f + 2 * i + 1 if gtt is None else gtt
        vvt = 100 * f + 2 * i + 2 if vvt is None else vvt
        c.writeback_tables(which, gtt, vvt)
        T.expect(w.gt, gch, w.vv, vch, which, gtt, vvt)
    if cols is not None:
        c.writeback_columns()
    c.synchronize()
    ch.pipe.read_feedback()
    T.check(f"frame {f} ({pattern})")
    return gch, vch


def make(seed, n_trees=60, headroom=600):
    sc = scenes.forest(n_trees=n_trees, levels=6, n_lights=24, seed=seed)
    ch = Churn(sc, headroom, seed=seed, visible_diff=False)
    T = Tables(ch.pipe.ctx, split(sc), np.random.default_rng(seed))
    return ch, T


def test_tables_match_the_oracle_on_dense_sparse_and_static_frames():
    """Four shuffled tables (plus an empty one for flat rows), column sinks registered beside them: every frame the tables
    hold exactly the oracle's results and ticks, and the column sinks still give what they gave before."""
    torch = pytest.importorskip("torch")
    ch, T = make(seed=3)
    try:
        c, sc = ch.pipe.ctx, ch.sc
        # the small tables come from one heap buffer: neighbouring columns share pages
        pages = lambda a: (a.ctypes.data // 4096, (a.ctypes.data + a.nbytes - 1) // 4096)
        assert pages(T.tabs[INNER].vv_ticks)[1] == pages(T.tabs[LEAVES].gt)[0]
        assert pages(T.tabs[LIGHTS].vv_ticks)[1] == pages(T.tabs[FLAT].gt)[0]
        # a few slots left unmapped in the middle of a table: never written
        T.map[LEAVES][[3, 40, 41]] = NONE
        for s in (3, 40, 41):
            c.set_table_rows(LEAVES, s, [NONE])
        N = c.max_entities
        W = (N + 31) // 32
        gt_h = torch.zeros((N, 16), dtype=torch.float32).pin_memory().numpy()
        gbits = torch.zeros(W, dtype=torch.int32).pin_memory().numpy().view(np.uint32)
        vbits = torch.zeros(W, dtype=torch.int32).pin_memory().numpy().view(np.uint32)
        vv_h = torch.zeros(N, dtype=torch.uint8).pin_memory().numpy()
        c.set_column_sinks(gt_h, gbits, vv_h, vbits)
        unpack = lambda b, n: np.unpackbits(b.view(np.uint8), bitorder="little")[:n]
        ever = np.zeros(sc.n, bool)
        for f, pattern in enumerate(["dense", "dense", "sparse", "static", "sparse", "dense", "static"]):
            gch, vch = run_frame(ch, T, f, pattern, cols=True)
            n = sc.n
            assert (unpack(gbits, n) == gch).all() and (unpack(vbits, n) == vch).all(), f
            ever |= gch.astype(bool)
            assert (gt_h[:n][ever].view(np.uint32) == affine3a(ch.world.gt[ever]).view(np.uint32)).all(), f
            assert (vv_h[:n] == ch.world.vv).all(), f
            if pattern == "static":
                assert not gch.any()
            if pattern == "sparse":
                assert 0 < gch.sum() < n // 4
        # split systems: GlobalTransform right after PROPAGATE, ViewVisibility after CULL, each with its own tick
        run_frame(ch, T, 9, "sparse", writebacks=((abi.WB_GLOBAL_TRANSFORM, 901, 0), (abi.WB_VIEW_VISIBILITY, 0, 902)))
        run_frame(ch, T, 10, "dense", writebacks=((abi.WB_GLOBAL_TRANSFORM, 1001, 0), (abi.WB_VIEW_VISIBILITY, 0, 1002)))
        c.set_column_sinks()
    finally:
        ch.close()


def test_archetype_moves_reallocation_edits_and_compaction():
    """Spawns, despawns and reparents move rows between archetypes (swap_remove plus a partial set_table_rows), the flat
    table grows to a new address, then the world is compacted on the device and the test leaves its tables alone."""
    ch, T = make(seed=5)
    try:
        c, sc = ch.pipe.ctx, ch.sc
        run_frame(ch, T, 0, "dense")
        flat_addr = T.tabs[FLAT].gt.ctypes.data
        for f in range(1, 7):
            ch.random_edit(n_despawn=6, n_flat=6, n_kids=4, n_reparent=3)
            follow_archetypes(ch, T)
            run_frame(ch, T, f, ["dense", "sparse", "static"][f % 3])
        assert T.tabs[FLAT].gt.ctypes.data != flat_addr, "the flat table never grew"
        assert c.topology_summary()[0] > c.topology_summary()[1], "no tombstones to compact"
        o2n = c.compact_topology().astype(np.int64)
        renumber(ch, o2n)
        T.map = [np.where(m != NONE, o2n[np.minimum(m, len(o2n) - 1)], NONE).astype(np.uint32) for m in T.map]
        for f in range(7, 10):
            run_frame(ch, T, f, ["dense", "sparse", "static"][f % 3])
        ch.random_edit(n_despawn=4, n_flat=8, n_kids=4, n_reparent=2)      # rows spawned after the compaction
        follow_archetypes(ch, T)
        run_frame(ch, T, 10, "dense")
        # set_topology unmaps every slot; the tables stay registered
        c.set_topology(sc.parent, sc.entity_bits)
        for m in T.map:
            m[:] = NONE
        ch.world.tchanged[:] = 1
        c.mark_transforms_changed(0, sc.n)
        run_frame(ch, T, 11, "dense")
    finally:
        ch.close()


def test_errors_leave_the_maps_as_they_were():
    ch, T = make(seed=7, n_trees=30)
    try:
        c = ch.pipe.ctx
        run_frame(ch, T, 0, "dense")
        leaves = T.tabs[LEAVES]
        cases = [
            (INVALID_ARG, lambda: c.set_table_rows(LEAVES, leaves.capacity - 1, [int(T.map[LEAVES][0]), 5])),   # past capacity
            (INVALID_ARG, lambda: c.set_table_rows(len(T.tabs), 0, [0])),                                       # no such table
            (INVALID_ARG, lambda: c.set_table_rows(ROOTS, 0, [ch.sc.n + 5])),                                   # no such row
        ]
        for code, call in cases:
            with pytest.raises(abi.B200VisError) as e:
                call()
            assert e.value.code == code, str(e.value)
        too_long = abi.Table(None, None, None, None, 9, 8)
        with pytest.raises(abi.B200VisError) as e:
            c.set_tables(T.tabs + [too_long])
        assert e.value.code == INVALID_ARG
        with pytest.raises(abi.B200VisError) as e:
            c.set_tables([abi.Table(None, None, None, None, 0, 0)] * (abi.MAX_TABLES + 1))
        assert e.value.code == CAPACITY
        run_frame(ch, T, 1, "dense")
        # a despawned row cannot be mapped, and the whole call is refused
        victim = int(T.map[LEAVES][0])
        ch.edit([victim], [], [], [], np.zeros((0, 10), np.float32))
        follow_archetypes(ch, T)
        keep = int(T.map[LEAVES][0])
        with pytest.raises(abi.B200VisError) as e:
            c.set_table_rows(LEAVES, 0, [keep, victim])
        assert e.value.code == INVALID_ARG
        run_frame(ch, T, 2, "dense")
        run_frame(ch, T, 3, "sparse")
    finally:
        ch.close()
    wide = abi.Context(64, world_size=2, rank=0)
    try:
        with pytest.raises(abi.B200VisError) as e:
            wide.set_tables([])
        assert e.value.code == UNSUPPORTED
        with pytest.raises(abi.B200VisError) as e:
            wide.writeback_tables()
        assert e.value.code == UNSUPPORTED
    finally:
        wide.close()
    fresh = abi.Context(64)
    try:
        with pytest.raises(abi.B200VisError) as e:
            fresh.writeback_tables()
        assert e.value.code == NOT_READY
    finally:
        fresh.close()


def test_pinned_memory_is_used_through_its_alias():
    """A table whose columns the caller pinned itself (torch's pin_memory): used as it is, not registered again."""
    torch = pytest.importorskip("torch")
    ch, T = make(seed=11, n_trees=20)
    try:
        old = T.tabs[LIGHTS]
        cap = old.capacity
        gt = torch.full((cap, 16), float("nan"), dtype=torch.float32).pin_memory().numpy()
        gtt = torch.full((cap,), 7, dtype=torch.int32).pin_memory().numpy().view(np.uint32)
        vv = torch.full((cap,), VV_SENTINEL, dtype=torch.uint8).pin_memory().numpy()
        vvt = torch.full((cap,), 7, dtype=torch.int32).pin_memory().numpy().view(np.uint32)
        new = abi.HostTable(gt, gtt, vv, vvt, old.len)
        for k in COLUMNS:
            raw(new, k)[:] = raw(old, k)
        T.tabs[LIGHTS] = new
        T.bufs[LIGHTS] = (gt, gtt, vv, vvt)
        ch.pipe.ctx.set_tables(T.tabs)
        for f, pattern in enumerate(["dense", "sparse", "dense"]):
            run_frame(ch, T, f, pattern)
    finally:
        ch.close()


def test_misaligned_columns_are_refused():
    """The kernel stores 16-byte matrices and 4-byte ticks: columns that cannot take them are refused, nothing changes."""
    ch, T = make(seed=13, n_trees=20)
    try:
        c = ch.pipe.ctx
        run_frame(ch, T, 0, "dense")
        t = T.tabs[LEAVES]
        for bad in (abi.Table(t.gt.ctypes.data + 4, None, None, None, 1, 1),
                    abi.Table(None, t.gt_ticks.ctypes.data + 2, None, None, 1, 1),
                    abi.Table(None, None, None, t.vv_ticks.ctypes.data + 1, 1, 1)):
            with pytest.raises(abi.B200VisError) as e:
                c.set_tables(T.tabs + [bad])
            assert e.value.code == INVALID_ARG
        run_frame(ch, T, 1, "sparse")
    finally:
        ch.close()


def test_queued_map_changes_reach_the_device_in_order():
    """Two rows of one table trade slots (a marker component added to one and removed from the other: len, pointers and
    capacity stay the same), several times over before one write-back; the queued changes land as the last call left them."""
    ch, T = make(seed=17, n_trees=20)
    try:
        c = ch.pipe.ctx
        run_frame(ch, T, 0, "dense")
        m = T.map[LEAVES]
        for a, b in ((0, 5), (5, 9), (1, 0), (9, 1)):
            ra, rb = int(m[a]), int(m[b])
            for k in COLUMNS:                              # the bytes travel with their entities
                col, mod = raw(T.tabs[LEAVES], k), T.model[LEAVES][k]
                col[[a, b]] = col[[b, a]]
                mod[[a, b]] = mod[[b, a]]
            m[a], m[b] = rb, ra
            c.set_table_rows(LEAVES, a, [rb])              # maps rb at a, unmaps it at b
            c.set_table_rows(LEAVES, b, [ra])
        run_frame(ch, T, 1, "dense")
        run_frame(ch, T, 2, "sparse")
    finally:
        ch.close()


def test_registrations_are_released():
    """set_tables([]) and the context's destruction unregister the memory the library registered: the caller can then
    register it itself."""
    torch = pytest.importorskip("torch")
    cudart = torch.cuda.cudart()
    tabs, buf = abi.host_tables([300, 40, 7])
    base, size = buf.ctypes.data, buf.nbytes
    page = (base + 4095) // 4096 * 4096

    def free_to_register():
        rc = int(cudart.cudaHostRegister(page, 4096, 0))
        if rc == 0:
            assert int(cudart.cudaHostUnregister(page)) == 0
        return rc == 0
    for release in ("set_tables", "destroy"):
        c = abi.Context(64)
        try:
            c.set_tables(tabs)
            if release == "set_tables":
                c.set_tables([])
        finally:
            c.close()
        assert free_to_register(), release
