"""The archetype-table write-back (b200vis_set_tables / b200vis_set_table_rows / b200vis_writeback_tables) stated slot by
slot, as include/b200vis.h states it and independent of the kernel, plus a driver that plays one scenario on the CPU oracle
and, given a device, on the library in step.

`Model` holds what every column of every registered table must hold:
- a GlobalTransform (glam Affine3A bits) and gt_tick only in slots [0, len) mapped to a row whose GlobalTransform changed,
  each only where its column is registered;
- a ViewVisibility byte where it differs from what the slot is known to hold.  What a slot is known to hold is kept per
  row, as the header words it: the byte last written for the row, or unknown after the row is mapped to a new slot, after
  its table's view_visibility column moves (NULL -> memory, memory -> NULL, memory -> other memory) and for rows that are
  new after a compaction.  So the model is exact for every slot;
- vv_tick where Changed<ViewVisibility> fires, where the vv_changed_ticks column is registered;
- nothing anywhere else: unmapped slots, slots at or past len, and the columns passed as NULL keep their bytes.

`Model(mutant=...)` swaps one rule for a plausible wrong one (MUTANTS).  A scenario tells a mutant apart when some table
content differs from the true model's at one of its checks; test_cpu_table_model.py shows on the CPU that every scenario
tells every mutant apart, so the device tests built from the same scenarios would catch a kernel or host that followed it.

`Run` plays a scenario: the scene on parity.OracleWorld's arrays (the C oracle's propagate and cull), the caller's tables
over plain numpy memory, and every true / mutant model; with device=True also the library, whose tables are compared with
the true model after b200vis_synchronize at every check."""
import numpy as np

import bevy_b200 as bb
from bevy_b200 import abi, scenes
import oracle as orc
from parity import IDENTITY, OracleWorld

NONE = abi.UNMAPPED
GT, VV = abi.WB_GLOBAL_TRANSFORM, abi.WB_VIEW_VISIBILITY
COLUMNS = ("gt", "gt_ticks", "vv", "vv_ticks")
ALL = frozenset(COLUMNS)
TICK_SENTINEL, VV_SENTINEL = 0xDEAD0001, 0xEE
UNKNOWN = 0xFF
DETACHED = 0xFFFFFFFE
F_NO_CPU_CULL = 0x20

MUTANTS = {
    "capacity": "slots [len, capacity) are written like the slots below len",
    "gt_tick_needs_gt": "gt_tick is stamped only where the GlobalTransform column is registered too",
    "vv_tick_needs_vv": "vv_tick is stamped only where the ViewVisibility column is registered too",
    "no_remap_reset": "a row mapped to a new slot keeps the byte its old slot was known to hold",
    "no_column_reset": "the rows of a table whose view_visibility column moved keep their known bytes",
}


def affine3a_bits(gt12):
    """[n, 12] x_axis, y_axis, z_axis, translation -> [n, 16] uint32 bits of glam Affine3A (Vec3A lanes, padding 0).  Bit
    copies, so NaN payloads are kept."""
    g = np.ascontiguousarray(gt12, np.float32).view(np.uint32).reshape(-1, 12)
    out = np.zeros((len(g), 16), np.uint32)
    for k in range(4):
        out[:, 4 * k:4 * k + 3] = g[:, 3 * k:3 * k + 3]
    return out


def raw(tab, name):
    a = getattr(tab, name)
    return a.view(np.uint32) if name == "gt" else a


def same_bits(a, b):
    """Bit equality, except that any NaN matches any NaN (the oracle's NaN payloads are the CPU's)."""
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


class Model:
    """The registered tables' contents as the header promises them.  `data[t][column]` are the model's copies of the caller's
    columns (the driver applies the caller's own writes to them), the slot -> row maps are kept back to back like the
    library's, and `known[r]` is the ViewVisibility byte row r's slot is known to hold (UNKNOWN: it gets written)."""

    def __init__(self, n_rows, mutant=None):
        assert mutant is None or mutant in MUTANTS
        self.mutant = mutant
        self.known = np.full(n_rows, UNKNOWN, np.uint8)
        self.loc = np.full(n_rows, -1, np.int64)            # row -> map entry
        self.tabs, self.data = [], []
        self.map, self.off = np.zeros(0, np.uint32), np.zeros(1, np.int64)

    def slots(self, t):
        return self.map[self.off[t]:self.off[t] + self.tabs[t]["cap"]]

    def set_tables(self, specs):
        """specs[t] = dict(len, cap, cols, vv_mem): vv_mem names the view_visibility memory (None when passed as NULL)."""
        off = np.concatenate([[0], np.cumsum([s["cap"] for s in specs])]).astype(np.int64)
        new = np.full(int(off[-1]), NONE, np.uint32)
        for t, s in enumerate(specs):
            if t >= len(self.tabs):
                continue
            keep = min(s["cap"], self.tabs[t]["cap"])
            new[off[t]:off[t] + keep] = self.slots(t)[:keep]
            if s["vv_mem"] != self.tabs[t]["vv_mem"] and self.mutant != "no_column_reset":
                r = new[off[t]:off[t] + keep]
                self.known[r[r != NONE]] = UNKNOWN
        self.tabs = [dict(s) for s in specs]
        self.map, self.off = new, off
        self.loc[:] = -1
        e = np.nonzero(new != NONE)[0]
        self.loc[new[e]] = e

    def set_rows(self, t, first, rows):
        rows = np.asarray(rows, np.int64)
        e0 = int(self.off[t]) + first
        for i, r in enumerate(rows.tolist()):
            e = e0 + i
            old = int(self.map[e])
            if old == r:
                continue
            if old != NONE:
                self.loc[old] = -1
            if r != NONE:
                if self.loc[r] >= 0:
                    self.map[self.loc[r]] = NONE
                self.loc[r] = e
                if self.mutant != "no_remap_reset":
                    self.known[r] = UNKNOWN
            self.map[e] = r

    def unmap_rows(self, rows):
        rows = np.asarray(rows, np.int64)
        e = self.loc[rows]
        self.map[e[e >= 0]] = NONE
        self.loc[rows] = -1

    def unmap_all(self):
        self.map[:] = NONE
        self.loc[:] = -1

    def renumber(self, o2n):
        """b200vis_compact_topology: the maps and the known bytes follow the rows; the rows past the new count are unknown."""
        keep = np.nonzero(o2n != NONE)[0]
        known = self.known.copy()
        known[:len(o2n)] = UNKNOWN
        known[o2n[keep]] = self.known[keep]
        self.known = known
        m = self.map != NONE
        self.map[m] = o2n[self.map[m]]
        self.loc[:] = -1
        e = np.nonzero(m)[0]
        self.loc[self.map[e]] = e

    def writeback(self, which, gt_tick, vv_tick, gt12, gch, vv, vch):
        for t, tab in enumerate(self.tabs):
            lim = tab["cap"] if self.mutant == "capacity" else tab["len"]
            m = self.slots(t)[:lim]
            s = np.nonzero(m != NONE)[0]
            r = m[s].astype(np.int64)
            d, cols = self.data[t], tab["cols"]
            if which & GT:
                c = gch[r] != 0
                if "gt" in cols:
                    d["gt"][s[c]] = affine3a_bits(gt12[r[c]])
                if "gt_ticks" in cols and ("gt" in cols or self.mutant != "gt_tick_needs_gt"):
                    d["gt_ticks"][s[c]] = gt_tick
            if which & VV:
                if "vv" in cols:
                    w = self.known[r] != vv[r]
                    d["vv"][s[w]] = vv[r[w]]
                    self.known[r[w]] = vv[r[w]]
                if "vv_ticks" in cols and ("vv" in cols or self.mutant != "vv_tick_needs_vv"):
                    d["vv_ticks"][s[vch[r] != 0]] = vv_tick


def fresh_tables(caps, lens):
    """Tables over one plain numpy buffer, every column sentinel-filled."""
    return abi.host_tables(caps, lens, gt_fill=np.nan, tick_fill=TICK_SENTINEL, vv_fill=VV_SENTINEL)


class Run:
    """One scenario: the oracle world, the caller's tables, the true model and every mutant; with device=True the library
    too.  Rows are the scene's rows; `alive` follows despawns."""

    def __init__(self, sc, device, static_opt=True, headroom=0, mutants=tuple(MUTANTS), seed=0):
        self.sc, self.device = sc, device
        self.world = OracleWorld(sc, static_opt)
        self.N = sc.n + headroom
        self.models = [Model(self.N)] + [Model(self.N, m) for m in mutants]
        self.rng = np.random.default_rng(seed)
        self.alive = np.ones(sc.n, bool)
        self.ext = np.zeros(sc.n, np.uint8)
        self.tabs, self.cols, self.vv_mem, self.bufs = [], [], [], []
        self.mem_ids = iter(range(1, 1 << 30))
        self.tick = 0
        self.separated = set()
        self.checks = 0
        self.sinks = None
        self.pipelined = False                              # frames enqueued back to back: no downloads until a check
        self.pipe = self.ctx = None
        if device:
            self.pipe = bb.VisibilityPipeline(sc, static_transform_optimizations=static_opt, max_entities=self.N)
            self.ctx = self.pipe.ctx

    def close(self):
        if self.pipe is not None:
            if self.sinks is not None:
                self.ctx.set_column_sinks()
            self.pipe.close()

    # ---- the caller's tables --------------------------------------------------------------------------------------------
    def add_tables(self, lens, caps=None, cols=None):
        """New tables at the end of the registry, in fresh memory; registered at once.  Returns their indices."""
        caps = list(lens) if caps is None else list(caps)
        tabs, buf = fresh_tables(caps, lens)
        self.bufs.append(buf)
        first = len(self.tabs)
        for i, tab in enumerate(tabs):
            self.tabs.append(tab)
            self.cols.append(ALL if cols is None else frozenset(cols[i]))
            self.vv_mem.append(next(self.mem_ids))
            for m in self.models:
                m.data.append({k: raw(tab, k).copy() for k in COLUMNS})
        self.register()
        return list(range(first, len(self.tabs)))

    def register(self):
        """b200vis_set_tables with every table's current columns, len and capacity."""
        specs = [dict(len=t.len, cap=t.capacity, cols=c, vv_mem=v if "vv" in c else None)
                 for t, c, v in zip(self.tabs, self.cols, self.vv_mem)]
        if self.ctx is not None:
            self.ctx.set_tables([t.desc(c) for t, c in zip(self.tabs, self.cols)])
        for m in self.models:
            m.set_tables(specs)

    def set_columns(self, t, cols):
        self.cols[t] = frozenset(cols)
        self.register()

    def new_vv_column(self, t):
        """Table t's ViewVisibility bytes move to fresh sentinel-filled memory (the caller's column was reallocated)."""
        tab = self.tabs[t]
        vv = np.full(max(tab.capacity, 1), VV_SENTINEL, np.uint8)[:tab.capacity]
        self.bufs.append(vv)
        tab.vv = vv
        self.vv_mem[t] = next(self.mem_ids)
        for m in self.models:
            m.data[t]["vv"] = vv.copy()
        self.register()

    def map(self, t, first, rows):
        rows = np.asarray(rows, np.uint32)
        if self.ctx is not None:
            self.ctx.set_table_rows(t, first, rows)
        for m in self.models:
            m.set_rows(t, first, rows)

    def fill(self, t, rows):
        """Table t's slots [0, len(rows)) hold `rows` in a shuffled order."""
        rows = self.rng.permutation(np.asarray(rows, np.uint32))
        assert len(rows) <= self.tabs[t].len
        if len(rows):
            self.map(t, 0, rows)
        return rows

    def row_at(self, t, s):
        return int(self.models[0].slots(t)[s])

    def where(self, r):
        e = int(self.models[0].loc[r])
        if e < 0:
            return None
        t = int(np.searchsorted(self.models[0].off, e, side="right")) - 1
        return t, e - int(self.models[0].off[t])

    def poke(self, t, s, k, value):
        """The caller (or another system) writes slot s of column k itself."""
        raw(self.tabs[t], k)[s] = value
        for m in self.models:
            m.data[t][k][s] = value

    def copy_slot(self, ta, sa, tb, sb):
        for k in COLUMNS:
            raw(self.tabs[tb], k)[sb] = raw(self.tabs[ta], k)[sa]
            for m in self.models:
                m.data[tb][k][sb] = m.data[ta][k][sa]

    def swap_remove(self, t, s):
        """Table::swap_remove: the last slot's bytes move into the hole and that row is mapped there (which unmaps the slot
        it left)."""
        tab = self.tabs[t]
        last = tab.len - 1
        if s != last:
            r = self.row_at(t, last)
            self.copy_slot(t, last, t, s)
            self.map(t, s, [r])
        tab.len -= 1

    def append(self, t, r, src=None, vv=None):
        """Row r joins table t at slot len: a spawn (GlobalTransform::IDENTITY, ViewVisibility::HIDDEN, ticks 0), or an
        archetype move whose bytes travel from `src`; `vv` re-inserts ViewVisibility with that byte."""
        tab = self.tabs[t]
        assert tab.len < tab.capacity
        d = tab.len
        if src is None:
            for k, v in (("gt", affine3a_bits(IDENTITY)[0]), ("gt_ticks", 0), ("vv", 0), ("vv_ticks", 0)):
                self.poke(t, d, k, v)
        else:
            self.copy_slot(src[0], src[1], t, d)
        if vv is not None:
            self.poke(t, d, "vv", vv)
        tab.len += 1
        self.map(t, d, [r])

    def move(self, r, t, vv=None):
        """An archetype move of row r to the end of table t; its old table swap_removes the hole."""
        a, s = self.where(r)
        self.append(t, r, src=(a, s), vv=vv)
        self.swap_remove(a, s)

    def leave(self, t):
        """Table t's last entity moves to a table without GlobalTransform: len drops, and since the plugin resends only
        slots [0, len) the slot past len stays mapped to that row."""
        r = self.row_at(t, self.tabs[t].len - 1)
        assert r != NONE
        self.tabs[t].len -= 1
        self.register()
        return r

    # ---- frames ----------------------------------------------------------------------------------------------------------
    def move_transforms(self, kind):
        """dense: every root moves (and the cameras); sparse: 8 roots; static: nothing."""
        sc = self.sc
        if kind == "static":
            return
        scenes.advance_cameras(sc, 0.05)
        if kind == "dense":
            rows, trs = scenes.mutate_roots(sc, self.tick)
        else:
            live = sc.roots[self.alive[sc.roots]]
            rows = np.sort(self.rng.choice(live, size=min(8, len(live)), replace=False)).astype(np.uint32)
            trs = sc.trs[rows].copy()
            trs[:, 0:3] += self.rng.uniform(-0.5, 0.5, (len(rows), 3)).astype(np.float32)
            sc.trs[rows] = trs
        self.upload(rows, trs)

    def upload(self, rows, trs):
        self.sc.trs[rows] = trs
        self.world.tchanged[rows] = 1
        if self.ctx is not None and len(rows):
            self.ctx.upload_transforms_scattered(rows, trs)

    def mark(self, rows, vals):
        """Another system writes GlobalTransforms (and their tick) into the rows' table slots, and the library is told."""
        rows = np.asarray(rows, np.uint32)
        vals = np.asarray(vals, np.float32).reshape(-1, 12)
        self.world.gt[rows] = vals
        self.ext[rows] = 1
        tick = self.next_tick()
        for r, bits in zip(rows.tolist(), affine3a_bits(vals)):
            at = self.where(r)
            if at is not None:
                self.poke(at[0], at[1], "gt", bits)
                self.poke(at[0], at[1], "gt_ticks", tick)
        if self.ctx is not None:
            self.ctx.write_global_transforms_scattered(rows, vals)

    def next_tick(self):
        self.tick += 1
        return 1000 + self.tick

    def planes(self):
        """update_frusta with the library's host functions, the way VisibilityPipeline.update_views builds them."""
        out = []
        for cam in self.sc.cameras:
            cfv = abi.host_perspective(cam.fov, cam.aspect, cam.near) if cam.clip_from_view is None \
                else np.ascontiguousarray(cam.clip_from_view, np.float32)
            out.append(abi.host_compute_frustum(cfv, cam.gt, cam.far))
        if self.pipe is not None:
            self.pipe.update_views(clusters=False)
        return np.stack(out)

    def _propagate(self):
        sc, w = self.sc, self.world
        ext = self.ext.copy()
        self.ext[:] = 0
        rc, gch = orc.propagate(sc.parent, sc.trs, w.gt, w.tchanged, w.static_opt, gt_ext_changed=ext)
        assert rc == 0
        w.tchanged[:] = 0
        if self.ctx is not None and not self.pipelined:
            gt, ch = self.ctx.download_global_transforms(0, sc.n)
            bad = ~same_bits(gt, w.gt).all(1)
            assert not bad.any(), f"GlobalTransform bits differ from the oracle on rows {np.nonzero(bad)[0][:8]}"
            assert (ch == gch).all(), f"Changed<GlobalTransform> differs from the oracle on rows {np.nonzero(ch != gch)[0][:8]}"
            w.gt[:] = gt                       # the device's own NaN payloads: the tables must receive exactly these bits
        return gch

    def _cull(self, planes):
        sc, w = self.sc, self.world
        vch, _ = orc.cull(w.gt, sc.bounds, sc.flags, sc.class_mask, sc.entity_bits, w.vv, planes, view_layers=sc.view_layers,
                          view_flags=sc.view_flags, layer_mask=sc.layer_mask, range_mask=sc.range_mask,
                          view_range_index=sc.view_range_index)
        if self.ctx is not None and not self.pipelined:
            vv, ch = self.ctx.download_view_visibility(0, sc.n)
            assert (vv == w.vv).all(), f"ViewVisibility differs from the oracle on rows {np.nonzero(vv != w.vv)[0][:8]}"
            assert (ch == vch).all(), f"Changed<ViewVisibility> differs from the oracle on rows {np.nonzero(ch != vch)[0][:8]}"
        return vch

    def writeback(self, which, gch=None, vch=None):
        gtt, vvt = self.next_tick(), self.next_tick()
        if self.ctx is not None:
            self.ctx.writeback_tables(which, gtt, vvt)
        w = self.world
        for m in self.models:
            m.writeback(which, gtt, vvt, w.gt, gch, w.vv, vch)

    def fused(self, check=True):
        """run(PROPAGATE | CULL) and one write-back of both columns."""
        planes = self.planes()
        if self.ctx is not None:
            self.ctx.run(abi.STAGE_PROPAGATE | abi.STAGE_CULL)
        gch = self._propagate()
        vch = self._cull(planes)
        self.writeback(GT | VV, gch, vch)
        if check:
            self.check("fused frame")
        return gch, vch

    def split(self, propagate_twice=False, check=True):
        """The plugin's frame: run(PROPAGATE) -> write-back of GlobalTransform with its own tick [twice on the first frame:
        PostStartup + PostUpdate] -> run(CULL) -> write-back of ViewVisibility with its own tick (and the column sinks'
        ViewVisibility when registered, as the plugin without the forked bevy does)."""
        for _ in range(2 if propagate_twice else 1):
            if self.ctx is not None:
                self.ctx.run(abi.STAGE_PROPAGATE)
            gch = self._propagate()
            self.writeback(GT, gch=gch)
            if check:
                self.check("split frame, GlobalTransform")
        planes = self.planes()
        if self.ctx is not None:
            self.ctx.run(abi.STAGE_CULL)
        vch = self._cull(planes)
        self.writeback(VV, vch=vch)
        if self.sinks is not None:
            self.ctx.writeback_columns(VV)
        if check:
            self.check("split frame, ViewVisibility")
            if self.sinks is not None:
                vv_h, vbits = self.sinks
                n = self.sc.n
                assert (vv_h[:n] == self.world.vv).all(), "column sink ViewVisibility differs from the oracle"
                assert (np.unpackbits(vbits.view(np.uint8), bitorder="little")[:n] == vch).all(), "column sink change bits differ"
        return vch

    def column_sinks(self):
        """The plugin without the forked bevy: ViewVisibility through the column sinks (device only)."""
        if self.ctx is None:
            return
        import torch
        N = self.ctx.max_entities
        vv_h = torch.zeros(N, dtype=torch.uint8).pin_memory().numpy()
        vbits = torch.zeros((N + 31) // 32, dtype=torch.int32).pin_memory().numpy().view(np.uint32)
        self.ctx.set_column_sinks(None, None, vv_h, vbits)
        self.sinks = (vv_h, vbits)

    def frame(self, shape, kind, **kw):
        self.move_transforms(kind)
        return self.split(**kw) if shape == "split" else self.fused(**kw)

    # ---- topology --------------------------------------------------------------------------------------------------------
    def despawn(self, rows):
        """b200vis_edit_topology despawning leaf rows (the library unmaps them); the oracle's rows become tombstones."""
        sc, w = self.sc, self.world
        d = np.asarray(rows, np.int64)
        assert not np.isin(d, sc.light_row).any() and not np.isin(sc.parent, d).any()
        if self.ctx is not None:
            self.ctx.edit_topology(d)
        sc.parent[d] = DETACHED; sc.flags[d] = F_NO_CPU_CULL; sc.class_mask[d] = 0
        w.vv[d] = 0; w.tchanged[d] = 0
        self.alive[d] = False
        if sc.roots is not None:
            sc.roots = sc.roots[~np.isin(sc.roots, d)]
        for m in self.models:
            m.unmap_rows(d)

    def compact(self):
        """b200vis_compact_topology: the tombstones go, the live rows keep their order (no visible list holds a tombstone
        after a frame with every view active).  The library renumbers the maps itself."""
        o2n = np.full(self.sc.n, NONE, np.uint32)
        o2n[self.alive] = np.arange(int(self.alive.sum()), dtype=np.uint32)
        if self.ctx is not None:
            got = self.ctx.compact_topology()
            assert (got == o2n).all(), "the compaction kept or moved rows differently"
        self._renumber(o2n)
        for m in self.models:
            m.renumber(o2n)
        return o2n

    def _renumber(self, o2n):
        sc, w = self.sc, self.world
        keep = np.nonzero(o2n != NONE)[0]
        p = sc.parent.astype(np.int64)
        real = p < sc.n
        p[real] = o2n[p[real]]
        sc.parent = p[keep].astype(np.uint32)
        for name in ("trs", "bounds", "flags", "class_mask", "entity_bits", "layer_mask", "range_mask"):
            if getattr(sc, name, None) is not None:
                setattr(sc, name, getattr(sc, name)[keep])
        sc.light_row = o2n[sc.light_row].astype(np.uint32)
        if sc.roots is not None:
            sc.roots = o2n[sc.roots].astype(np.uint32)
        w.gt, w.vv, w.tchanged = w.gt[keep], w.vv[keep], w.tchanged[keep]
        self.alive, self.ext = self.alive[keep], self.ext[keep]

    def set_topology(self):
        """The shim's fallback: the live rows renumbered through b200vis_set_topology (every slot unmapped, every column
        uploaded again), then every table's slots [0, len) resent with the new rows -- each row's known byte is another
        entity's now."""
        o2n = np.full(self.sc.n, NONE, np.uint32)
        o2n[self.alive] = np.arange(int(self.alive.sum()), dtype=np.uint32)
        old_maps = [self.models[0].slots(t)[:tab.len].copy() for t, tab in enumerate(self.tabs)]
        self._renumber(o2n)
        sc, w = self.sc, self.world
        w.tchanged[:] = 1
        if self.ctx is not None:
            c = self.ctx
            c.set_topology(sc.parent, sc.entity_bits)
            c.upload_transforms(0, sc.trs)
            c.upload_global_transforms(0, w.gt)
            c.upload_bounds(0, sc.bounds, sc.flags, sc.class_mask, sc.layer_mask, sc.range_mask)
            c.upload_view_visibility(0, w.vv)
            c.set_lights(sc.light_row, sc.light_range, sc.light_layers)
        for m in self.models:
            m.unmap_all()
        for t, old in enumerate(old_maps):
            if len(old):
                self.map(t, 0, np.where(old != NONE, o2n[np.minimum(old, len(o2n) - 1)], NONE))

    # ---- checks ----------------------------------------------------------------------------------------------------------
    def check(self, tag):
        """Device: every column of every table equals the true model's, bit for bit.  Both: which mutants differ here."""
        self.checks += 1
        true = self.models[0]
        if self.ctx is not None:
            self.ctx.synchronize()
            for t, tab in enumerate(self.tabs):
                for k in COLUMNS:
                    got, want = raw(tab, k), true.data[t][k]
                    diff = got != want
                    bad = np.nonzero(diff.any(1) if diff.ndim > 1 else diff)[0]
                    assert len(bad) == 0, (f"{tag} (check {self.checks}): table {t} column {k} differs at slots {bad[:6]} "
                                           f"(len {tab.len}, capacity {tab.capacity}, columns {sorted(self.cols[t])}, rows "
                                           f"{true.slots(t)[bad[:6]]}): got {got[bad[:2]].tolist()}, want {want[bad[:2]].tolist()}")
        for m in self.models[1:]:
            if m.mutant not in self.separated and any(
                    not np.array_equal(m.data[t][k], true.data[t][k]) for t in range(len(self.tabs)) for k in COLUMNS):
                self.separated.add(m.mutant)


# ---- scenarios: each plays on the CPU alone (device=False) or on the library too, and returns its closed Run ----------------
def archetypes(sc):
    """Rows split as Bevy's archetypes, as tests/test_gpu_table_writeback.py splits them: roots, inner nodes, leaves,
    lights, flat rows."""
    n = sc.n
    kids = np.zeros(n, np.int64)
    real = sc.parent < n
    np.add.at(kids, sc.parent[real].astype(np.int64), 1)
    light = np.zeros(n, bool)
    light[sc.light_row] = True
    kind = np.where(kids > 0, np.where(real, 1, 0), np.where(real, 2, 4))
    kind[light] = 3
    return [np.nonzero(kind == k)[0].astype(np.uint32) for k in range(5)]


def add_probes(run, rows):
    """Two tables every scenario carries so that each rule of the header is observable in it: one registered with only its
    two tick columns (GlobalTransform and ViewVisibility passed as NULL), and one whose last entity left for an
    unregistered table, so a mapped slot lies past len.  Returns the second."""
    k = len(rows) // 2
    a, b = run.add_tables([k, len(rows) - k], caps=[k, len(rows) - k + 8], cols=[("gt_ticks", "vv_ticks"), ALL])
    run.fill(a, rows[:k])
    run.fill(b, rows[k:])
    run.leave(b)
    return b


def reinsert_visible(run, t, k=6):
    """ViewVisibility re-inserted (ViewVisibility::HIDDEN) on k visible rows of table t: each row moves to a new slot whose
    byte is 0, so its known byte must be forgotten."""
    vis = [s for s in range(run.tabs[t].len) if run.world.vv[run.row_at(t, s)] & 1][:k]
    for s in vis:
        run.move(run.row_at(t, s), t, vv=0)
    return len(vis)


def forest_run(device, seed, n_trees=60, headroom=0, static_opt=True, probe=64):
    sc = scenes.forest(n_trees=n_trees, levels=6, n_lights=24, seed=seed)
    run = Run(sc, device, static_opt=static_opt, headroom=headroom, seed=seed)
    groups = archetypes(sc)
    pick = np.zeros(len(groups[2]), bool)
    pick[run.rng.choice(len(groups[2]), probe, replace=False)] = True      # leaves of many trees
    probes, groups[2] = groups[2][pick], groups[2][~pick]
    return run, groups, probes


def scenario_past_len(device):
    """Mapped slots at and past len, made the plugin's way; a len-0 table with mapped slots; a capacity-0 table."""
    run, groups, probes = forest_run(device, seed=21)
    try:
        leaves = groups[2]
        zero, groups[2] = leaves[:40], leaves[40:]
        tabs = run.add_tables([len(g) for g in groups], caps=[len(g) + 16 for g in groups])
        for t, g in zip(tabs, groups):
            run.fill(t, g)
        z, empty = run.add_tables([40, 0], caps=[48, 0])
        run.fill(z, zero)
        run.tabs[z].len = 0                                 # every entity left, the maps were never resent
        run.register()
        b = add_probes(run, probes)
        for t in (tabs[1], tabs[2], tabs[3]):               # INNER, LEAVES, LIGHTS each lose their last entity
            run.leave(t)
        for kind in ("dense", "sparse", "static", "dense"):
            run.frame("fused", kind)
        run.leave(tabs[2])                                  # a second slot past len, below the first
        assert reinsert_visible(run, b) and reinsert_visible(run, tabs[0])
        run.frame("fused", "static")
        run.new_vv_column(b)
        for kind in ("sparse", "static", "dense"):
            run.frame("fused", kind)
        assert run.tabs[empty].capacity == 0 and run.tabs[z].len == 0
        return run
    finally:
        run.close()


SUBSETS = [frozenset(c for i, c in enumerate(COLUMNS) if m >> i & 1) for m in range(16)]


def scenario_column_subsets(device):
    """Every one of the 16 subsets of the four columns across one registry; the subsets rotate between frames (NULL ->
    memory, memory -> NULL); a ViewVisibility column NULL over frames in which rows change visibility, then fresh
    sentinel-filled memory; then the plugin without the forked bevy: GlobalTransform tables with NULL ViewVisibility and
    the column sinks' ViewVisibility through writeback_columns_ex(WB_VIEW_VISIBILITY)."""
    run, groups, probes = forest_run(device, seed=22)
    try:
        rows = run.rng.permutation(np.concatenate(groups))
        parts = np.array_split(rows, 16)
        tabs = run.add_tables([len(p) for p in parts], caps=[len(p) + 4 for p in parts], cols=SUBSETS)
        for t, p in zip(tabs, parts):
            run.fill(t, p)
        b = add_probes(run, probes)
        for kind in ("dense", "sparse"):
            run.frame("fused", kind)
        for f in range(3):                                  # every table takes the next one's subset
            for i, t in enumerate(tabs):
                run.cols[t] = SUBSETS[(i + f + 1) % 16]
            run.register()
            run.frame("fused", ("dense", "static", "sparse")[f])
        full = tabs[15]
        run.set_columns(full, ALL)
        run.frame("fused", "dense")
        run.set_columns(full, ALL - {"vv"})                 # memory -> NULL while rows change visibility
        before = run.world.vv.copy()
        run.frame("fused", "dense")
        run.frame("fused", "dense")
        assert (run.world.vv != before).any()
        run.new_vv_column(full)                             # NULL -> fresh memory: every mapped slot gets its byte again
        run.set_columns(full, ALL)
        run.frame("fused", "static")
        assert (run.models[0].data[full]["vv"][:run.tabs[full].len] != VV_SENTINEL).all()
        assert reinsert_visible(run, b)
        run.frame("fused", "static")
        for t in tabs:                                      # the plugin without the forked bevy
            run.cols[t] = frozenset({"gt", "gt_ticks"})
        run.register()
        run.column_sinks()
        for kind in ("dense", "sparse", "static", "dense"):
            run.frame("split", kind)
        return run
    finally:
        run.close()


def late_view_scene(n_views):
    """tests/test_gpu_many_views.py's ring: views 0-7 render layer 2 only, the views past the eighth the default layer, so
    rows on layer 0 alone are seen only past the eighth view."""
    from test_gpu_many_views import _forest_ring
    sc = _forest_ring(n_cameras=n_views, n_trees=80)
    rng = np.random.default_rng(n_views)
    sc.layer_mask = rng.choice([1, 1, 3], sc.n).astype(np.uint64)
    sc.view_layers = np.array([2] * 8 + [1] * (n_views - 8), np.uint64)
    return sc


def scenario_plugin_frames(device, n_views=16, static_opt=True):
    """The plugin's frames (PROPAGATE twice on frame 0, then split frames with fused ones in between) with n_views views:
    rows seen only past the eighth view go 0 -> 1, stay, go 1 -> 0 as those views switch off, and come back; other systems
    write GlobalTransforms into roots and into inner rows whose children sit in other tables."""
    from test_gpu_split_stages import DEFAULT_SEQUENCE
    sc = late_view_scene(n_views)
    run = Run(sc, device, static_opt=static_opt, seed=23)
    try:
        groups = archetypes(sc)
        probes, groups[2] = groups[2][:64], groups[2][64:]
        tabs = run.add_tables([len(g) for g in groups], caps=[len(g) + 16 for g in groups])
        for t, g in zip(tabs, groups):
            run.fill(t, g)
        b = add_probes(run, probes)
        only_late = np.nonzero(sc.layer_mask == 1)[0]
        late_on = [1, 1, 1, 0, 0, 1, 1, 0, 1, 1, 1]
        sc.view_flags = np.full(n_views, bb.VIEW_ACTIVE, np.uint8)
        run.split(propagate_twice=True)
        seen = [int((run.world.vv[only_late] & 1).sum())]
        for f, (shape, kind) in enumerate(DEFAULT_SEQUENCE, start=1):
            sc.view_flags[8:] = bb.VIEW_ACTIVE if late_on[f] else 0
            if f in (2, 6):
                roots = run.rng.choice(sc.roots, 6, replace=False)
                inner = run.rng.choice(groups[1], 6, replace=False)
                rows = np.concatenate([roots, inner]).astype(np.uint32)
                vals = run.world.gt[rows].copy()
                vals[:, 9:12] += np.float32(0.75)
                run.mark(rows, vals)
            if f == 5:
                assert reinsert_visible(run, b) and reinsert_visible(run, tabs[2])
            if f == 8:
                run.new_vv_column(b)
            run.frame(shape, kind)
            seen.append(int((run.world.vv[only_late] & 1).sum()))
        assert seen[0] > 10 and seen[3] == 0 and seen[5] > 0, seen
        return run
    finally:
        run.close()


def scenario_pipelined(device):
    """Back-to-back run(PROPAGATE | CULL) frames, one table write-back enqueued per frame, no synchronize until the last."""
    run, groups, probes = forest_run(device, seed=24)
    try:
        tabs = run.add_tables([len(g) for g in groups], caps=[len(g) + 16 for g in groups])
        for t, g in zip(tabs, groups):
            run.fill(t, g)
        b = add_probes(run, probes)
        run.frame("fused", "dense")
        run.pipelined = True
        for kind in ("dense", "sparse", "dense", "static", "dense", "sparse"):
            run.frame("fused", kind, check=False)
        run.pipelined = False
        run.check("after the pipelined frames")
        assert reinsert_visible(run, b)
        run.pipelined = True
        for kind in ("static", "sparse"):
            run.frame("fused", kind, check=False)
        run.pipelined = False
        run.check("after the pipelined frames")
        run.new_vv_column(b)
        run.pipelined = True
        for kind in ("dense", "sparse", "dense"):
            run.frame("fused", kind, check=False)
        run.pipelined = False
        run.check("after the pipelined frames")
        return run
    finally:
        run.close()


EDGE_LENGTHS = (0, 1, 31, 32, 33, 127, 128, 129, 255, 256, 257)


def scenario_chunk_edges(device):
    """Table lengths around the 32-slot warp step and the 128-slot chunk, next to B200VIS_MAX_TABLES tables in all, most of
    them 1-3 slots, over shuffled maps: thousands of tables share the chunk -> table map."""
    run, groups, probes = forest_run(device, seed=25, n_trees=170)
    try:
        rows = run.rng.permutation(np.concatenate(groups))
        n_tiny = abi.MAX_TABLES - len(EDGE_LENGTHS) - 2
        tiny = run.rng.integers(1, 4, n_tiny)
        lens = list(EDGE_LENGTHS) + tiny.tolist()
        assert sum(lens) <= len(rows)
        caps = [n + int(run.rng.integers(0, 3)) for n in lens]
        tabs = run.add_tables(lens, caps=caps)
        o = 0
        for t, n in zip(tabs, lens):
            run.fill(t, rows[o:o + n])
            o += n
        b = add_probes(run, probes)
        assert len(run.tabs) == abi.MAX_TABLES
        for kind in ("dense", "sparse", "static", "dense"):
            run.frame("fused", kind)
        assert reinsert_visible(run, b) and reinsert_visible(run, tabs[len(EDGE_LENGTHS) - 1])
        run.frame("fused", "static")
        run.new_vv_column(b)
        run.frame("fused", "dense")
        return run
    finally:
        run.close()


def scenario_ieee(device):
    """propagate_reference.EdgeScene's frames through the tables: NaN rows, zero-sign-only changes, subnormals, overflow,
    and other systems writing -0 or NaN bits.  The matrices the tables receive are the device's own bits (NaN payloads
    included), which match the C oracle and the float32 restatement up to NaN payloads."""
    import propagate_reference as ref
    es = ref.EdgeScene(0)
    sc = es.scene
    want = ref.run_reference(es)
    run = Run(sc, device, seed=26)
    try:
        groups = archetypes(sc)
        probes, groups[2] = groups[2][:64], groups[2][64:]
        tabs = run.add_tables([len(g) for g in groups], caps=[len(g) + 16 for g in groups])
        for t, g in zip(tabs, groups):
            run.fill(t, g)
        b = add_probes(run, probes)
        for f, kind in enumerate(es.FRAMES):
            rows, trs = es.uploads(f)
            run.upload(rows, trs)
            mrows, mvals = es.marks(f, run.world.gt)
            if len(mrows):
                run.mark(mrows, mvals)
            if f == 3:
                assert reinsert_visible(run, b)
            if f == 5:
                run.new_vv_column(b)
            gch, _ = run.fused()
            gt_ref, ch_ref, _ = want[f]
            assert same_bits(run.world.gt, gt_ref).all() and (gch == ch_ref).all(), f"frame {f} {kind}"
            if kind == "first":
                with np.errstate(invalid="ignore"):
                    g = run.world.gt
                    assert np.isnan(g).any() and np.isinf(g).any() and ((g != 0) & (np.abs(g) < ref.TINY)).any()
        return run
    finally:
        run.close()


def scenario_queued_at_topology(device, op):
    """Map changes still queued when a topology call runs: a row moved twice, rows whose ViewVisibility was re-inserted, a
    row moved and then despawned; then edit_topology, compact_topology (the model renumbers with the returned map) or
    set_topology (every slot unmapped, every table resent with the new rows), with no write-back in between."""
    run, groups, probes = forest_run(device, seed=27, headroom=64)
    try:
        tabs = run.add_tables([len(g) for g in groups], caps=[len(g) + 64 for g in groups])
        for t, g in zip(tabs, groups):
            run.fill(t, g)
        b = add_probes(run, probes)
        run.frame("fused", "dense")
        kids = np.zeros(run.sc.n, np.int64)
        p = run.sc.parent
        np.add.at(kids, p[p < run.sc.n].astype(np.int64), 1)
        leaves = [r for r in groups[2].tolist() if kids[r] == 0]
        early = sorted(leaves[:: max(1, len(leaves) // 40)][:30])   # tombstones spread over the rows
        for r in early:
            t, s = run.where(r)
            run.despawn([r])
            run.swap_remove(t, s)
        run.register()
        run.frame("fused", "dense")
        leaves = [r for r in leaves if run.alive[r]]
        twice = leaves[5]
        run.move(twice, tabs[4])                            # LEAVES -> FLAT -> ROOTS
        run.move(twice, tabs[0])
        hidden = [r for r in leaves[10:] if not run.world.vv[r] & 1]
        doomed = hidden[0]
        run.move(doomed, tabs[4])
        vis = [r for r in leaves[10:] if run.world.vv[r] & 1][:8]
        for r in vis:
            run.move(r, tabs[2], vv=0)
        if op == "edit":
            t, s = run.where(doomed)
            run.despawn([doomed])
            run.swap_remove(t, s)
        run.register()                                      # the lens changed; set_tables flushes the queue itself
        if op != "edit":                                    # so queue more after it
            for r in vis[:4]:
                run.move(r, tabs[4], vv=0)
            run.move(twice, tabs[4])
            run.move(twice, tabs[2])
            t, s = run.where(doomed)
            run.despawn([doomed])
            run.swap_remove(t, s)
        if op == "compact":
            run.compact()
        elif op == "set_topology":
            run.set_topology()
        for kind in ("dense", "static", "sparse", "dense"):
            run.register()
            run.frame("fused", kind)
        run.new_vv_column(b)
        run.frame("fused", "dense")
        return run
    finally:
        run.close()


SCENARIOS = {
    "past_len": scenario_past_len,
    "column_subsets": scenario_column_subsets,
    "plugin_frames_16_views": lambda device: scenario_plugin_frames(device, 16),
    "plugin_frames_32_views_static_opt_off": lambda device: scenario_plugin_frames(device, 32, static_opt=False),
    "pipelined": scenario_pipelined,
    "chunk_edges": scenario_chunk_edges,
    "ieee": scenario_ieee,
    "queued_then_edit": lambda device: scenario_queued_at_topology(device, "edit"),
    "queued_then_compact": lambda device: scenario_queued_at_topology(device, "compact"),
    "queued_then_set_topology": lambda device: scenario_queued_at_topology(device, "set_topology"),
}
