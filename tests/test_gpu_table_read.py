"""b200vis_read_tables on the device: Transform and other systems' GlobalTransforms read straight from the caller's
archetype tables, in step with a twin context fed by the scattered uploads.

Every scenario runs two contexts on the same scene.  Context A registers its tables with input columns
(b200vis_set_tables_ex) and reads them (b200vis_read_tables).  Context B gets the sets the slot-by-slot model of
tests/table_read_model.py reads from A's tables, through b200vis_upload_transforms_scattered and
b200vis_write_global_transforms_scattered.  A "game system" writes Transforms and GlobalTransforms into the tables and
stamps their ticks; every slot it does not stamp holds bytes that differ from the device's (bypass_change_detection
writes), so a slot read by mistake shows.  After every frame A is checked against the C oracle (orc.propagate with
tchanged / gt_ext_changed), and A and B are compared bit for bit: the GlobalTransform column, both change-bit sets,
ViewVisibility, the visible lists and the tables both wrote back into."""
import os

import numpy as np
import pytest

import bevy_b200 as bb
from bevy_b200 import abi, scenes
import table_read_model as M
from parity import compare_frame
from test_gpu_compaction import renumber
from test_gpu_external_gt import oracle_marks
from test_gpu_table_writeback import COLUMNS, affine3a, raw, split
from test_gpu_topology_edits import Churn
from test_gpu_bench_scale import run_case

pytestmark = pytest.mark.gpu

NONE = abi.UNMAPPED
U32 = 0xFFFFFFFF
RD_ALL = abi.RD_TRANSFORM | abi.RD_GLOBAL_TRANSFORM
INVALID_ARG, NOT_READY, UNSUPPORTED = 1, 7, 8
BEVY = abi.BEVY_TRANSFORM_LAYOUT            # rotation @ 0, translation @ 16, scale @ 28, 48 bytes
PERMUTED = (48, 32, 12, 0)                  # scale @ 0, rotation @ 12, translation @ 32
PACKED = (40, 0, 12, 28)                    # translation, rotation, scale back to back, no padding


def qnan(payload):
    return np.uint32(0x7FC00000 | payload).view(np.float32)


class Twin:
    """Contexts A (reads its tables) and B (scattered uploads) on two copies of one scene, with the same edits."""

    def __init__(self, make_scene, seed, layout=BEVY, tick0=1000, no_inputs=(), no_gt=(), extra=(), headroom=24,
                 groups=None, churn_headroom=400, no_gt_ticks=(), past_len=None):
        self.a = Churn(make_scene(), churn_headroom, seed=seed)
        self.b = Churn(make_scene(), churn_headroom, seed=seed)          # the same diff state: the same compaction
        self.a.world.ext = np.zeros(self.a.sc.n, np.uint8)
        self.rng = np.random.default_rng(seed + 1000)
        self.layout, self.last, self.headroom = layout, tick0 & U32, headroom
        self.no_inputs, self.no_gt, self.extra = set(no_inputs), set(no_gt), list(extra)
        # no_gt_ticks: tables registered with global_transforms but no gt_changed_ticks (never read for GlobalTransform);
        # past_len {table: k}: the table's last k rows stay mapped at slots at or past len (never read, never written)
        self.no_gt_ticks, self.past_len = set(no_gt_ticks), dict(past_len or {})
        self.keep = []
        self.build(groups if groups is not None else split(self.a.sc))
        self.f = 0

    def close(self):
        self.a.close(); self.b.close()

    # ---- the tables ----
    def build(self, groups):
        """Fresh tables for every archetype group (a reallocation of every column), slots shuffled, plus the extra
        (len, capacity) tables, which stay unmapped."""
        caps = [len(g) + self.headroom for g in groups] + [c for _, c in self.extra]
        lens = [len(g) for g in groups] + [n for n, _ in self.extra]
        self.tabs_a, ba = abi.host_tables(caps, lens, tick_fill=self.last)
        self.tabs_b, bb_ = abi.host_tables(caps, lens, tick_fill=self.last)
        self.ins, bi = abi.host_table_inputs(caps, self.layout, tick_fill=self.last)
        self.maps = [np.full(c, NONE, np.uint32) for c in caps]
        for t, g in enumerate(groups):
            self.maps[t][:len(g)] = self.rng.permutation(np.asarray(g, np.uint32))
        self.register()
        self.keep = [ba, bb_, bi]                           # the old buffers are released after the registry moved
        for t, m in enumerate(self.maps):
            if self.tabs_a[t].len:
                for c in (self.a, self.b):
                    c.pipe.ctx.set_table_rows(t, 0, m[:self.tabs_a[t].len])
        if self.past_len:
            for t, k in self.past_len.items():
                self.tabs_a[t].len -= k
                self.tabs_b[t].len -= k
            self.register()

    def descs(self, tabs):
        return [t.desc(("vv", "vv_ticks") if i in self.no_gt else ("gt", "vv", "vv_ticks") if i in self.no_gt_ticks else COLUMNS)
                for i, t in enumerate(tabs)]

    def inputs(self):
        return [None if t in self.no_inputs else i for t, i in enumerate(self.ins)]

    def register(self):
        self.a.pipe.ctx.set_tables_ex(self.descs(self.tabs_a), self.inputs(), self.layout)
        self.b.pipe.ctx.set_tables(self.descs(self.tabs_b))

    def locate(self):
        out = {}
        for t, tab in enumerate(self.tabs_a):
            for s in np.nonzero(self.maps[t][:tab.len] != NONE)[0]:
                out[int(self.maps[t][s])] = (t, int(s))
        return out

    def model_tables(self):
        out = []
        for t, tab in enumerate(self.tabs_a):
            ins = None if t in self.no_inputs else self.ins[t]
            gt = t not in self.no_gt
            out.append(M.ModelTable(tab.len, tab.capacity, self.maps[t], trs=None if ins is None else ins.trs,
                                    trs_ticks=None if ins is None else ins.ticks, gt=tab.gt if gt else None,
                                    gt_ticks=tab.gt_ticks if gt and t not in self.no_gt_ticks else None))
        return out

    # ---- one frame ----
    def game(self, L, R, pattern, n_gt, which, ancient=False):
        """The other systems between two runs of the propagate system: Transforms and GlobalTransforms written with
        ticks in (L, R], everything else overwritten without a tick (bypass_change_detection)."""
        a, b, rng = self.a, self.b, self.rng
        where = self.locate()
        alive = a.alive
        for t, ins in enumerate(self.ins):                  # bypass writes: bytes that differ from the device's
            cap = self.tabs_a[t].capacity
            if not cap:
                continue
            ins.put(np.arange(cap), rng.uniform(-900, 900, (cap, 10)).astype(np.float32))
            ins.ticks[:] = (L - rng.integers(0, 40, cap)) & U32
            if ancient:                                     # after last_run, but older than MAX_CHANGE_AGE
                ins.ticks[rng.random(cap) < 0.5] = (L + 3) & U32
        for t, tab in enumerate(self.tabs_a):
            if tab.len < tab.capacity:                      # newer ticks on slots at and past len: never read
                self.ins[t].ticks[tab.len:] = self.newer_tick(L, R)
                tick, junk = self.newer_tick(L, R), rng.uniform(-50, 50, (tab.capacity - tab.len, 16)).astype(np.float32)
                for tabs in (self.tabs_a, self.tabs_b):
                    tabs[t].gt[tab.len:] = junk
                    tabs[t].gt_ticks[tab.len:] = tick
            if t in self.no_gt_ticks and tab.len:           # GlobalTransform bytes in a table without ticks: never read
                tick, junk = self.newer_tick(L, R), rng.uniform(-50, 50, (tab.len, 16)).astype(np.float32)
                for tabs in (self.tabs_a, self.tabs_b):
                    tabs[t].gt[:tab.len] = junk
                    tabs[t].gt_ticks[:tab.len] = tick
            if ancient and t not in self.no_gt and t not in self.no_gt_ticks and tab.len:
                sel = np.nonzero(rng.random(tab.len) < 0.5)[0]   # GlobalTransforms after last_run, older than the clamp
                junk = rng.uniform(-50, 50, (len(sel), 16)).astype(np.float32)
                for tabs in (self.tabs_a, self.tabs_b):
                    tabs[t].gt[sel] = junk
                    tabs[t].gt_ticks[sel] = (L + 3) & U32
        readable = [r for r, (t, _) in where.items() if t not in self.no_inputs and alive[r]]
        roots = set(a.sc.roots.tolist()) if a.sc.roots is not None else set()
        cand = np.array(sorted(r for r in readable if r in roots), np.int64)
        if not which & abi.RD_TRANSFORM or pattern == "static" or not len(cand):
            moved = np.zeros(0, np.int64)
        elif pattern == "dense":
            moved = cand
        else:
            moved = np.sort(rng.choice(cand, size=min(8, len(cand)), replace=False))
        trs = a.sc.trs[moved].copy()
        trs[:, 0:3] += rng.uniform(-0.5, 0.5, (len(moved), 3)).astype(np.float32)
        for sc in (a.sc, b.sc):
            sc.trs[moved] = trs
        a.world.tchanged[moved] = 1
        for r, v in zip(moved, trs):
            t, s = where[int(r)]
            self.ins[t].put([s], v[None])
            self.ins[t].ticks[s] = self.newer_tick(L, R)
        # GlobalTransforms other systems wrote, some with NaN payloads and -0
        gt_rows = np.zeros(0, np.int64)
        pool = np.array(sorted(r for r, (t, _) in where.items() if t not in self.no_gt | self.no_gt_ticks and alive[r]), np.int64)
        if which & abi.RD_GLOBAL_TRANSFORM and n_gt and len(pool):
            gt_rows = np.sort(rng.choice(pool, size=min(n_gt, len(pool)), replace=False))
            vals = a.world.gt[gt_rows] + rng.uniform(-0.5, 0.5, (len(gt_rows), 12)).astype(np.float32)
            vals[0, 1] = np.float32(-0.0)
            if len(gt_rows) > 2:
                vals[1, 4] = qnan(0x1234)
                vals[2, 11] = np.float32(-0.0)
            a.world.gt[gt_rows] = vals
            a.world.ext[gt_rows] = 1
            for r, v in zip(gt_rows, affine3a(vals)):
                t, s = where[int(r)]
                tick = self.newer_tick(L, R)
                for tabs in (self.tabs_a, self.tabs_b):
                    tabs[t].gt[s] = v
                    tabs[t].gt_ticks[s] = tick
        # bypass GlobalTransform writes (the same bytes on both sides: B's tables are compared with A's)
        rest = np.setdiff1d(pool, gt_rows)
        for r in rng.choice(rest, size=min(6, len(rest)), replace=False) if len(rest) else []:
            t, s = where[int(r)]
            junk = rng.uniform(-50, 50, 16).astype(np.float32)
            for tabs in (self.tabs_a, self.tabs_b):
                tabs[t].gt[s] = junk
        return set(moved.tolist()), set(gt_rows.tolist())

    def newer_tick(self, L, R):
        """A tick in (L, R] within 16 of R (so also younger than MAX_CHANGE_AGE)."""
        return (R - int(self.rng.integers(0, min((R - L) & U32, 16)))) & U32

    def frame(self, pattern="dense", n_gt=12, which=RD_ALL, step=10, ancient=False, kind="fused", check=True):
        a, b = self.a, self.b
        L = self.last
        R = (L + step) & U32
        moved, written = self.game(L, R, pattern, n_gt, which, ancient)
        got_t, got_g = M.read(self.model_tables(), self.layout, which, L, R)
        assert set(got_t) == moved and set(got_g) == written, "the scenario itself is off"
        (rt, tv), (rg, gv) = M.as_uploads(got_t, got_g)
        a.pipe.ctx.read_tables(which, L, R)
        if len(rt):
            b.pipe.ctx.upload_transforms_scattered(rt, tv)
        if len(rg):
            b.pipe.ctx.write_global_transforms_scattered(rg, gv)
        for c in (a, b):
            scenes.advance_cameras(c.sc, 0.05)
        if kind == "step":
            self.step_both()
        else:
            for c in (a, b):
                c.pipe.update_views()
            with oracle_marks(a.world):
                compare_frame(a.pipe, a.world, self.f)
            b.pipe.run_frame()
            b.pipe.read_feedback()
        for c in (a, b):
            c.pipe.ctx.writeback_tables(abi.WB_GLOBAL_TRANSFORM | abi.WB_VIEW_VISIBILITY, R, R)
            c.pipe.ctx.synchronize()
        self.last = R
        if check:
            self.compare()
        self.f += 1

    def step_both(self):
        """b200vis_step with zero changed rows on both sides (the rows came in through the read / the uploads)."""
        a, b = self.a, self.b
        for c in (a, b):
            sc = c.sc
            arr = (bb.CameraDesc * len(sc.cameras))()
            for v, cam in enumerate(sc.cameras):
                arr[v].global_transform[:] = cam.gt.tolist()
                arr[v].fov_y, arr[v].aspect, arr[v].near_z, arr[v].far_z = cam.fov, cam.aspect, cam.near, cam.far
                arr[v].layer_mask, arr[v].flags, arr[v].range_view_index = 1, bb.VIEW_ACTIVE, -1
            c.pipe.ctx.step(0, 0, 0, arr, len(sc.cameras), c.pipe.cluster_config, wait=True)
        a.pipe.update_views(clusters=False)
        with oracle_marks(a.world):
            compare_frame(a.pipe, a.world, self.f, cluster=False, run_device=False)

    def compare(self):
        a, b = self.a.pipe.ctx, self.b.pipe.ctx
        n, tag = self.a.sc.n, f"frame {self.f}"
        ga, ca = a.download_global_transforms(0, n)
        gb, cb = b.download_global_transforms(0, n)
        bad = np.nonzero((ga.view(np.uint32) != gb.view(np.uint32)).any(1))[0]
        assert not len(bad), f"{tag}: GlobalTransform bits differ from the scattered twin on rows {bad[:8]}"
        assert (ca == cb).all(), f"{tag}: Changed<GlobalTransform> differs on rows {np.nonzero(ca != cb)[0][:8]}"
        va, vca = a.download_view_visibility(0, n)
        vb, vcb = b.download_view_visibility(0, n)
        assert (va == vb).all() and (vca == vcb).all(), f"{tag}: ViewVisibility differs"
        for v in range(len(self.a.sc.cameras)):
            la, lb = a.download_visible(v), b.download_visible(v)
            assert len(la) == len(lb) and (la == lb).all(), f"{tag}: view {v} visible list differs"
        for t, (ta, tb) in enumerate(zip(self.tabs_a, self.tabs_b)):
            for k in COLUMNS:
                x, y = raw(ta, k), raw(tb, k)
                if not len(x):
                    continue
                d = np.nonzero((x != y).reshape(len(x), -1).any(1))[0]
                assert not len(d), f"{tag}: table {t} column {k} differs from the twin's at slots {d[:6]}"

    # ---- edits ----
    def edit(self, **kw):
        """The same random edit on both sides; the tables follow as fresh allocations (archetype moves + reserve)."""
        n0 = self.a.sc.n
        self.a.random_edit(**kw)
        self.b.random_edit(**kw)
        assert (self.a.sc.parent == self.b.sc.parent).all()
        self.a.world.ext = np.concatenate([self.a.world.ext, np.zeros(self.a.sc.n - n0, np.uint8)])
        self.a.world.ext[~self.a.alive] = 0
        groups = [[r for r in g if self.a.alive[r]] for g in split(self.a.sc)]
        self.build(groups)

    def compact(self):
        o2n = self.a.pipe.ctx.compact_topology().astype(np.int64)
        o2n_b = self.b.pipe.ctx.compact_topology().astype(np.int64)
        assert (o2n == o2n_b).all()
        keep = np.nonzero(o2n != NONE)[0]
        ext = np.zeros(len(keep), np.uint8); ext[o2n[keep]] = self.a.world.ext[keep]
        for c in (self.a, self.b):
            renumber(c, o2n)
        self.a.world.ext = ext
        self.maps = [np.where(m != NONE, o2n[np.minimum(m, len(o2n) - 1)], NONE).astype(np.uint32) for m in self.maps]


def forest(seed, n_trees=50):
    return lambda: scenes.forest(n_trees=n_trees, levels=6, n_lights=16, seed=seed)


@pytest.mark.parametrize("layout", [BEVY, PERMUTED, PACKED], ids=["bevy", "permuted", "packed40"])
def test_dense_sparse_and_static_frames(layout):
    tw = Twin(forest(3), seed=3, layout=layout)
    try:
        for pattern in ("dense", "dense", "sparse", "static", "sparse", "dense", "static", "sparse"):
            tw.frame(pattern)
        tw.frame("sparse", which=abi.RD_TRANSFORM)
        tw.frame("static", which=abi.RD_GLOBAL_TRANSFORM)
    finally:
        tw.close()


def test_ticks_across_the_wrap_and_past_max_change_age():
    tw = Twin(forest(5), seed=5, tick0=U32 - 25)
    try:
        for pattern in ("dense", "sparse", "dense", "sparse", "static"):   # this_run crosses 0 on the third frame
            tw.frame(pattern)
        tw.frame("sparse", step=M.MAX_CHANGE_AGE + 1000, ancient=True)    # last_run and the ticks at it: past the clamp
        tw.frame("sparse", step=7)
        tw.frame("dense")
    finally:
        tw.close()


def test_null_inputs_and_empty_tables():
    """One table without input columns, one without a GlobalTransform column, one with a GlobalTransform column but no
    ticks, newer mapped slots at and past len, a len-0 table and a capacity-0 table."""
    tw = Twin(forest(7), seed=7, no_inputs=(3,), no_gt=(2,), no_gt_ticks=(1,), past_len={0: 3, 2: 6},
              extra=[(0, 16), (0, 0)])
    try:
        for pattern in ("dense", "sparse", "static", "dense"):
            tw.frame(pattern)
    finally:
        tw.close()


def misaligned_inputs(tw):
    """Give every table a tick column at 4, 8, 12 or 0 bytes past a 16-byte boundary: the kernel's misaligned head."""
    ins = []
    for t, old in enumerate(tw.ins):
        cap = len(old.ticks)
        buf = np.zeros(cap * 4 + 64 + 4096, np.uint8)
        o = (-buf.ctypes.data) % 4096 + 4 * (t % 4)
        ticks = buf[o:o + cap * 4].view(np.uint32)
        ticks[:] = old.ticks
        ins.append(abi.HostInputs(old.trs, ticks, old.layout))
        tw.keep.append(buf)
    tw.ins = ins
    tw.register()


def test_lengths_around_warp_and_chunk_steps_beside_a_4096_slot_table():
    lengths = [0, 1, 2, 3, 5, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257]

    def scene():
        return scenes.many_cubes(4096 + sum(lengths), n_lights=4, seed=9)

    sc = scene()
    order = np.random.default_rng(9).permutation(sc.n)
    groups, o = [order[:4096].tolist()], 4096
    for n in lengths:
        groups.append(order[o:o + n].tolist()); o += n
    tw = Twin(scene, seed=9, groups=groups, headroom=3)
    try:
        tw.a.sc.roots = tw.b.sc.roots = np.arange(sc.n, dtype=np.uint32)    # every cube is a root
        misaligned_inputs(tw)
        for pattern in ("dense", "sparse", "dense", "static"):
            tw.frame(pattern, n_gt=40)
    finally:
        tw.close()


def test_queued_map_changes_moves_edits_and_compaction():
    tw = Twin(forest(11, n_trees=40), seed=11)
    try:
        tw.frame("dense")
        # two rows of one table trade slots, queued, right before the read: the bytes travel with their entities
        t = 2
        m = tw.maps[t]
        for x, y in ((0, 5), (5, 9), (1, 0)):
            rx, ry = int(m[x]), int(m[y])
            for tabs in (tw.tabs_a, tw.tabs_b):
                for k in COLUMNS:
                    col = raw(tabs[t], k)
                    col[[x, y]] = col[[y, x]]
            tw.ins[t].trs[[x, y]] = tw.ins[t].trs[[y, x]]
            tw.ins[t].ticks[[x, y]] = tw.ins[t].ticks[[y, x]]
            m[x], m[y] = ry, rx
            for c in (tw.a, tw.b):
                c.pipe.ctx.set_table_rows(t, x, [ry])
                c.pipe.ctx.set_table_rows(t, y, [rx])
        tw.frame("dense")
        for f in range(3):
            tw.edit(n_despawn=5, n_flat=5, n_kids=3, n_reparent=2)
            tw.frame(["dense", "sparse", "static"][f])
        tw.compact()
        tw.frame("sparse")
        tw.frame("dense")
    finally:
        tw.close()


def test_pipelined_frames_and_step_with_zero_changed_rows():
    tw = Twin(forest(13), seed=13)
    try:
        tw.frame("dense")
        for f in range(4):
            tw.frame("sparse", kind="step")
        # back-to-back STAGE_ALL frames: frame f is written, read and run without a write-back; frame f+1's read is
        # enqueued behind it with the columns left alone, so nothing is newer
        a, b = tw.a, tw.b
        L, R = tw.last, (tw.last + 10) & U32
        tw.game(L, R, "sparse", 12, RD_ALL)
        (rt, tv), (rg, gv) = M.as_uploads(*M.read(tw.model_tables(), tw.layout, RD_ALL, L, R))
        a.pipe.ctx.read_tables(RD_ALL, L, R)
        b.pipe.ctx.upload_transforms_scattered(rt, tv)
        b.pipe.ctx.write_global_transforms_scattered(rg, gv)
        for c in (a, b):
            scenes.advance_cameras(c.sc, 0.05)
            c.pipe.update_views()
        planes = np.stack([np.ctypeslib.as_array(v.half_spaces).reshape(6, 4).copy() for v in a.pipe.views])
        with oracle_marks(a.world):
            _, _, lists, _ = a.world.frame(planes)
        a.world.last_lists = [l if l is not None else a.world.last_lists[v] for v, l in enumerate(lists)]
        for c in (a, b):
            c.pipe.run_frame()
            c.pipe.read_feedback()
        L2, R2 = R, (R + 10) & U32
        a.pipe.ctx.read_tables(RD_ALL, L2, R2)
        for c in (a, b):
            scenes.advance_cameras(c.sc, 0.05)
            c.pipe.update_views()
        with oracle_marks(a.world):
            compare_frame(a.pipe, a.world, tw.f)
        b.pipe.run_frame(); b.pipe.read_feedback()
        for c in (a, b):
            c.pipe.ctx.writeback_tables(3, R2, R2)
            c.pipe.ctx.synchronize()
        tw.last = R2; tw.f += 1
        tw.compare()
        tw.frame("sparse")
    finally:
        tw.close()


def test_errors_leave_the_registry_as_it_was():
    tw = Twin(forest(17, n_trees=20), seed=17)
    try:
        c = tw.a.pipe.ctx
        tw.frame("dense")
        descs = tw.descs(tw.tabs_a)
        ins = tw.inputs()
        good = ins[0]
        cases = [
            (descs, ins, (48, 18, 0, 30)),                               # a field not 4-byte aligned
            (descs, ins, (48, 40, 0, 28)),                               # translation runs past stride
            (descs, ins, (48, 8, 0, 28)),                                # translation overlaps rotation
            (descs, ins, (46, 16, 0, 28)),                               # stride not 4-byte aligned
            (descs, ins, None),                                          # no layout
            (descs, [abi.TableInputs(good.trs.ctypes.data, None)] + ins[1:], BEVY),      # one pointer NULL
            (descs, [abi.TableInputs(None, good.ticks.ctypes.data)] + ins[1:], BEVY),
            (descs, [abi.TableInputs(good.trs.ctypes.data + 2, good.ticks.ctypes.data)] + ins[1:], BEVY),   # misaligned
            (descs, [abi.TableInputs(good.trs.ctypes.data, good.ticks.ctypes.data + 1)] + ins[1:], BEVY),
        ]
        for d, i, lay in cases:
            with pytest.raises(abi.B200VisError) as e:
                c.set_tables_ex(d, i, lay)
            assert e.value.code == INVALID_ARG, str(e.value)
        tw.frame("dense")
        tw.frame("sparse")
    finally:
        tw.close()
    fresh = abi.Context(64)
    try:
        with pytest.raises(abi.B200VisError) as e:
            fresh.read_tables()
        assert e.value.code == NOT_READY
        fresh.set_tables([])
        with pytest.raises(abi.B200VisError) as e:
            fresh.read_tables()
        assert e.value.code == NOT_READY
    finally:
        fresh.close()
    wide = abi.Context(64, world_size=2, rank=0)
    try:
        with pytest.raises(abi.B200VisError) as e:
            wide.read_tables()
        assert e.value.code == UNSUPPORTED
    finally:
        wide.close()


def test_input_registrations_are_released():
    torch = pytest.importorskip("torch")
    cudart = torch.cuda.cudart()
    tabs, _tb = abi.host_tables([50, 7])
    ins, buf = abi.host_table_inputs([300, 40])
    page = (buf.ctypes.data + 4095) // 4096 * 4096

    def free_to_register():
        rc = int(cudart.cudaHostRegister(page, 4096, 0))
        if rc == 0:
            assert int(cudart.cudaHostUnregister(page)) == 0
        return rc == 0
    for release in ("set_tables", "no_inputs", "destroy"):
        c = abi.Context(64)
        try:
            c.set_tables_ex(tabs, ins, BEVY)
            assert not free_to_register()                   # registered by the library
            if release == "set_tables":
                c.set_tables([])
            elif release == "no_inputs":
                c.set_tables_ex(tabs)
            if release != "destroy":
                assert free_to_register(), release
        finally:
            c.close()
        assert free_to_register(), release


def test_experiment_tile_kernel_is_unsupported_after_a_gt_read():
    run_case("import numpy as np, bevy_b200 as bb\n"
             "from bevy_b200 import abi\n"
             "sc = scenes.forest(n_trees=20, levels=5, n_lights=4)\n"
             "p = bb.VisibilityPipeline(sc)\n"
             "p.run_frame()\n"
             "tabs, buf = abi.host_tables([sc.n], tick_fill=5)\n"
             "ins, ibuf = abi.host_table_inputs([sc.n], tick_fill=5)\n"
             "p.ctx.set_tables_ex(tabs, ins, abi.BEVY_TRANSFORM_LAYOUT)\n"
             "p.ctx.set_table_rows(0, 0, np.arange(sc.n, dtype=np.uint32))\n"
             "p.ctx.read_tables(abi.RD_TRANSFORM, 5, 10)\n"
             "p.ctx.run(bb.STAGE_ALL)\n"
             "p.ctx.read_tables(abi.RD_GLOBAL_TRANSFORM, 10, 20)\n"
             "try:\n"
             "    p.ctx.run(bb.STAGE_ALL); raise SystemExit('run after a GlobalTransform read succeeded')\n"
             "except bb.B200VisError as e:\n"
             "    assert e.code == 8 and 'B200VIS_TILE_KERNEL=lean' in str(e), str(e)\n"
             "p.ctx.synchronize()\n"
             "p.close()\n", {"B200VIS_TILE_KERNEL": "lean"})


BENCH_SHARE = """
from test_gpu_table_read import Twin
make = lambda: scenes.forest(4903, 8, 512, seed=11)   # config #5 on 8 GPUs: one rank's 1,250,265 rows + 512 lights
tw = Twin(make, seed=31, churn_headroom=0, headroom=64)
try:
    chunks = sum((t.len + 127) // 128 for t in tw.tabs_a)
    assert chunks > 8 * 1184, chunks                  # the read's grid-stride loop goes round more than once
    tw.frame("dense", n_gt=200)
    tw.frame("sparse", n_gt=50)
finally:
    tw.close()
"""


def test_one_ranks_share_of_config5_in_shuffled_tables():
    # the case's interpreter loads the library this one does
    run_case(BENCH_SHARE, {k: os.environ[k] for k in ("B200VIS_LIB",) if k in os.environ}, timeout=1500)
