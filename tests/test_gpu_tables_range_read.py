"""b200vis_read_tables(RD_CULL_INPUTS) with b200vis_set_table_visibility_ranges attached: the VisibilityRange parameters
read straight from the caller's archetype tables, in step with a twin context fed by b200vis_upload_visibility_ranges.

Every scenario runs the twin of test_gpu_tables_cull_read.py.  Context A registers its tables with Transform inputs,
cull inputs and VisibilityRange columns and reads them.  Context B gets the bounds and flags the model of
tests/table_cull_model.py gives each row through b200vis_upload_bounds, and the range parameters the model of
tests/table_range_model.py gives each row through b200vis_upload_visibility_ranges (check_visibility_ranges as the
device evaluated it before this change).  The "game" overwrites every range column without a tick and stamps a few
slots with newer ticks.  After every frame A is checked against the C oracle (orc_check_visibility_ranges, the cull and
the point-light shadow pass with a LOD-origin range bit), and A and B are compared: the range masks, visible lists and
class masks, ViewVisibility, and the point, spot and cascade shadow lists."""
import os
import textwrap

import numpy as np
import pytest

from bevy_b200 import abi, scenes
import table_cull_model as CM
import table_range_model as RM
from parity import compare_frame
from test_gpu_bench_scale import run_case
from test_gpu_compaction import renumber
from test_gpu_external_gt import oracle_marks
from test_gpu_table_read import RD_ALL
from test_gpu_table_writeback import LIGHTS
import table_read_model as M
from test_gpu_tables_cull_read import (BASE, BOTH, FLAGS_ONLY, LIGHT, NFC, NOCPU, SPHERE, CullTwin, scene_with_shadows,
                                       visible_classes)

pytestmark = pytest.mark.gpu

NONE = abi.UNMAPPED
U32 = 0xFFFFFFFF
INVALID_ARG, NOT_READY, UNSUPPORTED = 1, 7, 8


class RangeTwin(CullTwin):
    """CullTwin whose context A also reads VisibilityRange columns from the tables in `ranged` (indices over the split's
    tables and the extra ones); those tables' cull inputs carry HAS_VIS_RANGE."""

    def __init__(self, make_scene, seed, struct="bevy", ranged=(0, 1, 2), **kw):
        self.struct, self.rlayout = struct, RM.abi_layout(struct)
        self.ranged, self.attached = set(ranged), True
        self.rgs = None
        self.se, self.ua = np.zeros((0, 2), np.uint32), np.zeros(0, np.uint8)
        self.rtold = set()
        self.extra_pos = None                               # range views past the cameras (more than 32 are dropped)
        super().__init__(make_scene, seed, **kw)
        for c in (self.a, self.b):                          # each culled view reads its own bit unless the scene says
            if c.sc.view_range_index is None:
                c.sc.view_range_index = np.arange(len(c.sc.cameras), dtype=np.int8)

    def build(self, groups):
        caps = [len(g) + self.headroom for g in groups] + [c for _, c in self.extra]
        self.rgs, buf = abi.host_table_ranges(caps, self.rlayout, tick_fill=getattr(self, "clast", self.last))
        super().build(groups)
        self.keep.append(buf)

    def register(self):
        if self.culls is not None:
            for t, c in enumerate(self.culls):
                c.flags = (c.flags | CM.F_RANGE) if t in self.ranged else (c.flags & ~CM.F_RANGE)
        super().register()
        if self.culls is not None and self.attached:
            self.attach()

    def attach(self):
        self.a.pipe.ctx.set_table_visibility_ranges([r if t in self.ranged else None for t, r in enumerate(self.rgs)], self.rlayout)

    def detach(self):
        """NULL, 0: the rows keep their parameters; the next attach is one after none."""
        self.attached, self.none = False, True
        self.a.pipe.ctx.set_table_visibility_ranges(None)

    def reattach(self):
        """After a detach, or a cull read while unattached, every ranged table is read in full; right after set_tables
        dropped the attachment, only tables whose entry changed are."""
        self.attached = True
        self.attach()
        if getattr(self, "none", False):
            for t in self.ranged:
                self.fresh[t][:] = True
        self.none = False

    def range_tables(self):
        return [RM.RangeTable(tab.len, tab.capacity, self.maps[t], self.fresh[t],
                              ranges=self.rgs[t].ranges if t in self.ranged and self.attached else None, ticks=self.rgs[t].ticks)
                for t, tab in enumerate(self.tabs_a)]

    def grow(self):
        n = self.a.sc.n
        if len(self.ua) < n:
            k = n - len(self.ua)
            self.se = np.concatenate([self.se, np.zeros((k, 2), np.uint32)])   # what an edit gives a new row
            self.ua = np.concatenate([self.ua, np.zeros(k, np.uint8)])

    def compact(self):
        """The Twin's device compaction, with the range state renumbered beside the rows."""
        o2n = self.a.pipe.ctx.compact_topology().astype(np.int64)
        o2n_b = self.b.pipe.ctx.compact_topology().astype(np.int64)
        assert (o2n == o2n_b).all()
        keep = np.nonzero(o2n != NONE)[0]
        ext = np.zeros(len(keep), np.uint8); ext[o2n[keep]] = self.a.world.ext[keep]
        for c in (self.a, self.b):
            renumber(c, o2n)
        self.a.world.ext = ext
        self.maps = [np.where(m != NONE, o2n[np.minimum(m, len(o2n) - 1)], NONE).astype(np.uint32) for m in self.maps]
        self.grow()
        se, ua = np.zeros((len(keep), 2), np.uint32), np.zeros(len(keep), np.uint8)
        se[o2n[keep]], ua[o2n[keep]] = self.se[keep], self.ua[keep]
        self.se, self.ua = se, ua

    def boundary(self, n_rows=6):
        """Rows of ranged tables whose distance to range view 0 is exactly start (in) or exactly end (out), use_aabb off,
        on a frame that moves nothing.  Returns (rows at start, rows at end)."""
        sc, gt = self.a.sc, self.a.world.gt
        p = np.asarray(self.range_pos()[0], np.float32)
        at_start, at_end = [], []
        for t in sorted(self.ranged):
            if CM.ARCHETYPES[self.arch_of(t)]["flags"] & CM.F_NO_CPU:
                continue
            for s in np.nonzero(self.maps[t][:self.tabs_a[t].len] != NONE)[0][:n_rows]:
                r = int(self.maps[t][s])
                m = gt[r, 9:12].astype(np.float32)
                dx, dy, dz = p - m
                d = np.sqrt(np.float32(np.float32(dx * dx + dy * dy) + dz * dz), dtype=np.float32)
                if len(at_start) <= len(at_end):
                    RM.put(self.rgs[t].ranges, self.struct, [s], [d], [d + np.float32(1000)], [0]); at_start.append(r)
                else:
                    RM.put(self.rgs[t].ranges, self.struct, [s], [np.float32(0)], [d], [0]); at_end.append(r)
                self.rgs[t].ticks[s] = (self.clast + 5) & U32
        return at_start, at_end

    def arch_of(self, t):
        k = len(self.tabs_a) - len(self.extra)
        return self.extra_archs[t - k] if t >= k else (LIGHT if t == LIGHTS else BASE)

    def range_pos(self):
        pos = np.stack([np.asarray(cam.gt, np.float32)[9:12] for cam in self.a.sc.cameras])
        return pos if self.extra_pos is None else np.concatenate([pos, self.extra_pos])

    def cframe(self, pattern="sparse", n_bounds=8, n_iv=4, n_ranges=8, which=RD_ALL, step=10, restore=True, items=False,
               nan=False, edge=False):
        """One frame, as CullTwin.cframe, with the range columns read on A and uploaded on B.  nan: two stamped slots get
        NaN margins.  edge: rows exactly at start / end of range view 0 (pass pattern='static', which=0)."""
        a, b = self.a, self.b
        L, R = self.last, (self.last + step) & U32
        Lc, Rc = self.clast, (self.clast + step + 3) & U32
        if not self.attached:                               # this cull read drops the kept entries (b200vis.h)
            self.none = True
        for c in (a, b):
            scenes.advance_cameras(c.sc, 0.05)
        moved, written = self.game(L, R, pattern, 12, which)
        tabs = self.cull_tables()
        CM.game(tabs, self.blayout, self.rng, Lc, Rc, n_bounds, n_iv)
        if restore:
            for t, fr in enumerate(self.fresh):
                self.restore(t, np.nonzero(fr[:self.tabs_a[t].len])[0])
        rtabs = self.range_tables()
        stamped = RM.game(rtabs, self.struct, self.rng, Lc, Rc, n_ranges)
        if nan and stamped:
            for t, s in stamped[:2]:
                RM.put(self.rgs[t].ranges, self.struct, [s], [np.float32(np.nan)], [np.float32(100)], [1])
            t, s = stamped[-1]
            RM.put(self.rgs[t].ranges, self.struct, [s], [np.float32(0)], [np.float32(np.nan)], [0])
        edges = self.boundary() if edge else ([], [])
        got_t, got_g = M.read(self.model_tables(), self.layout, which, L, R)
        assert set(got_t) == moved and set(got_g) == written, "the scenario itself is off"
        (rt, tv), (rg, gv) = M.as_uploads(got_t, got_g)
        sc = a.sc
        before = sc.flags.copy()
        before[np.asarray(sorted(moved), np.int64)] |= CM.F_TCHANGED
        bounds, flags, fresh = CM.read(tabs, self.blayout, Lc, Rc, sc.bounds.view(np.uint32), before)
        self.grow()
        right = RM.read(rtabs, self.struct, Lc, Rc, self.se, self.ua)
        for m in RM.MUTANTS:
            if not RM.same(right, RM.read(rtabs, self.struct, Lc, Rc, self.se, self.ua, mutant=m)):
                self.rtold.add(m)
        self.se, self.ua = right[0], right[1]
        a.pipe.ctx.read_tables(which, L, R)
        a.pipe.ctx.read_tables(abi.RD_CULL_INPUTS, Lc, Rc)
        if len(rt):
            b.pipe.ctx.upload_transforms_scattered(rt, tv)
        if len(rg):
            b.pipe.ctx.write_global_transforms_scattered(rg, gv)
        n = sc.n
        for s in (a.sc, b.sc):
            s.bounds[:] = bounds.view(np.float32)
            s.flags[:] = flags & (0xFF ^ CM.F_TCHANGED)
            s.range_se = self.se[:n].view(np.float32).copy()
            s.range_use_aabb = self.ua[:n].copy()
            s.range_view_pos = self.range_pos()[:32]           # check_visibility_ranges takes the first 32 views
            s.range_mask = np.zeros(n, np.uint32)
        self.fresh = fresh
        b.pipe.ctx.upload_bounds(0, b.sc.bounds, b.sc.flags, b.sc.class_mask)
        b.pipe.ctx.upload_visibility_ranges(0, b.sc.range_se, b.sc.range_use_aabb)
        for c in (a, b):
            c.pipe.ctx.set_visibility_range_views(self.range_pos())
            c.pipe.update_views()
        with oracle_marks(a.world):
            compare_frame(a.pipe, a.world, self.f)
        b.pipe.run_frame()
        b.pipe.read_feedback()
        b.pipe.check_point_light_mesh_visibility(b.sc.shadow_lights, b.sc.shadow_near_z, b.sc.shadow_lod_origin)
        pa, pb = a.pipe.ctx, b.pipe.ctx
        tag = f"frame {self.f}"
        ra, rb = pa.download_visibility_ranges(0, n), pb.download_visibility_ranges(0, n)
        assert (ra == rb).all(), f"{tag}: VisibleEntityRanges masks differ on rows {np.nonzero(ra != rb)[0][:8]}"
        assert (ra == a.sc.range_mask).all()
        if edge:
            assert all(ra[r] & 1 for r in edges[0]), f"{tag}: a row exactly at start_margin.start is out of range"
            assert not any(ra[r] & 1 for r in edges[1]), f"{tag}: a row exactly at end_margin.end is in range"
        for face in range(6):
            sa, sb = pa.download_shadow_visible(0, face), pb.download_shadow_visible(0, face)
            assert len(sa) == len(sb) and (sa == sb).all(), f"{tag}: point-light shadow face {face} differs"
        if items:
            self.items(pa, pb, tag)
        for c in (a, b):
            c.pipe.ctx.writeback_tables(abi.WB_GLOBAL_TRANSFORM | abi.WB_VIEW_VISIBILITY, R, R)
            c.pipe.ctx.synchronize()
        self.last, self.clast = R, Rc
        self.compare()
        for v in range(len(a.sc.cameras)):
            ca, cb = visible_classes(pa, v), visible_classes(pb, v)
            assert len(ca) == len(cb) and (ca == cb).all(), f"{tag}: view {v} class masks differ"
        self.f += 1

    def items(self, pa, pb, tag):
        """A point, a spot and a cascade item, all gated by range bit 0 (the shadow LOD origin / the cascade's view)."""
        sc = self.a.sc
        out = []
        for kind, o in ((0, 2), (1, 3)):
            row = int(sc.light_row[o])
            gt, _ = pa.download_global_transforms(row, 1, want_changed=False)
            fr = abi.host_point_light_frusta(gt[0], float(sc.light_range[o]))
            out.append(dict(kind=kind, light_row=row, range=float(sc.light_range[o]), range_view_index=0,
                            frusta=fr if kind == 0 else fr[o % 6]))
        hs = np.ctypeslib.as_array(self.a.pipe.views[0].half_spaces).reshape(6, 4).copy()
        out.append(dict(kind=2, range_view_index=0, frusta=hs))
        for c in (pa, pb):
            c.set_shadow_items(out)
            c.run_shadow_culling()
        for i, faces in ((0, range(6)), (1, range(1)), (2, range(1))):
            for face in faces:
                sa, sb = pa.download_shadow_visible(i, face), pb.download_shadow_visible(i, face)
                assert len(sa) == len(sb) and (sa == sb).all(), f"{tag}: shadow item {i} face {face} differs"


# ---- the scenarios (each in its own interpreter, as in test_gpu_tables_cull_read.py) ----

def scenario_frames(struct):
    tw = RangeTwin(scene_with_shadows(3), seed=3, struct=struct)
    try:
        tw.cframe("static", n_bounds=0, n_iv=0, n_ranges=0)   # the first read is a full one
        tw.cframe("static", n_bounds=0, n_iv=0, n_ranges=0)   # nothing newer: every bypass write is left alone
        tw.cframe("sparse", n_ranges=12, nan=True)
        tw.cframe("static", which=0, n_ranges=0, edge=True)   # exactly at start (in) and end (out)
        tw.cframe("dense", n_bounds=40, n_iv=20, n_ranges=30, items=True)
        return tw.rtold
    finally:
        tw.close()


def scenario_wrap():
    tw = RangeTwin(scene_with_shadows(5), seed=5, tick0=U32 - 40)
    try:
        for f in range(6):                                  # both tick pairs cross 0 on the way
            tw.cframe(["sparse", "static", "dense"][f % 3], n_ranges=10, items=f == 5)
        return tw.rtold
    finally:
        tw.close()


def scenario_moves():
    """Rows move out of a ranged table into unranged ones and into a ranged NoCpuCulling table and a ranged Sphere-only
    table (use_aabb without an Aabb), and back."""
    extra = (NFC, SPHERE, BOTH, NOCPU, FLAGS_ONLY)
    tw = RangeTwin(scene_with_shadows(7), seed=7, ranged=(2, 5 + 1, 5 + 2, 5 + 3), extra_archs=extra)
    try:
        tw.cframe("sparse")
        leaves, first_extra = 2, 5
        for k in range(len(extra)):
            for _ in range(3):
                tw.move(leaves, int(tw.rng.integers(0, tw.tabs_a[leaves].len)), first_extra + k)
        tw.cframe("sparse", restore=False)
        tw.cframe("static", n_bounds=0, n_iv=0)
        for k in (0, 1, 3):                                 # back into the ranged leaf table
            tw.move(first_extra + k, 0, leaves)
        tw.move(leaves, 1, 0)                               # out of it, into an unranged one
        tw.cframe("sparse", restore=False)
        tw.cframe("dense", items=True)
        return tw.rtold
    finally:
        tw.close()


def scenario_realloc():
    """Table reallocation, detach / re-attach, set_tables dropping the attachment (re-attached before and after a cull
    read, with a row moved from the unranged leaf table into a ranged one in between), edits and a device compaction."""
    tw = RangeTwin(scene_with_shadows(11), seed=11, ranged=(0, 1))
    try:
        tw.cframe("sparse")
        tw.build(tw.groups_now())                           # every table reallocated: read in full again
        tw.cframe("dense", n_bounds=0, n_iv=0, restore=False)
        tw.detach()                                         # detached: the rows keep their parameters
        tw.cframe("sparse", n_ranges=0)
        tw.reattach()
        tw.cframe("sparse", restore=False)
        tw.attached = False
        tw.register()                                       # set_tables drops the attachment ...
        tw.reattach()                                       # ... and attaching it again unchanged reads nothing in full
        tw.cframe("static", n_ranges=0)
        tw.attached = False
        tw.register()                                       # dropped again, and a row moves into a ranged table
        tw.move(2, 0, 1)
        tw.cframe("sparse", n_ranges=0)                     # a cull read before the re-attach: it gets no parameters
        tw.reattach()                                       # ... so the re-attach reads every ranged table in full
        tw.cframe("sparse")
        for f in range(2):
            tw.edit(n_despawn=5, n_flat=5, n_kids=3, n_reparent=2)
            tw.cframe(["sparse", "dense"][f])
        tw.compact()
        tw.cframe("sparse")
        tw.cframe("static", n_bounds=0, n_iv=0, items=True)
        return tw.rtold
    finally:
        tw.close()


def many_views_scene(n_cameras):
    def make():
        sc = scenes.many_cameras_lights(min(n_cameras, 16), forest_kwargs=dict(n_trees=60, levels=5))
        sc.trs[sc.roots, 0:3] *= np.float32(0.03)
        sc.cameras = (sc.cameras * 2)[:n_cameras]
        sc.shadow_lights = np.array([0], np.uint32)
        sc.shadow_caster = np.ones(sc.n, np.uint8); sc.shadow_caster[sc.light_row] = 0
        sc.shadow_near_z, sc.shadow_lod_origin = 0.1, 0
        sc.view_range_index = np.arange(n_cameras, dtype=np.int8)
        sc.view_range_index[1] = -1                         # a culled view outside the range map
        return sc
    return make


def scenario_views(n_cameras):
    tw = RangeTwin(many_views_scene(n_cameras), seed=13)
    try:
        if n_cameras == 32:                                 # 34 range views: the two past the 32nd are dropped
            tw.extra_pos = np.array([[0.0, 1.0, 0.0], [0.5, 0.5, 0.5]], np.float32)
        for f in range(3):
            tw.cframe(["static", "sparse", "dense"][f], n_ranges=12)
    finally:
        tw.close()


def scenario_errors():
    tw = RangeTwin(scene_with_shadows(17, n_trees=20), seed=17)
    try:
        c = tw.a.pipe.ctx
        tw.cframe("sparse")
        good = [r.desc() if t in tw.ranged else abi.TableVisibilityRanges() for t, r in enumerate(tw.rgs)]
        g0 = good[0]
        lay = tw.rlayout

        def with0(**kw):
            d = abi.TableVisibilityRanges(g0.ranges, g0.changed_ticks)
            for k, v in kw.items():
                setattr(d, k, v)
            return [d] + good[1:]
        unranged = max(set(range(len(good))) - tw.ranged)
        extra = list(good); extra[unranged] = g0
        missing = list(good); missing[0] = abi.TableVisibilityRanges()
        cases = [
            (good[:-1], lay),                               # n_tables differs from the registry's size
            (with0(changed_ticks=None), lay),               # half-NULL pair
            (with0(ranges=g0.ranges + 2), lay),             # misaligned
            (with0(changed_ticks=g0.changed_ticks + 1), lay),
            (extra, lay),                                   # a range column on a table without HAS_VIS_RANGE
            (missing, lay),                                 # HAS_VIS_RANGE without a range column
            (good, None),                                   # no layout
            (good, (20, 2, 12, 16)),                        # a float not 4-byte aligned
            (good, (22, 0, 12, 16)),                        # stride not 4-byte aligned
            (good, (16, 0, 12, 16)),                        # use_aabb past stride
            (good, (20, 0, 20, 16)),                        # end past stride
            (good, (20, 8, 8, 16)),                         # overlapping floats
            (good, (20, 0, 12, 14)),                        # use_aabb inside end
        ]
        for d, lay_ in cases:
            try:
                c.set_table_visibility_ranges(d, lay_)
            except abi.B200VisError as e:
                assert e.code == INVALID_ARG, str(e)
            else:
                raise AssertionError(f"set_table_visibility_ranges accepted {lay_}")
        # the cull inputs may not break the rule while ranges are attached
        for t, flip in ((0, True), (unranged, False)):
            descs = [x.desc() for x in tw.culls]
            descs[t].flags ^= CM.F_RANGE
            try:
                c.set_table_cull_inputs(descs, tw.blayout)
            except abi.B200VisError as e:
                assert e.code == INVALID_ARG, str(e)
            else:
                raise AssertionError(f"set_table_cull_inputs accepted table {t} with HAS_VIS_RANGE flipped")
        tw.cframe("sparse")                                 # the previous attachment stays in force
        tw.cframe("static", n_bounds=0, n_iv=0)
    finally:
        tw.close()
    for kw, code in (({}, NOT_READY), (dict(world_size=2, rank=0), UNSUPPORTED)):
        ctx = abi.Context(64, **kw)
        try:
            try:
                ctx.set_table_visibility_ranges([])
            except abi.B200VisError as e:
                assert e.code == code, str(e)
            else:
                raise AssertionError("set_table_visibility_ranges without a registry succeeded")
        finally:
            ctx.close()


def scenario_launches():
    """A cull read launches one kernel with or without ranges attached, and a frame launches the same number of kernels
    either way: the range read is an instantiation of the same kernel, and nothing new launches without it."""
    tw = RangeTwin(scene_with_shadows(19, n_trees=20), seed=19)
    try:
        tw.cframe("sparse")
        c = tw.a.pipe.ctx

        def count():
            c.synchronize()
            k0 = abi.kernel_launch_count()
            c.read_tables(abi.RD_CULL_INPUTS, tw.clast, tw.clast)
            k1 = abi.kernel_launch_count()
            tw.a.pipe.run_frame()
            tw.a.pipe.read_feedback()
            return k1 - k0, abi.kernel_launch_count() - k1
        with_ranges = count()
        c.set_table_visibility_ranges(None)
        without = count()
        assert with_ranges == without and with_ranges[0] == 1, (with_ranges, without)
    finally:
        tw.close()


def scenario_bench_world():
    def make():
        sc = scenes.forest(3922, 8, 256)                    # config #3: 1,000,366 rows in its four archetype tables
        sc.shadow_lights = np.array([0], np.uint32)
        sc.shadow_caster = np.ones(sc.n, np.uint8); sc.shadow_caster[sc.light_row] = 0
        sc.shadow_near_z, sc.shadow_lod_origin = 0.1, 0
        return sc
    tw = RangeTwin(make, seed=23, ranged=range(5), churn_headroom=0, headroom=64)
    try:
        tw.cframe("static", n_bounds=0, n_iv=0, n_ranges=0)   # every slot read in full: every row ranged
        tw.cframe("sparse", n_bounds=64, n_iv=32, n_ranges=64, items=True)
    finally:
        tw.close()


STRUCTS = ("bevy", "ua_first", "reversed")
# scenario -> the model mutants its frames must tell apart
EXPECT = {
    "frames_reversed": {"end_margin_start", "equal_tick_newer", "use_aabb_bit0"},
    "moves": {"ignore_fresh"},
    "realloc": {"ignore_fresh"},
}
CALLS = dict({f"frames_{s}": f"scenario_frames({s!r})" for s in STRUCTS},
             wrap="scenario_wrap()", moves="scenario_moves()", realloc="scenario_realloc()", views_9="scenario_views(9)",
             views_32="scenario_views(32)", errors="scenario_errors()", launches="scenario_launches()",
             pipeline_off="scenario_frames('bevy')", bench_world="scenario_bench_world()")
ENV = {"pipeline_off": {"B200VIS_PIPELINE": "0"}}


@pytest.mark.parametrize("name", list(CALLS))
def test_scenario(name):
    code = textwrap.dedent(f"""
        import test_gpu_tables_range_read as T
        told = T.{CALLS[name]}
        missing = T.EXPECT.get({name!r}, set()) - (told or set())
        assert not missing, f"the model mutants {{sorted(missing)}} were not told apart"
    """)
    env = {k: os.environ[k] for k in ("B200VIS_LIB",) if k in os.environ}
    env.update(ENV.get(name, {}))
    run_case(code, env, timeout=1500)
