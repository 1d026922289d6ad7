"""b200vis_read_tables(RD_CULL_INPUTS) on the device: Aabb, Sphere and InheritedVisibility read straight from the
caller's archetype tables, in step with a twin context fed by b200vis_upload_bounds.

Every scenario runs two contexts on the same scene (the Twin of test_gpu_table_read.py).  Context A registers its tables
with Transform inputs and cull inputs (b200vis_set_table_cull_inputs) and reads both, each with its own tick pair.
Context B gets the device state the slot-by-slot model of tests/table_cull_model.py gives each row, through
b200vis_upload_bounds, and the Transform set of tests/table_read_model.py through the scattered upload.  The "game"
(table_cull_model.game) overwrites every cull column with values that would flip visibility, without a tick, and stamps a
few slots with newer ticks; a slot that moved holds its entity's true values.  After every frame A is checked against the
C oracle, and A and B are compared bit for bit: visible lists and their class masks, ViewVisibility and its change bits,
the GlobalTransforms, the shadow-cull lists of one point light, and the tables both wrote back into."""
import ctypes as C
import os
import textwrap

import numpy as np
import pytest

from bevy_b200 import abi, scenes
import table_cull_model as CM
import table_read_model as M
from parity import compare_frame
from test_gpu_bench_scale import run_case
from test_gpu_external_gt import oracle_marks
from test_gpu_table_read import RD_ALL, Twin
from test_gpu_table_writeback import LIGHTS

pytestmark = pytest.mark.gpu

NONE = abi.UNMAPPED
U32 = 0xFFFFFFFF
INVALID_ARG, NOT_READY, UNSUPPORTED = 1, 7, 8
BASE, NFC, SPHERE, BOTH, NOCPU, LIGHT, IV_ONLY, FLAGS_ONLY = range(8)     # indices of CM.ARCHETYPES


def scene_with_shadows(seed, n_trees=40):
    def make():
        sc = scenes.forest(n_trees=n_trees, levels=6, n_lights=16, seed=seed)
        sc.shadow_lights = np.array([0], np.uint32)
        sc.shadow_caster = np.ones(sc.n, np.uint8); sc.shadow_caster[sc.light_row] = 0
        sc.shadow_near_z, sc.shadow_lod_origin = 0.1, 0
        return sc
    return make


def visible_classes(ctx, view):
    cnt = C.c_uint32(0)
    ctx._check(ctx._lib.b200vis_download_visible_classes(ctx._h, view, None, 0, C.byref(cnt)))
    out = np.zeros(max(cnt.value, 1), np.uint8)
    ctx._check(ctx._lib.b200vis_download_visible_classes(ctx._h, view, out.ctypes.data, len(out), C.byref(cnt)))
    return out[:cnt.value]


class CullTwin(Twin):
    """Twin whose context A also reads its cull inputs.  The light table has the point-light archetype of CM.ARCHETYPES,
    the other tables of the split the plain one; `extra_archs` adds empty tables of the given archetypes (targets of
    archetype moves)."""

    def __init__(self, make_scene, seed, blayout=CM.BEVY_LAYOUT, extra_archs=(), **kw):
        self.blayout, self.extra_archs = tuple(blayout), list(extra_archs)
        self.culls = None
        self.told = set()                                     # the mutants of CM.MUTANTS some frame's model state told apart
        super().__init__(make_scene, seed, extra=[(0, 48)] * len(extra_archs), **kw)
        self.clast = (self.last - 3) & U32
        self.restore_all()

    def build(self, groups):
        caps = [len(g) + self.headroom for g in groups] + [c for _, c in self.extra]
        self.culls, buf = abi.host_table_cull_inputs(caps, self.blayout, tick_fill=self.last)
        arch = [LIGHT if t == LIGHTS else BASE for t in range(len(groups))] + self.extra_archs
        for c, a in zip(self.culls, arch):
            c.has, c.flags = CM.ARCHETYPES[a]["has"], CM.ARCHETYPES[a]["flags"]
        self.fresh = [np.ones(c, bool) for c in caps]        # new columns: every table is read in full
        super().build(groups)
        self.held = [m.copy() for m in self.maps]
        self.keep.append(buf)
        if hasattr(self, "clast"):
            self.restore_all()

    def register(self):
        super().register()
        if self.culls is not None:
            self.a.pipe.ctx.set_table_cull_inputs(self.culls, self.blayout)

    def cull_tables(self):
        out = []
        for t, (tab, c) in enumerate(zip(self.tabs_a, self.culls)):
            pick = lambda name, a: a if name in c.has else None
            out.append(CM.CullTable(tab.len, tab.capacity, self.maps[t], self.fresh[t], aabb=pick("aabb", c.aabb),
                                    aabb_ticks=pick("aabb", c.aabb_ticks), sphere=pick("sphere", c.sphere),
                                    sphere_ticks=pick("sphere", c.sphere_ticks), iv=pick("iv", c.iv),
                                    iv_ticks=pick("iv", c.iv_ticks), flags=c.flags, held=self.held[t]))
        return out

    def groups_now(self):
        """The rows of the split's tables as they are mapped now (the extra tables left out)."""
        k = len(self.maps) - len(self.extra)
        return [[int(r) for r in m[:tab.len] if r != NONE] for m, tab in zip(self.maps[:k], self.tabs_a[:k])]

    def restore(self, t, slots):
        """The slots hold their entities' true values (what the device state says), ticks left as they are."""
        c, sc = self.culls[t], self.a.sc
        slots = np.asarray([s for s in slots if s < len(self.maps[t]) and self.maps[t][s] != NONE], np.int64)
        if not len(slots):
            return
        rows = self.maps[t][slots].astype(np.int64)
        b = sc.bounds[rows]
        CM.put(c.aabb, slots, ((self.blayout[1], b[:, 0:3]), (self.blayout[2], b[:, 3:6])))
        CM.put(c.sphere, slots, ((self.blayout[4], b[:, 0:3]), (self.blayout[5], b[:, 3:4])))
        c.iv[slots] = sc.flags[rows] & CM.F_INHERITED

    def restore_all(self):
        for t in range(len(self.culls)):
            self.restore(t, np.arange(self.tabs_a[t].len))

    def cframe(self, pattern="sparse", n_bounds=8, n_iv=4, which=RD_ALL, step=10, restore=True, spot=False):
        """One frame: the propagate reads its Transform set with (L, R], the cull reads its inputs with its own pair.
        restore: the fresh slots hold their entities' true values (else the game's bypass writes, so that a full read
        shows).  spot: also cull one point and one spot light through b200vis_set_shadow_items on both contexts and
        compare their lists (a pass the oracle world does not follow, so only on a scenario's last frame)."""
        a, b = self.a, self.b
        L, R = self.last, (self.last + step) & U32
        Lc, Rc = self.clast, (self.clast + step + 3) & U32
        moved, written = self.game(L, R, pattern, 12, which)
        tabs = self.cull_tables()
        CM.game(tabs, self.blayout, self.rng, Lc, Rc, n_bounds, n_iv)
        if restore:
            for t, fr in enumerate(self.fresh):
                self.restore(t, np.nonzero(fr[:self.tabs_a[t].len])[0])
        got_t, got_g = M.read(self.model_tables(), self.layout, which, L, R)
        assert set(got_t) == moved and set(got_g) == written, "the scenario itself is off"
        (rt, tv), (rg, gv) = M.as_uploads(got_t, got_g)
        sc = a.sc
        # the device flags at the cull read: the rows the Transform read just marked carry F_TCHANGED
        before = sc.flags.copy()
        before[np.asarray(sorted(moved), np.int64)] |= CM.F_TCHANGED
        right = CM.read(tabs, self.blayout, Lc, Rc, sc.bounds.view(np.uint32), before)
        for m in CM.MUTANTS:
            if not CM.same(right, CM.read(tabs, self.blayout, Lc, Rc, sc.bounds.view(np.uint32), before, mutant=m)):
                self.told.add(m)
        bounds, flags, fresh = right
        a.pipe.ctx.read_tables(which, L, R)
        a.pipe.ctx.read_tables(abi.RD_CULL_INPUTS, Lc, Rc)
        if len(rt):
            b.pipe.ctx.upload_transforms_scattered(rt, tv)
        if len(rg):
            b.pipe.ctx.write_global_transforms_scattered(rg, gv)
        for s in (a.sc, b.sc):
            s.bounds[:] = bounds.view(np.float32)
            s.flags[:] = flags & (0xFF ^ CM.F_TCHANGED)
        b.pipe.ctx.upload_bounds(0, b.sc.bounds, b.sc.flags, b.sc.class_mask)
        self.fresh = fresh
        for c in (a, b):
            scenes.advance_cameras(c.sc, 0.05)
            if getattr(c.sc, "range_se", None) is not None:
                c.sc.range_view_pos = np.stack([np.asarray(cam.gt, np.float32)[9:12] for cam in c.sc.cameras])
                c.pipe.ctx.set_visibility_range_views(c.sc.range_view_pos)
            c.pipe.update_views()
        with oracle_marks(a.world):
            compare_frame(a.pipe, a.world, self.f)
        b.pipe.run_frame()
        b.pipe.read_feedback()
        b.pipe.check_point_light_mesh_visibility(b.sc.shadow_lights, b.sc.shadow_near_z, b.sc.shadow_lod_origin)
        pa, pb = a.pipe.ctx, b.pipe.ctx
        tag = f"frame {self.f}"
        if getattr(sc, "range_se", None) is not None:
            ra, rb = pa.download_visibility_ranges(0, sc.n), pb.download_visibility_ranges(0, sc.n)
            assert (ra == rb).all(), f"{tag}: VisibleEntityRanges masks differ on rows {np.nonzero(ra != rb)[0][:8]}"
        for face in range(6):
            sa, sb = pa.download_shadow_visible(0, face), pb.download_shadow_visible(0, face)
            assert len(sa) == len(sb) and (sa == sb).all(), f"{tag}: point-light shadow face {face} differs"
        if spot:
            self.spot_and_point(pa, pb, tag)
        for c in (a, b):
            c.pipe.ctx.writeback_tables(abi.WB_GLOBAL_TRANSFORM | abi.WB_VIEW_VISIBILITY, R, R)
            c.pipe.ctx.synchronize()
        self.last, self.clast = R, Rc
        self.compare()
        for v in range(len(a.sc.cameras)):
            ca, cb = visible_classes(pa, v), visible_classes(pb, v)
            assert len(ca) == len(cb) and (ca == cb).all(), f"{tag}: view {v} class masks differ"
        self.f += 1

    def spot_and_point(self, pa, pb, tag):
        """check_point_light_mesh_visibility's point and spot halves (b200vis_set_shadow_items) on both contexts."""
        sc = self.a.sc
        items = []
        for kind, o in ((0, 2), (1, 3)):
            row = int(sc.light_row[o])
            gt, _ = pa.download_global_transforms(row, 1, want_changed=False)
            fr = abi.host_point_light_frusta(gt[0], float(sc.light_range[o]))
            items.append(dict(kind=kind, light_row=row, range=float(sc.light_range[o]), frusta=fr if kind == 0 else fr[o % 6]))
        for c in (pa, pb):
            c.set_shadow_items(items)
            c.run_shadow_culling()
        for i, faces in ((0, range(6)), (1, range(1))):
            for face in faces:
                sa, sb = pa.download_shadow_visible(i, face), pb.download_shadow_visible(i, face)
                assert len(sa) == len(sb) and (sa == sb).all(), f"{tag}: shadow item {i} face {face} differs"

    def move(self, src, s, dst):
        """An archetype move with swap_remove, on both contexts: the row of (src, s) to the end of dst, src's last row
        into s.  Columns keep their pointers; len changes, so the registry is sent again (the cull inputs re-attached)."""
        ta, tb_ = self.tabs_a, self.tabs_b
        row = int(self.maps[src][s])
        last = ta[src].len - 1
        d = ta[dst].len
        assert d < ta[dst].capacity
        moved_row = int(self.maps[src][last])
        for c in (self.a, self.b):
            c.pipe.ctx.set_table_rows(dst, d, [row])
            if s != last:
                c.pipe.ctx.set_table_rows(src, s, [moved_row])
            c.pipe.ctx.set_table_rows(src, last, [NONE])
        self.held[src] = self.maps[src].copy()
        self.maps[dst][d] = row
        self.maps[src][s] = moved_row if s != last else NONE
        self.maps[src][last] = NONE
        for t, k in ((dst, d), (src, s), (src, last)):
            self.fresh[t][k] = True
        for tabs in (ta, tb_):
            tabs[dst].len += 1
            tabs[src].len -= 1
        self.ins[dst].trs[d] = self.ins[src].trs[s]; self.ins[dst].ticks[d] = self.ins[src].ticks[s]
        if s != last:
            self.ins[src].trs[s] = self.ins[src].trs[last]; self.ins[src].ticks[s] = self.ins[src].ticks[last]
        self.register()

    def unmap(self, t, s):
        """Slot s of table t below len loses its row (an entity without a device row: GlobalTransform without Transform)."""
        for c in (self.a, self.b):
            c.pipe.ctx.set_table_rows(t, s, [NONE])
        self.held[t] = self.maps[t].copy()
        self.maps[t][s] = NONE
        self.fresh[t][s] = True

    def groups_now(self):
        """The rows of the split's tables as they are mapped now (the extra tables left out)."""
        k = len(self.maps) - len(self.extra)
        return [[int(r) for r in m[:tab.len] if r != NONE] for m, tab in zip(self.maps[:k], self.tabs_a[:k])]


# ---- the scenarios.  Each runs in a fresh interpreter (run_case), and the file sorts after the other table tests: the
# twins register and release many small host buffers, and what an earlier test leaves on the heap decides whether a
# later test's pageable array shares a page with one of its registrations, the hazard b200vis.h's page rules describe.  Each asserts the model mutants its frames tell
# apart (EXPECT); tests/test_cpu_table_cull_model.py checks that together they cover every mutant. ----

def scenario_frames(layout_name):
    tw = CullTwin(scene_with_shadows(3), seed=3, blayout=LAYOUTS[layout_name])
    try:
        tw.cframe("static", n_bounds=0, n_iv=0)             # the first read is a full one
        tw.cframe("static", n_bounds=0, n_iv=0)             # nothing newer: every poisoned slot is left alone
        tw.cframe("sparse", n_bounds=12, n_iv=0)
        tw.cframe("static", n_bounds=0, n_iv=10)
        tw.cframe("dense", n_bounds=40, n_iv=20, spot=True)
        return tw.told
    finally:
        tw.close()


def scenario_wrap():
    tw = CullTwin(scene_with_shadows(5), seed=5, tick0=U32 - 40)
    try:
        for f in range(6):                                  # both tick pairs cross 0 on the way
            tw.cframe(["sparse", "static", "dense"][f % 3], n_bounds=10, n_iv=6, spot=f == 5)
        return tw.told
    finally:
        tw.close()


def with_ranges(make):
    """The scene with VisibilityRange data on every row (it applies to the rows of the F_RANGE archetype)."""
    def make2():
        sc = make()
        rng = np.random.default_rng(99)
        start = rng.uniform(0, 60, sc.n).astype(np.float32)
        sc.range_se = np.stack([start, start + rng.uniform(0, 120, sc.n).astype(np.float32)], 1)
        sc.range_use_aabb = rng.integers(0, 2, sc.n).astype(np.uint8)
        sc.view_range_index = np.arange(len(sc.cameras), dtype=np.int8)
        sc.range_view_pos = np.stack([np.asarray(c.gt, np.float32)[9:12] for c in sc.cameras])
        sc.range_mask = np.zeros(sc.n, np.uint32)
        return sc
    return make2


def scenario_moves():
    """Rows move out of the leaf table into NoFrustumCulling, Sphere-only, Aabb + Sphere (VisibilityRange), NoCpuCulling,
    InheritedVisibility-only and flags-only tables, and back; an unmapped slot below len; two light rows trade slots;
    a table keeps mapped rows past len."""
    tw = CullTwin(with_ranges(scene_with_shadows(7)), seed=7, extra_archs=(NFC, SPHERE, BOTH, NOCPU, IV_ONLY, FLAGS_ONLY),
                  past_len={0: 3})
    try:
        for c in (tw.a, tw.b):
            c.pipe.ctx.upload_visibility_ranges(0, c.sc.range_se, c.sc.range_use_aabb)
            c.pipe.ctx.set_visibility_range_views(c.sc.range_view_pos)
        tw.cframe("sparse")
        leaves, first_extra = 2, 5
        for k in range(len(tw.extra_archs)):
            for _ in range(3):
                tw.move(leaves, int(tw.rng.integers(0, tw.tabs_a[leaves].len)), first_extra + k)
        tw.cframe("sparse", restore=False)                  # the moved rows' slots hold bypass writes: read in full
        tw.cframe("static", n_bounds=0, n_iv=0)
        for k in (1, 4, 5):                                 # back into the leaf table
            tw.move(first_extra + k, 0, leaves)
        tw.unmap(leaves, 4)
        lt = tw.maps[LIGHTS]                                # the shadow light's row trades slots with another light
        x, y = int(np.nonzero(lt == tw.a.sc.light_row[0])[0][0]), int(np.nonzero(lt == tw.a.sc.light_row[1])[0][0])
        rx, ry = int(lt[x]), int(lt[y])
        for c in (tw.a, tw.b):
            c.pipe.ctx.set_table_rows(LIGHTS, x, [ry])
            c.pipe.ctx.set_table_rows(LIGHTS, y, [rx])
        lt[x], lt[y] = ry, rx
        tw.fresh[LIGHTS][[x, y]] = True
        tw.cframe("sparse", restore=False)
        tw.cframe("dense", spot=True)
        return tw.told
    finally:
        tw.close()


def scenario_realloc():
    tw = CullTwin(scene_with_shadows(11), seed=11)
    try:
        tw.cframe("sparse")
        tw.build(tw.groups_now())                           # every table reallocated: read in full again
        tw.cframe("dense", n_bounds=0, n_iv=0, restore=False)   # ... over bypass writes and Changed<Transform> rows
        for f in range(2):
            tw.edit(n_despawn=5, n_flat=5, n_kids=3, n_reparent=2)
            tw.cframe(["sparse", "dense"][f])
        tw.compact()
        tw.cframe("sparse")
        tw.cframe("static", n_bounds=0, n_iv=0, spot=True)
        return tw.told
    finally:
        tw.close()


def scenario_errors():
    tw = CullTwin(scene_with_shadows(17, n_trees=20), seed=17)
    try:
        c = tw.a.pipe.ctx
        tw.cframe("sparse")
        good = [x.desc() for x in tw.culls]
        g0 = good[0]

        def with0(**kw):
            d = abi.TableCullInputs(*[getattr(g0, f) for f, _ in abi.TableCullInputs._fields_])
            for k, v in kw.items():
                setattr(d, k, v)
            return [d] + good[1:]
        lay = tw.blayout
        cases = [
            (good[:-1], lay),                                   # n_tables differs from the registry's size
            (with0(aabb_changed_ticks=None), lay),              # half-NULL pairs
            (with0(spheres=g0.aabbs), lay),
            (with0(iv_changed_ticks=None), lay),
            (with0(aabbs=g0.aabbs + 2), lay),                   # misaligned
            (with0(aabb_changed_ticks=g0.aabb_changed_ticks + 1), lay),
            (with0(flags=CM.F_INHERITED), lay),                 # derived bits are not passed
            (with0(flags=CM.F_AABB), lay),
            (with0(flags=0x80), lay),
            (good, None),                                       # no layout
            (good, (32, 2, 16, 32, 0, 16)),                     # a field not 4-byte aligned
            (good, (30, 0, 16, 32, 0, 16)),                     # stride not 4-byte aligned
            (good, (32, 0, 24, 32, 0, 16)),                     # half_extents past stride
            (good, (32, 0, 8, 32, 0, 16)),                      # overlapping fields
            (good, (32, 0, 16, 16, 0, 16)),                     # radius past stride
            (good, (32, 0, 16, 32, 0, 8)),                      # radius inside center
        ]
        for d, lay_ in cases:
            try:
                c.set_table_cull_inputs(d, lay_)
            except abi.B200VisError as e:
                assert e.code == INVALID_ARG, str(e)
            else:
                raise AssertionError(f"set_table_cull_inputs accepted {lay_}")
        tw.cframe("sparse")                                 # the previous inputs stay in force
        tw.cframe("static", n_bounds=0, n_iv=0)
    finally:
        tw.close()
    for kw, code in (({}, NOT_READY), (dict(world_size=2, rank=0), UNSUPPORTED)):
        ctx = abi.Context(64, **kw)
        try:
            for _ in range(2 if not kw else 1):
                try:
                    ctx.set_table_cull_inputs([])
                except abi.B200VisError as e:
                    assert e.code == code, str(e)
                else:
                    raise AssertionError("set_table_cull_inputs without a registry succeeded")
                if not kw:
                    ctx.set_tables([])                      # an empty registry is no registry either
        finally:
            ctx.close()


def scenario_bench_world():
    def make():
        sc = scenes.forest(3922, 8, 256)                    # config #3: 1,000,366 rows in its four archetype tables
        sc.shadow_lights = np.array([0], np.uint32)
        sc.shadow_caster = np.ones(sc.n, np.uint8); sc.shadow_caster[sc.light_row] = 0
        sc.shadow_near_z, sc.shadow_lod_origin = 0.1, 0
        return sc
    tw = CullTwin(make, seed=23, churn_headroom=0, headroom=64)
    try:
        tw.cframe("static", n_bounds=0, n_iv=0)             # every slot read in full
        tw.cframe("sparse", n_bounds=64, n_iv=32)
        tw.cframe("static", n_bounds=0, n_iv=0, spot=True)
    finally:
        tw.close()


LAYOUTS = {"bevy": CM.BEVY_LAYOUT, "permuted": CM.PERMUTED_LAYOUT, "packed": CM.PACKED_LAYOUT}
# scenario -> the model mutants its frames must tell apart
EXPECT = {
    "frames_permuted": {"packed_layout", "iv_by_aabb_tick"},
    "moves": {"sphere_over_aabb", "capacity", "unmapped", "fresh_by_ticks"},
    "realloc": {"fresh_by_ticks", "drop_tchanged"},
}
CALLS = {
    "frames_bevy": "scenario_frames('bevy')", "frames_permuted": "scenario_frames('permuted')",
    "frames_packed": "scenario_frames('packed')", "wrap": "scenario_wrap()", "moves": "scenario_moves()",
    "realloc": "scenario_realloc()", "errors": "scenario_errors()", "bench_world": "scenario_bench_world()",
}


@pytest.mark.parametrize("name", list(CALLS))
def test_scenario(name):
    code = textwrap.dedent(f"""
        import test_gpu_tables_cull_read as T
        told = T.{CALLS[name]}
        missing = T.EXPECT.get({name!r}, set()) - (told or set())
        assert not missing, f"the model mutants {{sorted(missing)}} were not told apart"
    """)
    # the case's interpreter loads the library this one does
    run_case(code, {k: os.environ[k] for k in ("B200VIS_LIB",) if k in os.environ}, timeout=1500)
