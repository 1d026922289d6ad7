"""Rows placed where the order of operations decides the verdict.

Camera cull: both the oracle and the kernels evaluate `plane . (c, 1) + r <= 0` in glam's order (pairwise dot4, no FMA,
`<=`).  Random scenes almost never put a row within a few ulps of a plane, so a kernel that summed left to right,
contracted an FMA or used `<` would still pass them.  Here every boundary row's `plane_dot_point + radius` (Sphere rows,
sphere-from-GT rows) or `plane_dot_point + relative_radius` (Aabb rows) is exactly 0 or one step either side of 0, with the
GlobalTransform coming out of the propagation through a rotated, non-uniformly scaled, mirrored parent.  Each scene also
proves, on the CPU, that it tells those three mutants apart from the real test.

Shadow cull: the block pre-pass of k_shadow_cull (casters just inside a cascade plane far from the origin, casters on a
light's range sphere) and the item loop's live-word jump and its items past 256."""
import numpy as np
import pytest

import bevy_b200 as bb
from bevy_b200 import scenes
from bevy_b200.scenes import Camera, Scene
import oracle as orc

from parity import OracleWorld, compare_frame
from test_gpu_bench_scale import run_case
from test_gpu_split_stages import same_bits, split_frame

pytestmark = pytest.mark.gpu

f32 = np.float32
IDENT9 = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1], f32)


# ---- float32 restatement of the camera test ------------------------------------------------------------------------------------
def plane_value(n, c, order="glam"):
    """n [4] . (c, 1): glam's (x + z) + (y + w); or a left-to-right sum; or one rounding of the exact sum (a contracted FMA)."""
    if order == "l2r":
        return ((n[0] * c[..., 0] + n[1] * c[..., 1]) + n[2] * c[..., 2]) + n[3]
    if order == "fma":
        d = n.astype(np.float64)
        return (d[0] * c[..., 0].astype(np.float64) + d[1] * c[..., 1].astype(np.float64) + d[2] * c[..., 2].astype(np.float64) + d[3]).astype(f32)
    return (n[0] * c[..., 0] + n[2] * c[..., 2]) + (n[1] * c[..., 1] + n[3] * f32(1.0))


def axes(gt):
    """m[.., i, j]: row i of the matrix (the kernels' g.r_i component j); gt is glam's [x_axis, y_axis, z_axis, translation]."""
    return gt[..., 0:9].reshape(gt.shape[:-1] + (3, 3)).swapaxes(-1, -2)


def aabb_centre_radius(gt, b, h):
    m, t = axes(gt), gt[..., 9:12]
    c = np.stack([((m[..., i, 0] * b[..., 0] + m[..., i, 1] * b[..., 1]) + m[..., i, 2] * b[..., 2]) + t[..., i] for i in range(3)], -1)
    v = [(m[..., i, 0] * h[..., 0] + m[..., i, 1] * h[..., 1]) + m[..., i, 2] * h[..., 2] for i in range(3)]
    return c, np.sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2])


def relative_radius(gt, h, n):
    m = axes(gt)
    d = [np.abs((n[0] * m[..., 0, j] + n[1] * m[..., 1, j]) + n[2] * m[..., 2, j]) for j in range(3)]
    return (d[0] * h[..., 0] + d[1] * h[..., 1]) + d[2] * h[..., 2]


def restated_visible(gt, bounds, flags, planes, order="glam", strict=False):
    """Frustum::intersects_sphere (5 planes) and, for Aabb rows, Frustum::intersects_obb: [V, n] bool."""
    with np.errstate(invalid="ignore", over="ignore"):            # the non-finite rows
        return _restated_visible(gt, bounds, flags, planes, order, strict)


def _restated_visible(gt, bounds, flags, planes, order, strict):
    le = (lambda a: a < f32(0.0)) if strict else (lambda a: a <= f32(0.0))
    has_aabb = (flags & bb.F_HAS_AABB) != 0
    c, r = aabb_centre_radius(gt, bounds[:, 0:3], bounds[:, 3:6])
    from_gt = (flags & bb.F_SPHERE_FROM_GT) != 0
    sc = np.where(from_gt[:, None], gt[:, 9:12], bounds[:, 0:3])
    c = np.where(has_aabb[:, None], c, sc)
    r = np.where(has_aabb, r, bounds[:, 3])
    tested = has_aabb | ((flags & bb.F_HAS_SPHERE) != 0)
    out = np.zeros((len(planes), len(gt)), bool)
    for v, pl in enumerate(planes):
        vis = np.ones(len(gt), bool)
        for k in range(5):
            vis &= ~le(plane_value(pl[k], c, order) + r)
        for k in range(5):
            obb = ~le(plane_value(pl[k], c, order) + relative_radius(gt, bounds[:, 3:6], pl[k]))
            vis &= np.where(has_aabb, obb, True)
        out[v] = np.where(tested, vis, True)
    return out


def view_planes(cameras):
    return np.stack([bb.host_compute_frustum(bb.host_perspective(c.fov, c.aspect, c.near), c.gt, c.far) for c in cameras])


# ---- the boundary scene --------------------------------------------------------------------------------------------------------
def _grid(x, steps):
    """x's float32 neighbours, -steps..steps ulps, per component: [(2*steps+1)^3, 3]."""
    x = np.asarray(x, f32)
    opts = []
    for i in range(3):
        o, lo, hi = [x[i]], x[i], x[i]
        for _ in range(steps):
            lo = np.nextafter(lo, f32(-np.inf), dtype=f32); hi = np.nextafter(hi, f32(np.inf), dtype=f32)
            o += [lo, hi]
        opts.append(np.array(o, f32))
    g = np.stack(np.meshgrid(*opts, indexing="ij"), -1).reshape(-1, 3)
    return g


def _pick(values):
    """Indices of a zero, the smallest positive and the largest negative value (what exists of them)."""
    out = []
    z = np.nonzero(values == 0)[0]
    if len(z):
        out.append(z[0])
    pos, neg = np.nonzero(values > 0)[0], np.nonzero(values < 0)[0]
    if len(pos):
        out.append(pos[np.argmin(values[pos])])
    if len(neg):
        out.append(neg[np.argmax(values[neg])])
    return out


class Builder:
    def __init__(self):
        self.parent, self.trs, self.bounds, self.flags = [], [], [], []

    def add(self, parent, trs, bounds, flags):
        self.parent.append(parent); self.trs.append(np.asarray(trs, f32)); self.bounds.append(np.asarray(bounds, f32))
        self.flags.append(flags)
        return len(self.parent) - 1

    def scene(self, name, cameras, shuffle=False, seed=0):
        n = len(self.parent)
        ent = np.arange(n, dtype=np.uint64) + np.uint64(3)
        if shuffle:
            ent = np.random.default_rng(seed).permutation(ent)
        return Scene(name, np.array(self.parent, np.uint32), np.stack(self.trs), np.stack(self.bounds), np.array(self.flags, np.uint8),
                     np.ones(n, np.uint8), ent, cameras=cameras, roots=None)


def boundary_rows(rng, planes, cameras, per_plane=2):
    """Trees (root, child) whose child sits on a camera plane: (root trs, child trs, child bounds, child flags) per tree."""
    out = []
    for v, cam in enumerate(cameras):
        eye = np.asarray(cam.gt[9:12], np.float64)
        fwd = -np.asarray(cam.gt[6:9], np.float64)
        for k in range(5):
            n = planes[v, k]
            for _ in range(per_plane):
                for kind in ("aabb", "sphere", "sphere_gt"):
                    q = scenes.random_unit_quats(rng, 1)[0]
                    s = rng.uniform(0.4, 2.5, 3) * np.where(rng.random(3) < 0.3, -1.0, 1.0)       # non-uniform, mirrored
                    root = np.concatenate([[0, 0, 0], q, s]).astype(f32)
                    child = np.concatenate([rng.uniform(-1, 1, 3), scenes.random_unit_quats(rng, 1)[0], rng.uniform(0.5, 1.5, 3)]).astype(f32)
                    g0 = orc.affine_mul(orc.affine_from_trs(root), orc.affine_from_trs(child))     # child GT with root translation 0
                    K = g0[9:12].copy()
                    bnd = np.zeros(6, f32)
                    if kind == "aabb":
                        bnd[0:3] = rng.uniform(-0.5, 0.5, 3); bnd[3:6] = rng.uniform(0.1, 1.0, 3)
                        flags = bb.F_INHERITED_VISIBLE | bb.F_HAS_AABB
                    else:
                        bnd[3] = rng.uniform(0.1, 1.5)
                        flags = bb.F_INHERITED_VISIBLE | bb.F_HAS_SPHERE | (bb.F_SPHERE_FROM_GT if kind == "sphere_gt" else 0)
                    # a point inside the frustum, moved onto plane k, then to where the chosen term is zero
                    p = eye + fwd * rng.uniform(3.0, 40.0) + rng.normal(scale=0.5, size=3)
                    nn = n[0:3].astype(np.float64)
                    p = p - nn * ((nn @ p + n[3]) / (nn @ nn))
                    if kind == "aabb":
                        c0, _ = aabb_centre_radius(g0[None], bnd[None, 0:3], bnd[None, 3:6])
                        term = float(relative_radius(g0[None], bnd[None, 3:6], n)[0])
                        c0 = c0[0].astype(np.float64) - K                     # the part of the centre that is not the translation
                    else:
                        c0, term = np.zeros(3), float(bnd[3])
                    target = p - nn * (term / (nn @ nn))
                    if kind == "sphere":                                      # world-space centre: search the centre itself
                        g = _grid(target, 3)
                        d = plane_value(n, g)
                    else:
                        t = _grid(target - c0 - K, 3)                         # root translations around the solution
                        T = (K[None, :] + t).astype(f32)                      # the child's translation: P.m3*L.t + P.t
                    if kind == "aabb":
                        gt = np.concatenate([np.tile(g0[0:9], (len(t), 1)), T], 1)
                        c, _ = aabb_centre_radius(gt, np.tile(bnd[0:3], (len(t), 1)), np.tile(bnd[3:6], (len(t), 1)))
                        vals = plane_value(n, c) + relative_radius(gt, np.tile(bnd[3:6], (len(t), 1)), n)
                        for i in _pick(vals):
                            r2 = root.copy(); r2[0:3] = t[i]
                            out.append((r2, child, bnd, flags))
                        continue
                    if kind == "sphere_gt":
                        d = plane_value(n, T)
                    # a sphere's radius is free: take it as -d of the nearest centre, so that d + r is exactly 0, and one
                    # step either side of that radius (the plane value itself is a multiple of the large operands' ulp)
                    i = int(np.argmin(np.abs(d + bnd[3])))
                    r0 = -d[i]
                    for r in (r0, np.nextafter(r0, f32(np.inf), dtype=f32), np.nextafter(r0, f32(-np.inf), dtype=f32)):
                        b2, r2 = bnd.copy(), root.copy()
                        b2[3] = r
                        if kind == "sphere":
                            b2[0:3] = g[i]
                        else:
                            r2[0:3] = t[i]
                        out.append((r2, child, b2, flags))
    return out


def boundary_scene(seed, offset, n_views=3, shuffle=False):
    rng = np.random.default_rng(seed)
    off = np.array([1.0, 0.37, -0.61]) / np.linalg.norm([1.0, 0.37, -0.61]) * offset
    cams = []
    for k in range(n_views):
        q = scenes.quat_mul(scenes.quat_axis("y", 0.8 * k), scenes.quat_axis("x", -0.15 * k))
        cams.append(Camera(gt=scenes.quat_to_gt(q, off + np.array([0.5 * k, 0.2, -0.3 * k])), quat=q, far=300.0))
    planes = view_planes(cams)
    trees = boundary_rows(rng, planes, cams)
    rng.shuffle(trees)
    B = Builder()
    ident = np.array([0, 0, 0, 0, 0, 0, 1, 1, 1, 1], f32)
    far_behind = lambda: np.concatenate([off - 5000.0 + rng.normal(size=3), [0, 0, 0, 1, 1, 1, 1]]).astype(f32)
    # roots first (no bounds: their warps never take the shortcut), children after them, so that a warp of children holds
    # only what is chosen for it; the non-finite trees go last
    bad = []
    for kind in ("nan_t", "inf_t", "inf_h", "nan_r"):
        t = trees[len(bad)]
        root, child, bnd, flags = t[0].copy(), t[1], t[2].copy(), t[3]
        if kind == "nan_t": root[1] = np.nan
        if kind == "inf_t": root[0] = np.inf
        if kind == "inf_h":
            bnd[3:6] = [np.inf, 0.5, 0.5]; flags = bb.F_INHERITED_VISIBLE | bb.F_HAS_AABB
        if kind == "nan_r":
            bnd[3] = np.nan; flags = bb.F_INHERITED_VISIBLE | bb.F_HAS_SPHERE
        bad.append((root, child, bnd, flags))
    trees = trees[len(bad):] + bad
    roots = [B.add(scenes.NO_PARENT, r, np.zeros(6, f32), bb.F_INHERITED_VISIBLE) for r, _, _, _ in trees]
    while len(B.parent) % 32:
        B.add(scenes.NO_PARENT, ident, np.zeros(6, f32), bb.F_INHERITED_VISIBLE)
    nb = len(trees) - len(bad)
    third = nb // 3
    # warps of boundary rows only
    for i in range(third):
        B.add(roots[i], trees[i][1], trees[i][2], trees[i][3])
    while len(B.parent) % 32:
        B.add(scenes.NO_PARENT, far_behind(), np.array([0, 0, 0, 0.5, 0.5, 0.5], f32), bb.F_INHERITED_VISIBLE | bb.F_HAS_AABB)
    # warps mixing boundary rows with rows far behind every camera (the warp shortcut must not fire)
    for i in range(third, nb):
        B.add(roots[i], trees[i][1], trees[i][2], trees[i][3])
        B.add(scenes.NO_PARENT, far_behind(), np.array([0, 0, 0, 0.5, 0.5, 0.5], f32), bb.F_INHERITED_VISIBLE | bb.F_HAS_AABB)
    while len(B.parent) % 32:
        B.add(scenes.NO_PARENT, far_behind(), np.array([0, 0, 0, 0.5, 0.5, 0.5], f32), bb.F_INHERITED_VISIBLE | bb.F_HAS_AABB)
    # warps of Sphere rows just outside one plane of view 0 (the shortcut should fire for them)
    n = planes[0, 0].astype(np.float64)
    eye, fwd = np.asarray(cams[0].gt[9:12], np.float64), -np.asarray(cams[0].gt[6:9], np.float64)
    for j in range(64):
        p = eye + fwd * (5.0 + j) ; p = p - n[0:3] * ((n[0:3] @ p + n[3]) / (n[0:3] @ n[0:3]))
        c = p - n[0:3] / np.linalg.norm(n[0:3]) * (0.5 + 1e-3 * (1.0 + np.abs(p).max()))
        B.add(scenes.NO_PARENT, ident, np.array([*c, 0.5, 0, 0], f32), bb.F_INHERITED_VISIBLE | bb.F_HAS_SPHERE)
    for i in range(nb, len(trees)):
        B.add(roots[i], trees[i][1], trees[i][2], trees[i][3])
    return B.scene(f"boundary_{offset:g}_{n_views}v", cams, shuffle=shuffle, seed=seed), planes


def check_sensitivity(sc, world):
    """The scene must tell a left-to-right dot, a contracted FMA and `<` apart from the real test (on the oracle's
    GlobalTransforms), and the restated real test must equal the oracle's lists."""
    planes = view_planes(sc.cameras)
    base = restated_visible(world.gt, sc.bounds, sc.flags, planes)
    for v in range(len(planes)):
        want = np.zeros(sc.n, bool); want[world.last_lists[v]] = True
        assert (base[v] == want).all(), f"view {v}: the float32 restatement disagrees with the oracle on rows {np.nonzero(base[v] != want)[0][:8]}"
    for name, kw in (("left-to-right dot", dict(order="l2r")), ("FMA-contracted dot", dict(order="fma")), ("'<' for '<='", dict(strict=True))):
        assert (restated_visible(world.gt, sc.bounds, sc.flags, planes, **kw) != base).any(), f"the scene cannot detect a {name}"


def boundary_frames(seed, offset, n_views=3, split=False, shuffle=False):
    sc, _ = boundary_scene(seed, offset, n_views, shuffle)
    pipe = bb.VisibilityPipeline(sc)
    world = OracleWorld(sc)
    try:
        for f in range(3):
            if f == 2:                                   # a Changed<Transform> frame that leaves every value as it was
                rows = np.arange(0, sc.n, 7, dtype=np.uint32)
                pipe.ctx.upload_transforms_scattered(rows, sc.trs[rows])
                world.tchanged[rows] = 1
            if split:
                split_frame(pipe, world, f)
            else:
                pipe.update_views()
                pipe.run_frame()
                rc, want = orc.propagate(sc.parent, sc.trs, world.gt, world.tchanged, world.static_opt)
                world.tchanged[:] = 0
                gt, ch = pipe.ctx.download_global_transforms(0, sc.n)
                bad = ~same_bits(gt, world.gt).all(1)
                assert not bad.any(), f"frame {f}: GlobalTransform bits differ on rows {np.nonzero(bad)[0][:8]}"
                assert (ch == want).all()
                compare_frame(pipe, world, f, check_gt=False, run_device=False)
            if f == 0:
                assert np.isnan(world.gt).any() and np.isinf(world.gt).any()
                check_sensitivity(sc, world)
    finally:
        pipe.close()


CASES = [(31, 0.0, 3), (32, 1e3, 3), (33, 1e5, 3), (34, 1e3, 7), (35, 0.0, 8)]


@pytest.mark.parametrize("seed,offset,n_views", CASES)
def test_rows_on_camera_planes_split_cull(seed, offset, n_views):
    """Kernel 1c (CULL without PROPAGATE), rows in Entity order (k_cull<SIMPLE>) and shuffled (k_cull<false>)."""
    boundary_frames(seed, offset, n_views, split=True)
    boundary_frames(seed, offset, n_views, split=True, shuffle=True)


FUSED = {"default": {}, "lean": {"B200VIS_TILE_KERNEL": "lean"},
         "lean_sphere_reject": {"B200VIS_TILE_KERNEL": "lean", "B200VIS_LEAN_PROBE": "8"},
         "warp": {"B200VIS_TILE_KERNEL": "warp", "B200VIS_WARP_VARIANT": "2p"}, "classic": {"B200VIS_TILE_KERNEL": "classic"}}


@pytest.mark.parametrize("variant", list(FUSED))
def test_rows_on_camera_planes_fused(variant):
    """The fused tile pass of each kernel, every case, in its own interpreter."""
    run_case("from test_gpu_cull_boundaries import boundary_frames, CASES\n"
             "for seed, offset, views in CASES:\n"
             "    boundary_frames(seed, offset, views)\n"
             "    boundary_frames(seed, offset, views, shuffle=True)", FUSED[variant])


# ---- shadow culling ------------------------------------------------------------------------------------------------------------
def shadow_scene(casters, others, lights_listed, lights_unlisted):
    """Roots only: caster rows (world centre, half extents), other meshes, and light rows (no bounds: the camera lists a light
    row iff it is visible).  Returns (scene, caster mask, light rows listed, light rows not listed)."""
    B = Builder()
    for c, h in casters:
        B.add(scenes.NO_PARENT, np.concatenate([c, [0, 0, 0, 1, 1, 1, 1]]), np.concatenate([[0, 0, 0], h]), bb.F_INHERITED_VISIBLE | bb.F_HAS_AABB)
    for c in others:
        B.add(scenes.NO_PARENT, np.concatenate([c, [0, 0, 0, 1, 1, 1, 1]]), [0, 0, 0, 0.5, 0.5, 0.5], bb.F_INHERITED_VISIBLE | bb.F_HAS_AABB)
    listed = [B.add(scenes.NO_PARENT, np.concatenate([p, [0, 0, 0, 1, 1, 1, 1]]), np.zeros(6), bb.F_INHERITED_VISIBLE) for p in lights_listed]
    unlisted = [B.add(scenes.NO_PARENT, np.concatenate([p, [0, 0, 0, 1, 1, 1, 1]]), np.zeros(6), 0) for p in lights_unlisted]
    sc = B.scene("shadow", [scenes._camera(0.0)])
    caster = np.zeros(sc.n, np.uint8); caster[:len(casters)] = 1
    return sc, caster, np.array(listed, np.uint32), np.array(unlisted, np.uint32)


def shadow_frame(sc, caster, items):
    """One camera frame then the shadow items (dicts as Context.set_shadow_items takes, with frusta from the oracle), device
    against oracle: every (item, face) list, ViewVisibility and its change flags.  Returns the rows listed per item."""
    pipe = bb.VisibilityPipeline(sc)
    world = OracleWorld(sc)
    try:
        pipe.ctx.upload_shadow_casters(0, caster)
        planes = view_planes(sc.cameras)
        pipe.update_views()
        pipe.ctx.run(bb.STAGE_PROPAGATE | bb.STAGE_CULL)
        pipe.ctx.set_shadow_items(items)
        pipe.ctx.run_shadow_culling()
        orc.propagate(sc.parent, sc.trs, world.gt, world.tchanged, True)
        orc.set_defer_mark_newly_hidden(True)
        try:
            vv_changed, lists = orc.cull(world.gt, sc.bounds, sc.flags, sc.class_mask, sc.entity_bits, world.vv, planes)
        finally:
            orc.set_defer_mark_newly_hidden(False)
        listed = set(np.concatenate(lists).tolist())
        seen = []
        for i, it in enumerate(items):
            if it["kind"] == 2:
                want = orc.check_dir_light_mesh_visibility(world.gt, sc.bounds, sc.flags, caster, sc.entity_bits, world.vv, vv_changed,
                                                           [(np.asarray(it["frusta"], f32)[None], 1, -1)])[0]
            elif it["light_row"] not in listed:                  # the light is in no view's VisibleEntities: not processed
                want = [np.zeros(0, np.uint32)] * 6
            else:
                row = it["light_row"]
                sphere = np.concatenate([world.gt[row, 9:12], [it["range"]]]).astype(f32)[None]
                fn = orc.check_point_light_mesh_visibility if it["kind"] == 0 else orc.check_spot_light_mesh_visibility
                r = fn(world.gt, sc.bounds, sc.flags, caster, sc.entity_bits, world.vv, vv_changed, sphere,
                       np.asarray(it["frusta"], f32)[None], lod_origin_index=-1, light_layers=np.array([1], np.uint64))
                want = r[0] if it["kind"] == 0 else [r[0]]
            got_any = []
            for face, rows in enumerate(want):
                got = pipe.ctx.download_shadow_visible(i, face)
                assert len(got) == len(rows) and (got == rows).all(), f"item {i} ({it['kind']}) face {face}: {len(got)} vs {len(rows)} rows"
                got_any += list(got)
            seen.append(len(got_any))
        orc.mark_newly_hidden(sc.flags, world.vv, vv_changed)
        vv, vch = pipe.ctx.download_view_visibility(0, sc.n)
        assert (vv == world.vv).all(), f"ViewVisibility differs on rows {np.nonzero(vv != world.vv)[0][:8]}"
        assert (vch == vv_changed).all(), "Changed<ViewVisibility> differs"
        return seen
    finally:
        pipe.close()


def test_cascade_planes_through_point_casters_far_from_the_origin():
    """One zero-extent caster per 256-row block, 3e4 to 1e6 from the origin, just inside plane 0 of its own cascade (within
    a few ulps); the other 255 rows of each block are not casters.  The caster is reached; an absolute pre-pass margin
    skipped exactly these."""
    from test_cpu_shadow_prepass import cascade_skips_absolute_margin, point_casters_on_cascade_planes
    rng = np.random.default_rng(3)
    chosen = []
    for offset in (3e4, 1e5, 3e5, 1e6):
        planes, c, keep = point_casters_on_cascade_planes(rng, offset)
        old = cascade_skips_absolute_margin(c, c, np.zeros(len(c), f32), planes)
        idx = np.nonzero(old & keep)[0][:12]                     # reachable, and skipped by the absolute margin
        idx = np.concatenate([idx, np.nonzero(keep & ~old)[0][:4], np.nonzero(~keep)[0][:4]])
        chosen += [(planes[i], c[i]) for i in idx]
    assert len(chosen) >= 40
    B_rows = []                                                  # each caster opens a 256-row block of 255 non-casters
    for fr, c in chosen:
        B_rows.append(("caster", c))
        B_rows += [("other", c + np.float32(3.0))] * 255
    Bd = Builder()
    for kind, c in B_rows:
        Bd.add(scenes.NO_PARENT, np.concatenate([c, [0, 0, 0, 1, 1, 1, 1]]).astype(f32),
               np.array([0, 0, 0, 0, 0, 0] if kind == "caster" else [0, 0, 0, 0.5, 0.5, 0.5], f32), bb.F_INHERITED_VISIBLE | bb.F_HAS_AABB)
    sc = Bd.scene("far_casters", [scenes._camera(0.0)])
    caster = np.array([k == "caster" for k, _ in B_rows], np.uint8)
    items = [dict(kind=2, range_view_index=-1, layer_mask=1, frusta=fr) for fr, _ in chosen]
    seen = shadow_frame(sc, caster, items)
    assert sum(s > 0 for s in seen) >= 30


def unit(x):
    return x / np.linalg.norm(x)


def _sphere_boundary_casters(rng, light, r, direction_fn, k):
    """Zero-extent casters at distance ~r from `light` with d_sq - r * d exactly 0 or one step either side."""
    out = []
    for _ in range(k):
        u = direction_fn()
        g = _grid(light + u * r, 2)
        v = (g - light).astype(f32)
        d_sq = (v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2]
        vals = d_sq - r * np.sqrt(d_sq)
        out += [g[i] for i in _pick(vals)]
    return out


def test_casters_on_point_and_spot_light_range_spheres():
    rng = np.random.default_rng(9)
    lights = [np.array([20.0 * i, 5.0, -30.0], f32) + f32(1e3 * (i % 2)) for i in range(8)]
    ranges = [f32(x) for x in rng.uniform(2.0, 15.0, 8)]
    casters = []
    items_spec = []
    for i, (p, r) in enumerate(zip(lights, ranges)):
        gt = np.concatenate([IDENT9, p]).astype(f32)
        fr6 = orc.point_light_frusta(gt, r, 0.1)
        if i % 2 == 0:                                                             # point light: any direction
            dirs = lambda: unit(rng.normal(size=3))
            kind, fr = 0, fr6
        else:                                                                      # spot light: directions inside its frustum
            def dirs(p=p, r=r, fr=fr6[1]):
                while True:
                    u = unit(rng.normal(size=3))
                    if all(plane_value(fr[k], (p + u * (0.9 * r)).astype(f32)) > 0 for k in range(6)):
                        return u
            kind, fr = 1, fr6[1]
        for c in _sphere_boundary_casters(rng, p.astype(np.float64), float(r), dirs, 12):
            casters.append((c, np.zeros(3, f32)))
        items_spec.append((kind, r, fr))
    sc, caster, listed, _ = shadow_scene(casters, [], lights, [])
    items = [dict(kind=k, light_row=int(listed[i]), range=float(r), range_view_index=-1, layer_mask=1, frusta=fr)
             for i, (k, r, fr) in enumerate(items_spec)]
    seen = shadow_frame(sc, caster, items)
    assert all(s > 0 for s in seen)


@pytest.mark.parametrize("count", [31, 32, 33, 255, 256, 257, 300])
def test_only_one_item_reaches_the_casters(count):
    """`count` items of which only the one at index 0, 31, 32, 255, 256 or the last reaches any row: the live-word jump of
    the pre-tested first 256 items, and the items past 256 that are always live.  Past 256, point and spot items whose
    light is in no view's list would reach every caster: they must stay empty."""
    rng = np.random.default_rng(count)
    casters = [(rng.normal(scale=4.0, size=3).astype(f32), rng.uniform(0.2, 0.8, 3).astype(f32)) for _ in range(1024)]
    far = [np.array([1e4 + 10.0 * i, 0.0, 0.0], f32) for i in range(count)]
    near = [np.array([0.5, 0.0, 0.0], f32)]
    unlisted = [np.array([0.1 * (i % 7), 0.0, 0.0], f32) for i in range(count)]       # among the casters
    sc, caster, listed, not_listed = shadow_scene(casters, [], far + near, unlisted)
    for live in sorted({i for i in (0, 31, 32, 255, 256, count - 1) if i < count}):
        items = []
        for i in range(count):
            kind = i % 2
            if i == live:
                row, rg = int(listed[-1]), 60.0
            elif i >= 256 and i % 3 == 0:
                row, rg = int(not_listed[i]), 60.0
            else:
                row, rg = int(listed[i]), 1.0
            p = np.concatenate([IDENT9, sc.trs[row, 0:3]]).astype(f32)
            fr6 = orc.point_light_frusta(p, rg, 0.1)
            items.append(dict(kind=kind, light_row=row, range=rg, range_view_index=-1, layer_mask=1, frusta=fr6 if kind == 0 else fr6[0]))
        seen = shadow_frame(sc, caster, items)
        assert seen[live] > 0 and sum(seen) == seen[live], (live, [i for i, s in enumerate(seen) if s])
