"""VisibilityRange rows placed where the order of operations decides the verdict (SURVEY.md 8(f) N4a), proved on the CPU.

check_visibility_ranges (crates/bevy_camera/src/visibility/range.rs:230-284) keeps view bit v of a row when
`start <= |view_v - model_position| < end`, with glam's float32 `Vec3A::length`: `sqrtf((dx*dx + dy*dy) + dz*dz)`.  Random
distances almost never land within an ulp of a threshold, so a kernel with `>` for `>=`, `<=` for `<`, another summation
order, a contracted FMA, squared distances against squared thresholds, or the sphere centre as the model position of a
Sphere row would still pass them.  `range_scene` builds a hierarchy (rotated, non-uniformly scaled and mirrored parents, at
a world offset), takes the frame-0 GlobalTransforms from the oracle, and sets each row's (start, end) to the float32
distance to one view, or one step either side of it.  `check_range_sensitivity` proves that the scene tells every one of
those mutants apart from the real test; the GPU file runs the same scenes on the device."""
import numpy as np
import pytest

import bevy_b200 as bb
from bevy_b200 import scenes
from bevy_b200.scenes import Camera
import oracle as orc

f32 = np.float32
N_RANGE_VIEWS = 36                     # > 32: bit 31 is used, views 32.. are ignored
CAMERA_RANGE_INDEX = [0, 1, 2, -1]     # cameras 0-2 read range views 0-2; camera 3 reads none
MUTANTS = ("gt_for_ge", "le_for_lt", "sum_yz_first", "fma", "squared", "sphere_centre")


# ---- float32 restatement of check_visibility_ranges ----------------------------------------------------------------------------
def model_position(gt, bounds, flags, use_aabb, mutant=None):
    """(use_aabb, Some(aabb)) => transform_point3a(aabb.center), else the translation (range.rs:263-268).  The
    "sphere_centre" mutant takes a Sphere row's centre instead, as a kernel that dropped `has_aabb` would."""
    m = gt[:, 0:9].reshape(-1, 3, 3)          # m[:, axis, component]
    b = bounds[:, 0:3]
    tp = np.stack([((m[:, 0, k] * b[:, 0] + m[:, 1, k] * b[:, 1]) + m[:, 2, k] * b[:, 2]) + gt[:, 9 + k] for k in range(3)], 1)
    has_aabb = (flags & bb.F_HAS_AABB) != 0
    pos = np.where(((use_aabb != 0) & has_aabb)[:, None], tp, gt[:, 9:12])
    if mutant == "sphere_centre":
        sphere = ((use_aabb != 0) & ~has_aabb & ((flags & bb.F_HAS_SPHERE) != 0))[:, None]
        centre = np.where(((flags & bb.F_SPHERE_FROM_GT) != 0)[:, None], gt[:, 9:12], b)
        pos = np.where(sphere, centre, pos)
    return pos.astype(f32)


def distances(view_pos, pos, order="glam"):
    """[n_views, n] float32 distance: glam's ((dx*dx + dy*dy) + dz*dz) then sqrtf, or dx*dx + (dy*dy + dz*dz), or one
    rounding of the exact sum (a contracted FMA); order "squared" returns the squared glam sum, not its root."""
    d = (view_pos[:, None, :] - pos[None, :, :]).astype(f32)
    dx, dy, dz = d[..., 0], d[..., 1], d[..., 2]
    if order == "sum_yz_first":
        s = dx * dx + (dy * dy + dz * dz)
    elif order == "fma":
        e = d.astype(np.float64)
        s = ((e[..., 0] * e[..., 0] + e[..., 1] * e[..., 1]) + e[..., 2] * e[..., 2]).astype(f32)
    else:
        s = (dx * dx + dy * dy) + dz * dz
    return s if order == "squared" else np.sqrt(s)


def restated_masks(gt, bounds, flags, range_se, use_aabb, view_pos, mutant=None):
    """VisibleEntityRanges value per row (0 = no entry) under the real test or one mutant."""
    pos = model_position(gt, bounds, flags, use_aabb, mutant)
    vp = np.asarray(view_pos, f32)[:32]
    order = mutant if mutant in ("sum_yz_first", "fma", "squared") else "glam"
    d = distances(vp, pos, order)
    s, e = range_se[:, 0][None], range_se[:, 1][None]
    if mutant == "squared":
        vis = (d >= s * s) & (d < e * e)
    elif mutant == "gt_for_ge":
        vis = (d > s) & (d < e)
    elif mutant == "le_for_lt":
        vis = (d >= s) & (d <= e)
    else:
        vis = (d >= s) & (d < e)
    mask = (vis.astype(np.uint64) << np.arange(len(vp), dtype=np.uint64)[:, None]).sum(0).astype(np.uint32)
    in_query = ((flags & bb.F_HAS_VIS_RANGE) != 0) & ((flags & bb.F_NO_CPU_CULLING) == 0)
    return np.where(in_query, mask, np.uint32(0))


# ---- the boundary scene --------------------------------------------------------------------------------------------------------
def range_views(sc, extra, frame):
    """Range views in view-query order: the first three cameras, then the extra positions rotated by `frame` places, so that
    each boundary view moves to another bit between frames (into bit 32, out of it, and through bit 31)."""
    cams = np.stack([np.asarray(c.gt[9:12], f32) for c in sc.cameras[:3]])
    return np.concatenate([cams, np.roll(extra, frame, axis=0)]).astype(f32)


def range_scene(seed, offset, n_trees=48):
    """Returns (scene, extra view positions).  Every row gets range parameters; the flags decide which are in the query."""
    rng = np.random.default_rng(seed)
    base = np.array([0.6, -0.2, 0.77]) / np.linalg.norm([0.6, -0.2, 0.77]) * offset
    cams = []
    for k in range(4):
        q = scenes.quat_mul(scenes.quat_axis("y", 0.05 * k), scenes.quat_axis("x", -0.03 * k))
        cams.append(Camera(gt=scenes.quat_to_gt(q, base + np.array([1.5 * k - 2.0, 0.3 * k, 4.0 - k])), quat=q, far=400.0))
    parent, trs, bounds, flags, use_aabb = [], [], [], [], []
    kinds = []

    def add(p, t, kind):
        parent.append(p); trs.append(np.asarray(t, f32))
        b = np.zeros(6, f32)
        fl = bb.F_INHERITED_VISIBLE | bb.F_HAS_VIS_RANGE
        ua = 1
        if kind in ("aabb", "aabb_translation", "no_range", "no_cpu_culling"):
            b[0:3] = rng.uniform(-0.6, 0.6, 3); b[3:6] = rng.uniform(0.1, 0.8, 3)
            fl |= bb.F_HAS_AABB
            ua = 0 if kind == "aabb_translation" else 1
        else:                                    # Sphere with use_aabb set: the model position is the translation
            b[3] = rng.uniform(0.1, 1.0)
            fl |= bb.F_HAS_SPHERE
        if kind == "no_range":
            fl &= ~bb.F_HAS_VIS_RANGE
        if kind == "no_cpu_culling":
            fl |= bb.F_NO_CPU_CULLING
        bounds.append(b); flags.append(fl); use_aabb.append(ua); kinds.append(kind)
        return len(parent) - 1

    cycle = ["aabb", "aabb_translation", "sphere", "aabb", "aabb_translation", "sphere", "no_range", "no_cpu_culling"]
    for i in range(n_trees):
        q = scenes.random_unit_quats(rng, 1)[0]
        s = rng.uniform(0.4, 2.5, 3) * np.where(rng.random(3) < 0.3, -1.0, 1.0)       # non-uniform, mirrored
        t = base + np.array([rng.uniform(-10, 10), rng.uniform(-5, 5), -rng.uniform(12, 70)])
        root = add(scenes.NO_PARENT, np.concatenate([t, q, s]), cycle[i % len(cycle)])
        for j in range(3):
            ct = np.concatenate([rng.uniform(-2, 2, 3), scenes.random_unit_quats(rng, 1)[0], rng.uniform(0.5, 1.5, 3)])
            child = add(root, ct, cycle[(i + j + 1) % len(cycle)])
            if j == 0:
                add(child, np.concatenate([rng.uniform(-1, 1, 3), scenes.random_unit_quats(rng, 1)[0], rng.uniform(0.5, 1.5, 3)]),
                    cycle[(i + 5) % len(cycle)])
    # point lights among the rows: shadow items whose LOD origin is range view 0
    lights = [add(scenes.NO_PARENT, np.concatenate([base + np.array([rng.uniform(-6, 6), rng.uniform(-3, 3), -rng.uniform(20, 50)]),
                                                    [0, 0, 0, 1, 1, 1, 1]]), "light") for _ in range(4)]
    n = len(parent)
    sc = scenes.Scene(f"ranges_{offset:g}", np.array(parent, np.uint32), np.stack(trs), np.stack(bounds), np.array(flags, np.uint8),
                      np.full(n, scenes.CLASS_MESH, np.uint8), rng.permutation(n).astype(np.uint64) + np.uint64(5), cameras=cams,
                      roots=None)
    lr = np.array(lights, np.uint32)
    sc.light_row, sc.light_range = lr, rng.uniform(25.0, 60.0, len(lr)).astype(f32)
    sc.class_mask[lr] = scenes.CLASS_LIGHT
    sc.flags[lr] = bb.F_INHERITED_VISIBLE | bb.F_HAS_SPHERE | bb.F_SPHERE_FROM_GT     # lights have no VisibilityRange
    sc.bounds[lr] = 0.0; sc.bounds[lr, 3] = sc.light_range
    sc.view_range_index = np.array(CAMERA_RANGE_INDEX, np.int8)
    sc.shadow_lights = np.arange(len(lr), dtype=np.uint32)
    sc.shadow_caster = np.ones(n, np.uint8); sc.shadow_caster[lr] = 0
    sc.shadow_near_z = 0.1
    sc.shadow_lod_origin = 0
    extra = (base + rng.uniform(-40, 40, (N_RANGE_VIEWS - 3, 3))).astype(f32)

    # frame-0 GlobalTransforms from the oracle, then the thresholds
    gt = np.tile(np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], f32), (n, 1))
    rc, _ = orc.propagate(sc.parent, sc.trs, gt, np.ones(n, np.uint8), True)
    assert rc == 0
    ua = np.array(use_aabb, np.uint8)
    vp = range_views(sc, extra, 0)
    sphere_rows = np.array([k == "sphere" for k in kinds])
    # a Sphere row's centre (free data) 3 units further from some view than its translation, see below
    pos = model_position(gt, sc.bounds, sc.flags, ua)
    d = {o: distances(vp, pos, o) for o in ("glam", "sum_yz_first", "fma", "squared")}
    se = np.zeros((n, 2), f32)
    steps = ["start_eq", "start_up", "start_down", "end_eq", "end_up", "end_down"]
    up = lambda x: np.nextafter(x, f32(np.inf), dtype=f32)
    down = lambda x: np.nextafter(x, f32(-np.inf), dtype=f32)
    for r in range(n):
        step = steps[(r // 2) % len(steps)]
        # candidate boundary views: the cameras' range views for half the rows (the visible lists then depend on the bit);
        # for the rest view 31, the ignored views past 32, or any counted view
        cand = [np.arange(3), [31], np.arange(32, N_RANGE_VIEWS), np.arange(32), np.arange(32)][0 if r % 2 == 0 else 1 + (r // 2) % 4]
        best, best_score = cand[0], -1
        for v in cand:
            g = d["glam"][v, r]
            t = {"start_eq": g, "start_up": up(g), "start_down": down(g), "end_eq": g, "end_up": up(g), "end_down": down(g)}[step]
            if step.startswith("start"):
                s_, e_ = t, f32(t * f32(4.0) + f32(50.0))
            else:
                s_, e_ = f32(0.0), t
            real = (g >= s_) & (g < e_)
            score = int(((d["sum_yz_first"][v, r] >= s_) & (d["sum_yz_first"][v, r] < e_)) != real) \
                + int(((d["fma"][v, r] >= s_) & (d["fma"][v, r] < e_)) != real) \
                + int(((d["squared"][v, r] >= s_ * s_) & (d["squared"][v, r] < e_ * e_)) != real)
            if score > best_score:
                best, best_score, se[r] = v, score, (s_, e_)
        if sphere_rows[r]:
            # the translation sits on a threshold, the sphere centre 3 units from it along the same line, on the other side
            g = d["glam"][best, r]
            into_range = -3.0 if r % 3 == 0 else 3.0
            dirv = (pos[r].astype(np.float64) - vp[best]) / max(float(g), 1e-6)
            sc.bounds[r, 0:3] = (pos[r] + dirv * into_range).astype(f32)
            se[r] = (f32(0.0), g) if r % 3 == 0 else (g, g + f32(1.0))
    sc.range_se = se
    sc.range_use_aabb = ua
    sc.range_view_pos = vp
    sc.range_mask = np.zeros(n, np.uint32)
    return sc, extra


def check_range_sensitivity(sc, gt):
    """The restated real test equals the oracle on these GlobalTransforms, and each mutant changes at least one mask bit."""
    want = orc.check_visibility_ranges(gt, sc.bounds, sc.flags, sc.range_se, sc.range_use_aabb, sc.range_view_pos)
    base = restated_masks(gt, sc.bounds, sc.flags, sc.range_se, sc.range_use_aabb, sc.range_view_pos)
    bad = np.nonzero(base != want)[0]
    assert not len(bad), f"the float32 restatement disagrees with the oracle on rows {bad[:8]}"
    flipped = {}
    for m in MUTANTS:
        diff = restated_masks(gt, sc.bounds, sc.flags, sc.range_se, sc.range_use_aabb, sc.range_view_pos, m) != base
        assert diff.any(), f"the scene cannot detect the {m} mutant"
        flipped[m] = int(diff.sum())
    # the camera-indexed bits are used, bit 31 is set somewhere, and rows outside the query read 0
    assert (want & 0x7).any() and (want >> 31).any()
    out = ((sc.flags & bb.F_HAS_VIS_RANGE) == 0) | ((sc.flags & bb.F_NO_CPU_CULLING) != 0)
    assert out.any() and not want[out].any()
    return flipped


RANGE_CASES = [(41, 0.0), (42, 1e3), (43, 1e5)]


@pytest.mark.parametrize("seed,offset", RANGE_CASES)
def test_range_scene_detects_every_mutant_of_check_visibility_ranges(seed, offset):
    sc, extra = range_scene(seed, offset)
    gt = np.tile(np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], f32), (sc.n, 1))
    orc.propagate(sc.parent, sc.trs, gt, np.ones(sc.n, np.uint8), True)
    check_range_sensitivity(sc, gt)
    for frame in (1, 2):                          # the rotated view orders keep the boundaries, at other bits
        sc.range_view_pos = range_views(sc, extra, frame)
        for m in ("gt_for_ge", "le_for_lt"):
            assert (restated_masks(gt, sc.bounds, sc.flags, sc.range_se, sc.range_use_aabb, sc.range_view_pos, m)
                    != restated_masks(gt, sc.bounds, sc.flags, sc.range_se, sc.range_use_aabb, sc.range_view_pos)).any()
