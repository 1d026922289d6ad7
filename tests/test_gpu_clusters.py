"""The cluster stage (assign_objects_to_clusters, point lights) on the device, across projections, cluster configs, light
counts (and so kernel paths), placements on and around cluster planes, eight views, index overflow and the kernel
switches.  Every case runs several frames with the Clusters feedback closed, is compared bit for bit with the oracle
(tests/parity.py compare_frame: dims, offsets, indices, farthest_z bits, index count) and holds the device's lists to the
float64 reference of tests/cluster_reference.py."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import bevy_b200 as bb
from bevy_b200 import scenes
from cluster_cases import PROJECTIONS, lights_around, make_camera
from cluster_reference import check_grid, check_view
from parity import ClusterSpec, OracleWorld, compare_frame, run_parity

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
IDENT = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], np.float32)


def scene_of(cams, pos, ranges, screen=(1920, 1080), n_mesh=256, seed=0, name="clusters"):
    """A few hundred cubes (so the cull stage has work) plus point lights at `pos` with `ranges`."""
    rng = np.random.default_rng(seed)
    t = rng.uniform(-80, 80, (n_mesh, 3)).astype(np.float32)
    parent = np.full(n_mesh, scenes.NO_PARENT, np.uint32)
    bounds = np.zeros((n_mesh, 6), np.float32); bounds[:, 3:6] = 0.5
    cols = (parent, scenes._trs(t), bounds, np.full(n_mesh, scenes.F_INHERITED_VISIBLE | scenes.F_HAS_AABB, np.uint8),
            np.full(n_mesh, scenes.CLASS_MESH, np.uint8))
    cols, light_row = scenes._append_lights(cols, np.asarray(pos, np.float32).reshape(-1, 3), np.asarray(ranges, np.float32))
    parent, trs, bounds, flags, cls = cols
    return scenes.Scene(name, parent, trs, bounds, flags, cls, scenes._entity_bits(len(parent)), light_row,
                        np.asarray(ranges, np.float32), list(cams), screen=screen)


def lights_for(cams, n, seed):
    """n lights spread over the cameras' view volumes (some behind / straddling / containing the camera)."""
    rng = np.random.default_rng(seed)
    per = [lights_around(c, rng, max(n // len(cams) + 1, 8), c.clip_from_view is not None) for c in cams]
    lights = np.concatenate(per)[:n]
    return lights[:, :3], lights[:, 3]


def reference_check(spec):
    """on_frame hook: every clustered view's grid and lists against the float64 reference."""
    seen = []

    def on_frame(pipe, world, f):
        sc = pipe.scene
        lights = np.concatenate([world.gt[sc.light_row, 9:12], sc.light_range[:, None]], 1)
        eligible = (world.vv[sc.light_row] & 1).astype(bool)
        rng = np.random.default_rng(f)
        for v, cam in enumerate(sc.cameras):
            cv = pipe.cluster_views[v]
            fb = world.fb_used[v]
            ortho_near = cam.near if cam.clip_from_view is not None else None
            check_grid(spec, cam.gt, ortho_near, fb["far"], fb["cnt"], cv.enabled, cv.dims, cv.near_z, cv.far_z)
            if not cv.enabled:
                continue
            cfv = cam.clip_from_view if cam.clip_from_view is not None else bb.host_perspective(cam.fov, cam.aspect, cam.near)
            el = eligible if sc.light_layers is None else eligible & ((sc.light_layers & np.uint64(1)) != 0)
            off, idx = pipe.ctx.download_clusters(v)
            seen.append(check_view(cv.dims, cv.near_z, cv.far_z, cv.is_orthographic, cfv, cam.gt, cam.far, lights, el,
                                   off, idx, rng))
    on_frame.seen = seen
    return on_frame


def run(scene, spec=None, frames=3, animate=True, before_frame=None):
    spec = spec or ClusterSpec(screen=scene.screen)
    hook = reference_check(spec)
    run_parity(scene, frames=frames, animate=animate, cluster_spec=spec, before_frame=before_frame, on_frame=hook)
    return hook.seen


def ortho_cam(l=-40.0, r=40.0, b=-22.5, t=22.5, near=0.0, yaw=0.0, pos=(0.0, 0.0, 0.0)):
    q = scenes.quat_axis("y", yaw)
    return scenes.Camera(gt=scenes.quat_to_gt(q, pos), near=near, quat=q,
                         clip_from_view=scenes.orthographic_clip_from_view(l, r, b, t, near))


# ---- projections ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("proj", list(PROJECTIONS) + ["mixed", "scaled_uniform", "scaled_nonuniform", "mirrored"])
def test_projections(proj):
    rng = np.random.default_rng(5)
    scale = {"scaled_uniform": (2.0, 2.0, 2.0), "scaled_nonuniform": (0.5, 1.5, 0.75), "mirrored": (-1.0, 1.0, 1.0)}.get(proj)
    if proj == "mixed":
        cams = [make_camera(PROJECTIONS[p], rng) for p in ("persp_45_16x9", "ortho_near0", "persp_90_1x1", "ortho_near2")]
    else:
        cams = [make_camera(PROJECTIONS.get(proj, PROJECTIONS["persp_45_16x9"]), rng, scale or (1.0, 1.0, 1.0))]
    pos, rg = lights_for(cams, 300, 11)
    seen = run(scene_of(cams, pos, rg, name=proj), animate=scale is None)   # the animation rebuilds unit-scale transforms
    assert sum(p for p, _ in seen) > 1000 and sum(e for _, e in seen) > 100


# ---- cluster configs (each with a perspective and an orthographic view) -----------------------------------------------------
CONFIGS = {
    "none": ClusterSpec(kind="none"),
    "zero_viewport": ClusterSpec(screen=(0, 1080)),
    "single": ClusterSpec(kind="single"),
    "xyz_1_1_1": ClusterSpec(kind="xyz", dims=(1, 1, 1)),
    "xyz_16_9_24": ClusterSpec(kind="xyz", dims=(16, 9, 24)),
    "xyz_64_32_2": ClusterSpec(kind="xyz", dims=(64, 32, 2)),
    "xyz_1_1_1024_unstaged": ClusterSpec(kind="xyz", dims=(1, 1, 1024)),    # nx + ny + nz > 512: planes read from global memory
    "fixedz_one_slice": ClusterSpec(z_slices=1),
    "fixedz_slices_over_total": ClusterSpec(total=16, z_slices=40),
    "far_constant": ClusterSpec(far_z_constant=80.0),
    "screen_1x1": ClusterSpec(screen=(1, 1)),
    "screen_7x3": ClusterSpec(screen=(7, 3)),
    "screen_1080x1920": ClusterSpec(screen=(1080, 1920)),
    "screen_3840x2160": ClusterSpec(screen=(3840, 2160)),
}


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_configs(cfg):
    rng = np.random.default_rng(7)
    cams = [make_camera(PROJECTIONS["persp_45_16x9"], rng), make_camera(PROJECTIONS["ortho_near2"], rng)]
    pos, rg = lights_for(cams, 200, 13)
    spec = CONFIGS[cfg]
    sc = scene_of(cams, pos, rg, screen=spec.screen, name=cfg)
    seen = run(sc, spec)
    if cfg in ("none", "zero_viewport"):
        assert not seen
    else:
        assert sum(p for p, _ in seen) > 200


def test_dynamic_resizing_shrinks_and_restores_the_grid():
    """Index count above the bindings' max_indices shrinks x/y next frame; once it falls back the grid grows again."""
    rng = np.random.default_rng(9)
    cams = [make_camera(PROJECTIONS["persp_45_16x9"], rng), make_camera(PROJECTIONS["ortho_near0"], rng)]
    pos, rg = lights_for(cams, 400, 17)
    big, small = np.maximum(rg, 4.0) * 2, np.minimum(rg, 0.2)
    sc = scene_of(cams, pos, big, name="dynamic")
    spec = ClusterSpec(max_indices=6000)
    dims = []
    schedule = [big, big, small, small, big]

    def before(pipe, world, f):
        sc.light_range[:] = schedule[f]
        sc.bounds[sc.light_row, 3] = schedule[f]
        pipe.ctx.set_lights(sc.light_row, sc.light_range)
        pipe.ctx.upload_bounds(int(sc.light_row[0]), sc.bounds[sc.light_row], sc.flags[sc.light_row], sc.class_mask[sc.light_row])
        dims.append([tuple(cv.dims) for cv in pipe.cluster_views])

    run(sc, spec, frames=len(schedule), before_frame=before)
    # frame f's grid follows frame f-1's count: full, shrunk, shrunk, full again (per view)
    for v in range(2):
        d = [dims[f][v] for f in range(1, len(schedule))]       # grids as set up for frames 0..3
        assert d[1][0] * d[1][1] < d[0][0] * d[0][1] and d[3] == d[0], d


# ---- light counts (kernel paths) ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 31, 33, 1024, 3200, 3201, 6400, 6401])
def test_light_counts(n):
    """<= 3200 lights: the 8-CTA fused kernel; 3201 .. 6400: 16 CTAs; above: the three-kernel split path."""
    rng = np.random.default_rng(n)
    cams = [make_camera(PROJECTIONS["persp_45_16x9"], rng), make_camera(PROJECTIONS["ortho_near0"], rng)]
    if n == 0:                                        # lights exist, none is visible: all far behind both cameras
        pos, rg = np.array([[0.0, 0.0, 5000.0], [0.0, 5000.0, 0.0]]), np.array([1.0, 1.0])
    else:
        pos, rg = lights_for(cams, n, n + 1)
    sc = scene_of(cams, pos, rg, name=f"L{n}")
    before = bb.abi.kernel_launch_count()
    seen = run(sc, frames=2, animate=False)
    print(f"{n} lights: {(bb.abi.kernel_launch_count() - before) / 2:.1f} launches per frame")
    if n >= 31:
        assert sum(p for p, _ in seen) > 1000


# ---- placements on and around cluster planes ----------------------------------------------------------------------------
def _planes(cam, spec, far=None):
    """The host's plane tables and z thresholds for an identity-rotation camera, used only to PLACE lights."""
    cfv = cam.clip_from_view if cam.clip_from_view is not None else bb.host_perspective(cam.fov, cam.aspect, cam.near)
    fr = bb.host_compute_frustum(cfv, cam.gt, cam.far)
    fb = bb.ClusterFeedback()
    if far is not None:
        fb.has_farthest_z, fb.farthest_z = 1, far
    cv, scratch = bb.host_cluster_view_setup(spec.abi_config(), cam.gt, cfv, fr, 1, fb)
    d = cv.dims
    xp = np.ctypeslib.as_array(cv.x_planes, (4097 * 4,))[:(d[0] + 1) * 4].reshape(-1, 4).copy()
    yp = np.ctypeslib.as_array(cv.y_planes, (4097 * 4,))[:(d[1] + 1) * 4].reshape(-1, 4).copy()
    zp = np.ctypeslib.as_array(cv.z_planes, (4097 * 4,))[:(d[2] + 1) * 4].reshape(-1, 4).copy()
    thr = bb.host_z_slice_thresholds(np.array(cv.cluster_factors, np.float32), d[2], bool(cv.is_orthographic))
    del scratch
    return xp, yp, zp, thr


def test_orthographic_lights_on_and_tangent_to_cluster_planes():
    """Identity camera, dyadic coordinates: view space is world space exactly, so centres sit exactly on x / y / z
    planes and spheres exactly touch them (the x walk's strict `> 0`, the y distance's sign, the z projection)."""
    cam = ortho_cam(-64.0, 64.0, -32.0, 32.0, near=0.0)
    cam.gt = IDENT.copy()
    spec = ClusterSpec(kind="xyz", dims=(16, 8, 8), far_z_constant=128.0, dynamic_resizing=False)
    xp, yp, zp, thr = _planes(cam, spec)
    xs, ys, zs = xp[1:-1, 3], yp[1:-1, 3], np.array([p[3] / p[2] for p in zp[1:-1]], np.float32)
    pos, rg = [], []
    for i, x in enumerate(xs):
        for r in (0.0, 0.5, 2.0):
            y, z = ys[i % len(ys)] + np.float32(1.25), -np.float32(10 + 12 * (i % 8)) - np.float32(0.375)
            pos += [(x, y, z), (x + np.float32(r), y, z), (x - np.float32(r), y, z)]; rg += [r, r, r]
    for j, y in enumerate(ys):
        for r in (0.5, 2.0):
            x, z = xs[j % len(xs)] + np.float32(0.75), -np.float32(20 + 10 * j)
            pos += [(x, y, z), (x, y + np.float32(r), z), (x, y - np.float32(r), z)]; rg += [r, r, r]
    for k, z in enumerate(zs):
        for r in (0.5, 4.0):
            x, y = xs[k % len(xs)] + np.float32(3.0), ys[k % len(ys)] - np.float32(2.0)
            pos += [(x, y, z), (x, y, z + np.float32(r)), (x, y, z - np.float32(r))]; rg += [r, r, r]
    # range 5, 3 from a y plane: the sphere projected onto that plane has radius sqrtf(25 - 9) = 4 exactly and touches the
    # x plane 4 away, inside the box's cluster range (the box reaches 5 away), so the x walk meets `-dx + r == 0` / `dx + r == 0`
    for i, x in enumerate(xs):
        if x == 0:
            continue
        y, z = ys[(i + 2) % len(ys)], -np.float32(16 * (i % 8) + 8)
        for sx in (4.0, -4.0):
            for sy in (3.0, -3.0):
                pos.append((x + np.float32(sx), y + np.float32(sy), z)); rg.append(5.0)
    seen = run(scene_of([cam], pos, rg, name="ortho_planes"), spec, frames=2, animate=False)
    assert sum(p for p, _ in seen) > 500


def test_perspective_lights_on_slice_thresholds_and_the_near_plane():
    """Centres exactly on the host's z thresholds (view_z_to_z_slice's `>=`), on the near plane (NDC z == 1 exactly:
    z_center is Some), behind the camera and straddling its near plane (seen by a second camera facing backwards),
    containing the camera, range 0, and one light that covers every cluster."""
    cam = scenes.Camera(gt=IDENT.copy(), quat=np.array([0.0, 0.0, 0.0, 1.0]))
    back = scenes.Camera(gt=scenes.quat_to_gt(scenes.quat_axis("y", math.pi), (0.0, 0.0, 0.0)), quat=scenes.quat_axis("y", math.pi))
    spec = ClusterSpec(far_z_constant=200.0, dynamic_resizing=False)
    _, _, _, thr = _planes(cam, spec)
    rng = np.random.default_rng(21)
    pos, rg = [], []
    for k, u in enumerate(thr):
        for j in range(3):
            pos.append((rng.uniform(-0.3, 0.3) * u, rng.uniform(-0.2, 0.2) * u, -u)); rg.append([0.0, 0.05 * u, 0.3 * u][j])
    near = np.float32(0.1)
    for _ in range(96):                                                   # on the near plane
        pos.append((rng.uniform(-0.12, 0.12), rng.uniform(-0.07, 0.07), -near)); rg.append(rng.uniform(0.005, 0.3))
    for _ in range(24):                                                   # behind the camera / straddling the near plane
        pos.append((rng.uniform(-3, 3), rng.uniform(-2, 2), rng.uniform(-0.2, 6.0))); rg.append(rng.uniform(0.1, 4.0))
    pos += [(0.25, -0.5, 0.75), (0.0, 0.0, -30.0)]; rg += [3.0, 1e4]      # contains the camera; covers every cluster
    pos = np.array(pos, np.float32)
    seen = run(scene_of([cam, back], pos, rg, name="persp_planes"), spec, frames=2, animate=False)
    assert sum(p for p, _ in seen) > 1000


# ---- eight views --------------------------------------------------------------------------------------------------------
def test_eight_views():
    """kMaxViews views, every one clustered: views 6 and 7 are never rejected by the cull stage's warp-level test."""
    rng = np.random.default_rng(3)
    cams = []
    for k in range(8):
        c = make_camera(PROJECTIONS["ortho_near0" if k % 3 == 2 else "persp_45_16x9"], rng)
        q = scenes.quat_axis("y", k * math.pi / 4)
        c.gt, c.quat = scenes.quat_to_gt(q, (0.0, 0.0, 0.0)), q
        cams.append(c)
    pos, rg = lights_for(cams, 77 * 8, 5)                              # not a multiple of 32
    seen = run(scene_of(cams, pos, rg, name="eight_views"), frames=3)
    assert len(seen) == 3 * 8 and all(p > 0 for p, _ in seen)


# ---- index overflow -----------------------------------------------------------------------------------------------------
def test_index_overflow_is_flagged_and_clears():
    rng = np.random.default_rng(12)
    cams = [make_camera(PROJECTIONS["persp_45_16x9"], rng)]
    pos, rg = lights_for(cams, 300, 8)
    rg = np.maximum(rg, 3.0)
    sc = scene_of(cams, pos, rg, name="overflow")
    spec = ClusterSpec(far_z_constant=150.0, dynamic_resizing=False)
    cap = 2000
    pipe = bb.VisibilityPipeline(sc, max_cluster_indices=cap, cluster_config=spec.abi_config())
    world = OracleWorld(sc, cluster_kwargs=spec.oracle_kwargs())
    try:
        planes = np.stack([np.ctypeslib.as_array(v.half_spaces).reshape(6, 4).copy() for v in pipe.views])
        _, _, _, clusters = world.frame(planes)
        total = clusters[0][0].total_index_count
        assert total > cap
        pipe.run_frame()
        st = pipe.read_feedback()
        assert st.cluster_index_overflow[0] == 1 and st.cluster_index_count[0] == total
        with pytest.raises(bb.B200VisError) as e:
            pipe.ctx.download_clusters(0)
        assert e.value.code == 6                                       # B200VIS_ERR_CAPACITY
        sc.light_range[:] = 0.25                                       # next frame: fewer indices
        sc.bounds[sc.light_row, 3] = 0.25
        pipe.ctx.set_lights(sc.light_row, sc.light_range)
        pipe.ctx.upload_bounds(int(sc.light_row[0]), sc.bounds[sc.light_row], sc.flags[sc.light_row], sc.class_mask[sc.light_row])
        pipe.update_views()
        st = compare_frame(pipe, world, 1)
        assert st.cluster_index_overflow[0] == 0
        reference_check(spec)(pipe, world, 1)
    finally:
        pipe.close()


# ---- kernel switches (read once per process: one interpreter per case) ----------------------------------------------------
def switch_scenes():
    """A 1080p default scene and an orthographic XYZ scene, through whichever cluster kernel the environment selects."""
    rng = np.random.default_rng(1)
    cams = [make_camera(PROJECTIONS["persp_45_16x9"], rng), make_camera(PROJECTIONS["persp_90_1x1"], rng)]
    pos, rg = lights_for(cams, 700, 2)
    run(scene_of(cams, pos, rg, name="default_1080p"))
    cams = [make_camera(PROJECTIONS["ortho_near2"], rng)]
    pos, rg = lights_for(cams, 500, 3)
    run(scene_of(cams, pos, rg, name="ortho_xyz"), ClusterSpec(kind="xyz", dims=(24, 12, 14)))


SWITCHES = {
    "split": {"B200VIS_CLUSTER_KERNEL": "split"},
    "ctas_2": {"B200VIS_CLUSTER_CTAS": "2"},
    "ctas_4": {"B200VIS_CLUSTER_CTAS": "4"},
    "ctas_16": {"B200VIS_CLUSTER_CTAS": "16"},
    "no_branch": {"B200VIS_CLUSTER_BRANCH": "0"},
    "serial": {"B200VIS_PIPELINE": "0"},
}


@pytest.mark.parametrize("switch", list(SWITCHES))
def test_kernel_switches(switch):
    e = {k: v for k, v in os.environ.items() if not k.startswith("B200VIS_") or k == "B200VIS_LIB"}
    e.update(SWITCHES[switch])
    prog = (f"import sys; sys.path.insert(0, {ROOT!r}); sys.path.insert(0, {HERE!r})\n"
            "import test_gpu_clusters as t\nt.switch_scenes()\n")
    res = subprocess.run([sys.executable, "-c", prog], env=e, capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, f"{SWITCHES[switch]}\n{res.stdout[-2000:]}\n{res.stderr[-4000:]}"


def test_update_views_fast_refuses_an_explicit_projection():
    """b200vis_camera_desc has no projection field: the fast path must not silently cluster an orthographic camera as a
    perspective one."""
    sc = scene_of([ortho_cam()], [(0.0, 0.0, -10.0)], [1.0], name="fast_ortho")
    pipe = bb.VisibilityPipeline(sc)
    try:
        with pytest.raises(ValueError):
            pipe.update_views_fast()
    finally:
        pipe.close()
