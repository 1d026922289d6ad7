"""The reference has NO test for cluster membership (SURVEY.md 4), so the oracle's restatement of the
iterative sphere refinement is cross-checked by geometry: every cluster that truly intersects the light's
view-space sphere must be listed (no false negatives), and everything listed must lie inside the
conservative cluster range of the light's view-space AABB.  The later tests apply the float64 reference of
tests/cluster_reference.py, which builds its froxels without the oracle's plane tables, across projections and configs."""
import math
import zlib

import numpy as np
import pytest

import oracle as orc
from bevy_b200 import scenes
from cluster_cases import PROJECTIONS, SPECS, lights_around, make_camera
from cluster_reference import check_grid, check_view
from parity import ClusterSpec


def _setup(seed, n_lights=40):
    rng = np.random.default_rng(seed)
    q = scenes.quat_mul(scenes.quat_axis("y", rng.uniform(0, 6.28)), scenes.quat_axis("x", rng.uniform(-0.5, 0.5)))
    cam = scenes.quat_to_gt(q, rng.uniform(-5, 5, 3))
    cfv = orc.perspective(math.pi / 4, 16 / 9, 0.1)
    fr = orc.compute_frustum(cfv, cam, 1000.0)
    inv = orc.affine_inverse(cam)
    # lights in front of the camera (view space), then to world space
    pv = np.stack([rng.uniform(-30, 30, n_lights), rng.uniform(-15, 15, n_lights), -rng.uniform(1, 120, n_lights)], 1)
    R = cam[:9].reshape(3, 3).T.astype(np.float64)      # columns x,y,z
    pw = (pv @ R.T + cam[9:12]).astype(np.float32)
    rng_l = np.exp(rng.uniform(math.log(0.5), math.log(25.0), n_lights)).astype(np.float32)
    lights = np.concatenate([pw, rng_l[:, None]], 1).astype(np.float32)
    vin = orc.default_cluster_view_in(cam, cfv, fr, last_farthest_z=150.0)
    return vin, lights, inv, cfv


def test_refinement_has_no_false_negatives_and_stays_in_aabb_range():
    for seed in range(6):
        vin, lights, inv, cfv = _setup(seed)
        out, offsets, idx, planes = orc.assign_lights_to_clusters(vin, lights, want_planes=True)
        dx, dy, dz = out.dims
        xp, yp, zp = [p.astype(np.float64) for p in planes]
        member = np.zeros((dx * dy * dz, len(lights)), bool)
        for c in range(dx * dy * dz):
            member[c, idx[offsets[c]:offsets[c + 1]]] = True
        assert out.total_index_count == member.sum()
        m = inv.astype(np.float64)
        Rm = np.stack([m[0:3], m[3:6], m[6:9]], 1)
        rngs = np.random.default_rng(seed + 100)
        for li, (x, y, z, r) in enumerate(lights.astype(np.float64)):
            cv = Rm @ np.array([x, y, z]) + m[9:12]
            # sample points inside the sphere; the cluster containing each sample must list the light
            pts = rngs.normal(size=(300, 3)); pts /= np.linalg.norm(pts, axis=1, keepdims=True)
            pts = cv + pts * (rngs.uniform(0, 1, (300, 1)) ** (1 / 3)) * r * 0.999
            for p in pts:
                if p[2] >= -1e-3:
                    continue
                # cluster coordinates of the point from the plane tables (inside-facing normals)
                ix = np.nonzero((xp[:, [0, 2]] @ p[[0, 2]]) >= 0)[0]
                iy = np.nonzero((yp[:, [1, 2]] @ p[[1, 2]]) >= 0)[0]
                if len(ix) == 0 or len(iy) == 0 or len(ix) > dx or len(iy) > dy:
                    continue                               # outside the screen
                cx, cy = ix.max(), iy.max()
                depth = -p[2]
                zs = -zp[:, 3] * np.sign(zp[:, 2]) if False else np.array([(-zp[k, 3] / zp[k, 2]) for k in range(dz + 1)])
                below = np.nonzero(-zs <= depth)[0]
                if len(below) == 0 or below.max() >= dz:
                    continue                               # beyond the far slice
                cz = below.max()
                c = (cy * dx + cx) * dz + cz
                assert member[c, li], f"seed {seed}: light {li} misses cluster {(cx, cy, cz)}"


def test_total_index_count_and_farthest_z_are_consistent():
    vin, lights, inv, cfv = _setup(11)
    out, offsets, idx, _ = orc.assign_lights_to_clusters(vin, lights)
    assert offsets[-1] == out.total_index_count == len(idx)
    m = inv.astype(np.float64)
    far = max(0.0, max(-(m[2] * x + m[5] * y + m[8] * z + m[11]) + r for x, y, z, r in lights.astype(np.float64)))
    assert abs(out.farthest_z - far) < 1e-3 * max(1.0, far)


def test_lights_out_of_frustum_or_wrong_layer_are_skipped():
    vin, lights, _, _ = _setup(5, 10)
    out_all, _, idx_all, _ = orc.assign_lights_to_clusters(vin, lights)
    layers = np.ones(len(lights), np.uint64); layers[::2] = 2      # view is on layer 0 only
    out, offsets, idx, _ = orc.assign_lights_to_clusters(vin, lights, layers)
    assert set(idx.tolist()) <= set(range(1, len(lights), 2))
    behind = lights.copy(); behind[:, :3] = 1e6
    out_b, off_b, idx_b, _ = orc.assign_lights_to_clusters(vin, behind)
    assert out_b.total_index_count == 0 and out_b.farthest_z == 0.0


# ---- the float64 reference against the oracle: projections x cluster configs --------------------------------------------
def run_oracle_view(spec, cam, lights, frames=2):
    """The oracle on one view over `frames` frames with the Clusters feedback closed; every frame is held to the reference."""
    cfv = cam.clip_from_view if cam.clip_from_view is not None else orc.perspective(cam.fov, cam.aspect, cam.near)
    fr = orc.compute_frustum(cfv, cam.gt, cam.far)
    ortho_near = cam.near if cam.clip_from_view is not None else None
    far, cnt = None, None
    rng = np.random.default_rng(7)
    checked = [0, 0]
    outs = []
    for _ in range(frames):
        vin = orc.default_cluster_view_in(cam.gt, cfv, fr, last_farthest_z=far, last_index_count=cnt, **spec.oracle_kwargs())
        out, offsets, idx, _ = orc.assign_lights_to_clusters(vin, lights)
        check_grid(spec, cam.gt, ortho_near, far, cnt, not out.cleared, out.dims, out.near, out.far)
        if not out.cleared:
            assert bool(out.is_orthographic) == (ortho_near is not None)
            p, e = check_view(out.dims, out.near, out.far, out.is_orthographic, cfv, cam.gt, cam.far, lights,
                              np.ones(len(lights), bool), offsets, idx, rng)
            checked[0] += p; checked[1] += e
        far, cnt = out.farthest_z, out.total_index_count
        outs.append(out)
    return outs, checked


@pytest.mark.parametrize("proj", list(PROJECTIONS))
@pytest.mark.parametrize("spec", list(SPECS))
def test_reference_holds_the_oracle_across_projections_and_configs(spec, proj):
    rng = np.random.default_rng(zlib.crc32(f"{spec}/{proj}".encode()))
    cam = make_camera(PROJECTIONS[proj], rng)
    lights = lights_around(cam, rng, 160, "ortho" in PROJECTIONS[proj])
    outs, checked = run_oracle_view(SPECS[spec], cam, lights)
    assert checked[0] > 100 and checked[1] > 10, checked           # the check was not vacuous
    if spec == "dynamic_resizing":
        assert outs[0].total_index_count > 300 and np.prod(outs[1].dims[:2]) < np.prod(outs[0].dims[:2])


@pytest.mark.parametrize("proj", ["persp_45_16x9", "ortho_near2"])
@pytest.mark.parametrize("scale", [(2.0, 2.0, 2.0), (0.5, 1.5, 0.75), (-1.0, 1.0, 1.0)])
def test_reference_holds_the_oracle_for_scaled_cameras(proj, scale):
    rng = np.random.default_rng(31)
    cam = make_camera(PROJECTIONS[proj], rng, scale)
    lights = lights_around(cam, rng, 120, "ortho" in proj)
    _, checked = run_oracle_view(ClusterSpec(), cam, lights)
    assert checked[0] > 100 and checked[1] > 10, checked


def test_zero_sized_viewport_and_config_none_clear_the_clusters():
    rng = np.random.default_rng(3)
    cam = make_camera(PROJECTIONS["persp_45_16x9"], rng)
    lights = lights_around(cam, rng, 20, False)
    for spec in (ClusterSpec(kind="none"), ClusterSpec(screen=(0, 1080)), ClusterSpec(screen=(1920, 0))):
        outs, _ = run_oracle_view(spec, cam, lights, frames=1)
        assert outs[0].cleared and outs[0].total_index_count == 0


@pytest.mark.parametrize("proj", list(PROJECTIONS))
def test_host_grid_setup_follows_the_config_rules(proj):
    """The device's per-view constants come from the host's cluster_view_setup: its dims, first slice depth and far z
    are held to the float64 config rules for every config, with and without feedback, for unit and scaled cameras."""
    import bevy_b200 as bb
    rng = np.random.default_rng(zlib.crc32(proj.encode()))
    for scale in ((1.0, 1.0, 1.0), (0.5, 1.5, 0.75), (-1.0, 1.0, 2.0)):
        cam = make_camera(PROJECTIONS[proj], rng, scale)
        cfv = cam.clip_from_view if cam.clip_from_view is not None else bb.host_perspective(cam.fov, cam.aspect, cam.near)
        fr = bb.host_compute_frustum(cfv, cam.gt, cam.far)
        for spec in SPECS.values():
            for far, cnt in ((None, None), (137.25, 900), (3.5, 40000)):
                fb = bb.ClusterFeedback()
                if far is not None:
                    fb.has_farthest_z, fb.farthest_z, fb.has_index_count, fb.index_count = 1, far, 1, cnt
                cv, _ = bb.host_cluster_view_setup(spec.abi_config(), cam.gt, cfv, fr, 1, fb)
                ortho_near = cam.near if cam.clip_from_view is not None else None
                check_grid(spec, cam.gt, ortho_near, far, cnt, cv.enabled, cv.dims, cv.near_z, cv.far_z)
                assert not cv.enabled or bool(cv.is_orthographic) == (ortho_near is not None)
