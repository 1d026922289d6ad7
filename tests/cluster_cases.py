"""Cameras, light sets and cluster configs shared by the cluster tests (tests/test_oracle_cluster.py on the CPU,
tests/test_gpu_clusters.py on the device)."""
import math

import numpy as np

from bevy_b200 import scenes
from parity import ClusterSpec

PROJECTIONS = {
    "persp_45_16x9": dict(fov=math.pi / 4, aspect=16 / 9),
    "persp_90_1x1": dict(fov=math.pi / 2, aspect=1.0),
    "persp_20_4x3": dict(fov=math.radians(20), aspect=4 / 3),
    "ortho_near0": dict(ortho=(-40.0, 40.0, -22.5, 22.5), near=0.0),
    "ortho_near2": dict(ortho=(-15.0, 25.0, -10.0, 12.0), near=2.0),
}
SPECS = {
    "fixedz_default": ClusterSpec(),
    "single": ClusterSpec(kind="single"),
    "xyz_1_1_1": ClusterSpec(kind="xyz", dims=(1, 1, 1)),
    "xyz_16_9_24": ClusterSpec(kind="xyz", dims=(16, 9, 24)),
    "xyz_64_32_2": ClusterSpec(kind="xyz", dims=(64, 32, 2)),
    "xyz_1_1_1024": ClusterSpec(kind="xyz", dims=(1, 1, 1024)),
    "fixedz_one_slice": ClusterSpec(z_slices=1),
    "fixedz_slices_over_total": ClusterSpec(total=16, z_slices=40),
    "far_constant": ClusterSpec(far_z_constant=80.0),
    "screen_1x1": ClusterSpec(screen=(1, 1)),
    "screen_7x3": ClusterSpec(screen=(7, 3)),
    "screen_1080x1920": ClusterSpec(screen=(1080, 1920)),
    "screen_3840x2160": ClusterSpec(screen=(3840, 2160)),
    "dynamic_resizing": ClusterSpec(max_indices=300),
}


def make_camera(proj, rng, scale=(1.0, 1.0, 1.0)):
    """A camera at a random pose with the projection PROJECTIONS[...] describes; `scale` multiplies its axes."""
    q = scenes.quat_mul(scenes.quat_axis("y", rng.uniform(0, 6.28)), scenes.quat_axis("x", rng.uniform(-0.5, 0.5)))
    gt = scenes.quat_to_gt(q, rng.uniform(-5, 5, 3))
    gt[0:3] *= scale[0]; gt[3:6] *= scale[1]; gt[6:9] *= scale[2]
    if "ortho" in proj:
        l, r, b, t = proj["ortho"]
        return scenes.Camera(gt=gt, near=proj["near"], quat=q, clip_from_view=scenes.orthographic_clip_from_view(l, r, b, t, proj["near"]))
    return scenes.Camera(gt=gt, fov=proj["fov"], aspect=proj["aspect"], quat=q)


def lights_around(cam, rng, n, ortho):
    """Lights in and around the view volume, some straddling or behind the camera, ranges 0.05 .. 30 (and a few 0)."""
    depth = np.concatenate([np.exp(rng.uniform(math.log(0.3), math.log(200.0), n - n // 8)), rng.uniform(-10, 1, n // 8)])
    ext = 1.3 * (40.0 if ortho else np.maximum(np.abs(depth), 1.0) * 0.8)
    pv = np.stack([rng.uniform(-1, 1, n) * ext, rng.uniform(-1, 1, n) * ext * 0.6, -depth], 1)
    M = cam.gt[:9].reshape(3, 3).T.astype(np.float64)
    pw = pv @ M.T + cam.gt[9:12]
    r = np.exp(rng.uniform(math.log(0.05), math.log(30.0), n))
    r[::17] = 0.0
    return np.concatenate([pw, r[:, None]], 1).astype(np.float32)
