"""More than eight views per context: the scene generator, the oracle's per-view independence on a 16-view cull, the
new C entry points and the argument checks that run before any device is touched."""
import math
import os
import re

import numpy as np
import pytest

import bevy_b200 as bb
from bevy_b200 import abi, scenes
import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_many_cameras_lights_restates_the_example():
    sc = scenes.many_cameras_lights()
    f32 = np.float32
    assert sc.n == 2 + 5 and len(sc.cameras) == 16 and sc.screen == (480, 270)
    # circle base: Circle::new(4.0), rotated -pi/2 about X; unit cube at (0, 0.5, 0)
    np.testing.assert_allclose(sc.bounds[0, 3:6], (4.0, 4.0, 0.0))
    np.testing.assert_allclose(sc.trs[0, 3:7], (-math.sin(math.pi / 4), 0, 0, math.cos(math.pi / 4)), atol=1e-7)
    np.testing.assert_allclose(sc.trs[1, 0:3], (0.0, 0.5, 0.0)); np.testing.assert_allclose(sc.bounds[1, 3:6], 0.5)
    # NUM_LIGHTS = 5 point lights, range 20 (PointLight::default), at (sin a * 4, 2, cos a * 4)
    assert len(sc.light_row) == 5 and (sc.light_range == 20.0).all()
    for i, r in enumerate(sc.light_row):
        a = f32(i) / f32(5) * f32(math.pi) * f32(2)
        np.testing.assert_allclose(sc.trs[r, 0:3], (math.sin(a) * 4, 2.0, math.cos(a) * 4), atol=1e-6)
        assert sc.flags[r] & scenes.F_SPHERE_FROM_GT and sc.bounds[r, 3] == 20.0
    # 16 cameras on the radius-4 circle at height 2.5, looking at the origin, 480x270 viewports
    for i, cam in enumerate(sc.cameras):
        a = f32(i) / f32(16) * f32(math.pi) * f32(2)
        np.testing.assert_allclose(cam.gt[9:12], (math.sin(a) * 4, 2.5, math.cos(a) * 4), atol=1e-6)
        fwd = -cam.gt[6:9]                                   # -Z axis of the camera
        np.testing.assert_allclose(fwd, -cam.gt[9:12] / np.linalg.norm(cam.gt[9:12]), atol=1e-6)
        assert abs(cam.aspect - 16.0 / 9.0) < 1e-6 and cam.fov == math.pi / 4
    # rotate_around(ZERO, rotation_y): the cameras stay on their circle and keep looking at the origin
    scenes.rotate_cameras(sc, 0.3)
    for cam in sc.cameras:
        assert abs(np.hypot(cam.gt[9], cam.gt[11]) - 4.0) < 1e-5 and cam.gt[10] == np.float32(2.5)
        np.testing.assert_allclose(-cam.gt[6:9], -cam.gt[9:12] / np.linalg.norm(cam.gt[9:12]), atol=1e-5)
    wide = scenes.many_cameras_lights(forest_kwargs=dict(n_trees=10, levels=4))
    assert wide.n == 7 + 10 * 15 and (wide.roots >= 7).all() and (wide.parent[7:][wide.parent[7:] != scenes.NO_PARENT] >= 7).all()


def _sixteen_view_state(seed):
    sc = scenes.many_cameras_lights(forest_kwargs=dict(n_trees=40, levels=5))
    sc.trs[sc.roots, 0:3] *= np.float32(0.02)               # the forest inside the camera ring
    rng = np.random.default_rng(seed)
    n, V = sc.n, len(sc.cameras)
    gt = np.tile(np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], np.float32), (n, 1))
    assert orc.propagate(sc.parent, sc.trs, gt, np.ones(n, np.uint8), True)[0] == 0
    planes = np.stack([orc.compute_frustum(orc.perspective(c.fov, c.aspect, c.near), c.gt, c.far) for c in sc.cameras])
    layer_mask = rng.choice([1, 1, 2, 3], n).astype(np.uint64)
    view_layers = rng.choice([1, 3, 2], V).astype(np.uint64)
    view_flags = np.full(V, bb.VIEW_ACTIVE, np.uint8); view_flags[[3, 11]] = 0; view_flags[12] |= bb.VIEW_NO_CPU_CULLING
    vv = rng.integers(0, 4, n).astype(np.uint8)
    return sc, gt, planes, layer_mask, view_layers, view_flags, vv


@pytest.mark.parametrize("seed", [0, 1])
def test_oracle_sixteen_view_cull_is_the_union_of_one_view_culls(seed):
    sc, gt, planes, layer_mask, view_layers, view_flags, vv0 = _sixteen_view_state(seed)
    vv = vv0.copy()
    _, lists = orc.cull(gt, sc.bounds, sc.flags, sc.class_mask, sc.entity_bits, vv, planes, view_layers=view_layers,
                        view_flags=view_flags, layer_mask=layer_mask)
    any_vis = np.zeros(sc.n, bool)
    listed = 0
    for v in range(len(sc.cameras)):
        one = vv0.copy()
        _, l1 = orc.cull(gt, sc.bounds, sc.flags, sc.class_mask, sc.entity_bits, one, planes[v:v + 1],
                         view_layers=view_layers[v:v + 1], view_flags=view_flags[v:v + 1], layer_mask=layer_mask)
        if lists[v] is None:
            assert l1[0] is None and not view_flags[v] & bb.VIEW_ACTIVE
            continue
        assert np.array_equal(lists[v], l1[0]), f"view {v}"
        any_vis |= (one & 1).astype(bool)
        listed += len(l1[0])
    assert listed > 100
    assert np.array_equal((vv & 1).astype(bool), any_vis)


def test_new_entry_points_are_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "b200vis.h")).read()
    assert re.search(r"#define B200VIS_MAX_CAMERAS\s+32u", hdr) and re.search(r"#define B200VIS_MAX_VIEWS\s+8u", hdr)
    assert abi.MAX_CAMERAS == 32 and abi.MAX_VIEWS == 8 and len(abi.FrameStats().visible_count) == 8
    lib = bb.load_library()
    for name in ("b200vis_download_view_stats", "b200vis_set_view_stats_sink"):
        assert re.search(r"B200VIS_API\s+int32_t\s+%s\s*\(" % name, hdr), name
        assert name in abi.EXPORTED_SYMBOLS and hasattr(lib, name), name


@pytest.mark.parametrize("max_views,world_size", [(0, 1), (33, 1), (9, 2), (32, 4)])
def test_view_limits_are_checked_before_the_device(max_views, world_size):
    with pytest.raises(bb.B200VisError) as e:
        bb.Context(16, max_views=max_views, world_size=world_size)
    assert e.value.code == 1
