"""No GPU needed: the RenderLayers model of tests/light_layers_reference.py against the reference's own tests
(render_layers.rs:252-360, their expected values copied as data), and the full-RenderLayers restatements of the cluster and
shadow stages built on the block-0 oracle:
- with every block 1..3 empty they give exactly what the block-0 oracle calls give;
- moving every light, view and entity layer k to k + 64 j (j = 1..3) leaves every cluster list, index count, farthest z,
  shadow list and ViewVisibility byte unchanged.
And include/b200vis.h, compiled as C with -Wall -Wextra -Werror, declares b200vis_set_light_render_layers_ext and
b200vis_set_shadow_item_render_layers_ext with the argument types the Python signatures pass; the library exports both."""
import os
import subprocess

import numpy as np
import pytest

import light_layers_reference as LR
import oracle as orc
from bevy_b200 import abi, scenes
from light_layers_reference import RenderLayers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64 = np.uint64


# ---- the model, pinned on render_layers.rs's tests -----------------------------------------------------------------------
# rendering_mask_sanity (:256-331): (layers, expected blocks)
SANITY_BLOCKS = [([0], [1]), ([1], [2]), ([0, 1], [3]), ([0, 2345], None)]
SANITY_2345 = dict(len=37, block0=1, block36=2199023255552)
# (a, b, intersects)
SANITY_INTERSECTS = [([0, 2345], [0], True), ([1], [1], True), ([0, 3], [3], True), ([0], [0], True), ([0], [1], False),
                     ([], [], False)]
ROUNDTRIP = [[0, 2, 16, 30], [0, 5, 17, 55, 999, 1025, 1026]]
# render_layer_ops (:336-347): a = [2, 4, 6], b = [1, 2, 3, 4, 5]
OPS = dict(a=[2, 4, 6], b=[1, 2, 3, 4, 5], union=[1, 2, 3, 4, 5, 6], inter=[2, 4], xor=[1, 3, 5, 6])
MANY = [(1 << 64) - 1]


def test_rendering_mask_sanity():
    for layers, blocks in SANITY_BLOCKS[:3]:
        assert RenderLayers.from_layers(layers).blocks == blocks
        assert len(RenderLayers.from_layers(layers).blocks) == 1
    assert RenderLayers.layer(0).with_(1).without(0).blocks == [2]
    l = RenderLayers.layer(0).with_(2345)
    assert len(l.blocks) == SANITY_2345["len"] and l.blocks[0] == SANITY_2345["block0"] and l.blocks[36] == SANITY_2345["block36"]
    for a, b, want in SANITY_INTERSECTS:
        assert RenderLayers.from_layers(a).intersects(RenderLayers.from_layers(b)) == want, (a, b)
    assert RenderLayers.layer(0).intersects(RenderLayers([1]))
    assert RenderLayers.default().intersects(RenderLayers.default())
    assert not RenderLayers.none().intersects(RenderLayers.none())
    for layers in ROUNDTRIP:
        assert RenderLayers.from_layers(layers).iter() == layers


def test_render_layer_ops():
    a, b = RenderLayers.from_layers(OPS["a"]), RenderLayers.from_layers(OPS["b"])
    assert a | b == RenderLayers.from_layers(OPS["union"])
    assert a & b == RenderLayers.from_layers(OPS["inter"])
    assert a ^ b == RenderLayers.from_layers(OPS["xor"])
    many = RenderLayers(MANY)
    assert RenderLayers.none() & many == RenderLayers.none()
    assert RenderLayers.none() | many == many
    assert RenderLayers.none() ^ many == many


def test_render_layer_shrink():
    layers = RenderLayers.from_layers([1, 77])
    assert len(layers.blocks) == 2
    assert len(layers.without(77).blocks) == 1


def test_intersects_is_the_zip_over_the_common_prefix():
    """A block one side lacks never matches; the array form agrees with the model on blocks 0..3."""
    assert not RenderLayers.from_layers([70]).intersects(RenderLayers.from_layers([6]))
    assert not RenderLayers([0, 4]).intersects(RenderLayers([0]))
    rng = np.random.default_rng(0)
    for _ in range(300):
        a = RenderLayers.from_layers(rng.choice(256, rng.integers(0, 4), replace=False).tolist())
        b = RenderLayers.from_layers(rng.choice(256, rng.integers(0, 4), replace=False).tolist())
        assert LR.intersects(a.blocks4(), b.blocks4()) == a.intersects(b)
    with pytest.raises(ValueError):
        RenderLayers.layer(256).blocks4()


# ---- the restatements ------------------------------------------------------------------------------------------------------
def random_layers(rng, n, j=0, hi=8):
    """[n, 4] blocks: default, none(), or a few layers of 0..hi-1 -- all moved up by 64 j."""
    out = np.zeros((n, 4), U64)
    kind = rng.integers(0, 4, n)
    for i in range(n):
        if kind[i] == 0:
            ls = [0]
        elif kind[i] == 1:
            ls = []
        else:
            ls = rng.choice(hi, rng.integers(1, 3), replace=False).tolist()
        out[i] = RenderLayers.from_layers([k + 64 * j for k in ls]).blocks4()
    return out


def world(seed=3):
    sc = scenes.forest(n_trees=24, levels=5, n_lights=48, seed=seed)
    gt = np.tile(orc.IDENTITY_GT, (sc.n, 1))
    orc.propagate(sc.parent, sc.trs, gt, np.ones(sc.n, np.uint8))
    planes = []
    for cam in sc.cameras:
        planes.append(orc.compute_frustum(orc.perspective(cam.fov, cam.aspect, cam.near), cam.gt, cam.far))
    vv = np.zeros(sc.n, np.uint8)
    orc.cull(gt, sc.bounds, sc.flags, sc.class_mask, sc.entity_bits, vv, np.stack(planes))
    return sc, gt, vv, planes


def clusters(sc, gt, vv, planes, light_blocks, view_blocks, full):
    vis = np.nonzero(vv[sc.light_row] & 1)[0]
    lights = np.concatenate([gt[sc.light_row[vis], 9:12], sc.light_range[vis, None]], 1).astype(np.float32)
    out = []
    for v, cam in enumerate(sc.cameras):
        fb = dict(far=None, cnt=None)
        for _ in range(3):                                   # the Clusters feedback loop
            vin = orc.default_cluster_view_in(cam.gt, orc.perspective(cam.fov, cam.aspect, cam.near), planes[v],
                                              view_layers=int(view_blocks[v][0]), last_farthest_z=fb["far"],
                                              last_index_count=fb["cnt"])
            if full:
                o, off, idx, _ = LR.assign_lights_to_clusters(vin, lights, light_blocks[vis], view_blocks[v])
            else:
                o, off, idx, _ = orc.assign_lights_to_clusters(vin, lights, np.ascontiguousarray(light_blocks[vis, 0]))
            fb = dict(far=o.farthest_z, cnt=o.total_index_count)
            out.append((tuple(o.dims), off, vis[idx], o.total_index_count, np.float32(o.farthest_z).view(np.uint32)))
    return out


def same_clusters(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x[0] == y[0] and (x[1] == y[1]).all() and len(x[2]) == len(y[2]) and (x[2] == y[2]).all()
        assert x[3] == y[3] and x[4] == y[4]


def shadows(sc, gt, vv0, row_blocks, item_blocks, full):
    """Point, spot and cascade items over the lights; returns every list and the ViewVisibility bytes / change flags."""
    caster = np.ones(sc.n, np.uint8); caster[sc.light_row] = 0
    vv, ch = vv0.copy(), np.zeros(sc.n, np.uint8)
    pts, spots = np.arange(0, 12), np.arange(12, 20)
    sph = lambda o: np.concatenate([gt[sc.light_row[o], 9:12], sc.light_range[o, None] * 4]).astype(np.float32)
    fr = lambda o: orc.point_light_frusta(gt[sc.light_row[o]], sc.light_range[o] * 4)
    casc = [(np.stack([orc.point_light_frusta(np.concatenate([np.eye(3, dtype=np.float32).ravel(), [0, 0, 0]]).astype(np.float32),
                                              r)[c] for c in range(2)]), -1) for r in (60.0, 200.0)]
    kw = dict(range_mask=None)
    res = []
    ib = np.asarray(item_blocks, U64)
    if full:
        res += LR.check_point_light_mesh_visibility(gt, sc.bounds, sc.flags, caster, sc.entity_bits, vv, ch,
                                                    np.stack([sph(o) for o in pts]), np.stack([fr(o) for o in pts]),
                                                    row_blocks, ib[:12], **kw)
        res += LR.check_spot_light_mesh_visibility(gt, sc.bounds, sc.flags, caster, sc.entity_bits, vv, ch,
                                                   np.stack([sph(o) for o in spots]), np.stack([fr(o)[o % 6] for o in spots]),
                                                   row_blocks, ib[12:20], **kw)
        res += LR.check_dir_light_mesh_visibility(gt, sc.bounds, sc.flags, caster, sc.entity_bits, vv, ch,
                                                  [(f, ib[20 + i], vri) for i, (f, vri) in enumerate(casc)], row_blocks, **kw)
    else:
        lm = np.ascontiguousarray(row_blocks[:, 0])
        res += orc.check_point_light_mesh_visibility(gt, sc.bounds, sc.flags, caster, sc.entity_bits, vv, ch,
                                                     np.stack([sph(o) for o in pts]), np.stack([fr(o) for o in pts]),
                                                     layer_mask=lm, light_layers=np.ascontiguousarray(ib[:12, 0]), **kw)
        res += orc.check_spot_light_mesh_visibility(gt, sc.bounds, sc.flags, caster, sc.entity_bits, vv, ch,
                                                    np.stack([sph(o) for o in spots]), np.stack([fr(o)[o % 6] for o in spots]),
                                                    layer_mask=lm, light_layers=np.ascontiguousarray(ib[12:20, 0]), **kw)
        res += orc.check_dir_light_mesh_visibility(gt, sc.bounds, sc.flags, caster, sc.entity_bits, vv, ch,
                                                   [(f, int(ib[20 + i, 0]), vri) for i, (f, vri) in enumerate(casc)],
                                                   layer_mask=lm, **kw)
    flat = []
    for r in res:
        flat += [np.asarray(x) for x in r] if isinstance(r, list) else [np.asarray(r)]
    return flat, vv, ch


def same_shadows(a, b):
    la, vva, cha = a
    lb, vvb, chb = b
    assert len(la) == len(lb) and all(len(x) == len(y) and (x == y).all() for x, y in zip(la, lb))
    assert (vva == vvb).all() and (cha == chb).all()


def test_empty_blocks_give_the_block0_oracle_exactly():
    sc, gt, vv, planes = world()
    rng = np.random.default_rng(5)
    lb, vb, rb = random_layers(rng, len(sc.light_row)), random_layers(rng, 4), random_layers(rng, sc.n)
    vb[1] = RenderLayers.layer(1).blocks4()
    a, b = clusters(sc, gt, vv, planes, lb, vb, True), clusters(sc, gt, vv, planes, lb, vb, False)
    same_clusters(a, b)
    assert sum(x[3] for x in a) > 0
    ib = random_layers(rng, 22)
    sa, sb = shadows(sc, gt, vv, rb, ib, True), shadows(sc, gt, vv, rb, ib, False)
    same_shadows(sa, sb)
    assert sum(len(x) for x in sa[0]) > 0


@pytest.mark.parametrize("j", [1, 2, 3])
def test_shifting_every_layer_by_whole_blocks_changes_nothing(j):
    sc, gt, vv, planes = world()
    rng = np.random.default_rng(9)
    lb, vb, rb, ib = random_layers(rng, len(sc.light_row)), random_layers(rng, 4), random_layers(rng, sc.n), random_layers(rng, 22)
    vb[1] = RenderLayers.layer(2).blocks4()                  # a view with no default layer
    base = clusters(sc, gt, vv, planes, lb, vb, True)
    moved = clusters(sc, gt, vv, planes, LR.shifted(lb, j), LR.shifted(vb, j), True)
    same_clusters(base, moved)
    assert any(len(x[2]) for x in base) and any(x[3] != y[3] for x, y in zip(base, clusters(
        sc, gt, vv, planes, np.zeros_like(lb), vb, True)))      # the layers decide something
    same_shadows(shadows(sc, gt, vv, rb, ib, True), shadows(sc, gt, vv, LR.shifted(rb, j), LR.shifted(ib, j), True))
    # the block-0 oracle, by contrast, loses the shifted layers
    if j:
        lost = clusters(sc, gt, vv, planes, LR.shifted(lb, j), LR.shifted(vb, j), False)
        assert sum(x[3] for x in lost) == 0


# ---- the C header and the library ----------------------------------------------------------------------------------------
SRC = r"""
#include <stdio.h>
#include "b200vis.h"
int main(void) {
    int32_t (*lights_fn)(b200vis_ctx *, uint32_t, const uint64_t *) = b200vis_set_light_render_layers_ext;
    int32_t (*items_fn)(b200vis_ctx *, uint32_t, const uint64_t *) = b200vis_set_shadow_item_render_layers_ext;
    printf("%d\n", (lights_fn != 0) + (items_fn != 0));
    return 0;
}
"""


def test_header_declares_the_entry_points(tmp_path):
    src = tmp_path / "decl.c"
    src.write_text(SRC)
    cmd = ["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(src)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    for name in ("b200vis_set_light_render_layers_ext", "b200vis_set_shadow_item_render_layers_ext"):
        argtypes = abi._SIGNATURES[name][1]
        assert len(argtypes) == 3 and argtypes[1] is abi.C.c_uint32


def test_entry_points_are_exported():
    names = ("b200vis_set_light_render_layers_ext", "b200vis_set_shadow_item_render_layers_ext")
    for name in names:
        assert name in abi.EXPORTED_SYMBOLS
    lib = os.path.join(ROOT, "bevy_b200", "libb200vis.so")
    if not os.path.exists(lib):
        pytest.skip("libb200vis.so is not built")
    syms = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True, check=True).stdout.split()
    assert all(n in syms for n in names)
