"""RenderLayers past the first 64 layers, for the light stages (TEST INFRASTRUCTURE).

`RenderLayers` models crates/bevy_camera/src/visibility/render_layers.rs: a list of 64-bit blocks, `with` / `without`
(which shrinks trailing zero blocks), `shrink`, the block-wise operators and `intersects`, which ANDs the blocks of the
common prefix (:121-135).  Its `as_ptr()` shortcut (:124) never changes the outcome at the call sites restated here:
- assign_objects_to_clusters clones each light's layers into its assignment data (assign.rs:204), so the light's pointer
  is never the view's;
- in the light systems (bevy_light/src/lib.rs:437, 611, 703) both pointers are equal only when both sides fall back to
  the `DEFAULT_LAYERS` static (layer 0), and then the block-wise AND (1 & 1) is true as well.
So `intersects` below is the zip alone.

The oracle (oracle/bevy_oracle.c) restates the cluster and shadow stages with block 0 only.  The functions here restate
them over blocks 0..3 through it, exactly: the layer test of those stages is a yes / no per (light, view) or per
(light, entity) pair and nothing else reads the layers, so each view (clusters) or each light (shadows) is run on its
own with the pair's answer as a one-bit block 0 (1 = intersects, 0 = does not) on one side and 1 on the other.  Every
other input is passed through unchanged, and the per-light loops of the shadow restatements are independent apart from
set_visible(), which is idempotent and order-free.
"""
import numpy as np

import oracle as orc

U64 = np.uint64


class RenderLayers:
    """render_layers.rs:20-23: SmallVec<[u64; 1]>; an instance always has at least one block."""

    def __init__(self, blocks=(0,)):
        self.blocks = [int(b) for b in blocks] or [0]

    @staticmethod
    def layer(n):
        return RenderLayers().with_(n) if n >= 64 else RenderLayers([1 << n])

    @staticmethod
    def none():
        return RenderLayers([0])

    @staticmethod
    def default():
        return RenderLayers([1])

    @staticmethod
    def from_layers(layers):
        r = RenderLayers.none()
        for n in layers:
            r = r.with_(n)
        return r

    def with_(self, n):
        b = list(self.blocks)
        b += [0] * max(0, n // 64 + 1 - len(b))
        b[n // 64] |= 1 << (n % 64)
        return RenderLayers(b)

    def without(self, n):
        b = list(self.blocks)
        i = n // 64
        if i < len(b):
            b[i] &= ~(1 << (n % 64)) & 0xFFFFFFFFFFFFFFFF
            if i == len(b) - 1:
                return RenderLayers(b).shrink()
        return RenderLayers(b)

    def shrink(self):
        b = list(self.blocks)
        while len(b) > 1 and b[-1] == 0:
            b.pop()
        return RenderLayers(b)

    def iter(self):
        return [k * 64 + i for k, w in enumerate(self.blocks) for i in range(64) if (w >> i) & 1]

    def intersects(self, other):
        return any(a & b for a, b in zip(self.blocks, other.blocks))

    def _combine(self, other, f):
        n = max(len(self.blocks), len(other.blocks))
        pad = lambda b: b + [0] * (n - len(b))
        return RenderLayers([f(a, b) for a, b in zip(pad(self.blocks), pad(other.blocks))])

    def __and__(self, other):
        return self._combine(other, lambda a, b: a & b).shrink()

    def __or__(self, other):
        return self._combine(other, lambda a, b: a | b)

    def __xor__(self, other):
        return self._combine(other, lambda a, b: a ^ b).shrink()

    def __eq__(self, other):
        return self.blocks == other.blocks

    def blocks4(self):
        """Blocks 0..3 (layers 0..255) as the device takes them: block 0 for the layer_mask arguments, blocks 1..3 for the
        *_render_layers_ext calls.  A set layer past 255 is an error, as in the plugin."""
        if any(self.blocks[4:]):
            raise ValueError(f"RenderLayers {self.iter()} has a layer past 255")
        return np.array((self.blocks + [0, 0, 0])[:4], U64)


def intersects(a, b):
    """Block-wise RenderLayers::intersects over [..., 4] uint64 arrays (broadcasting)."""
    return ((np.asarray(a, U64) & np.asarray(b, U64)) != 0).any(-1)


def shifted(blocks, j):
    """Every layer k of blocks 0..3 moved to k + 64 j (blocks past 3 must be empty)."""
    b = np.asarray(blocks, U64)
    if j:
        assert not b[..., 4 - j:].any(), "a layer would move past 255"
    return np.roll(b, j, axis=-1) if j else b.copy()


def assign_lights_to_clusters(view_in, lights, light_blocks, view_blocks, **kw):
    """orc.assign_lights_to_clusters with the whole RenderLayers test of assign.rs:489: lights [L, 4], light_blocks [L, 4],
    view_blocks [4].  view_in.view_layers is ignored."""
    hit = intersects(np.asarray(light_blocks, U64).reshape(-1, 4), np.asarray(view_blocks, U64)[None]).astype(U64)
    view_in.view_layers = 1
    return orc.assign_lights_to_clusters(view_in, lights, hit, **kw)


def _per_light(fn, n_lights, row_blocks, light_blocks):
    rb = np.asarray(row_blocks, U64)
    return [fn(l, intersects(rb, np.asarray(light_blocks, U64)[l][None]).astype(U64)) for l in range(n_lights)]


def check_point_light_mesh_visibility(gt, bounds, flags, caster, entity_bits, vv, vv_changed, light_sphere, frusta,
                                      row_blocks, light_blocks, range_mask=None, lod_origin_index=-1):
    """lib.rs:517-668 (point half) with the whole RenderLayers test of :611.  Returns [light][face] row lists."""
    ls = np.asarray(light_sphere, np.float32).reshape(-1, 4); fr = np.asarray(frusta, np.float32).reshape(-1, 6, 6, 4)
    one = np.ones(1, U64)
    return _per_light(lambda l, lm: orc.check_point_light_mesh_visibility(
        gt, bounds, flags, caster, entity_bits, vv, vv_changed, ls[l:l + 1], fr[l:l + 1], layer_mask=lm, range_mask=range_mask,
        lod_origin_index=lod_origin_index, light_layers=one)[0], len(ls), row_blocks, light_blocks)


def check_spot_light_mesh_visibility(gt, bounds, flags, caster, entity_bits, vv, vv_changed, light_sphere, frusta,
                                     row_blocks, light_blocks, range_mask=None, lod_origin_index=-1):
    """lib.rs:670-748 with the whole RenderLayers test of :703.  Returns one row list per light."""
    ls = np.asarray(light_sphere, np.float32).reshape(-1, 4); fr = np.asarray(frusta, np.float32).reshape(-1, 6, 4)
    one = np.ones(1, U64)
    return _per_light(lambda l, lm: orc.check_spot_light_mesh_visibility(
        gt, bounds, flags, caster, entity_bits, vv, vv_changed, ls[l:l + 1], fr[l:l + 1], layer_mask=lm, range_mask=range_mask,
        lod_origin_index=lod_origin_index, light_layers=one)[0], len(ls), row_blocks, light_blocks)


def check_dir_light_mesh_visibility(gt, bounds, flags, caster, entity_bits, vv, vv_changed, items, row_blocks,
                                    range_mask=None):
    """lib.rs:342-510 with the whole RenderLayers test of :437: items = [(cascade frusta [C, 6, 4], light blocks [4],
    view_range_index)].  Returns [item][cascade] row lists."""
    return _per_light(lambda l, lm: orc.check_dir_light_mesh_visibility(
        gt, bounds, flags, caster, entity_bits, vv, vv_changed, [(items[l][0], 1, items[l][2])], layer_mask=lm,
        range_mask=range_mask)[0], len(items), row_blocks, [it[1] for it in items])
