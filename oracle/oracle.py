"""ctypes/numpy wrapper over libbevy_oracle.so (TEST INFRASTRUCTURE).

Every function mirrors one exported C function of oracle/bevy_oracle.c, which
cites the reference file:line it restates.
"""
import ctypes as C
import os
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
NO_PARENT = 0xFFFFFFFF
DETACHED = 0xFFFFFFFE

F_INHERITED_VISIBLE = 0x01
F_HAS_AABB = 0x02
F_HAS_SPHERE = 0x04
F_NO_FRUSTUM_CULLING = 0x08
F_HAS_VIS_RANGE = 0x10
F_NO_CPU_CULLING = 0x20
F_SPHERE_FROM_GT = 0x40
F_TRANSFORM_CHANGED = 0x80
VIEW_ACTIVE = 0x01
VIEW_NO_CPU_CULLING = 0x02


def build(force=False):
    """Compile the oracle with the committed Makefile (gcc, no FMA contraction)."""
    subprocess.check_call(["make", "-s", "-C", _HERE] + (["-B"] if force else []))   # no-op when up to date


_lib = None
_lib_mt = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(os.path.join(_HERE, "libbevy_oracle.so"))
        _declare(_lib)
    return _lib


def lib_mt():
    global _lib_mt
    if _lib_mt is None:
        build()
        _lib_mt = C.CDLL(os.path.join(_HERE, "libbevy_oracle_mt.so"))
        _declare(_lib_mt)
        _lib_mt.orc_mt_threads.restype = C.c_int
        _lib_mt.orc_mt_set_threads.argtypes = [C.c_int]
        _lib_mt.orc_mt_prepare.restype = C.c_int
        _lib_mt.orc_mt_prepare.argtypes = [C.c_uint32, C.POINTER(C.c_uint32)]
    return _lib_mt


class ClusterViewIn(C.Structure):
    _fields_ = [
        ("config_kind", C.c_uint32), ("cfg_dims", C.c_uint32 * 3),
        ("cfg_total", C.c_uint32), ("cfg_z_slices", C.c_uint32),
        ("first_slice_depth", C.c_float), ("far_z_mode", C.c_uint32),
        ("far_z_constant", C.c_float), ("dynamic_resizing", C.c_uint32),
        ("screen_w", C.c_uint32), ("screen_h", C.c_uint32),
        ("view_cluster_bindings_max_indices", C.c_uint32),
        ("camera_gt", C.c_float * 12), ("clip_from_view", C.c_float * 16),
        ("frustum", C.c_float * 24), ("view_layers", C.c_uint64),
        ("has_last_farthest_z", C.c_uint32), ("last_farthest_z", C.c_float),
        ("has_last_index_count", C.c_uint32), ("last_index_count", C.c_uint32),
    ]


class ClusterViewOut(C.Structure):
    _fields_ = [
        ("cleared", C.c_uint32), ("tile_size", C.c_uint32 * 2), ("dims", C.c_uint32 * 3),
        ("near", C.c_float), ("far", C.c_float), ("is_orthographic", C.c_uint32),
        ("cluster_factors", C.c_float * 2), ("view_from_world", C.c_float * 16),
        ("view_from_world_scale", C.c_float * 3), ("view_from_world_scale_max", C.c_float),
        ("total_index_count", C.c_uint32), ("farthest_z", C.c_float),
    ]


def _p(a, t):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _declare(l):
    l.orc_frustum_intersects_sphere.restype = C.c_int
    l.orc_frustum_intersects_sphere.argtypes = [C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_float, C.c_int]
    l.orc_frustum_intersects_obb.restype = C.c_int
    l.orc_frustum_intersects_obb.argtypes = [C.POINTER(C.c_float)] * 4 + [C.c_int, C.c_int]
    l.orc_frustum_intersects_obb_identity.restype = C.c_int
    l.orc_frustum_intersects_obb_identity.argtypes = [C.POINTER(C.c_float)] * 3
    l.orc_frustum_contains_aabb.restype = C.c_int
    l.orc_frustum_contains_aabb.argtypes = [C.POINTER(C.c_float)] * 4
    l.orc_sphere_intersects_obb.restype = C.c_int
    l.orc_sphere_intersects_obb.argtypes = [C.POINTER(C.c_float), C.c_float] + [C.POINTER(C.c_float)] * 3
    l.orc_perspective_infinite_reverse_rh.argtypes = [C.c_float, C.c_float, C.c_float, C.POINTER(C.c_float)]
    l.orc_compute_frustum.argtypes = [C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_float, C.POINTER(C.c_float)]
    l.orc_propagate.restype = C.c_int
    l.orc_propagate.argtypes = [C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_float), C.POINTER(C.c_float),
                                C.POINTER(C.c_uint8), C.POINTER(C.c_uint8), C.c_int, C.POINTER(C.c_uint8)]
    l.orc_cull.restype = C.c_int
    l.orc_cull.argtypes = [C.c_uint32, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_uint8),
                           C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_uint8),
                           C.POINTER(C.c_uint64), C.POINTER(C.c_uint8), C.POINTER(C.c_uint8),
                           C.c_uint32, C.POINTER(C.c_float), C.POINTER(C.c_uint64), C.POINTER(C.c_uint8),
                           C.POINTER(C.c_int8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    l.orc_assign_lights_to_clusters.restype = C.c_int
    l.orc_assign_lights_to_clusters.argtypes = [C.POINTER(ClusterViewIn), C.c_uint32, C.POINTER(C.c_float),
                                                C.POINTER(C.c_uint64), C.POINTER(ClusterViewOut),
                                                C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_uint32,
                                                C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float)]
    l.orc_cluster_dimensions_for_screen_size.argtypes = [C.c_uint32, C.POINTER(C.c_uint32), C.c_uint32, C.c_uint32,
                                                         C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32)]
    l.orc_clusters_update.argtypes = [C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                      C.POINTER(C.c_uint32)]
    l.orc_logf.restype = C.c_float
    l.orc_logf.argtypes = [C.c_float]
    l.orc_powf.restype = C.c_float
    l.orc_powf.argtypes = [C.c_float, C.c_float]
    l.orc_view_z_to_z_slice.restype = C.c_uint32
    l.orc_view_z_to_z_slice.argtypes = [C.POINTER(C.c_float), C.c_uint32, C.c_float, C.c_int]
    l.orc_set_defer_mark_newly_hidden.argtypes = [C.c_int]
    l.orc_mark_newly_hidden.argtypes = [C.c_uint32, C.POINTER(C.c_uint8), C.POINTER(C.c_uint8), C.POINTER(C.c_uint8)]
    l.orc_point_light_frusta.argtypes = [C.POINTER(C.c_float), C.c_float, C.c_float, C.POINTER(C.c_float)]
    l.orc_check_point_light_mesh_visibility.restype = C.c_int
    l.orc_check_point_light_mesh_visibility.argtypes = [
        C.c_uint32, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_uint8), C.POINTER(C.c_uint8),
        C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint8),
        C.POINTER(C.c_uint8), C.c_uint32, C.POINTER(C.c_float), C.POINTER(C.c_uint64), C.POINTER(C.c_float),
        C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    l.orc_check_spot_light_mesh_visibility.restype = C.c_int
    l.orc_check_spot_light_mesh_visibility.argtypes = l.orc_check_point_light_mesh_visibility.argtypes
    l.orc_check_dir_light_mesh_visibility.restype = C.c_int
    l.orc_check_dir_light_mesh_visibility.argtypes = [
        C.c_uint32, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_uint8), C.POINTER(C.c_uint8),
        C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_uint8), C.POINTER(C.c_uint8),
        C.c_uint32, C.POINTER(C.c_int32), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_float),
        C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    if hasattr(l, "orc_update_cpu_culled_entities"):   # bevy_oracle_next.c (not part of the MT baseline library)
        U64P, U32P, U8P = C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_uint8)
        l.orc_sort_pairs_by_main.argtypes = [U64P, U64P, C.c_uint32]
        l.orc_update_cpu_culled_entities.argtypes = [U64P, U64P, C.c_uint32, U64P, U64P, C.c_uint32,
                                                     U64P, U64P, U32P, U64P, U64P, U32P]
        l.orc_entity_pair_is_visible.restype = C.c_int
        l.orc_entity_pair_is_visible.argtypes = [U64P, U64P, C.c_uint32, C.c_uint64, C.c_uint64]
        l.orc_cluster_bindings.argtypes = [C.c_uint32, U32P, U32P, U32P, C.c_uint32, C.c_int, U32P, U32P, U32P, U32P]
        l.orc_check_visibility_ranges.argtypes = [C.c_uint32, C.POINTER(C.c_float), C.POINTER(C.c_float), U8P,
                                                  C.POINTER(C.c_float), U8P, C.c_uint32, C.POINTER(C.c_float), U32P]
        l.orc_visibility_propagate.restype = C.c_int
        l.orc_visibility_propagate.argtypes = [C.c_uint32, U32P, U8P, U8P, U8P, C.c_uint32, U32P, C.c_uint32, U32P]
    for name in ("orc_half_space_new", "orc_affine_from_trs", "orc_affine_inverse", "orc_mat4_inverse"):
        getattr(l, name).argtypes = [C.POINTER(C.c_float)] * 2
    for name in ("orc_affine_mul", "orc_mat4_mul"):
        getattr(l, name).argtypes = [C.POINTER(C.c_float)] * 3


FP = C.POINTER(C.c_float)
_SCRATCH = {}


def _scratch(name, shape, dtype):
    """Reusable output buffers, so timing the oracle does not time numpy allocations."""
    key = (name, tuple(shape), np.dtype(dtype).str)
    buf = _SCRATCH.get(key)
    if buf is None:
        buf = _SCRATCH[key] = np.zeros(shape, dtype)
    return buf


# ---- small helpers ---------------------------------------------------------
def half_space_new(nd):
    nd = _f32(nd); out = np.zeros(4, np.float32)
    lib().orc_half_space_new(_p(nd, C.c_float), _p(out, C.c_float)); return out


def frustum_from_half_spaces(rows):
    """6 literal Vec4s -> HalfSpace::new each (as the reference tests build a Frustum)."""
    return np.stack([half_space_new(r) for r in rows]).astype(np.float32)


def affine_from_trs(trs):
    trs = _f32(trs); out = np.zeros(12, np.float32)
    lib().orc_affine_from_trs(_p(trs, C.c_float), _p(out, C.c_float)); return out


def affine_mul(a, b):
    a = _f32(a); b = _f32(b); out = np.zeros(12, np.float32)
    lib().orc_affine_mul(_p(a, C.c_float), _p(b, C.c_float), _p(out, C.c_float)); return out


def affine_inverse(a):
    a = _f32(a); out = np.zeros(12, np.float32)
    lib().orc_affine_inverse(_p(a, C.c_float), _p(out, C.c_float)); return out


def mat4_inverse(m):
    m = _f32(m); out = np.zeros(16, np.float32)
    lib().orc_mat4_inverse(_p(m, C.c_float), _p(out, C.c_float)); return out


def intersects_sphere(planes, center, radius, intersect_far):
    planes = _f32(planes); center = _f32(center)
    return bool(lib().orc_frustum_intersects_sphere(_p(planes, C.c_float), _p(center, C.c_float),
                                                    C.c_float(radius), int(intersect_far)))


def intersects_obb(planes, center, half, gt12, near, far):
    planes = _f32(planes); center = _f32(center); half = _f32(half); gt12 = _f32(gt12)
    return bool(lib().orc_frustum_intersects_obb(_p(planes, C.c_float), _p(center, C.c_float), _p(half, C.c_float),
                                                 _p(gt12, C.c_float), int(near), int(far)))


def intersects_obb_identity(planes, center, half):
    planes = _f32(planes); center = _f32(center); half = _f32(half)
    return bool(lib().orc_frustum_intersects_obb_identity(_p(planes, C.c_float), _p(center, C.c_float),
                                                          _p(half, C.c_float)))


def contains_aabb(planes, center, half, gt12):
    planes = _f32(planes); center = _f32(center); half = _f32(half); gt12 = _f32(gt12)
    return bool(lib().orc_frustum_contains_aabb(_p(planes, C.c_float), _p(center, C.c_float), _p(half, C.c_float),
                                                _p(gt12, C.c_float)))


def sphere_intersects_obb(sc, sr, center, half, gt12):
    sc = _f32(sc); center = _f32(center); half = _f32(half); gt12 = _f32(gt12)
    return bool(lib().orc_sphere_intersects_obb(_p(sc, C.c_float), C.c_float(sr), _p(center, C.c_float),
                                                _p(half, C.c_float), _p(gt12, C.c_float)))


def perspective(fov_y, aspect, near):
    out = np.zeros(16, np.float32)
    lib().orc_perspective_infinite_reverse_rh(C.c_float(fov_y), C.c_float(aspect), C.c_float(near), _p(out, C.c_float))
    return out


def compute_frustum(clip_from_view, camera_gt12, far):
    cfv = _f32(clip_from_view); g = _f32(camera_gt12); out = np.zeros((6, 4), np.float32)
    lib().orc_compute_frustum(_p(cfv, C.c_float), _p(g, C.c_float), C.c_float(far), _p(out, C.c_float))
    return out


IDENTITY_GT = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], np.float32)


# ---- stages ------------------------------------------------------------------
def propagate(parent, trs, gt, tchanged, static_opt=True, gt_ext_changed=None, mt=False):
    """Returns (rc, changed); gt is updated in place."""
    n = len(parent)
    parent = np.ascontiguousarray(parent, np.uint32)
    trs = _f32(trs)
    assert gt.dtype == np.float32 and gt.flags.c_contiguous
    tchanged = np.ascontiguousarray(tchanged, np.uint8)
    changed = np.zeros(n, np.uint8)
    l = lib_mt() if mt else lib()
    fn = l.orc_propagate_mt if mt else l.orc_propagate
    rc = fn(n, _p(parent, C.c_uint32), _p(trs, C.c_float), _p(gt, C.c_float), _p(tchanged, C.c_uint8),
            _p(None if gt_ext_changed is None else np.ascontiguousarray(gt_ext_changed, np.uint8), C.c_uint8),
            int(bool(static_opt)), _p(changed, C.c_uint8))
    return rc, changed


def cull(gt, bounds, flags, class_mask, entity_bits, vv, view_planes, view_layers=None, view_flags=None,
         layer_mask=None, range_mask=None, view_range_index=None, mt=False):
    """Returns (vv_changed, [visible rows per view or None for inactive views]); vv updated in place."""
    n = len(flags)
    gt = _f32(gt); bounds = _f32(bounds)
    flags = np.ascontiguousarray(flags, np.uint8)
    class_mask = np.ascontiguousarray(class_mask, np.uint8)
    entity_bits = np.ascontiguousarray(entity_bits, np.uint64)
    assert vv.dtype == np.uint8 and vv.flags.c_contiguous
    view_planes = _f32(view_planes).reshape(-1, 6, 4)
    V = view_planes.shape[0]
    view_layers = np.ones(V, np.uint64) if view_layers is None else np.ascontiguousarray(view_layers, np.uint64)
    view_flags = np.full(V, VIEW_ACTIVE, np.uint8) if view_flags is None else np.ascontiguousarray(view_flags, np.uint8)
    if layer_mask is not None:
        layer_mask = np.ascontiguousarray(layer_mask, np.uint64)
    if range_mask is not None:
        range_mask = np.ascontiguousarray(range_mask, np.uint32)
    if view_range_index is not None:
        view_range_index = np.ascontiguousarray(view_range_index, np.int8)
    vv_changed = np.zeros(n, np.uint8)
    rows = _scratch("cull_rows", (V, max(n, 1)), np.uint32)      # reused across calls: no per-frame 16 MB allocation
    counts = np.zeros(V, np.uint32)
    l = lib_mt() if mt else lib()
    fn = l.orc_cull_mt if mt else l.orc_cull
    rc = fn(n, _p(gt, C.c_float), _p(bounds, C.c_float), _p(flags, C.c_uint8), _p(layer_mask, C.c_uint64),
            _p(range_mask, C.c_uint32), _p(class_mask, C.c_uint8), _p(entity_bits, C.c_uint64),
            _p(vv, C.c_uint8), _p(vv_changed, C.c_uint8), V, _p(view_planes, C.c_float),
            _p(view_layers, C.c_uint64), _p(view_flags, C.c_uint8), _p(view_range_index, C.c_int8),
            _p(rows, C.c_uint32), _p(counts, C.c_uint32))
    assert rc == 0
    lists = [None if counts[v] == 0xFFFFFFFF else rows[v, :counts[v]].copy() for v in range(V)]
    return vv_changed, lists


def set_render_layers_ext(entity_ext=None, view_ext=None):
    """RenderLayers blocks 1..3 (layers 64..255) for the following cull() calls: entity_ext [n, 3], view_ext [V, 3] uint64; the
    arrays are kept alive here.  None switches the extension off."""
    global _layers_ext_keep
    fn = lib().orc_set_render_layers_ext
    fn.restype = None
    if entity_ext is None or view_ext is None:
        _layers_ext_keep = None
        fn(None, None)
        return
    e = np.ascontiguousarray(entity_ext, np.uint64); v = np.ascontiguousarray(view_ext, np.uint64)
    _layers_ext_keep = (e, v)
    fn(_p(e, C.c_uint64), _p(v, C.c_uint64))


_layers_ext_keep = None


def visible_entities_by_class(visible_rows, class_mask, entity_bits):
    """VisibleEntities::entities of one view: {class k: sorted rows} (orc_visible_entities_by_class)."""
    vis = np.ascontiguousarray(visible_rows, np.uint32)
    class_mask = np.ascontiguousarray(class_mask, np.uint8)
    entity_bits = np.ascontiguousarray(entity_bits, np.uint64)
    m = len(vis)
    out = np.zeros((8, max(m, 1)), np.uint32)
    cnt = np.zeros(8, np.uint32)
    fn = lib().orc_visible_entities_by_class
    fn.restype = None
    fn(m, _p(vis, C.c_uint32), _p(class_mask, C.c_uint8), _p(entity_bits, C.c_uint64), _p(out, C.c_uint32), _p(cnt, C.c_uint32))
    return {k: out[k, :cnt[k]].copy() for k in range(8) if cnt[k]}


def default_cluster_view_in(camera_gt12, clip_from_view, frustum, screen=(1920, 1080), view_layers=1,
                            config_kind=3, cfg_dims=(0, 0, 0), total=4096, z_slices=24, first_slice_depth=5.0,
                            far_z_mode=0, far_z_constant=0.0, dynamic_resizing=True, max_indices=16384,
                            last_farthest_z=None, last_index_count=None):
    """ClusterConfig::default() = FixedZ{4096, 24, first_slice_depth 5.0, MaxClusterableObjectRange, dynamic}
    (crates/bevy_light/src/cluster/mod.rs:297-307)."""
    v = ClusterViewIn()
    v.config_kind = config_kind
    for i in range(3):
        v.cfg_dims[i] = cfg_dims[i]
    v.cfg_total = total; v.cfg_z_slices = z_slices
    v.first_slice_depth = first_slice_depth; v.far_z_mode = far_z_mode; v.far_z_constant = far_z_constant
    v.dynamic_resizing = int(dynamic_resizing)
    v.screen_w, v.screen_h = screen
    v.view_cluster_bindings_max_indices = max_indices
    for i, x in enumerate(_f32(camera_gt12).ravel()):
        v.camera_gt[i] = x
    for i, x in enumerate(_f32(clip_from_view).ravel()):
        v.clip_from_view[i] = x
    for i, x in enumerate(_f32(frustum).ravel()):
        v.frustum[i] = x
    v.view_layers = view_layers
    v.has_last_farthest_z = int(last_farthest_z is not None)
    v.last_farthest_z = 0.0 if last_farthest_z is None else last_farthest_z
    v.has_last_index_count = int(last_index_count is not None)
    v.last_index_count = 0 if last_index_count is None else last_index_count
    return v


def assign_lights_to_clusters(view_in, lights, light_layers=None, indices_cap=None, want_planes=False):
    """lights: [L,4] = (x,y,z,range) of the VISIBLE point lights in query order.
    Returns (out struct, offsets[n_clusters+1], indices, planes or None)."""
    lights = _f32(lights).reshape(-1, 4)
    L = lights.shape[0]
    if light_layers is not None:
        light_layers = np.ascontiguousarray(light_layers, np.uint64)
    out = ClusterViewOut()
    offsets = np.zeros(4097, np.uint32)
    cap = indices_cap if indices_cap is not None else max(4096 * max(L, 1), 1)
    cap = min(cap, 1 << 28)
    indices = _scratch("cluster_indices", (cap,), np.uint32)
    xp = _scratch("xp", (4098, 4), np.float32); yp = _scratch("yp", (4098, 4), np.float32); zp = _scratch("zp", (4098, 4), np.float32)
    rc = lib().orc_assign_lights_to_clusters(C.byref(view_in), L, _p(lights, C.c_float), _p(light_layers, C.c_uint64),
                                             C.byref(out), _p(offsets, C.c_uint32), _p(indices, C.c_uint32), cap,
                                             _p(xp, C.c_float), _p(yp, C.c_float), _p(zp, C.c_float))
    if rc != 0:
        raise RuntimeError(f"orc_assign_lights_to_clusters rc={rc}")
    nc = out.dims[0] * out.dims[1] * out.dims[2]
    planes = None
    if want_planes and not out.cleared:
        planes = (xp[:out.dims[0] + 1].copy(), yp[:out.dims[1] + 1].copy(), zp[:out.dims[2] + 1].copy())
    return out, offsets[:nc + 1].copy(), indices[:offsets[nc]].copy(), planes


def cluster_dimensions_for_screen_size(kind, dims, total, z_slices, w, h):
    d = (C.c_uint32 * 3)(*dims); out = (C.c_uint32 * 3)()
    lib().orc_cluster_dimensions_for_screen_size(kind, d, total, z_slices, w, h, out)
    return tuple(out)


def clusters_update(w, h, req):
    r = (C.c_uint32 * 3)(*req); tile = (C.c_uint32 * 2)(); dims = (C.c_uint32 * 3)()
    lib().orc_clusters_update(w, h, r, tile, dims)
    return tuple(tile), tuple(dims)


# ---- SURVEY.md section 8(f) rows (bevy_oracle_next.c) -------------------------------------------------
VIS_INHERITED, VIS_HIDDEN, VIS_VISIBLE, VIS_NO_COMPONENTS = 0, 1, 2, 4


def _u64(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


def sort_pairs_by_main(render, main):
    """collect_visible_cpu_culled_entities_for_subview's sort (view/visibility/mod.rs:425-427)."""
    render, main = _u64(render).copy(), _u64(main).copy()
    lib().orc_sort_pairs_by_main(_p(render, C.c_uint64), _p(main, C.c_uint64), len(main))
    return render, main


def update_cpu_culled_entities(old_render, old_main, new_render, new_main):
    """RenderVisibleEntitiesClass::update_cpu_culled_entities -> (added_render, added_main, removed_render, removed_main)."""
    o_r, o_m, n_r, n_m = _u64(old_render), _u64(old_main), _u64(new_render), _u64(new_main)
    a_r, a_m = np.zeros(len(n_m), np.uint64), np.zeros(len(n_m), np.uint64)
    r_r, r_m = np.zeros(len(o_m), np.uint64), np.zeros(len(o_m), np.uint64)
    na, nr = C.c_uint32(0), C.c_uint32(0)
    U = C.c_uint64
    lib().orc_update_cpu_culled_entities(_p(o_r, U), _p(o_m, U), len(o_m), _p(n_r, U), _p(n_m, U), len(n_m),
                                         _p(a_r, U), _p(a_m, U), C.byref(na), _p(r_r, U), _p(r_m, U), C.byref(nr))
    return a_r[:na.value], a_m[:na.value], r_r[:nr.value], r_m[:nr.value]


def entity_pair_is_visible(render, main, entity, main_entity):
    render, main = _u64(render), _u64(main)
    return bool(lib().orc_entity_pair_is_visible(_p(render, C.c_uint64), _p(main, C.c_uint64), len(main),
                                                 int(entity), int(main_entity)))


def cluster_bindings(offsets, indices, gpu_index_of_light=None, storage=True):
    """Clusters (CSR) -> ViewClusterBindings buffers: (offsets_and_counts, index_lists, n_offsets, n_indices).
    `gpu_index_of_light[o]` is light ordinal o's entity_to_index; an ordinal past its end gets the dummy index !0."""
    offsets = np.ascontiguousarray(offsets, np.uint32)
    indices = np.ascontiguousarray(indices, np.uint32)
    n = len(offsets) - 1
    if storage:
        oc = np.zeros((n, 8), np.uint32)
        il = np.zeros(max(int(offsets[-1]), 1), np.uint32)
    else:
        oc = np.zeros(4096, np.uint32)
        il = np.zeros(4096, np.uint32)
    gi = None if gpu_index_of_light is None else np.ascontiguousarray(gpu_index_of_light, np.uint32)
    no, ni = C.c_uint32(0), C.c_uint32(0)
    U = C.c_uint32
    lib().orc_cluster_bindings(n, _p(offsets, U), _p(indices, U), None if gi is None else _p(gi, U),
                               0 if gi is None else len(gi), int(bool(storage)),
                               _p(oc, U), _p(il, U), C.byref(no), C.byref(ni))
    if storage:
        il = il[:ni.value]
    return oc, il, no.value, ni.value


def check_visibility_ranges(gt, bounds, flags, range_se, use_aabb, view_pos):
    """check_visibility_ranges -> per-row u32 view bitmask (0 = no VisibleEntityRanges entry)."""
    gt, bounds = _f32(gt), _f32(bounds)
    flags = np.ascontiguousarray(flags, np.uint8)
    range_se, view_pos = _f32(range_se), _f32(view_pos).reshape(-1, 3)
    use_aabb = np.ascontiguousarray(use_aabb, np.uint8)
    out = np.zeros(len(flags), np.uint32)
    lib().orc_check_visibility_ranges(len(flags), _p(gt, C.c_float), _p(bounds, C.c_float), _p(flags, C.c_uint8),
                                      _p(range_se, C.c_float), _p(use_aabb, C.c_uint8), len(view_pos),
                                      _p(view_pos, C.c_float), _p(out, C.c_uint32))
    return out


def visibility_propagate(parent, vis, inherited, changed_rows, removed_rows=()):
    """visibility_propagate_system: returns (inherited, changed) after one run."""
    parent = np.ascontiguousarray(parent, np.uint32)
    vis = np.ascontiguousarray(vis, np.uint8)
    inh = np.ascontiguousarray(inherited, np.uint8).copy()
    ch = np.zeros(len(parent), np.uint8)
    cr = np.ascontiguousarray(changed_rows, np.uint32)
    rr = np.ascontiguousarray(removed_rows, np.uint32)
    rc = lib().orc_visibility_propagate(len(parent), _p(parent, C.c_uint32), _p(vis, C.c_uint8), _p(inh, C.c_uint8),
                                        _p(ch, C.c_uint8), len(cr), _p(cr, C.c_uint32), len(rr), _p(rr, C.c_uint32))
    assert rc == 0
    return inh, ch


# ---- N3: shadow-view culling for point lights (bevy_oracle.c) ----------------------------------------
def set_defer_mark_newly_hidden(on):
    """Make cull() stop before mark_newly_hidden_entities_invisible so the light-visibility systems can run in between."""
    lib().orc_set_defer_mark_newly_hidden(int(bool(on)))


def mark_newly_hidden(flags, vv, vv_changed):
    flags = np.ascontiguousarray(flags, np.uint8)
    assert vv.dtype == np.uint8 and vv_changed.dtype == np.uint8 and vv.flags.c_contiguous and vv_changed.flags.c_contiguous
    lib().orc_mark_newly_hidden(len(flags), _p(flags, C.c_uint8), _p(vv, C.c_uint8), _p(vv_changed, C.c_uint8))


def point_light_frusta(light_gt12, light_range, shadow_map_near_z=0.1):
    """update_point_light_frusta for one light -> [6 faces][6 half spaces][4]."""
    g = _f32(light_gt12)
    out = np.zeros((6, 6, 4), np.float32)
    lib().orc_point_light_frusta(_p(g, C.c_float), float(light_range), float(shadow_map_near_z), _p(out, C.c_float))
    return out


def check_point_light_mesh_visibility(gt, bounds, flags, caster, entity_bits, vv, vv_changed, light_sphere, frusta,
                                      layer_mask=None, range_mask=None, lod_origin_index=-1, light_layers=None):
    """check_point_light_mesh_visibility (point lights): vv / vv_changed are updated in place; returns the per
    (light, face) sorted row lists as a list of 6-lists."""
    gt, bounds = _f32(gt), _f32(bounds)
    flags = np.ascontiguousarray(flags, np.uint8); caster = np.ascontiguousarray(caster, np.uint8)
    bits = np.ascontiguousarray(entity_bits, np.uint64)
    ls = _f32(light_sphere).reshape(-1, 4); fr = _f32(frusta).reshape(-1, 6, 6, 4)
    n, L = len(flags), len(ls)
    lm = None if layer_mask is None else np.ascontiguousarray(layer_mask, np.uint64)
    rm = None if range_mask is None else np.ascontiguousarray(range_mask, np.uint32)
    ll = None if light_layers is None else np.ascontiguousarray(light_layers, np.uint64)
    rows = np.zeros((max(L, 1) * 6, max(n, 1)), np.uint32); cnt = np.zeros(max(L, 1) * 6, np.uint32)
    rc = lib().orc_check_point_light_mesh_visibility(
        n, _p(gt, C.c_float), _p(bounds, C.c_float), _p(flags, C.c_uint8), _p(caster, C.c_uint8), _p(lm, C.c_uint64),
        _p(rm, C.c_uint32), int(lod_origin_index), _p(bits, C.c_uint64), _p(vv, C.c_uint8), _p(vv_changed, C.c_uint8), L,
        _p(ls, C.c_float), _p(ll, C.c_uint64), _p(fr, C.c_float), _p(rows, C.c_uint32), _p(cnt, C.c_uint32))
    assert rc == 0
    return [[rows[l * 6 + k, :cnt[l * 6 + k]].copy() for k in range(6)] for l in range(L)]


def check_spot_light_mesh_visibility(gt, bounds, flags, caster, entity_bits, vv, vv_changed, light_sphere, frusta,
                                     layer_mask=None, range_mask=None, lod_origin_index=-1, light_layers=None):
    """Spot-light half of check_point_light_mesh_visibility: one frustum [6, 4] per light; returns one row list per light."""
    gt, bounds = _f32(gt), _f32(bounds)
    flags = np.ascontiguousarray(flags, np.uint8); caster = np.ascontiguousarray(caster, np.uint8)
    bits = np.ascontiguousarray(entity_bits, np.uint64)
    ls = _f32(light_sphere).reshape(-1, 4); fr = _f32(frusta).reshape(-1, 6, 4)
    n, L = len(flags), len(ls)
    lm = None if layer_mask is None else np.ascontiguousarray(layer_mask, np.uint64)
    rm = None if range_mask is None else np.ascontiguousarray(range_mask, np.uint32)
    ll = None if light_layers is None else np.ascontiguousarray(light_layers, np.uint64)
    rows = np.zeros((max(L, 1), max(n, 1)), np.uint32); cnt = np.zeros(max(L, 1), np.uint32)
    rc = lib().orc_check_spot_light_mesh_visibility(
        n, _p(gt, C.c_float), _p(bounds, C.c_float), _p(flags, C.c_uint8), _p(caster, C.c_uint8), _p(lm, C.c_uint64),
        _p(rm, C.c_uint32), int(lod_origin_index), _p(bits, C.c_uint64), _p(vv, C.c_uint8), _p(vv_changed, C.c_uint8), L,
        _p(ls, C.c_float), _p(ll, C.c_uint64), _p(fr, C.c_float), _p(rows, C.c_uint32), _p(cnt, C.c_uint32))
    assert rc == 0
    return [rows[l, :cnt[l]].copy() for l in range(L)]


def check_dir_light_mesh_visibility(gt, bounds, flags, caster, entity_bits, vv, vv_changed, items, layer_mask=None,
                                    range_mask=None):
    """items: list of (cascade frusta [C, 6, 4], light_layers, view_range_index) per (directional light, view) pair;
    returns a list (per item) of lists (per cascade) of rows."""
    gt, bounds = _f32(gt), _f32(bounds)
    flags = np.ascontiguousarray(flags, np.uint8); caster = np.ascontiguousarray(caster, np.uint8)
    bits = np.ascontiguousarray(entity_bits, np.uint64)
    n = len(flags)
    ncasc = np.array([len(np.asarray(f).reshape(-1, 6, 4)) for f, _, _ in items], np.uint32)
    fr = _f32(np.concatenate([np.asarray(f, np.float32).reshape(-1, 6, 4) for f, _, _ in items])) if len(items) else np.zeros((0, 6, 4), np.float32)
    ll = np.array([l for _, l, _ in items], np.uint64); vri = np.array([v for _, _, v in items], np.int32)
    lm = None if layer_mask is None else np.ascontiguousarray(layer_mask, np.uint64)
    rm = None if range_mask is None else np.ascontiguousarray(range_mask, np.uint32)
    tot = int(ncasc.sum())
    rows = np.zeros((max(tot, 1), max(n, 1)), np.uint32); cnt = np.zeros(max(tot, 1), np.uint32)
    rc = lib().orc_check_dir_light_mesh_visibility(
        n, _p(gt, C.c_float), _p(bounds, C.c_float), _p(flags, C.c_uint8), _p(caster, C.c_uint8), _p(lm, C.c_uint64),
        _p(rm, C.c_uint32), _p(bits, C.c_uint64), _p(vv, C.c_uint8), _p(vv_changed, C.c_uint8), len(items),
        _p(vri, C.c_int32), _p(ll, C.c_uint64), _p(ncasc, C.c_uint32), _p(fr, C.c_float), _p(rows, C.c_uint32), _p(cnt, C.c_uint32))
    assert rc == 0
    out, k = [], 0
    for c in ncasc:
        out.append([rows[k + j, :cnt[k + j]].copy() for j in range(int(c))]); k += int(c)
    return out
