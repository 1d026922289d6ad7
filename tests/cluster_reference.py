"""A float64 geometric reference for the cluster stage (assign_objects_to_clusters, point lights), independent of the plane
tables the host and the oracle build: froxel boundaries come straight from the formulas of the reference, evaluated in float64.

* x and y: at NDC 2i/d - 1 (ndc_position_to_cluster, crates/bevy_light/src/cluster/assign.rs:922-941; y index 0 is the top).
* z, perspective: slice 0 ends at view depth 0 ... near, slice k >= 1 starts at near * (far/near)^((k-1)/(zs-1))
  (z_slice_to_view_z, assign.rs:903-920).  z, orthographic: linear from near to far.

Two properties are checked for every view:

1. No false negatives: points sampled inside each light's sphere (<= 0.999 r) land in a froxel that lists the light.  Points
   within a relative 1e-4 of a froxel boundary, behind the camera or its near plane, beyond its far plane, outside the
   screen or past the last slice are skipped.  In perspective views only the lights whose centre keeps its row across
   the sphere's depth range are held to it: the reference itself can miss rows of the others (`_rows_stay_put`).
2. Bounded over-inclusion: for a light whose view-space box c +- r * |scale| lies entirely in front of the camera, every
   froxel that lists it, dilated by a relative 1e-4, overlaps that box on each axis: its x and y NDC intervals overlap
   the box's projection, its depth interval the box's depth range.  The froxels at the edges of the grid reach to
   infinity outwards, because the reference clamps NDC to [-1, 1] and slice indices to [0, zs - 1] (assign.rs:922-941,
   1046-1062).  The bound is per axis, not a 3D intersection: the reference walks the box's cluster range
   (assign.rs:504-526, 606-678) and refines it one axis at a time against the sphere or its projection onto the
   z plane, then the y plane (project_to_plane_z / _y, assign.rs:1094-1134), so a froxel whose y row touches the sphere
   at another depth than its own slice stays listed.  Lights that straddle view z = 0 get property 1 only: their NDC
   box is clamped (assign.rs:980-1036).

`expected_grid` evaluates the config rules (ClusterConfig::dimensions_for_screen_size, crates/bevy_light/src/cluster/mod.rs:
311-347, Clusters::update :398-416, the far-z and first-slice rules and dynamic resizing of assign.rs:341-410) in float64,
so that the dims, near and far a view reports can be held to them before the froxels are built from them."""
import math

import numpy as np

REL = 1e-4


def _near_int(v):
    r = round(v)
    return v != r and abs(v - r) <= 1e-6 * max(abs(v), 1.0), r


def _floor(v):
    """floor of a float64 value the float32 rules may have landed on either side of an integer."""
    near, r = _near_int(v)
    return {r - 1, r} if near else {math.floor(v)}


def _ceil(v):
    near, r = _near_int(v)
    return {r, r + 1} if near else {math.ceil(v)}


def _requested(spec):
    w, h = spec.screen
    if spec.kind == "single":
        return {(1, 1, 1)}
    if spec.kind == "xyz":
        return {tuple(int(d) for d in spec.dims)}
    aspect = w / h
    zs = min(spec.z_slices, spec.total)
    per_layer = spec.total / zs
    y = math.sqrt(per_layer / aspect)
    out = set()
    for x in _floor(y * aspect):
        for yi in _floor(y):
            if x == 0:
                out |= {(1, p, zs) for p in _floor(per_layer)}
            elif yi == 0:
                out |= {(p, 1, zs) for p in _floor(per_layer)}
            else:
                out.add((x, yi, zs))
    return out


def expected_grid(spec, cam_gt, ortho_near=None, last_far=None, last_count=None):
    """(set of possible dims, first_slice_depth, far_z) the config rules give in float64, or None if clustering is off.
    `ortho_near` is the near distance of an orthographic projection (None: perspective); `last_far` / `last_count` are
    the Clusters feedback of the view's previous frame (None: absent)."""
    w, h = spec.screen
    if spec.kind == "none" or w == 0 or h == 0:
        return None
    dims = set()
    for req in _requested(spec):
        reqs = {req}
        if spec.kind in ("xyz", "fixedz") and spec.dynamic_resizing and last_count is not None and last_count > spec.max_indices:
            xy = math.sqrt(spec.max_indices / last_count)
            reqs = {(max(a, 1), max(b, 1), req[2]) for a in _floor(req[0] * xy) for b in _floor(req[1] * xy)}
        for rx, ry, rz in reqs:
            for tx in _ceil(w / rx):
                for ty in _ceil(h / ry):
                    tx_, ty_ = max(tx, 1), max(ty, 1)
                    for dx in _ceil(w / tx_):
                        for dy in _ceil(h / ty_):
                            dims.add((max(dx, 1), max(dy, 1), max(rz, 1)))
    gt = np.asarray(cam_gt, np.float64)
    inv_scale_z = 1.0 / np.linalg.norm(gt[6:9])
    if spec.kind == "single" or spec.far_z_constant is None:
        far = 1000.0 if last_far is None else float(last_far)
    else:
        far = float(spec.far_z_constant)
    cfg_first = 0.0 if spec.kind == "single" else spec.first_slice_depth
    zs = next(iter(dims))[2]
    if ortho_near is not None:
        first = ortho_near
    elif zs == 1:
        first = max(cfg_first, far)
    else:
        first = cfg_first
    first *= inv_scale_z
    return dims, first, max(far, first)


def check_grid(spec, cam_gt, ortho_near, last_far, last_count, enabled, dims, near, far):
    """Holds a view's reported grid (enabled, dims, near, far) to expected_grid."""
    exp = expected_grid(spec, cam_gt, ortho_near, last_far, last_count)
    if exp is None:
        assert not enabled, "clustering should be off (ClusterConfig::None or a zero-sized viewport)"
        return
    assert enabled
    e_dims, e_near, e_far = exp
    assert tuple(int(d) for d in dims) in e_dims, f"dims {tuple(dims)} not in {sorted(e_dims)}"
    assert abs(near - e_near) <= 1e-5 * max(abs(e_near), 1e-3), f"near {near} vs {e_near}"
    assert abs(far - e_far) <= 1e-5 * abs(e_far), f"far {far} vs {e_far}"


def z_boundaries(dz, near, far, ortho):
    """View depth (-view z) of the dz + 1 slice boundaries, float64."""
    k = np.arange(dz + 1, dtype=np.float64)
    if ortho:
        return near + (far - near) * k / dz
    b = np.zeros(dz + 1)
    e = (k[1:] - 1) / (dz - 1) if dz > 1 else np.ones(1)     # one slice: [0, far) (first = max(first, far))
    b[1:] = near * (far / near) ** e
    return b


def _view_frame(cam_gt):
    g = np.asarray(cam_gt, np.float64)
    M = g[:9].reshape(3, 3).T                           # columns: x_axis, y_axis, z_axis
    return np.linalg.inv(M), g[9:12], 1.0 / np.linalg.norm(M, axis=0)


def _row_class(ndy, dy):
    """y_center of the reference (assign.rs:593-603): None above the screen (-1 here), dims.y + 1 below, else the row."""
    row = np.minimum(np.floor((1 - ndy) * 0.5 * dy), dy - 1)
    return np.where(ndy > 1, -1, np.where(ndy < -1, dy + 1, row))


def _rows_stay_put(lights, P, Minv, t, inv_scale, dy, B):
    """Perspective views: the lights whose sphere the reference refines without false negatives.  It classifies the
    light's row once, from the centre's NDC (y_center, assign.rs:583-603), but tests rows against the sphere projected onto
    a slice's z plane (assign.rs:606-645), whose centre sits at another depth, where NDC y = P11 y / depth may fall in
    another row: a row that holds the projected centre but is farther from the plane it is tested against is then
    skipped.  That cannot happen when the centre's row is the same at every depth the sphere is projected to (the slice
    boundaries within its depth range, B[1] onwards), and the centre is in front of the camera and of the near plane
    (z_center is Some, :588-592; behind the camera the centre's NDC is mirrored)."""
    c = (lights[:, :3] - t) @ Minv.T
    r = lights[:, 3] * np.abs(inv_scale).max()
    u = -c[:, 2]

    def ndc_y(depth):
        return (P[1, 1] * c[:, 1] - P[1, 2] * depth + P[1, 3]) / (-P[3, 2] * depth + P[3, 3])

    in_front = (u > 0) & ((-P[2, 2] * u + P[2, 3]) / np.where(u > 0, u, 1.0) <= 1.0)
    ud = np.where(in_front, u, 1.0)
    lo, hi = np.minimum(ud, np.maximum(ud - r, B[1] if len(B) > 1 else ud)), ud + r
    ys = [ndc_y(d) for d in (lo, ud, hi)]
    same = (_row_class(ys[0], dy) == _row_class(ys[1], dy)) & (_row_class(ys[2], dy) == _row_class(ys[1], dy))
    off_edge = np.ones(len(c), bool)
    for y in ys:                                        # not within REL of a row boundary either
        f = (1 - y) * 0.5 * dy
        off_edge &= np.abs(f - np.round(f)) > REL * dy * 0.5
    return in_front & same & off_edge


def check_view(dims, near, far, ortho, clip_from_view, cam_gt, cam_far, lights, eligible, offsets, indices, rng, samples=40):
    """Checks one view's cluster lists (offsets [nc+1], indices = light ordinals) against the geometry.
    lights: [L, 4] world (x, y, z, range) of every light; eligible: [L] bool, the lights the view's clustering sees
    (ViewVisibility set, on the view's render layers).  Returns (points checked, entries checked)."""
    dx, dy, dz = (int(d) for d in dims)
    nc = dx * dy * dz
    L = len(lights)
    offsets = np.asarray(offsets, np.int64)[:nc + 1]
    indices = np.asarray(indices, np.int64)
    assert offsets[0] == 0 and (np.diff(offsets) >= 0).all() and offsets[-1] == len(indices), "offsets are not a CSR"
    cl = np.repeat(np.arange(nc), np.diff(offsets))
    if len(indices):
        assert indices.max() < L and eligible[indices].all(), "a listed light is not visible / not on the view's layers"
        same = cl[1:] == cl[:-1]
        assert (np.diff(indices)[same] > 0).all(), "a cluster's lights are not in ascending (push) order"
    listed = np.unique(cl * L + indices)
    P = np.asarray(clip_from_view, np.float64).reshape(4, 4).T          # row-major clip_from_view
    assert P[0, 1] == P[1, 0] == P[3, 0] == P[3, 1] == 0.0
    Minv, t, inv_scale = _view_frame(cam_gt)
    fwd = -np.asarray(cam_gt, np.float64)[6:9]
    fwd /= np.linalg.norm(fwd)
    B = z_boundaries(dz, near, far, ortho)
    lights = np.asarray(lights, np.float64)

    # ---- 1. no false negatives
    li = np.nonzero(eligible)[0]
    if P[3, 3] == 0.0:
        li = li[_rows_stay_put(lights[li], P, Minv, t, inv_scale, dy, B)]
    n_pts = 0
    if len(li):
        d = rng.normal(size=(len(li), samples, 3))
        d /= np.linalg.norm(d, axis=2, keepdims=True)
        rad = lights[li, 3, None] * 0.999 * rng.uniform(0, 1, (len(li), samples)) ** (1 / 3)
        rad[:, 0] = 0.0                                                  # the centre itself
        pw = lights[li, None, :3] + d * rad[..., None]
        owner = np.repeat(li, samples)
        pw = pw.reshape(-1, 3)
        v = (pw - t) @ Minv.T
        clip = v @ P[:, :3].T + P[:, 3]
        w = clip[:, 3]
        ok = w > 0
        wd = np.where(ok, w, 1.0)
        ndx, ndy, ndz = clip[:, 0] / wd, clip[:, 1] / wd, clip[:, 2] / wd
        u = -v[:, 2]
        ok &= (np.abs(ndx) < 1 - REL) & (np.abs(ndy) < 1 - REL) & (ndz < 1 - REL)     # on screen, beyond the near plane
        ok &= (pw - t) @ fwd < cam_far * (1 - REL)                                      # before the far plane
        fx, fy = (ndx + 1) * 0.5 * dx, (1 - ndy) * 0.5 * dy
        ok &= (np.abs(fx - np.round(fx)) > REL * dx * 0.5) & (np.abs(fy - np.round(fy)) > REL * dy * 0.5)
        iz = np.searchsorted(B, u, side="right") - 1
        ok &= (iz >= 0) & (iz < dz)
        tol = REL * np.abs(B) + 1e-7 * B[-1]
        ok &= (np.abs(u[:, None] - B[None, :]) > tol[None, :]).all(1)
        ix = np.clip(np.floor(fx).astype(np.int64), 0, dx - 1)
        iy = np.clip(np.floor(fy).astype(np.int64), 0, dy - 1)
        c = (iy * dx + ix) * dz + np.clip(iz, 0, dz - 1)
        hit = np.isin(c * L + owner, listed)
        bad = np.nonzero(ok & ~hit)[0]
        assert len(bad) == 0, (f"{len(bad)} sampled points miss their froxel's list, e.g. light {owner[bad[:4]]} at froxel "
                               f"{[(int(ix[b]), int(iy[b]), int(iz[b])) for b in bad[:4]]}, view depth {u[bad[:4]]}, ndc {ndx[bad[:4]]}, {ndy[bad[:4]]}")
        n_pts = int(ok.sum())

    # ---- 2. bounded over-inclusion (lights whose view-space box is entirely in front of the camera)
    n_ent = 0
    if len(indices):
        lc = (lights[indices, :3] - t) @ Minv.T
        half = lights[indices, 3, None] * inv_scale[None, :]
        front = lc[:, 2] + half[:, 2] < 0
        lc, half, cf = lc[front], half[front], cl[front]
        z = cf % dz
        x = (cf // dz) % dx
        y = cf // (dz * dx)
        ulo = np.where(z == 0, -np.inf, B[z] - REL * B[z] - 1e-7 * B[-1])
        uhi = np.where(z == dz - 1, np.inf, B[np.minimum(z + 1, dz)] * (1 + REL) + 1e-7 * B[-1])
        a0 = np.where(x == 0, -np.inf, 2.0 * x / dx - 1 - 2 * REL)
        a1 = np.where(x == dx - 1, np.inf, 2.0 * (x + 1) / dx - 1 + 2 * REL)
        b0 = np.where(y == dy - 1, -np.inf, 1 - 2.0 * (y + 1) / dy - 2 * REL)
        b1 = np.where(y == 0, np.inf, 1 - 2.0 * y / dy + 2 * REL)
        # the NDC range of the box over its 8 corners (in front of the camera: exactly the range of its projection)
        corners = lc[:, None, :] + half[:, None, :] * np.array([[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)])
        cc = corners @ P[:, :3].T + P[:, 3]
        nx_, ny_ = cc[..., 0] / cc[..., 3], cc[..., 1] / cc[..., 3]
        feasible = (a0 <= nx_.max(1)) & (a1 >= nx_.min(1)) & (b0 <= ny_.max(1)) & (b1 >= ny_.min(1))
        feasible &= (ulo <= -(lc[:, 2] - half[:, 2])) & (uhi >= -(lc[:, 2] + half[:, 2]))
        bad = np.nonzero(~feasible)[0]
        assert len(bad) == 0, (f"{len(bad)} listed froxels lie outside their light's box on some axis, e.g. light "
                               f"{indices[front][bad[:4]]} in froxel {[(int(x[b]), int(y[b]), int(z[b])) for b in bad[:4]]}")
        n_ent = int(front.sum())
    return n_pts, n_ent
