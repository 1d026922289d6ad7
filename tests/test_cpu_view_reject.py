"""The warp-level view rejection of the tile kernel (kernels.cu: warp_view_reject_sphere / warp_view_reject_lean) is a shortcut in
front of Frustum::intersects_sphere (crates/bevy_camera/src/primitives.rs:255-268): it may only reject a view for a warp when the
exact test rejects that view for EVERY row of the warp.  The device code cannot run here; this restates both bounds in float32
numpy, operation for operation, and checks that property (and that the shortcut is not vacuous) on warps of rows the way the
scenes lay them out: 32 neighbours, far away from most frusta, plus adversarial cases right at a plane."""
import numpy as np
import pytest

f32 = np.float32
OFFSET_DIR = np.array([0.6, -0.48, 0.64])           # unit length: world offsets go along this direction
OFFSETS = (0.0, 1e4, 1e5, 1e6)                       # the scaled margin must hold far from the origin too


def exact_rejects(planes, c, r):
    """intersects_sphere, per row: True where some of the 5 planes has dot4(plane, (c, 1)) + r <= 0 (glam order)."""
    out = np.zeros(len(c), bool)
    for n in planes:
        d = (n[0] * c[:, 0] + n[2] * c[:, 2]) + (n[1] * c[:, 1] + n[3] * f32(1.0))
        out |= (d + r) <= f32(0.0)
    return out


def sphere_rejects(planes, c, r):
    """warp_view_reject_sphere for one view: a plane the warp's bounding sphere is behind."""
    x0, y0, z0 = c[0]
    mine = ((np.abs(c[:, 0] - x0) + np.abs(c[:, 1] - y0)) + np.abs(c[:, 2] - z0)) + np.abs(r)
    rmax = mine.max()
    for n in planes:
        vlen = max(f32(np.sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2])) * f32(1.000001), f32(1.0))
        reach = f32(vlen * rmax)
        d = ((n[0] * x0 + n[1] * y0) + n[2] * z0) + n[3]
        mag = ((abs(n[0] * x0) + abs(n[1] * y0)) + abs(n[2] * z0)) + (abs(n[3]) + reach)
        if (d + reach) + (f32(1e-5) * mag + f32(1e-6)) < f32(0.0):
            return True
    return False


def box_rejects(planes, c, r):
    """warp_view_reject_lean for one view: a plane the warp's bounding box (+ largest radius) is behind."""
    lo, hi, r1 = c.min(0), c.max(0), r.max()
    for n in planes:
        m = ((max(n[0] * lo[0], n[0] * hi[0]) + max(n[1] * lo[1], n[1] * hi[1])) + max(n[2] * lo[2], n[2] * hi[2])) + n[3]
        mag = ((abs(n[0]) * max(abs(lo[0]), abs(hi[0])) + abs(n[1]) * max(abs(lo[1]), abs(hi[1]))) +
               abs(n[2]) * max(abs(lo[2]), abs(hi[2]))) + (abs(n[3]) + abs(r1))
        if (m + r1) + (f32(1e-5) * mag + f32(1e-6)) < f32(0.0):
            return True
    return False


def random_frustum(rng, normalised=True, offset=0.0):
    """Five half spaces (normal, d) of a perspective-like frustum at a random pose `offset` from the origin (along a fixed
    diagonal); optionally with un-normalised normals."""
    q = rng.normal(size=(3, 3)); q, _ = np.linalg.qr(q)
    eye = rng.uniform(-300, 300, 3) + offset * OFFSET_DIR
    a, b = np.tan(rng.uniform(0.2, 0.7)), np.tan(rng.uniform(0.15, 0.5))
    local = [(1, 0, -a), (-1, 0, -a), (0, 1, -b), (0, -1, -b), (0, 0, -1)]      # L R B T near (looking down -z)
    planes = []
    for k, v in enumerate(local):
        n = q @ (np.array(v, float) / np.linalg.norm(v))
        d = -n @ eye - (0.1 if k == 4 else 0.0)
        s = 1.0 if normalised else rng.uniform(0.05, 20.0)
        planes.append(np.array([n[0] * s, n[1] * s, n[2] * s, d * s], f32))
    return planes


@pytest.mark.parametrize("normalised", [True, False])
def test_warp_shortcuts_never_reject_a_view_the_exact_test_keeps(normalised):
    """Near the origin and far from it (world offsets up to 1e6), where the margin must grow with the coordinates."""
    for k, offset in enumerate(OFFSETS):
        _warp_shortcuts_at(np.random.default_rng((7 if normalised else 8) + 100 * k), normalised, offset)


def _warp_shortcuts_at(rng, normalised, offset):
    hits = {"sphere": 0, "box": 0}
    trials = 0
    for _ in range(400):
        planes = random_frustum(rng, normalised, offset)
        for spread in (0.5, 4.0, 40.0, 400.0):
            centre = rng.uniform(-500, 500, 3) + offset * OFFSET_DIR
            c = (centre + rng.normal(scale=spread, size=(32, 3))).astype(f32)
            r = rng.uniform(0.0, 1.5, 32).astype(f32)
            if rng.random() < 0.1:
                r[rng.integers(32)] = f32(-0.5)          # a user-provided negative Sphere radius
            ex = exact_rejects(planes, c, r)
            trials += 1
            for name, fn in (("sphere", sphere_rejects), ("box", box_rejects)):
                if fn(planes, c, r):
                    hits[name] += 1
                    assert ex.all(), f"{name} bound rejected a warp with a row the exact test keeps (world offset {offset:g})"
    # the shortcut has to fire for most far-away warps, or it is worthless
    assert hits["sphere"] > trials // 3 and hits["box"] > trials // 3, (offset, hits, trials)


def test_rows_just_inside_a_plane_are_never_rejected():
    for k, offset in enumerate(OFFSETS):
        _rows_just_inside_at(np.random.default_rng(11 + 100 * k), offset)


def _rows_just_inside_at(rng, offset):
    kept = 0
    for _ in range(300):
        planes = random_frustum(rng, True, offset)
        n = planes[rng.integers(5)].astype(np.float64)
        # a tight warp whose first row touches the plane from outside by less than its radius: the exact test keeps it.  The
        # warp starts from a point inside the frustum (on its axis, in front of the apex the four side planes share) moved onto
        # the plane, so that the other four planes keep it
        side = np.array(planes[:4], np.float64)
        eye = np.linalg.lstsq(side[:, :3], -side[:, 3], rcond=None)[0]
        p0 = eye + np.asarray(planes[4][:3], np.float64) * rng.uniform(1.0, 100.0)
        p0 -= n[:3] * ((n[:3] @ p0 + n[3]) / (n[:3] @ n[:3]))          # onto the plane
        # far from the origin the float32 grid is coarser than the 1e-4 / 1e-3 steps used near it: scale them with it
        sp = float(np.spacing(f32(np.abs(p0).max())))
        r = np.full(32, max(0.5, 16 * sp), f32)
        c = (p0 - n[:3] * (r[0] - max(1e-4, 8 * sp)) + rng.normal(scale=max(1e-3, sp), size=(32, 3))).astype(f32)
        ex = exact_rejects([planes[k] for k in range(5)], c, r)
        if not ex.all():
            kept += 1
            assert not sphere_rejects(planes, c, r), f"world offset {offset:g}"
            assert not box_rejects(planes, c, r), f"world offset {offset:g}"
    assert kept > 200, (offset, kept)          # most warps do keep a row: the check is not vacuous at any offset
