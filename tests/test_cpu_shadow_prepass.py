"""The block pre-pass of the shadow cull (kernels.cu: k_shadow_cull) is a shortcut in front of the exact per-row tests: for each
(CTA, item) pair it builds an axis-aligned box around the world-space centres of the CTA's bounded caster rows plus the
largest OBB reach E1, and skips the item for the whole CTA when the item's range sphere, or one of a cascade's half spaces,
cannot reach that box.  It may only skip a pair when the exact tests (Sphere::intersects_obb, primitives.rs:219-226, and
Frustum::intersects_obb, primitives.rs:272-294, as the same kernel's per-row loop evaluates them) fail for every eligible row
of the CTA.  The device code cannot run here; this restates the pre-pass and the exact tests in float32 numpy, operation for
operation, and checks that property and that the pre-pass is not vacuous."""
import numpy as np
import pytest

f32 = np.float32
CASCADE_PLANES = (0, 1, 2, 3, 5)          # a cascade skips its near plane (lib.rs:455-458)


# ---- rows ----------------------------------------------------------------------------------------------------------------------
def centres_and_e1(M, T, b, h):
    """World centre (transform_point3a of the Aabb centre) and E1 = sum_i |h_i| * |axis_i|_1 per row, in the kernel's order.
    M [..., 3, 3] with M[.., i, j] = row i of the matrix (g.r_i component j), T [..., 3], b / h [..., 3]."""
    c = [((M[..., i, 0] * b[..., 0] + M[..., i, 1] * b[..., 1]) + M[..., i, 2] * b[..., 2]) + T[..., i] for i in range(3)]
    a = np.abs(M)
    col = [(a[..., 0, j] + a[..., 1, j]) + a[..., 2, j] for j in range(3)]
    e1 = (np.abs(h[..., 0]) * col[0] + np.abs(h[..., 1]) * col[1]) + np.abs(h[..., 2]) * col[2]
    return np.stack(c, -1), e1


def block_box(c, e1, eligible):
    """(lo, hi, E1, usable): the reduction over the CTA's bounded rows; usable = False when an eligible row is not finite
    (the kernel switches skipping off for such a CTA)."""
    fin = np.isfinite(((c[:, 0] + c[:, 1]) + c[:, 2]) + e1)
    if (eligible & ~fin).any():
        return None, None, None, False
    ok = eligible & fin
    if not ok.any():
        return None, None, None, True
    return c[ok].min(0), c[ok].max(0), e1[ok].max(), True


# ---- the pre-pass --------------------------------------------------------------------------------------------------------------
# lo / hi [..., 3] and e1 [...] broadcast against the items: one box for many items, or one box per item
def sphere_skips(lo, hi, e1, s, r):
    """Point / spot items: the range sphere (s [k, 3], r [k]) cannot reach the box grown by E1."""
    d = [np.maximum(np.maximum(lo[..., i] - s[:, i], s[:, i] - hi[..., i]), f32(0.0)) for i in range(3)]
    reach = (r + e1) * f32(1.001) + f32(1e-3)
    return (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2] > reach * reach


def _plane_max(n, lo, hi):
    """The plane value of the box corner farthest along n, summed ((x + y) + z) + w."""
    return ((np.maximum(n[:, 0] * lo[..., 0], n[:, 0] * hi[..., 0]) + np.maximum(n[:, 1] * lo[..., 1], n[:, 1] * hi[..., 1])) +
            np.maximum(n[:, 2] * lo[..., 2], n[:, 2] * hi[..., 2])) + n[:, 3]


def _l1(n):
    return (np.abs(n[:, 0]) + np.abs(n[:, 1])) + np.abs(n[:, 2])


def cascade_skips(lo, hi, e1, planes):
    """Cascade items (planes [k, 6, 4]): a half space no point of the box reaches, even grown by E1.  The margin scales with
    the operands of the box's plane value (1e-5 of their magnitude, as in warp_view_reject), so it covers the rounding of the
    exact plane_dot_point(..) + relative_radius at any world offset."""
    skip = np.zeros(len(planes), bool)
    ax = [np.maximum(np.abs(lo[..., i]), np.abs(hi[..., i])) for i in range(3)]
    for k in CASCADE_PLANES:
        n = planes[:, k]
        m = _plane_max(n, lo, hi)
        reach = e1 * _l1(n)
        mag = ((np.abs(n[:, 0]) * ax[0] + np.abs(n[:, 1]) * ax[1]) + np.abs(n[:, 2]) * ax[2]) + (np.abs(n[:, 3]) + reach)
        skip |= (m + reach) + (f32(1e-5) * mag + f32(1e-6)) < f32(0.0)
    return skip


def cascade_skips_absolute_margin(lo, hi, e1, planes):
    """The cascade test of earlier versions: an absolute margin of 1e-3 that does not grow with the world coordinates."""
    skip = np.zeros(len(planes), bool)
    for k in CASCADE_PLANES:
        n = planes[:, k]
        skip |= _plane_max(n, lo, hi) + (e1 * f32(1.001) + f32(1e-3)) * _l1(n) < f32(0.0)
    return skip


# ---- the exact per-row tests ---------------------------------------------------------------------------------------------------
def _dot3(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def exact_sphere(M, c, h, s, r):
    """Sphere::intersects_obb per (item, row): d_sq <= radius * d + relative_radius(v).  Returns [k, rows]."""
    v = c[None, :, :] - s[:, None, :]
    d_sq = (v[..., 0] * v[..., 0] + v[..., 1] * v[..., 1]) + v[..., 2] * v[..., 2]
    d = np.sqrt(d_sq)
    a = [np.abs(_dot3(v, M[None, :, :, j])) for j in range(3)]          # v . axis_j
    rr = (a[0] * h[:, 0] + a[1] * h[:, 1]) + a[2] * h[:, 2]
    return d_sq <= r[:, None] * d + rr


def exact_cascade(M, c, h, planes):
    """Frustum::intersects_obb without the near plane per (item, row), in the kernel's order.  Returns [k, rows]."""
    inside = np.ones((len(planes), len(c)), bool)
    for k in CASCADE_PLANES:
        n = planes[:, None, k, :]
        a = [np.abs(_dot3(n, M[None, :, :, j])) for j in range(3)]
        prr = (a[0] * h[:, 0] + a[1] * h[:, 1]) + a[2] * h[:, 2]
        dot = (n[..., 0] * c[:, 0] + n[..., 2] * c[:, 2]) + (n[..., 1] * c[:, 1] + n[..., 3] * f32(1.0))
        inside &= ~(dot + prr <= f32(0.0))
    return inside


# ---- inputs --------------------------------------------------------------------------------------------------------------------
def random_matrices(rng, k):
    """Rotation x non-uniform scale, some mirrored, some nearly flat, as propagation produces them."""
    q, _ = np.linalg.qr(rng.normal(size=(k, 3, 3)))
    s = rng.uniform(0.3, 2.0, (k, 3))
    s[rng.random(k) < 0.15] *= -1.0
    s[rng.random(k) < 0.05, rng.integers(0, 3)] = 1e-4
    return (q * s[:, None, :]).astype(f32)


def half_extents(rng, k):
    h = rng.uniform(0.0, 2.0, (k, 3))
    pick = rng.random(k)
    h[pick < 0.2] = 0.0                                         # zero extent: a point caster
    h[(pick >= 0.2) & (pick < 0.3)] *= 1e-6                     # tiny
    h[(pick >= 0.3) & (pick < 0.4)] *= -1.0                     # negative (a user-provided Aabb)
    return h.astype(f32)


def unit(rng, k):
    n = rng.normal(size=(k, 3))
    return n / np.linalg.norm(n, axis=1, keepdims=True)


def cta(rng, layout, offset):
    """256 rows of one CTA: (M, T, local centre b, half extents h, eligible)."""
    k = 256
    centre = unit(rng, 1)[0] * offset
    if layout == "tree":
        T = centre + rng.normal(scale=3.0, size=(k, 3))
    else:                                                      # scattered over a 400-unit cube
        T = centre + rng.uniform(-200.0, 200.0, (k, 3))
    M = random_matrices(rng, k)
    b = rng.uniform(-1.0, 1.0, (k, 3)).astype(f32)
    b[rng.random(k) < 0.3] = 0.0
    h = half_extents(rng, k)
    eligible = rng.random(k) < rng.choice([0.2, 0.8, 1.0])
    if layout == "single":
        eligible[:] = False
        eligible[rng.integers(k)] = True
    return M, T.astype(f32), b, h, eligible


def planes_through(rng, points, n_planes=6, jitter_ulps=4):
    """Cascade frusta whose every plane passes (to a few ulps of w) through one of `points`, unnormalised normals included."""
    k = len(points)
    planes = np.zeros((k, n_planes, 4), f32)
    for p in range(n_planes):
        n = unit(rng, k) * np.where(rng.random(k) < 0.3, rng.uniform(0.05, 20.0, k), 1.0)[:, None]
        n = n.astype(f32)
        w = -(n.astype(np.float64) * points.astype(np.float64)).sum(1)
        w = w.astype(f32)
        steps = rng.integers(-jitter_ulps, jitter_ulps + 1, k)
        w = np.array([np.float32(x) if s == 0 else _ulps(x, int(s)) for x, s in zip(w, steps)], f32)
        planes[:, p, 0:3] = n
        planes[:, p, 3] = w
    return planes


def _ulps(x, s):
    x = np.float32(x)
    for _ in range(abs(s)):
        x = np.nextafter(x, np.float32(np.inf if s > 0 else -np.inf), dtype=np.float32)
    return x


def items_for(rng, c, eligible, lo, hi, e1):
    """Point / spot spheres and cascade frusta aimed at this CTA: near the box, at its boundary and through its rows."""
    rows = np.nonzero(eligible)[0]
    pick = c[rng.choice(rows, 16)]
    span = np.maximum(hi - lo, f32(1.0))
    s = np.concatenate([pick,                                                  # a light exactly at a row centre
                        lo + rng.uniform(-1.0, 2.0, (16, 3)) * span,
                        pick + unit(rng, 16) * rng.uniform(0.5, 30.0, (16, 1))]).astype(f32)
    r = rng.uniform(0.0, 30.0, len(s)).astype(f32)
    r[rng.random(len(s)) < 0.15] = 0.0                                         # range 0
    r[rng.random(len(s)) < 0.1] *= -1.0                                        # negative range
    # ranges that put a row's centre at the sphere boundary
    on = rng.random(len(s)) < 0.3
    r[on] = np.linalg.norm((pick[rng.integers(0, 16, on.sum())] - s[on]).astype(np.float64), axis=1).astype(f32)
    planes = np.concatenate([planes_through(rng, pick), planes_through(rng, lo + rng.random((8, 3)).astype(f32) * span)])
    return s, r, planes


def check_cta(rng, M, T, b, h, eligible):
    """Returns (pairs tested, pairs skipped); asserts that no skipped pair has an eligible row the exact tests keep."""
    c, e1r = centres_and_e1(M, T, b, h)
    lo, hi, e1, usable = block_box(c, e1r, eligible)
    if not usable or lo is None:
        return 0, 0
    s, r, planes = items_for(rng, c, eligible, lo, hi, e1)
    el = np.nonzero(eligible)[0]
    sk = sphere_skips(lo, hi, e1, s, r)
    keep = exact_sphere(M[el], c[el], h[el], s, r).any(1)
    bad = sk & keep
    assert not bad.any(), f"sphere pre-pass skipped a reachable item: light {s[bad][0]} range {r[bad][0]}, box {lo}..{hi}, E1 {e1}"
    skc = cascade_skips(lo, hi, e1, planes)
    keepc = exact_cascade(M[el], c[el], h[el], planes).any(1)
    badc = skc & keepc
    assert not badc.any(), f"cascade pre-pass skipped a reachable item: frustum {planes[badc][0].tolist()}, box {lo}..{hi}, E1 {e1}"
    return len(s) + len(planes), int(sk.sum() + skc.sum())


@pytest.mark.parametrize("offset", [0.0, 1e3, 1e4, 3e4, 1e5, 1e6])
@pytest.mark.parametrize("layout", ["tree", "scattered", "single"])
def test_pre_pass_never_skips_an_item_some_row_passes(layout, offset):
    rng = np.random.default_rng(int(offset) % 1000 + {"tree": 1, "scattered": 2, "single": 3}[layout])
    tested = 0
    for _ in range(40):
        t, _s = check_cta(rng, *cta(rng, layout, offset))
        tested += t
    assert tested > 1000


def point_casters_on_cascade_planes(rng, offset, k=200_000):
    """One zero-extent caster per CTA (the box collapses to a point) lying within an ulp or two of a cascade plane, at
    `offset` from the origin.  Returns (planes [k, 6, 4], centre [k, 3], E1 [k], exact-keeps [k])."""
    n = unit(rng, k).astype(f32)
    p = unit(rng, k) * offset + rng.normal(scale=10.0, size=(k, 3))
    w = (-(n.astype(np.float64) * p).sum(1)).astype(f32)
    c = (p + n * rng.uniform(-4e-7, 4e-7, (k, 1)) * max(offset, 1.0)).astype(f32)
    planes = np.zeros((k, 6, 4), f32)
    planes[:, :, 0:3] = -n[:, None, :]                       # every other plane keeps the caster well inside...
    planes[:, :, 3] = f32(1e9)
    planes[:, 0, 0:3] = n                                    # ...but plane 0 goes through it
    planes[:, 0, 3] = w
    M = np.broadcast_to(np.eye(3, dtype=f32), (k, 3, 3))
    h = np.zeros((k, 3), f32)
    keep = np.ones(k, bool)
    for kk in CASCADE_PLANES:
        nk = planes[:, kk]
        dot = (nk[:, 0] * c[:, 0] + nk[:, 2] * c[:, 2]) + (nk[:, 1] * c[:, 1] + nk[:, 3] * f32(1.0))
        keep &= ~(dot <= f32(0.0))
    return planes, c, np.zeros(k, f32), keep, M, h


@pytest.mark.parametrize("offset", [0.0, 1e3, 1e4, 3e4, 1e5, 1e6])
@pytest.mark.parametrize("layout", ["tree", "scattered", "single"])
def test_pre_pass_never_skips_an_item_some_row_passes(layout, offset):
    """CTAs of one tree, of scattered rows and of a single eligible caster; rotated, scaled and mirrored matrices; zero, tiny
    and negative half extents; lights at a row centre, on a row's range boundary, of range 0 and negative; cascade planes
    through rows and through the box."""
    rng = np.random.default_rng(int(offset) % 1000 + {"tree": 1, "scattered": 2, "single": 3}[layout])
    tested = 0
    for _ in range(40):
        tested += check_cta(rng, *cta(rng, layout, offset))[0]
    assert tested > 1000


def point_casters_on_cascade_planes(rng, offset, k=200_000):
    """k CTAs, each with one zero-extent caster (so the box is that point and E1 = 0) lying within a few ulps of plane 0 of
    its cascade frustum, at `offset` from the origin; the other planes hold the caster well inside.
    Returns (planes [k, 6, 4], centres [k, 3], whether the exact test keeps each caster [k])."""
    n = unit(rng, k).astype(f32)
    p = unit(rng, k) * offset + rng.normal(scale=10.0, size=(k, 3))
    w = (-(n.astype(np.float64) * p).sum(1)).astype(f32)
    c = (p + n * rng.uniform(-4e-7, 4e-7, (k, 1)) * max(offset, 1.0)).astype(f32)
    planes = np.zeros((k, 6, 4), f32)
    planes[:, :, 0:3] = -n[:, None, :]
    planes[:, :, 3] = f32(1e9)
    planes[:, 0, 0:3] = n
    planes[:, 0, 3] = w
    M = np.broadcast_to(np.eye(3, dtype=f32), (k, 3, 3))
    keep = np.ones(k, bool)
    for kk in CASCADE_PLANES:
        nk = planes[:, kk]
        dot = (nk[:, 0] * c[:, 0] + nk[:, 2] * c[:, 2]) + (nk[:, 1] * c[:, 1] + nk[:, 3] * f32(1.0))
        keep &= ~(dot <= f32(0.0))
    # the same through the general restatement, for a sample (rows = one caster each)
    for i in range(0, k, k // 50):
        assert exact_cascade(M[i:i + 1], c[i:i + 1], np.zeros((1, 3), f32), planes[i:i + 1])[0, 0] == keep[i]
    return planes, c, keep


@pytest.mark.parametrize("offset", [0.0, 1e3, 1e4, 3e4, 1e5, 1e6])
def test_point_casters_just_inside_a_cascade_plane_are_never_skipped(offset):
    rng = np.random.default_rng(17 + int(offset) % 97)
    planes, c, keep = point_casters_on_cascade_planes(rng, offset)
    assert keep.sum() > len(keep) // 4 and (~keep).sum() > len(keep) // 4      # both sides of the plane are well populated
    skip = cascade_skips(c, c, np.zeros(len(c), f32), planes)
    bad = np.nonzero(skip & keep)[0]
    assert len(bad) == 0, f"{len(bad)} reachable casters skipped, e.g. plane {planes[bad[0], 0].tolist()} centre {c[bad[0]].tolist()}"


@pytest.mark.parametrize("offset", [1e5, 1e6])
def test_an_absolute_cascade_margin_skips_reachable_casters_far_from_the_origin(offset):
    """What the scaled margin fixes: with the absolute 1e-3 margin, the box's ((x + y) + z) + w and the exact test's
    (x + z) + (y + w) differ by more than the margin once world coordinates reach ~3e4, and casters the exact test keeps
    are skipped.  This is the regression the inputs above are built to catch."""
    rng = np.random.default_rng(17 + int(offset) % 97)
    planes, c, keep = point_casters_on_cascade_planes(rng, offset)
    old = cascade_skips_absolute_margin(c, c, np.zeros(len(c), f32), planes)
    assert (old & keep).sum() > 0


def test_pre_pass_skips_most_pairs_on_a_bench_forest():
    """Not vacuous: on the bench's layout (one tree per CTA, roots spread over 1000^3) nearly every (CTA, point light) and
    (CTA, cascade) pair is skipped (a CTA of 256 rows spans two 255-row trees)."""
    import oracle as orc
    from bevy_b200 import scenes
    sc = scenes.forest(n_trees=256, levels=8, n_lights=64)
    gt = np.tile(np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], f32), (sc.n, 1))
    rc, _ = orc.propagate(sc.parent, sc.trs, gt, np.ones(sc.n, np.uint8), True)
    assert rc == 0
    M = gt[:, 0:9].reshape(-1, 3, 3).transpose(0, 2, 1)       # columns are the axes: M[r, i, j] = axis_j[i]
    T = gt[:, 9:12]
    s = T[sc.light_row]
    r = sc.light_range.astype(f32)
    ident = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1], f32)
    planes = np.stack([orc.point_light_frusta(np.concatenate([ident, np.asarray(cam.gt[9:12], f32) + f32(5.0 * c_)]), rr, 0.1)[k % 6]
                       for k, cam in enumerate(sc.cameras) for c_, rr in enumerate((25.0, 80.0))])
    n_mesh = sc.n - len(sc.light_row)
    pairs = skipped = 0
    for b0 in range(0, n_mesh - 255, 256):
        rows = slice(b0, b0 + 256)
        c, e1r = centres_and_e1(M[rows], T[rows], sc.bounds[rows, 0:3], sc.bounds[rows, 3:6])
        lo, hi, e1, usable = block_box(c, e1r, np.ones(256, bool))
        assert usable
        sk, skc = sphere_skips(lo, hi, e1, s, r), cascade_skips(lo, hi, e1, planes)
        el = np.arange(256)
        assert not (sk & exact_sphere(M[rows][el], c, sc.bounds[rows, 3:6], s, r).any(1)).any()
        assert not (skc & exact_cascade(M[rows][el], c, sc.bounds[rows, 3:6], planes).any(1)).any()
        pairs += len(s) + len(planes); skipped += int(sk.sum() + skc.sum())
    assert skipped > 0.6 * pairs, (skipped, pairs)
