"""Plain references of the propagate stage, and the edge scenes that hold the oracle and the kernels to them.

Written from bevy_transform's systems.rs and glam's SSE2 source, independently of oracle/:
- `propagate`: numpy float32, one rounding per ufunc, so every GlobalTransform bit is the reference's:
  Mat3A::from_quat, the scale applied to the columns, Affine3A * Affine3A in glam's operation order; set_if_neq with
  IEEE `!=` (+0 == -0 keeps the stored bits, NaN != NaN reports a change every visit) and children computed from the
  stored value; roots with children written unconditionally (with the static optimisations: only in a dirty tree); flat
  rows written on Changed<Transform> only; detached rows never; mark_dirty_trees as the ancestor closure of the changed
  rows.  `mutants` switches in one of the mistakes a kernel could make; the edge scenes must tell every one of them apart.
- `reference64`: the same algebra in float64 (glam's from_quat formula as written, so zero and non-unit quaternions keep
  their meaning), with the same product evaluated on absolute values, and the per-entry error bound of the float32
  evaluation (`bound`).

Light rows (F_SPHERE_FROM_GT) stay finite: what glam's Vec3 and Vec3A min/max do with a NaN light position in
cluster_space_clusterable_object_aabb cannot be restated here, so non-finite lights are out of scope.
"""
import itertools

import numpy as np

from bevy_b200 import abi, scenes
from bevy_b200.scenes import Scene

NO_PARENT, DETACHED = 0xFFFFFFFF, 0xFFFFFFFE
f32 = np.float32
TINY = np.finfo(f32).tiny                      # 2^-126: below it a float32 is subnormal
U = 2.0 ** -24                                 # unit roundoff of float32
ETA = 2.0 ** -150                              # largest absolute error of one product rounded into the subnormal range

# the mistakes a kernel could make that the edge scenes must detect (bit or Changed flag)
EDGE_MUTANTS = ("bitwise_neq", "children_from_new", "ftz", "fma_translation", "pw_first", "one_minus_yy_minus_zz")
# algebra mistakes the float64 bound must reject by a wide margin
ALGEBRA_MUTANTS = ("transposed_quat", "swap_parent_child", "scale_rows", "quat_sign")


class Ops:
    """float32 +, -, * (one rounding each); with flush-to-zero, subnormal inputs and outputs become zeros of their sign."""

    def __init__(self, ftz=False):
        self.ftz = ftz

    def _f(self, x):
        x = np.asarray(x, f32)
        return np.where(np.abs(x) < TINY, x * f32(0), x) if self.ftz else x

    def mul(self, a, b):
        return self._f(self._f(a) * self._f(b))

    def add(self, a, b):
        return self._f(self._f(a) + self._f(b))

    def sub(self, a, b):
        return self._f(self._f(a) - self._f(b))


# ---- float32 restatement ---------------------------------------------------------------------------------------------------
def from_quat(q, o, mutants=()):
    """Mat3A::from_quat: the columns (X, Y, Z), each [m, 3]."""
    x, y, z, w = (q[:, i:i + 1] for i in range(4))
    x2, y2, z2 = o.add(x, x), o.add(y, y), o.add(z, z)
    xx, xy, xz = o.mul(x, x2), o.mul(x, y2), o.mul(x, z2)
    yy, yz, zz = o.mul(y, y2), o.mul(y, z2), o.mul(z, z2)
    wx, wy, wz = o.mul(w, x2), o.mul(w, y2), o.mul(w, z2)
    one = f32(1.0)
    if "one_minus_yy_minus_zz" in mutants:
        d = (o.sub(o.sub(one, yy), zz), o.sub(o.sub(one, xx), zz), o.sub(o.sub(one, xx), yy))
    else:
        d = (o.sub(one, o.add(yy, zz)), o.sub(one, o.add(xx, zz)), o.sub(one, o.add(xx, yy)))
    X = [d[0], o.add(xy, wz), o.sub(xz, wy)]
    if "quat_sign" in mutants:
        X[1] = o.sub(xy, wz)
    Y = [o.sub(xy, wz), d[1], o.add(yz, wx)]
    Z = [o.add(xz, wy), o.sub(yz, wx), d[2]]
    cols = [np.concatenate(c, 1) for c in (X, Y, Z)]
    if "transposed_quat" in mutants:
        m = np.stack(cols, 1)                   # [m, col, row]
        cols = [m[:, :, i] for i in range(3)]
    return cols


def local_affine(trs, o, mutants=()):
    """Transform::compute_affine = Affine3A::from_scale_rotation_translation: [m, 12] (x_axis, y_axis, z_axis, t)."""
    trs = np.asarray(trs, f32)
    X, Y, Z = from_quat(trs[:, 3:7], o, mutants)
    s = trs[:, 7:10]
    if "scale_rows" in mutants:
        X, Y, Z = o.mul(X, s), o.mul(Y, s), o.mul(Z, s)
    else:
        X, Y, Z = o.mul(X, s[:, 0:1]), o.mul(Y, s[:, 1:2]), o.mul(Z, s[:, 2:3])
    return np.concatenate([X, Y, Z, trs[:, 0:3]], 1)


def _fma(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(f32)


def affine_mul(P, L, o, mutants=()):
    """Affine3A * Affine3A: matrix3 = P.m3 * L.m3 with mul_vec3a = ((X*v.x) + (Y*v.y)) + (Z*v.z) lane-wise;
    translation = P.m3 * L.t + P.t."""
    if "swap_parent_child" in mutants:
        P, L = L, P
    PX, PY, PZ, PT = P[:, 0:3], P[:, 3:6], P[:, 6:9], P[:, 9:12]

    def mv(v):
        return o.add(o.add(o.mul(PX, v[:, 0:1]), o.mul(PY, v[:, 1:2])), o.mul(PZ, v[:, 2:3]))
    cols = [mv(L[:, 0:3]), mv(L[:, 3:6]), mv(L[:, 6:9])]
    t = L[:, 9:12]
    if "fma_translation" in mutants:
        T = o.add(_fma(PZ, t[:, 2:3], _fma(PY, t[:, 1:2], o.mul(PX, t[:, 0:1]))), PT)
    elif "pw_first" in mutants:
        T = o.add(o.add(o.add(PT, o.mul(PX, t[:, 0:1])), o.mul(PY, t[:, 1:2])), o.mul(PZ, t[:, 2:3]))
    else:
        T = o.add(mv(t), PT)
    return np.concatenate(cols + [T], 1)


def mark_dirty_trees(parent, tchanged):
    """The changed rows and all their ancestors."""
    n = len(parent)
    real = parent < n
    p = np.where(real, parent, 0).astype(np.int64)
    dirty = np.asarray(tchanged, bool).copy()
    cur = dirty & real
    while cur.any():
        up = np.zeros(n, bool)
        up[p[cur]] = True
        up &= ~dirty
        dirty |= up
        cur = up & real
    return dirty


def propagate(parent, trs, gt, tchanged, static_opt=True, gt_ext_changed=None, mutants=(), mutant_rows=None):
    """sync_simple_transforms + mark_dirty_trees + propagate_parent_transforms; gt [n, 12] float32 is updated in place.
    gt_ext_changed marks rows whose GlobalTransform another system changed since the last run (is_changed() of the
    parent).  mutant_rows [n] bool confines 'children_from_new' to these children (one kind of parent hand-over).
    Returns Changed<GlobalTransform> [n] bool."""
    parent = np.asarray(parent, np.uint32)
    n = len(parent)
    o = Ops(ftz="ftz" in mutants)
    real = parent < n
    p = np.where(real, parent, 0).astype(np.int64)
    has_kids = np.zeros(n, bool)
    has_kids[p[real]] = True
    tch = np.asarray(tchanged, bool)
    ext = np.zeros(n, bool) if gt_ext_changed is None else np.asarray(gt_ext_changed, bool)
    dirty = mark_dirty_trees(parent, tch) if static_opt else np.ones(n, bool)
    changed = np.zeros(n, bool)
    root = parent == NO_PARENT
    with np.errstate(all="ignore"):
        written = (root & ~has_kids & tch) | (root & has_kids & dirty)       # roots are written unconditionally
        gt[written] = local_affine(trs[written], o, mutants)
        changed[written] = True
        fresh = gt.copy()                     # every row's newly computed matrix, written or not
        frontier = root & has_kids & dirty
        while True:
            cand = real & frontier[p]
            if not cand.any():
                break
            visit = cand & (dirty | (changed | ext)[p])
            rows = np.nonzero(visit)[0]
            P = gt[p[rows]]
            if "children_from_new" in mutants:
                new = np.ones(len(rows), bool) if mutant_rows is None else mutant_rows[rows]
                P[new] = fresh[p[rows[new]]]
            g = affine_mul(P, local_affine(trs[rows], o, mutants), o, mutants)
            fresh[rows] = g
            old = gt[rows]
            if "bitwise_neq" in mutants:
                neq = (g.view(np.uint32) != old.view(np.uint32)).any(1)
            else:
                neq = (g != old).any(1)
            gt[rows[neq]] = g[neq]
            changed[rows[neq]] = True
            frontier = visit
    return changed


# ---- float64 reference and the error bound ---------------------------------------------------------------------------------
K_LOCAL = 4      # roundings on the longest path to an entry of Transform::compute_affine: x*y2, the sum, 1 - sum, the scale
K_MUL = 4        # roundings of one Affine3A product entry: a product and two sums (matrix), one more sum (translation: + P.t)


def k_of_depth(d):
    """Roundings a row at hierarchy depth d (root = 0) accumulates: its own local matrix, and per level above it one local
    matrix and one product.  The bound uses gamma(k) = k u / (1 - k u), which also covers the second-order terms."""
    return K_LOCAL * (d + 1) + K_MUL * d


def _local64(trs):
    """(value, absolute-value evaluation, underflow count) of compute_affine in float64: [m, 12] each."""
    t = trs.astype(np.float64)
    out = []
    for absval in (False, True):
        q = np.abs(t[:, 3:7]) if absval else t[:, 3:7]
        s = np.abs(t[:, 7:10]) if absval else t[:, 7:10]
        x, y, z, w = (q[:, i:i + 1] for i in range(4))
        pm = (lambda a, b: a + b) if absval else (lambda a, b: a - b)
        xx, xy, xz, yy, yz, zz = x * 2 * x, x * 2 * y, x * 2 * z, y * 2 * y, y * 2 * z, z * 2 * z
        wx, wy, wz = w * 2 * x, w * 2 * y, w * 2 * z
        X = [pm(1.0, yy + zz), xy + wz, pm(xz, wy)]
        Y = [pm(xy, wz), pm(1.0, xx + zz), yz + wx]
        Z = [xz + wy, pm(yz, wx), pm(1.0, xx + yy)]
        cols = [np.concatenate(c, 1) * s[:, j:j + 1] for j, c in enumerate((X, Y, Z))]
        out.append(np.concatenate(cols + [np.abs(t[:, 0:3]) if absval else t[:, 0:3]], 1))
    # two products that can round into the subnormal range before the scale (both scaled by |s| after), one after it
    s = np.abs(t[:, 7:10])
    c = np.concatenate([np.repeat(2.0 * s[:, j:j + 1] + 1.0, 3, 1) for j in range(3)] + [np.zeros((len(t), 3))], 1)
    return out[0], out[1], c


def _mul64(P, L):
    PX, PY, PZ, PT = P[:, 0:3], P[:, 3:6], P[:, 6:9], P[:, 9:12]
    mv = lambda v: PX * v[:, 0:1] + PY * v[:, 1:2] + PZ * v[:, 2:3]
    return np.concatenate([mv(L[:, 0:3]), mv(L[:, 3:6]), mv(L[:, 6:9]), mv(L[:, 9:12]) + PT], 1)


def reference64(parent, trs):
    """Every row under a root, from the Transforms alone: (g64, m64, c64, depth, reached).  m64 is the same products on
    absolute values; c64 counts the products that can round into the subnormal range, each carried to the row through the
    absolute values of the later factors."""
    parent = np.asarray(parent, np.uint32)
    n = len(parent)
    real = parent < n
    p = np.where(real, parent, 0).astype(np.int64)
    g, m, c = (np.full((n, 12), np.nan) for _ in range(3))
    depth = np.full(n, -1, np.int64)
    with np.errstate(all="ignore"):
        lg, lm, lc = _local64(np.asarray(trs, f32))
        level = parent == NO_PARENT
        g[level], m[level], c[level] = lg[level], lm[level], lc[level]
        depth[level] = 0
        d = 0
        while True:
            d += 1
            rows = np.nonzero(real & level[p])[0]
            if not len(rows):
                break
            P = p[rows]
            g[rows] = _mul64(g[P], lg[rows])
            m[rows] = _mul64(m[P], lm[rows])
            # |P| c_L + c_P |L| (+ c_P.t in the translation), and the entry's own three products
            mP = m[P].copy()
            mP[:, 9:12] = 0.0
            c[rows] = _mul64(mP, lc[rows]) + _mul64(c[P], lm[rows]) + 3.0
            depth[rows] = d
            level = np.zeros(n, bool)
            level[rows] = True
    return g, m, c, depth, depth >= 0


def bound(m64, c64, depth):
    k = k_of_depth(np.maximum(depth, 0)).astype(np.float64)[:, None]
    gamma = k * U / (1.0 - k * U)
    return gamma * m64 + (1.0 + gamma) * c64 * ETA


def bound_violation(g32, parent, trs):
    """max over finite entries of |g32 - g64| / bound, and the number of entries checked."""
    g64, m64, c64, depth, reached = reference64(parent, trs)
    with np.errstate(all="ignore"):
        g32 = g32.astype(np.float64)
        ok = reached[:, None] & np.isfinite(g32) & np.isfinite(g64) & np.isfinite(m64) & np.isfinite(c64)
        b = bound(m64, c64, depth)
        r = np.where(ok, np.abs(g32 - g64) / np.maximum(b, 1e-300), 0.0)
    return float(r.max()), int(ok.sum())


# ---- the edge scene --------------------------------------------------------------------------------------------------------
KINDS = ("zero_scale", "zero_quat", "nan_t", "nan_q", "nan_s", "subnormal", "overflow", "quat_norms", "offsets")


def _row(t=(0, 0, 0), q=(0, 0, 0, 1), s=(1, 1, 1)):
    return np.array([*t, *q, *s], f32)


def _quat_with_x_axis_signs(rng, signs):
    """A random unit quaternion whose rotation's x_axis has the given component signs."""
    while True:
        q = scenes.random_unit_quats(rng, 1)[0]
        X = scenes.quat_to_gt(q, (0, 0, 0))[0:3]
        if (np.sign(X) == signs).all() and (np.abs(X) > 0.1).all():
            return q


def probe_chain(kind, rng):
    """One probe chain, head first: [(trs of frame 0, trs of the zero-sign frame or None)].  The head's parent has an
    identity rotation (the chain's ancestors are made so), so zero signs reach the product unchanged."""
    rq = lambda: scenes.random_unit_quats(rng, 1)[0]
    rt = lambda a=2.0: rng.uniform(-a, a, 3)
    if kind == "zero_scale":
        # C's x column is recomputed as -0 where +0 is stored: equal, so kept; D (rewritten: its z scale changes) reads
        # C's row 0 = (+-0, 0, 0): x_axis signs (+, -, -) make its row 0 zero signs depend on which C it multiplies
        dq = _quat_with_x_axis_signs(rng, np.array([1.0, -1.0, -1.0]))
        return [(_row(), None),
                (_row(t=(0, 0.5, 0), s=(0, 1, 1)), _row(t=(0, 0.5, 0), s=(-0.0, 1, 1))),
                (_row(t=rt(), q=dq), None),
                (_row(t=rt(), q=rq()), None)]
    if kind == "zero_quat":
        return [(_row(t=(0, 0, 0)), _row(t=(-0.0, 0, -0.0))),
                (_row(q=(0, 0, 0, 1), s=(1, 0, 1)), _row(q=(-0.0, 0, -0.0, 1), s=(1, -0.0, 1))),
                (_row(q=(0, -0.0, 0, -1), t=(0, 1, 0)), _row(q=(-0.0, 0, 0, -1), t=(0, 1, -0.0))),
                (_row(t=rt(), q=rq()), None)]
    if kind in ("nan_t", "nan_q", "nan_s"):
        a = _row(t=rt(), q=rq(), s=rng.uniform(0.5, 1.5, 3))
        a[{"nan_t": 1, "nan_q": 3, "nan_s": 9}[kind]] = np.nan
        return [(_row(t=rt(), q=rq()), None), (a, None), (_row(t=rt(), q=rq()), None), (_row(t=rt(), q=rq()), None)]
    if kind == "subnormal":
        # products of 1e-20 and 1e-20 land at ~1e-40 (subnormal), then ~1e-46 (below the subnormal range)
        return [(_row(s=(1e-20, 1e-20, 1e-20)), None),
                (_row(t=rt(), q=rq(), s=rng.uniform(0.5, 2.0, 3) * 1e-20), None),
                (_row(t=rt(), q=rq(), s=(1e-40, 0.7, 1.0)), None),
                (_row(t=rt(), q=rq(), s=(1e-6, 1e-6, 1e-6)), None)]
    if kind == "overflow":
        # 1e20 at two levels overflows the matrix to +-Inf; an identity child multiplies Inf by 0 (NaN), its translation
        # sums +Inf and -Inf (NaN); a translation of 3e38 added to 3e38 overflows on its own
        return [(_row(t=(3e38, 0, 0), q=rq(), s=(1e20, 1e20, 1e20)), None),
                (_row(t=(3e38, 1, 1), q=rq(), s=(1e20, 1e20, 1e20)), None),
                (_row(t=(1, 2, 3)), None),
                (_row(t=rt(), q=rq()), None)]
    if kind == "quat_norms":
        return [(_row(t=rt(), q=(0, 0, 0, 0), s=(1.5, 0.5, 1)), None),
                (_row(t=rt(), q=rq() * 1e-3), None),
                (_row(t=rt(), q=rq() * 1e3), None),
                (_row(t=rt(), q=rq() * 1e-3, s=(1e-6, 1e-6, 1e-6)), None)]
    if kind == "offsets":
        off = rng.normal(size=3)
        off = off / np.linalg.norm(off) * 10.0 ** rng.uniform(5, 7)
        return [(_row(t=off, q=rq()), None), (_row(t=rt(50.0), q=rq()), None), (_row(t=rt(50.0), q=rq(), s=(1.3, 0.7, 1.1)), None),
                (_row(t=rt(50.0), q=rq()), None)]
    raise ValueError(kind)


def tiles_of(desc, n):
    """The tile of every row, from a plan's tile descriptors (columns 0, 1 = first row, rows)."""
    out = np.full(n, -1, np.int64)
    for t, (base, nr) in enumerate(desc[:, 0:2].tolist()):
        out[base:base + nr] = t
    return out


def _binary_tree(n_levels):
    per = (1 << n_levels) - 1
    loc = np.arange(per)
    return np.where(loc == 0, -1, (loc - 1) // 2)


def _fanout_tree(fanout=(4, 4, 3, 3, 2, 2)):
    """Config #1's tree shape (benches/bevy_transform/propagate.rs), BFS order: local parent per row."""
    par, cur = [-1], [0]
    for fo in fanout:
        nxt = []
        for q in cur:
            for _ in range(fo):
                nxt.append(len(par)); par.append(q)
        cur = nxt
    return np.array(par)


class EdgeScene:
    """Probe chains inside complete 255-node BFS trees, config #1-shaped trees, a 700-deep and a 40-deep chain, next to flat rows,
    detached rows and finite light rows; with the frame inputs the edge tests run.

    frames: 0 first write; 1 the probes' zero components flip sign (values unchanged) and D of the zero_scale chains
    changes its z scale; 2 half of the NaN chains re-upload their Transforms (visited again), half not; 3 static;
    4 another system writes -0 or NaN bits into probe parents; 5 static."""
    FRAMES = ("first", "zero_signs", "nan_revisit", "static", "marks", "static")

    def __init__(self, seed=0, n_binary=45, n_fanout=4):
        rng = np.random.default_rng(seed)
        parent, origin = [], []
        for _ in range(n_binary):
            lp = _binary_tree(8); b = len(parent)
            parent += [NO_PARENT if x < 0 else b + x for x in lp]; origin.append(("binary", b, lp))
        for _ in range(n_fanout):
            lp = _fanout_tree(); b = len(parent)
            parent += [NO_PARENT if x < 0 else b + x for x in lp]; origin.append(("fanout", b, lp))
        b = len(parent)
        parent += [NO_PARENT] + list(range(b, b + 699)); origin.append(("chain", b, None))
        self.chain_base = b
        b40 = len(parent)
        parent += [NO_PARENT] + list(range(b40, b40 + 39))            # one tile of 40 levels
        n_flat = len(parent)
        parent += [NO_PARENT] * 24
        parent += [DETACHED] * 5
        n = len(parent)
        parent = np.array(parent, np.uint32)
        trs = np.zeros((n, 10), f32)
        trs[:, 0:3] = rng.uniform(-2, 2, (n, 3)); trs[:, 3:7] = scenes.random_unit_quats(rng, n)
        trs[:, 7:10] = rng.uniform(0.5, 1.5, (n, 1))
        roots = np.nonzero(parent == NO_PARENT)[0]
        ang = rng.uniform(0, 2 * np.pi, len(roots))
        trs[roots, 0] = np.cos(ang) * rng.uniform(15, 90, len(roots)); trs[roots, 2] = np.sin(ang) * rng.uniform(15, 90, len(roots))
        trs[roots, 1] = rng.uniform(-5, 5, len(roots))
        trs[self.chain_base + 1:self.chain_base + 700, 0:3] *= f32(0.05)      # keep the deep chain near its root
        bounds = np.zeros((n, 6), f32); bounds[:, 3:6] = rng.uniform(0.25, 0.75, (n, 3))
        flags = np.full(n, scenes.F_INHERITED_VISIBLE | scenes.F_HAS_AABB, np.uint8)
        self.flip = {}                                 # row -> trs of the zero-sign frame
        self.nan_rows = []                             # (row, revisit in frame 2)
        self.mark_parents = []                         # rows with children whose GlobalTransform is written in frame 4
        self.probe_edges = []                          # (parent row, child row) inside a chain
        taken = np.zeros(n, bool)
        kinds = itertools.cycle(KINDS)
        # the tile plan of the final rows (the light rows are appended as roots): where a parent is in another tile
        desc, _ = abi.host_tile_plan(np.concatenate([parent, np.full(8, NO_PARENT, np.uint32)]))
        tile_of = tiles_of(desc, n + 8)[:n]
        crosses = np.zeros(n, bool)
        crosses[parent < n] = tile_of[parent[parent < n]] != tile_of[parent < n]

        def place(path, s, kind, identity_ancestors=True):
            rows = path[s:s + 4]
            chain = probe_chain(kind, rng)[:len(rows)]
            if taken[rows].any() or (identity_ancestors and taken[path[:s]].any()):
                return False
            if identity_ancestors:                   # identity rotation and scale above the chain, translations only
                trs[path[:s], 3:10] = [0, 0, 0, 1, 1, 1, 1]
            for i, (r, (t0, t1)) in enumerate(zip(rows, chain)):
                trs[r] = t0
                taken[r] = True
                if t1 is not None:
                    self.flip[int(r)] = t1
                if i % 2:
                    bounds[r] = [0, 0, 0, rng.uniform(0.3, 1.5), 0, 0]; flags[r] = scenes.F_INHERITED_VISIBLE | scenes.F_HAS_SPHERE
                if i:
                    self.probe_edges.append((int(rows[i - 1]), int(r)))
            if kind == "zero_scale" and len(rows) >= 3:
                d = trs[rows[2]].copy(); d[9] = f32(1.25)
                self.flip[int(rows[2])] = d
            if kind.startswith("nan"):
                self.nan_rows.append((int(rows[1]), len(self.nan_rows) % 2 == 0))
            if kind in ("zero_scale", "zero_quat", "offsets") and len(rows) >= 3:
                self.mark_parents.append(int(rows[1]))
            return True

        def path_to(b, lp, leaf):
            out = [leaf]
            while lp[out[-1]] >= 0:
                out.append(lp[out[-1]])
            return [b + x for x in out[::-1]]

        starts = (0, 1, 3, 4, 5, 2)
        for i, (what, b, lp) in enumerate(origin):
            if what == "binary":
                s = starts[i % len(starts)]
                leaf = int(rng.integers(127, 255))
                place(path_to(b, lp, leaf), s, next(kinds))
            elif what == "fanout":
                # a zero_scale chain whose C -> D edge crosses into a later pass, first
                depth = np.zeros(len(lp), np.int64)
                for x in range(1, len(lp)):
                    depth[x] = depth[lp[x]] + 1
                cand = [x for x in range(len(lp)) if crosses[b + x] and depth[x] >= 2]
                if cand:
                    leaf = cand[0]
                    while (lp == leaf).any():
                        leaf = int(np.nonzero(lp == leaf)[0][0])
                    assert place(path_to(b, lp, leaf), int(depth[cand[0]]) - 2, "zero_scale")
                leaves = np.arange(len(lp) - 576, len(lp))           # depth 6
                for s in (1, 2, 3):
                    kind = next(kinds)
                    assert any(place(path_to(b, lp, int(rng.choice(leaves))), s, kind) for _ in range(50))
        # the deep chain: a zero_scale chain whose C -> D edge is the first pass boundary, the other kinds further down
        chain = np.arange(self.chain_base, self.chain_base + 700)
        bounds_at = np.nonzero(crosses[chain])[0]
        assert len(bounds_at) >= 2 and bounds_at[0] >= 2
        assert place(list(chain), int(bounds_at[0]) - 2, "zero_scale")
        for s, kind in zip(range(int(bounds_at[0]) + 130, 700, 130), ("quat_norms", "offsets", "subnormal", "nan_t")):
            assert place(list(chain), s, kind, identity_ancestors=False)
        assert place(list(range(b40, b40 + 40)), 20, "zero_scale")
        # flat rows: translations with zero components that flip sign (written unconditionally on Changed<Transform>)
        for r in range(n_flat, n_flat + 24):
            t = trs[r].copy(); t[3:7] = [0, 0, 0, 1]; t[1] = 0.0
            trs[r] = t
            f = t.copy(); f[1] = -0.0
            if r % 2:
                f[4] = -0.0
            self.flip[r] = f
        sc = Scene(f"propagate_edges_{seed}", parent, trs, bounds, flags, np.full(n, scenes.CLASS_MESH, np.uint8),
                   np.arange(n, dtype=np.uint64) + np.uint64(1), cameras=scenes.four_cameras(), roots=roots.astype(np.uint32))
        lpos = scenes.fibonacci_sphere(8, 40.0).astype(f32)
        cols, light_row = scenes._append_lights((sc.parent, sc.trs, sc.bounds, sc.flags, sc.class_mask), lpos,
                                                np.linspace(5.0, 30.0, 8).astype(f32))
        sc.parent, sc.trs, sc.bounds, sc.flags, sc.class_mask = cols
        sc.entity_bits = np.arange(sc.n, dtype=np.uint64) + np.uint64(1)
        sc.light_row, sc.light_range = light_row, np.linspace(5.0, 30.0, 8).astype(f32)
        for c in sc.cameras:
            c.far = 200.0
        self.scene = sc

    def uploads(self, f):
        """(rows, trs) whose Transform is uploaded (Changed<Transform>) before frame f; also applied to the scene."""
        kind = self.FRAMES[f]
        if kind == "zero_signs":
            rows = np.array(sorted(self.flip), np.uint32)
            trs = np.stack([self.flip[r] for r in rows])
        elif kind == "nan_revisit":
            rows = np.array([r for r, again in self.nan_rows if again], np.uint32)
            trs = self.scene.trs[rows].copy()
        else:
            return np.zeros(0, np.uint32), np.zeros((0, 10), f32)
        self.scene.trs[rows] = trs
        return rows, trs

    def marks(self, f, gt):
        """(rows, values) another system writes before frame f: a probe parent's stored GlobalTransform with its zeros
        negated, or with a NaN translation."""
        if self.FRAMES[f] != "marks":
            return np.zeros(0, np.uint32), np.zeros((0, 12), f32)
        rows = np.array(self.mark_parents, np.uint32)
        vals = gt[rows].copy()
        for i in range(len(rows)):
            if i % 3 == 2:
                vals[i, 10] = np.nan
            else:
                z = vals[i] == 0
                vals[i, z] = -vals[i, z]
        return rows, vals


def run_reference(es, static_opt=True, mutants=(), frames=None, mutant_rows=None):
    """The edge scene's frames through the float32 restatement: [(gt, changed, the frame's Transforms)] per frame."""
    sc = es.scene
    trs0 = sc.trs.copy()
    try:
        gt = np.tile(np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], f32), (sc.n, 1))
        tch = np.ones(sc.n, bool)
        out = []
        for f in range(len(es.FRAMES) if frames is None else frames):
            rows, _ = es.uploads(f)
            tch[rows] = True
            mrows, mvals = es.marks(f, gt)
            ext = np.zeros(sc.n, bool)
            gt[mrows] = mvals
            ext[mrows] = True
            ch = propagate(sc.parent, sc.trs, gt, tch, static_opt, ext, mutants, mutant_rows)
            tch[:] = False
            out.append((gt.copy(), ch, sc.trs.copy()))
        return out
    finally:
        sc.trs[:] = trs0
