"""The C oracle's propagate against an independent numpy float32 restatement (tests/propagate_reference.py), bit for bit,
on random forests and on the edge scenes (signed zeros, NaN, subnormals, overflow, zero and non-unit quaternions, world
offsets); the float32 results against a float64 reference within a rounding-count bound; and proof, in numpy, that the
edge scenes detect the kernel mistakes they are there for, including children computed from a parent's new matrix on each
single kind of parent hand-over of the tile kernels."""
import numpy as np
import pytest

from bevy_b200 import abi, scenes
import oracle as orc
import propagate_reference as ref

NO_PARENT, DETACHED = ref.NO_PARENT, ref.DETACHED
tiles_of = ref.tiles_of
T_EXT_PARENT = 1 << 30


def same_bits(a, b):
    """Bit equality, except that any NaN matches any NaN; +0 and -0 differ."""
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def random_forest(seed):
    """Random topological forest with flat rows, detached rows, zero scales and mutated Transforms between frames."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(200, 3000))
    parent = np.full(n, NO_PARENT, np.uint32)
    for r in range(1, n):
        k = rng.random()
        if k < 0.1:
            continue
        if k < 0.13:
            parent[r] = DETACHED
            continue
        parent[r] = rng.integers(max(0, r - int(rng.integers(1, 200))), r)
    trs = np.zeros((n, 10), np.float32)
    trs[:, 0:3] = rng.uniform(-50, 50, (n, 3)); trs[:, 3:7] = scenes.random_unit_quats(rng, n)
    trs[:, 7:10] = rng.uniform(-1.5, 1.5, (n, 3))
    trs[rng.random(n) < 0.02, 7] = 0.0
    return parent, trs


def oracle_frames(parent, trs_per_frame, tch_per_frame, static_opt, ext_per_frame=None):
    gt = np.tile(orc.IDENTITY_GT, (len(parent), 1))
    out = []
    for f, (trs, tch) in enumerate(zip(trs_per_frame, tch_per_frame)):
        ext = None
        if ext_per_frame is not None:
            rows, vals = ext_per_frame(f, gt)
            gt[rows] = vals
            ext = np.zeros(len(parent), np.uint8); ext[rows] = 1
        rc, ch = orc.propagate(parent, trs, gt, tch, static_opt, gt_ext_changed=ext)
        assert rc == 0
        out.append((gt.copy(), ch.astype(bool)))
    return out


def assert_same(got, want, what):
    for f, ((g, c), (wg, wc)) in enumerate(zip(got, want)):
        bad = ~same_bits(g, wg).all(1)
        assert not bad.any(), f"{what} frame {f}: GlobalTransform bits differ on rows {np.nonzero(bad)[0][:8]}"
        assert (c == wc).all(), f"{what} frame {f}: Changed<GlobalTransform> differs on rows {np.nonzero(c != wc)[0][:8]}"


# ---- the oracle against the restatement --------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("static_opt", [True, False])
def test_oracle_matches_restatement_on_random_forests(seed, static_opt):
    parent, trs0 = random_forest(seed)
    rng = np.random.default_rng(seed + 100)
    n = len(parent)
    trs_f, tch_f = [trs0], [np.ones(n, np.uint8)]
    for f in range(1, 4):
        trs = trs_f[-1].copy()
        tch = (rng.random(n) < 0.05).astype(np.uint8)
        trs[tch == 1, 0:3] += rng.uniform(-1, 1, (int(tch.sum()), 3)).astype(np.float32)
        trs_f.append(trs); tch_f.append(tch)
    want = oracle_frames(parent, trs_f, tch_f, static_opt)
    gt = np.tile(orc.IDENTITY_GT, (n, 1))
    got = []
    for trs, tch in zip(trs_f, tch_f):
        ch = ref.propagate(parent, trs, gt, tch, static_opt)
        got.append((gt.copy(), ch))
    assert_same(got, want, f"random forest {seed}")
    r, checked = ref.bound_violation(got[-1][0], parent, trs_f[-1])
    assert checked > 0 and r <= 1.0, f"float32 result exceeds the float64 bound by {r:.3g}x"


@pytest.fixture(scope="module")
def edge():
    return ref.EdgeScene(seed=0)


def edge_oracle(es, static_opt):
    sc = es.scene
    trs0 = sc.trs.copy()
    try:
        trs_f, tch_f = [], []
        for f in range(len(es.FRAMES)):
            rows, _ = es.uploads(f)
            tch = np.ones(sc.n, np.uint8) if f == 0 else np.zeros(sc.n, np.uint8)
            tch[rows] = 1
            trs_f.append(sc.trs.copy()); tch_f.append(tch)
    finally:
        sc.trs[:] = trs0
    return oracle_frames(sc.parent, trs_f, tch_f, static_opt, ext_per_frame=es.marks)


@pytest.mark.parametrize("static_opt", [True, False])
def test_oracle_matches_restatement_on_edge_scene(edge, static_opt):
    want = edge_oracle(edge, static_opt)
    got = [(g, c) for g, c, _ in ref.run_reference(edge, static_opt)]
    assert_same(got, want, "edge scene")
    g0 = got[0][0]
    with np.errstate(invalid="ignore"):
        sub = (g0 != 0) & (np.abs(g0) < ref.TINY)
    assert np.isnan(g0).any() and np.isinf(g0).any() and sub.any()
    assert (np.signbit(g0) & (g0 == 0)).any()


def test_edge_scene_values(edge):
    """The scene reaches what it is there for: subnormal results, Inf, NaN from Inf * 0 and Inf - Inf, kept zero signs."""
    got = ref.run_reference(edge, True)
    g0, c1 = got[0][0], got[1][1]
    with np.errstate(invalid="ignore"):
        assert ((g0 != 0) & (np.abs(g0) < ref.TINY)).sum() >= 20
    assert np.isinf(g0[:, 0:9]).any() and np.isinf(g0[:, 9:12]).any()
    assert np.isnan(g0[:, 0:9]).any() and np.isnan(g0[:, 9:12]).any()
    # the zero-sign frame: rows whose only new input is a zero sign are visited and keep their bits
    flipped = np.array(sorted(edge.flip), np.int64)
    kept = flipped[~c1[flipped]]
    assert len(kept) >= 5
    # NaN rows: re-uploaded ones report a change again, the others' trees stay clean; a static frame changes nothing
    c2 = got[2][1]
    assert c2[[r for r, a in edge.nan_rows if a]].all() and not c2[[r for r, a in edge.nan_rows if not a]].any()
    assert not got[3][1].any() and not got[5][1].any()


@pytest.mark.parametrize("static_opt", [True, False])
@pytest.mark.parametrize("mutant", ref.EDGE_MUTANTS)
def test_edge_scene_detects_mutant(edge, static_opt, mutant):
    base = ref.run_reference(edge, static_opt)
    mut = ref.run_reference(edge, static_opt, mutants=(mutant,))
    diff = [int((~same_bits(g, mg).all(1) | (c != mc)).sum()) for (g, c, _), (mg, mc, _) in zip(base, mut)]
    assert sum(diff) > 0, f"the edge scene cannot detect '{mutant}'"


# ---- float64 bound -------------------------------------------------------------------------------------------------------------
def test_bound_holds_on_edge_scene(edge):
    for static_opt in (True, False):
        for f, (g, _, trs) in enumerate(ref.run_reference(edge, static_opt)):
            if edge.FRAMES[f] != "marks":                # a written NaN stays until its tree is propagated again
                r, checked = ref.bound_violation(g, edge.scene.parent, trs)
                assert checked > 100000 and r <= 1.0, f"frame {f}: float32 result exceeds the float64 bound by {r:.3g}x"


@pytest.mark.parametrize("mutant", ref.ALGEBRA_MUTANTS)
def test_bound_rejects_algebra_mistakes(edge, mutant):
    """A transposed from_quat, parent and child swapped, the scale on rows, a quaternion sign error: each exceeds the
    float64 bound by at least 100x, on the edge scene and on a random forest."""
    g = ref.run_reference(edge, True, mutants=(mutant,), frames=1)[0][0]
    r, _ = ref.bound_violation(g, edge.scene.parent, edge.scene.trs)
    assert r >= 100.0, f"'{mutant}' exceeds the bound by only {r:.3g}x on the edge scene"
    parent, trs = random_forest(7)
    gt = np.tile(orc.IDENTITY_GT, (len(parent), 1))
    ref.propagate(parent, trs, gt, np.ones(len(parent), bool), True, mutants=(mutant,))
    r, _ = ref.bound_violation(gt, parent, trs)
    assert r >= 100.0, f"'{mutant}' exceeds the bound by only {r:.3g}x on a random forest"


# ---- the probes sit on every edge type of the tile kernels -------------------------------------------------------------------
HAND_OVERS = ("cross_pass", "top_levels", "scout_levels", "syncwarp", "named_barrier", "more_than_8_levels", "warp_slot")


def hand_overs(parent):
    """How each row receives its parent's GlobalTransform, by the CTA-per-tile and warp-per-tile plans: kind -> [n] bool.
    cross_pass: the parent is in a tile of an earlier pass (read from HBM at level 0).  top_levels: 1L walks the tile's
    depths < top_levels in registers when top_levels >= 2.  scout_levels: the scout kernel's scout warps walk depths
    < top_levels for any top_levels >= 1 (the same rows as top_levels while every in-tile child has depth >= 1, kept
    apart so that a planner change cannot merge them unseen).  syncwarp / named_barrier: the level loop of a tile of 2..8
    levels.  more_than_8_levels: the CTA-wide walk.  warp_slot: the warp kernel's parent slots."""
    n = len(parent)
    desc, topo = abi.host_tile_plan(parent)
    tile_of, wtile = tiles_of(desc, n), tiles_of(abi.host_warp_plan(parent)[0], n)
    out = {k: np.zeros(n, bool) for k in HAND_OVERS}
    for c in np.nonzero(parent < n)[0]:
        p = int(parent[c])
        _, _, n_levels, wsm, top, lo, hi, _ = desc[tile_of[c]].tolist()
        if wtile[p] == wtile[c]:
            out["warp_slot"][c] = True
        if tile_of[p] != tile_of[c]:
            assert topo[c] & T_EXT_PARENT
            out["cross_pass"][c] = True
            continue
        lvl = (int(topo[c]) >> 9) & 0x1FF
        out["more_than_8_levels"][c] = n_levels > 8
        out["top_levels"][c] = top >= 2 and lvl < top
        out["scout_levels"][c] = top >= 1 and lvl < top
        if 2 <= n_levels <= 8 and (wsm >> lvl) & 1:
            out["syncwarp"][c] = True                      # the level loop's __syncwarp (1b; 1L without the register walk)
        elif 2 <= n_levels <= 8 and (lo | hi) and lvl >= max(top, 1):
            out["named_barrier"][c] = True
    return out


@pytest.fixture(scope="module")
def edge_hand_overs(edge):
    return hand_overs(edge.scene.parent)


def test_probe_edges_cover_every_hand_over(edge, edge_hand_overs):
    children = np.array([c for _, c in edge.probe_edges])
    missing = [k for k in HAND_OVERS if not edge_hand_overs[k][children].any()]
    assert not missing, f"no probe edge is handed over by {missing}"


@pytest.mark.parametrize("static_opt", [True, False])
@pytest.mark.parametrize("kind", HAND_OVERS)
def test_edge_scene_detects_new_matrix_on_each_hand_over(edge, edge_hand_overs, kind, static_opt):
    """Children computed from the parent's new matrix instead of its kept bits, on this one kind of hand-over only,
    changes a GlobalTransform bit or a Changed flag: a kernel that got the kept bits wrong on just that path is seen."""
    base = ref.run_reference(edge, static_opt)
    mut = ref.run_reference(edge, static_opt, mutants=("children_from_new",), mutant_rows=edge_hand_overs[kind])
    diff = sum(int((~same_bits(g, mg).all(1) | (c != mc)).sum()) for (g, c, _), (mg, mc, _) in zip(base, mut))
    assert diff > 0, f"the edge scene cannot tell kept bits from new bits on the '{kind}' hand-over"
