"""Pins orc_propagate's gt_ext_changed input (a GlobalTransform another system wrote since the propagate system last ran)
to the rule of propagate_descendants_unchecked (crates/bevy_transform/src/systems.rs:706-724): a child is skipped only if
static optimisations are on, its tree is clean and NOT p_global_transform.is_changed() -- and is_changed() is true when
propagation wrote the parent in this run or another system wrote it before.  So a marked row that propagation visits hands
its children "changed" even when set_if_neq keeps its bits; a marked row it does not visit keeps the written value and hands
nothing.  The expected matrices come from orc.propagate with every row changed, so no matrix product is restated here."""
import numpy as np

import oracle as orc

NO = orc.NO_PARENT
# 0 R (root)   1 A (R)   2 S (R)   3 P (A)   4 C1 (P)   5 C2 (P)   6 G (C1)   7 Q (root)   8 Q1 (Q)   9 Q2 (Q1)   10 L (lone root)
R, A, S, P, C1, C2, G, Q, Q1, Q2, L = range(11)
PARENT = np.array([NO, R, R, A, P, P, C1, NO, Q, Q1, NO], np.uint32)
N = len(PARENT)


def random_trs(rng, n):
    trs = np.zeros((n, 10), np.float32)
    trs[:, 0:3] = rng.uniform(-3, 3, (n, 3))
    q = rng.normal(size=(n, 4)).astype(np.float32)
    trs[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    trs[:, 7:10] = rng.uniform(0.5, 2.0, (n, 3))
    return trs


def full(trs):
    """Every row propagated: what each row's GlobalTransform is once everything has been recomputed."""
    gt = np.tile(orc.IDENTITY_GT, (N, 1))
    rc, _ = orc.propagate(PARENT, trs, gt, np.ones(N, np.uint8), True)
    assert rc == 0
    return gt


def setup(seed=1):
    """A converged world (gt = the full propagation of trs0), then S's Transform changes: R's tree is dirty, and only the
    rows that depend on S have new values in F1."""
    rng = np.random.default_rng(seed)
    trs0 = random_trs(rng, N)
    trs1 = trs0.copy()
    trs1[S] = random_trs(rng, 1)[0]
    tchanged = np.zeros(N, np.uint8)
    tchanged[S] = 1
    return trs1, full(trs0), full(trs1), tchanged


def run(trs, gt, tchanged, marks=(), static_opt=True):
    ext = np.zeros(N, np.uint8)
    ext[list(marks)] = 1
    gt = gt.copy()
    rc, changed = orc.propagate(PARENT, trs, gt, tchanged.copy(), static_opt, gt_ext_changed=ext)
    assert rc == 0
    return gt, changed


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def written(rng):
    return rng.uniform(-5, 5, 12).astype(np.float32)


def test_marked_parent_recomputed_to_its_written_bits_repropagates_children():
    trs, F0, F1, tch = setup()
    rng = np.random.default_rng(7)
    gt = F0.copy()
    gt[A] = F1[A]                                        # TransformHelper-style write: the bits propagation will compute
    for r in (P, C1, C2, G):
        gt[r] = written(rng)                             # stale descendants: they only change if A hands "changed" down
    got, ch = run(trs, gt, tch, marks=[A])
    assert (bits(got) == bits(F1)).all()
    assert ch[A] == 0, "set_if_neq keeps A's bits: its own Changed<GlobalTransform> must not fire"
    assert ch[[R, S, P, C1, C2, G]].all()
    # without the mark, A hands nothing down and its subtree keeps the stale values
    got0, ch0 = run(trs, gt, tch)
    assert (bits(got0[[P, C1, C2, G]]) == bits(gt[[P, C1, C2, G]])).all()
    assert not ch0[[A, P, C1, C2, G]].any()


def test_marked_row_not_visited_keeps_written_value():
    trs, F0, F1, tch = setup()
    gt = F0.copy()
    w = written(np.random.default_rng(3))
    gt[P] = w                                            # A is visited but unchanged, P's subtree is clean: P is not visited
    got, ch = run(trs, gt, tch, marks=[P])
    assert (bits(got[P]) == bits(w)).all()
    assert (bits(got[[C1, C2, G]]) == bits(F0[[C1, C2, G]])).all(), "the children of an unvisited row are untouched"
    assert not ch[[A, P, C1, C2, G]].any()
    assert (bits(got[[R, S]]) == bits(F1[[R, S]])).all() and ch[[R, S]].all()


def test_mark_in_clean_tree_does_nothing():
    trs, F0, F1, tch = setup()
    rng = np.random.default_rng(4)
    gt = F0.copy()
    gt[Q1] = written(rng)
    gt[Q] = written(rng)
    gt[L] = written(rng)
    got, ch = run(trs, gt, tch, marks=[Q, Q1, L])
    assert (bits(got[[Q, Q1, L]]) == bits(gt[[Q, Q1, L]])).all()
    assert (bits(got[Q2]) == bits(F0[Q2])).all()
    assert not ch[[Q, Q1, Q2, L]].any()
    got0, ch0 = run(trs, gt, tch)
    assert (bits(got) == bits(got0)).all() and (ch == ch0).all()


def test_static_optimisations_off_marks_are_irrelevant():
    trs, F0, F1, tch = setup()
    rng = np.random.default_rng(5)
    gt = F0.copy()
    for r in (A, P, C1, Q1, L):
        gt[r] = written(rng)
    everything = [r for r in range(N)]
    for marks in ([A], [P, Q1], [L, Q], everything):
        got, ch = run(trs, gt, tch, marks=marks, static_opt=False)
        got0, ch0 = run(trs, gt, tch, static_opt=False)
        assert (bits(got) == bits(got0)).all() and (ch == ch0).all()
    assert (bits(got0[:L]) == bits(F1[:L])).all()


def test_marked_root_with_children_is_overwritten_as_always():
    trs, F0, F1, tch = setup()
    rng = np.random.default_rng(6)
    gt = F0.copy()
    gt[R] = written(rng)                                 # R's tree is dirty: the root is rewritten from its Transform
    got, ch = run(trs, gt, tch, marks=[R])
    got0, ch0 = run(trs, gt, tch)
    assert (bits(got[R]) == bits(F1[R])).all() and ch[R] == 1
    assert (bits(got) == bits(got0)).all() and (ch == ch0).all()
    gt[Q] = written(rng)                                 # Q's tree is clean: Q keeps the written value, its children are not visited
    got, ch = run(trs, gt, tch, marks=[Q])
    assert (bits(got[Q]) == bits(gt[Q])).all() and not ch[[Q, Q1, Q2]].any()
    assert (bits(got[[Q1, Q2]]) == bits(F0[[Q1, Q2]])).all()
