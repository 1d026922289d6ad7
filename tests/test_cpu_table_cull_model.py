"""The table cull-read model (tests/table_cull_model.py) on a machine without a GPU: its rules on hand-made slots, and the
frame sequence tests/test_gpu_tables_cull_read.py runs (the archetype tables of M.ARCHETYPES, the shared `game`, a first
full read, static and sparse frames, archetype moves, unmapped slots, mapped slots past len, rows marked
Changed<Transform>) telling every wrong rule of the model apart from the right one."""
import numpy as np
import pytest

import table_cull_model as M

U32 = 0xFFFFFFFF
NONE = M.UNMAPPED


def world(rng, layout, n=200, headroom=8):
    """Tables of every archetype over numpy memory, rows 0..n-1 spread over them, every slot fresh (just attached)."""
    sa, ss = layout[0], layout[3]
    groups = np.array_split(rng.permutation(n).astype(np.uint32), len(M.ARCHETYPES))
    tables = []
    for g, arch in zip(groups, M.ARCHETYPES):
        cap = len(g) + headroom
        rows = np.full(cap, NONE, np.uint32); rows[:len(g)] = g
        has = arch["has"]
        col = lambda name, shape, dt=np.uint8: np.zeros(shape, dt) if name in has else None
        tables.append(M.CullTable(len(g), cap, rows, np.ones(cap, bool),
                                  aabb=col("aabb", (cap, sa)), aabb_ticks=col("aabb", cap, np.uint32),
                                  sphere=col("sphere", (cap, ss)), sphere_ticks=col("sphere", cap, np.uint32),
                                  iv=col("iv", cap), iv_ticks=col("iv", cap, np.uint32), flags=arch["flags"]))
    return tables


def move(tables, src, s, dst):
    """An archetype move with swap_remove: the row of (src, s) to the end of dst, src's last row into s."""
    a, b = tables[src], tables[dst]
    row = a.rows[s]
    b.rows[b.len] = row; b.fresh[b.len] = True; b.len += 1
    last = a.len - 1
    a.held = a.rows.copy()
    a.rows[s] = a.rows[last]; a.fresh[s] = True
    a.rows[last] = NONE; a.fresh[last] = True; a.len -= 1


def frames(layout, seed=5):
    """Yields (tables, last_run, this_run, bounds, flags) before each read of the GPU test's sequence."""
    rng = np.random.default_rng(seed)
    n = 200
    tables = world(rng, layout, n)
    bounds = rng.integers(0, 2**31, (n, 6), dtype=np.uint32)
    flags = np.zeros(n, np.uint8)
    L = U32 - 30                                             # this_run crosses the u32 wrap on the fourth frame
    for f in range(9):
        R = (L + 10) & U32
        M.game(tables, layout, rng, L, R)
        if f == 3:
            move(tables, 0, 2, 1)                            # into NoFrustumCulling
            move(tables, 1, 0, 2)                            # into Sphere only
            move(tables, 2, 1, 3)                            # into Aabb + Sphere
            move(tables, 3, 0, 4)                            # into NoCpuCulling
            move(tables, 0, 0, 6)                            # into InheritedVisibility only
            move(tables, 1, 1, 7)                            # into flags only
        if f == 5:                                           # an unmapped slot below len, a mapped slot past len
            t = tables[0]
            t.held = t.rows.copy()
            t.rows[1] = NONE; t.fresh[1] = True
            t.rows[t.len] = t.held[1]; t.fresh[t.len] = True
        if f in (3, 6):                                      # rows whose Transform was read earlier in the frame
            flags[rng.choice(n, 40, replace=False)] |= M.F_TCHANGED
        yield tables, L, R, bounds, flags
        bounds, flags, fresh = M.read(tables, layout, L, R, bounds, flags)
        for t, fr in zip(tables, fresh):
            t.fresh = fr
        L = R


@pytest.mark.parametrize("layout", [M.BEVY_LAYOUT, M.PERMUTED_LAYOUT], ids=["bevy", "permuted"])
def test_every_mutant_is_told_apart(layout):
    told = {m: False for m in M.MUTANTS}
    for tables, L, R, bounds, flags in frames(layout):
        right = M.read(tables, layout, L, R, bounds, flags)
        for m in M.MUTANTS:
            told[m] |= not M.same(right, M.read(tables, layout, L, R, bounds, flags, mutant=m))
    missing = [m for m, t in told.items() if not t]
    if layout == M.PERMUTED_LAYOUT:
        assert not missing, f"no frame tells {missing} apart"
    else:                                                    # Bevy's layout differs from the packed one only in padding
        assert set(missing) <= {"packed_layout"}, missing


def test_rules_on_one_slot():
    lay = M.BEVY_LAYOUT
    cap = 4
    aabb = np.zeros((cap, 32), np.uint8); sph = np.zeros((cap, 32), np.uint8)
    M.put(aabb, [0], ((0, [[1, 2, 3]]), (16, [[4, 5, 6]])))
    M.put(sph, [0], ((0, [[7, 8, 9]]), (16, [[10]])))
    ticks = np.full(cap, 100, np.uint32)
    iv = np.array([1, 0, 0, 0], np.uint8)
    rows = np.array([0, NONE, NONE, NONE], np.uint32)
    bounds, flags = np.zeros((1, 6), np.uint32), np.array([M.F_TCHANGED | M.F_INHERITED], np.uint8)

    def one(fresh, aabb_=aabb, sph_=sph, iv_ticks=ticks, fl=M.F_NO_FRUSTUM):
        t = M.CullTable(1, cap, rows, np.array([fresh, 0, 0, 0], bool), aabb=aabb_, aabb_ticks=ticks, sphere=sph_,
                        sphere_ticks=ticks, iv=iv, iv_ticks=iv_ticks, flags=fl)
        return M.read([t], lay, 100, 110, bounds, flags)
    b, f, fr = one(True)                                     # full: Aabb over Sphere, flags rebuilt, F_TCHANGED kept
    assert (b[0].view(np.float32) == [1, 2, 3, 4, 5, 6]).all()
    assert f[0] == M.F_TCHANGED | M.F_NO_FRUSTUM | M.F_AABB | M.F_INHERITED and not fr[0].any()
    b, f, _ = one(True, aabb_=None)                          # Sphere only: radius then two zeros
    assert (b[0].view(np.float32) == [7, 8, 9, 10, 0, 0]).all() and f[0] & M.F_SPHERE
    b, f, _ = one(False)                                     # nothing newer, not fresh: unchanged
    assert (b == bounds).all() and (f == flags).all()
    b, f, _ = one(False, iv_ticks=np.full(cap, 105, np.uint32))   # InheritedVisibility newer: bit 0 only
    assert (b == bounds).all() and f[0] == M.F_TCHANGED | M.F_INHERITED
    b, f, _ = one(True, aabb_=None, sph_=None, fl=0)         # InheritedVisibility only: bounds kept, flags rebuilt
    assert (b == bounds).all() and f[0] == M.F_TCHANGED | M.F_INHERITED
    t = M.CullTable(1, cap, rows, np.ones(cap, bool), flags=M.F_NO_CPU)   # flags only: bounds kept
    b, f, _ = M.read([t], lay, 100, 110, bounds, flags)
    assert (b == bounds).all() and f[0] == M.F_TCHANGED | M.F_NO_CPU
    t = M.CullTable(1, cap, rows, np.ones(cap, bool))        # an entry with nothing: the table is not read
    b, f, fr = M.read([t], lay, 100, 110, bounds, flags)
    assert (f == flags).all() and fr[0].all()


def test_the_gpu_scenarios_cover_every_mutant():
    """Each GPU scenario asserts, on the device run, that its frames tell the mutants of its EXPECT entry apart; together
    they cover every mutant of the model."""
    import test_gpu_tables_cull_read as G
    assert set().union(*G.EXPECT.values()) == set(M.MUTANTS)
    assert set(G.EXPECT) <= set(G.CALLS)
