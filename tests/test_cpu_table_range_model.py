"""The table range-read model (tests/table_range_model.py) on a machine without a GPU: its rules on hand-made slots, and a
frame sequence like the one tests/test_gpu_tables_range_read.py runs (ranged and unranged tables, the shared `game`, a
first full read, tick wrap, archetype moves into and out of a ranged table, a changed table entry, use_aabb bytes other
than 0 and 1) telling every wrong rule of the model apart from the right one."""
import numpy as np
import pytest

import table_range_model as M

U32 = 0xFFFFFFFF
NONE = M.UNMAPPED


def world(rng, struct, n=120, headroom=8):
    """Three tables, rows 0..n-1 spread over them: two with a VisibilityRange column, one without; every slot fresh."""
    stride = M.STRUCTS[struct]["stride"]
    groups = np.array_split(rng.permutation(n).astype(np.uint32), 3)
    tables = []
    for k, g in enumerate(groups):
        cap = len(g) + headroom
        rows = np.full(cap, NONE, np.uint32); rows[:len(g)] = g
        ranged = k != 2
        tables.append(M.RangeTable(len(g), cap, rows, np.ones(cap, bool),
                                   ranges=np.zeros((cap, stride), np.uint8) if ranged else None,
                                   ticks=np.zeros(cap, np.uint32) if ranged else None))
    return tables


def move(tables, src, s, dst):
    """An archetype move with swap_remove: the row of (src, s) to the end of dst, src's last row into s."""
    a, b = tables[src], tables[dst]
    row = a.rows[s]
    b.rows[b.len] = row; b.fresh[b.len] = True; b.len += 1
    last = a.len - 1
    a.rows[s] = a.rows[last]; a.fresh[s] = True
    a.rows[last] = NONE; a.fresh[last] = True; a.len -= 1


def frames(struct, seed=3):
    """Yields (tables, last_run, this_run, se, ua) before each read."""
    rng = np.random.default_rng(seed)
    n = 120
    tables = world(rng, struct, n)
    se = rng.integers(0, 2**31, (n, 2), dtype=np.uint32)
    ua = rng.integers(0, 2, n).astype(np.uint8)
    L = U32 - 25                                             # this_run crosses the u32 wrap on the third frame
    for f in range(8):
        R = (L + 10) & U32
        M.game(tables, struct, rng, L, R)
        if f == 3:
            move(tables, 0, 1, 2)                            # out of a ranged table
            move(tables, 2, 0, 1)                            # into a ranged table
        if f == 5:                                           # table 1's range column reallocated: read in full
            tables[1].fresh[:] = True
        yield tables, L, R, se, ua
        se, ua, fresh = M.read(tables, struct, L, R, se, ua)
        for t, fr in zip(tables, fresh):
            t.fresh = fr
        L = R


@pytest.mark.parametrize("struct", list(M.STRUCTS))
def test_every_mutant_is_told_apart(struct):
    told = {m: False for m in M.MUTANTS}
    for tables, L, R, se, ua in frames(struct):
        right = M.read(tables, struct, L, R, se, ua)
        for m in M.MUTANTS:
            told[m] |= not M.same(right, M.read(tables, struct, L, R, se, ua, mutant=m))
    missing = [m for m, t in told.items() if not t]
    assert not missing, f"no frame tells {missing} apart"


def test_rules_on_one_slot():
    st = "bevy"
    cap = 4
    col = np.zeros((cap, 20), np.uint8)
    M.put(col, st, [0], [2.0], [9.0], [2], margins=[[3.0, 8.0]])
    ticks = np.full(cap, 100, np.uint32)
    rows = np.array([0, NONE, NONE, NONE], np.uint32)
    se0, ua0 = np.zeros((1, 2), np.uint32), np.zeros(1, np.uint8)

    def one(fresh, L=100, R=110, t=ticks):
        tb = M.RangeTable(1, cap, rows, np.array([fresh, 0, 0, 0], bool), ranges=col, ticks=t)
        return M.read([tb], st, L, R, se0, ua0)
    se, ua, fr = one(True)                                   # full: start_margin.start, end_margin.end, use_aabb != 0
    assert (se[0].view(np.float32) == [2.0, 9.0]).all() and ua[0] == 1 and not fr[0].any()
    se, ua, _ = one(False)                                   # tick == last_run: not newer, not fresh: unchanged
    assert (se == se0).all() and (ua == ua0).all()
    se, ua, _ = one(False, t=np.full(cap, 101, np.uint32))   # newer tick: read
    assert (se[0].view(np.float32) == [2.0, 9.0]).all() and ua[0] == 1
    se, _, _ = one(False, L=U32 - 2, R=5, t=np.full(cap, 1, np.uint32))   # newer across the wrap
    assert (se[0].view(np.float32) == [2.0, 9.0]).all()
    tb = M.RangeTable(1, cap, rows, np.ones(cap, bool))      # no range column: the table is not read
    se, ua, fr = M.read([tb], st, 100, 110, se0, ua0)
    assert (se == se0).all() and fr[0].all()
    for mutant, want in (("end_margin_start", [2.0, 8.0]), ("use_aabb_bit0", None)):
        tb = M.RangeTable(1, cap, rows, np.array([1, 0, 0, 0], bool), ranges=col, ticks=ticks)
        se, ua, _ = M.read([tb], st, 100, 110, se0, ua0, mutant=mutant)
        if want is not None:
            assert (se[0].view(np.float32) == want).all()
        else:
            assert ua[0] == 0


def test_the_gpu_scenarios_cover_every_mutant():
    """Each GPU scenario asserts, on the device run, that its frames tell the mutants of its EXPECT entry apart; together
    they cover every mutant of the model."""
    import test_gpu_tables_range_read as G
    assert set().union(*G.EXPECT.values()) == set(M.MUTANTS)
    assert set(G.EXPECT) <= set(G.CALLS)
