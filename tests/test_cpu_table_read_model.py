"""The table-read model (tests/table_read_model.py) on a machine without a GPU: Tick::is_newer_than on the values of
Bevy's own change-tick tests, and scenarios that tell every wrong rule of the model apart from the right one."""
import numpy as np
import pytest

import table_read_model as M

MAX = M.MAX_CHANGE_AGE
U32 = 0xFFFFFFFF

# (tick, last_run, this_run, newer), from crates/bevy_ecs/src/change_detection/mod.rs's tests
BEVY_TICKS = [
    (1, 0, 1, True),                                        # change_expiration: spawned after the system last ran
    (1, 1, (1 + MAX) & U32, False),                         # change_expiration: both MAX_CHANGE_AGE old -> MAX > MAX fails
    (0, U32, 1, True),                                      # change_tick_wraparound: last_run u32::MAX, world wrapped to 1
    (1, 0, (1 + MAX + M.CHECK_TICK_THRESHOLD) & U32, False),   # change_tick_scan: both ages past the clamp
]


def test_max_change_age_is_bevys():
    assert MAX == 3_258_167_296


@pytest.mark.parametrize("tick,last_run,this_run,newer", BEVY_TICKS)
def test_is_newer_than_on_bevys_tick_tests(tick, last_run, this_run, newer):
    assert bool(M.is_newer(tick, last_run, this_run)) is newer


def test_is_newer_than_edges():
    assert not M.is_newer(100, 100, 105)                     # a tick equal to last_run (the write-back's own stamp)
    assert M.is_newer(101, 100, 105) and M.is_newer(105, 100, 105)
    assert not M.is_newer(99, 100, 105)
    assert M.is_newer(3, U32 - 2, 5)                         # this_run across the wrap, the tick after it
    assert M.is_newer(U32, U32 - 2, 5)                       # ... and before it
    assert not M.is_newer(U32 - 2, U32 - 2, 5)


def layout_bytes(cap, layout, vals10, rng):
    stride, t, r, s = layout
    b = rng.integers(0, 256, (cap, stride), dtype=np.uint8)
    v = np.ascontiguousarray(vals10, np.float32).view(np.uint8).reshape(cap, 40)
    for o, a, e in ((t, 0, 12), (r, 12, 28), (s, 28, 40)):
        b[:, o:o + e - a] = v[:, a:e]
    return b


def scenario(kind, rng):
    """(tables, layout, which, last_run, this_run) for one scenario."""
    layout = (48, 16, 0, 28)
    last, this = 1000, 1010
    cap, n = 64, 40
    rows = np.full(cap, M.UNMAPPED, np.uint32)
    rows[:n] = rng.permutation(n)
    held = rows.copy()
    ticks = np.full(cap, last, np.uint32)
    gt_ticks = np.full(cap, last, np.uint32)
    newer = rng.random(cap) < 0.3
    ticks[newer] = last + 5
    gt_ticks[rng.random(cap) < 0.3] = last + 7
    gt = rng.standard_normal((cap, 16)).astype(np.float32)
    vals = rng.standard_normal((cap, 10)).astype(np.float32)
    tbl = dict(trs=layout_bytes(cap, layout, vals, rng), trs_ticks=ticks, gt=gt, gt_ticks=gt_ticks)
    which = M.RD_TRANSFORM | M.RD_GLOBAL_TRANSFORM
    if kind == "wrap":                                      # this_run past the u32 wrap, last_run before it
        last, this = U32 - 3, 6
        ticks[:] = U32 - 3; ticks[newer] = 2
        gt_ticks[:] = U32 - 3
    elif kind == "ancient":                                 # last_run and every tick older than MAX_CHANGE_AGE
        this = (last + MAX + 500) & U32
        ticks[:] = last + 3                                 # younger than last_run, both ages past the clamp
        gt_ticks[:] = last + 3
    elif kind == "own_stamp":                               # most ticks equal last_run
        pass
    elif kind == "past_len":                                # newer ticks and mapped rows at and past len
        rows[n:] = np.arange(n, cap)
        held = rows.copy()
        ticks[n:] = last + 5
    elif kind == "unmapped":                                # rows unmapped below len, their slots newer
        held = rows.copy()
        rows[[2, 7, 11]] = M.UNMAPPED
        ticks[[2, 7, 11]] = last + 5
    elif kind == "gt_no_ticks":
        tbl["gt_ticks"] = None
    tables = [M.ModelTable(n, cap, rows, held=held, **tbl)]
    return tables, layout, which, last, this


KINDS = ("plain", "wrap", "ancient", "own_stamp", "past_len", "unmapped", "gt_no_ticks")


def test_every_mutant_is_told_apart():
    rng = np.random.default_rng(7)
    cases = [scenario(k, rng) for k in KINDS]
    for mutant in M.MUTANTS:
        differs = [k for k, c in zip(KINDS, cases) if not M.same(M.read(*c), M.read(*c, mutant=mutant))]
        assert differs, f"no scenario tells the {mutant!r} mutant apart"


def test_reads_follow_the_rules():
    rng = np.random.default_rng(3)
    tables, layout, which, last, this = scenario("plain", rng)
    t = tables[0]
    trs, gt = M.read(tables, layout, which, last, this)
    want_t = {int(t.rows[s]) for s in range(t.len) if t.trs_ticks[s] == last + 5}
    want_g = {int(t.rows[s]) for s in range(t.len) if t.gt_ticks[s] == last + 7}
    assert set(trs) == want_t and set(gt) == want_g
    for s in range(t.len):
        r = int(t.rows[s])
        if r in gt:
            assert (gt[r] == t.gt[s].view(np.uint32).reshape(4, 4)[:, :3].reshape(12)).all()
    only_t = M.read(tables, layout, M.RD_TRANSFORM, last, this)
    assert only_t[0].keys() == trs.keys() and not only_t[1]
