"""The table write-back scenarios of tests/test_gpu_table_writeback_edges.py, played on the CPU oracle alone: each one must
tell every wrong rule of tests/table_model.py (MUTANTS) apart from the header's, in at least one slot at one of its checks.
So the device tests are shown, without a device, to fail for a kernel or host that followed any of those rules."""
import numpy as np
import pytest

import table_model as tm


@pytest.mark.parametrize("name", list(tm.SCENARIOS))
def test_scenario_separates_every_mutant(name):
    run = tm.SCENARIOS[name](device=False)
    assert run.checks > 0
    missed = set(tm.MUTANTS) - run.separated
    assert not missed, f"{name} cannot tell these rules from the header's: {sorted(missed)}"


def test_the_model_writes_nothing_past_len_or_into_null_columns():
    """The rules themselves on a hand-made registry: slots past len, unmapped slots and NULL columns keep their bytes; a
    remap and a column change make the known byte unknown."""
    m = tm.Model(8)
    data = lambda cap: {"gt": np.zeros((cap, 16), np.uint32), "gt_ticks": np.zeros(cap, np.uint32),
                        "vv": np.full(cap, tm.VV_SENTINEL, np.uint8), "vv_ticks": np.zeros(cap, np.uint32)}
    m.data = [data(4), data(4)]
    m.set_tables([dict(len=2, cap=4, cols=tm.ALL, vv_mem=1), dict(len=4, cap=4, cols=frozenset({"gt_ticks"}), vv_mem=None)])
    m.set_rows(0, 0, [3, 5, 6])                              # slot 2 is past len
    m.set_rows(1, 0, [0, tm.NONE, 1])
    gt = np.arange(8 * 12, dtype=np.float32).reshape(8, 12)
    ones = np.ones(8, np.uint8)
    vv = np.array([1, 1, 0, 1, 0, 3, 1, 0], np.uint8)
    m.writeback(tm.GT | tm.VV, 7, 9, gt, ones, vv, ones)
    assert (m.data[0]["gt"][:2] == tm.affine3a_bits(gt[[3, 5]])).all() and not m.data[0]["gt"][2:].any()
    assert m.data[0]["vv"].tolist() == [1, 3, tm.VV_SENTINEL, tm.VV_SENTINEL] and m.data[0]["vv_ticks"].tolist() == [9, 9, 0, 0]
    assert m.data[1]["gt_ticks"].tolist() == [7, 0, 7, 0] and not m.data[1]["gt"].any() and not m.data[1]["vv_ticks"].any()
    m.data[0]["vv"][0] = 0                                   # a stale byte the model knows nothing about: kept
    m.writeback(tm.VV, 7, 10, gt, ones, vv, 0 * ones)
    assert m.data[0]["vv"][0] == 0
    m.set_rows(0, 1, [3])                                    # row 3 moves: its byte is written again
    m.writeback(tm.VV, 7, 10, gt, ones, vv, 0 * ones)
    assert m.data[0]["vv"][1] == 1 and m.map[0] == tm.NONE
    mut = tm.Model(8, "capacity")
    mut.data = [data(4)]
    mut.set_tables([dict(len=1, cap=4, cols=tm.ALL, vv_mem=1)])
    mut.set_rows(0, 0, [2, 4])
    mut.writeback(tm.GT, 1, 1, gt, ones, vv, ones)
    assert mut.data[0]["gt_ticks"].tolist() == [1, 1, 0, 0]
