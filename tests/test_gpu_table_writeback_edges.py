"""The archetype-table write-back at its edges, on the device, checked through the tables only against the slot-by-slot
model of tests/table_model.py after b200vis_synchronize: mapped slots at and past len, every subset of NULL columns and
columns that come and go, the plugin's split frames with 16 and 32 views and other systems' GlobalTransforms, pipelined
frames, table lengths at the warp and chunk steps next to B200VIS_MAX_TABLES tables, the IEEE edge scene bit for bit, map
changes still queued when a topology call runs, and one rank's share of bench config #5, whose chunks outnumber the
write-back grid's warps.  tests/test_cpu_table_model.py shows on the CPU that each scenario would catch each of the model's
wrong rules."""
import os

import pytest

import table_model as tm
from test_gpu_bench_scale import run_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", list(tm.SCENARIOS))
def test_tables_match_the_model(name):
    run = tm.SCENARIOS[name](device=True)
    assert run.checks > 0


BENCH_SHARE = """
import numpy as np
import table_model as tm
sc = scenes.forest(4903, 8, 512, seed=11)           # config #5 on 8 GPUs: one rank's 1,250,265 rows + 512 lights
run = tm.Run(sc, True, mutants=(), seed=31)
try:
    groups = tm.archetypes(sc)
    tabs = run.add_tables([len(g) for g in groups], caps=[len(g) + 64 for g in groups])
    for t, g in zip(tabs, groups):
        run.fill(t, g)
    chunks = sum((run.tabs[t].len + 127) // 128 for t in tabs)
    assert chunks > 8 * 1184, chunks                 # the write-back's grid-stride loop goes round more than once
    run.frame("fused", "dense")
    run.frame("fused", "sparse")
finally:
    run.close()
"""


def test_one_ranks_share_of_config5_in_five_shuffled_tables():
    # the case's interpreter loads the library this one does
    run_case(BENCH_SHARE, {k: os.environ[k] for k in ("B200VIS_LIB",) if k in os.environ}, timeout=900)
