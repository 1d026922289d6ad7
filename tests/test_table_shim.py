"""The table write-back without Python: tests/table_shim.c registers malloc'd, Bevy-native archetype tables filled in spawn
order (not the planned row order) through include/b200vis.h, has the GPU write both components and both changed_ticks
columns into them, and checks every frame against the CPU oracle."""
import ctypes as C
import json
import os
import subprocess
import sys

import pytest

from bevy_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_table_shim(out):
    sys.path.insert(0, ROOT)
    import oracle
    oracle.build()
    cmd = ["gcc", "-O2", "-std=gnu11", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "table_shim.c"), "-o", out,
           "-L" + os.path.join(ROOT, "bevy_b200"), "-lb200vis", "-L" + os.path.join(ROOT, "oracle"), "-lbevy_oracle", "-lm",
           "-Wl,-rpath," + os.path.join(ROOT, "bevy_b200"), "-Wl,-rpath," + os.path.join(ROOT, "oracle")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr


def test_table_struct_layout_matches_ctypes(tmp_path):
    """No GPU needed: the harness compiles as C11 with -Wall -Wextra -Werror, links against libb200vis.so, and the C layout
    of b200vis_table is the one abi.Table declares."""
    exe = str(tmp_path / "table_shim")
    build_table_shim(exe)
    res = subprocess.run([exe, "--sizeof"], capture_output=True, text=True, timeout=60)
    assert res.returncode == 0, res.stderr
    lay = json.loads(res.stdout)
    assert lay["sizeof"] == C.sizeof(abi.Table)
    for name, _ in abi.Table._fields_:
        assert lay[name] == getattr(abi.Table, name).offset, name


@pytest.mark.gpu
def test_table_shim_matches_the_oracle(tmp_path):
    exe = str(tmp_path / "table_shim")
    build_table_shim(exe)
    res = subprocess.run([exe, "200", "6", "4"], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and "TABLE_SHIM OK" in res.stdout, res.stdout[-2000:] + res.stderr[-2000:]
    stats = json.loads([l for l in res.stdout.splitlines() if l.startswith("{")][-1])
    assert stats["entities"] == 200 * 63 + 48 and stats["rows_out_of_spawn_order"] > 0


@pytest.mark.gpu
def test_table_shim_at_bench_scale_reports_host_costs(tmp_path):
    """3922 trees of 255 (1,000,158 entities): prints the time per frame of the step and of the wait for the write-back."""
    exe = str(tmp_path / "table_shim")
    build_table_shim(exe)
    res = subprocess.run([exe, "3922", "8", "3"], capture_output=True, text=True, timeout=900)
    assert res.returncode == 0 and "TABLE_SHIM OK" in res.stdout, res.stdout[-2000:] + res.stderr[-2000:]
    print(res.stdout[-600:])
