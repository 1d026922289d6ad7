"""The plugin's VisibilityRange sequence without Python: tests/table_range_shim.c registers malloc'd, Bevy-native archetype
tables (one of them with a VisibilityRange column), attaches the ranges with the layout Rust's size_of / offset_of! give,
sets the range views from ShadowLodOrigin entities and the cameras (take(32), so one camera has range_view_index -1),
culls with a NULL range mask after a tick-driven table read, moves entities into and out of the ranged table, and checks
the range masks and every view's visible rows against the CPU oracle every frame."""
import ctypes as C
import json
import os
import subprocess
import sys

import pytest

from bevy_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_shim(out):
    sys.path.insert(0, ROOT)
    import oracle
    oracle.build()
    cmd = ["gcc", "-O2", "-std=gnu11", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "table_range_shim.c"), "-o", out,
           "-L" + os.path.join(ROOT, "bevy_b200"), "-lb200vis", "-L" + os.path.join(ROOT, "oracle"), "-lbevy_oracle", "-lm",
           "-Wl,-rpath," + os.path.join(ROOT, "bevy_b200"), "-Wl,-rpath," + os.path.join(ROOT, "oracle")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr


def test_range_layouts(tmp_path):
    """No GPU needed: the shim compiles as C11 with -Wall -Wextra -Werror and links against libb200vis.so; its
    VisibilityRange is the 20 bytes of abi.BEVY_VISIBILITY_RANGE_LAYOUT's guess, and b200vis_visibility_range_layout has
    the layout abi.VisibilityRangeLayout declares."""
    exe = str(tmp_path / "table_range_shim")
    build_shim(exe)
    res = subprocess.run([exe, "--sizeof"], capture_output=True, text=True, timeout=60)
    assert res.returncode == 0, res.stderr
    lay = json.loads(res.stdout)
    assert lay["visibility_range"] == abi.BEVY_VISIBILITY_RANGE_LAYOUT[0]
    L = abi.VisibilityRangeLayout
    assert lay["layout"] == [C.sizeof(L), L.start.offset, L.end.offset, L.use_aabb.offset]


@pytest.mark.gpu
def test_table_range_shim_matches_the_oracle(tmp_path):
    exe = str(tmp_path / "table_range_shim")
    build_shim(exe)
    res = subprocess.run([exe, "120", "6", "5"], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and "TABLE_RANGE_SHIM OK" in res.stdout, res.stdout[-2000:] + res.stderr[-2000:]
    stats = json.loads([line for line in res.stdout.splitlines() if line.startswith("{")][-1])
    # the scenario exercises what it claims: rows in range, ranged rows culled visible, moves, stamped and bypassed edits
    assert stats["in_range"] > 0 and stats["ranged_visible"] > 0
    assert stats["moved_in"] > 0 and stats["stamped"] > 0 and stats["bypassed"] > 0
