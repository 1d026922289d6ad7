"""A frame with no per-entity host work in either direction, in plain C: tests/table_io_shim.c keeps Bevy-native archetype
tables (Transform with rotation first, GlobalTransform, ViewVisibility and their changed_ticks), has the GPU read the
changed Transforms and other systems' GlobalTransforms from them and write the results back, and checks every frame
against the CPU oracle."""
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
           os.path.join(ROOT, "tests", "table_io_shim.c"), "-o", out,
           "-L" + os.path.join(ROOT, "bevy_b200"), "-lb200vis", "-L" + os.path.join(ROOT, "oracle"), "-lbevy_oracle", "-lm",
           "-Wl,-rpath," + os.path.join(ROOT, "bevy_b200"), "-Wl,-rpath," + os.path.join(ROOT, "oracle")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr


def test_input_struct_layouts_match_ctypes(tmp_path):
    """No GPU needed: the shim compiles as C11 with -Wall -Wextra -Werror, links against libb200vis.so, and the C layouts
    of b200vis_transform_layout and b200vis_table_inputs are the ones abi declares."""
    exe = str(tmp_path / "table_io_shim")
    build_shim(exe)
    res = subprocess.run([exe, "--sizeof"], capture_output=True, text=True, timeout=60)
    assert res.returncode == 0, res.stderr
    lay = json.loads(res.stdout)
    for key, struct in (("layout", abi.TransformLayout), ("inputs", abi.TableInputs)):
        assert lay[key]["sizeof"] == C.sizeof(struct), key
        for name, _ in struct._fields_:
            assert lay[key][name] == getattr(struct, name).offset, (key, name)


@pytest.mark.gpu
def test_table_io_shim_matches_the_oracle(tmp_path):
    exe = str(tmp_path / "table_io_shim")
    build_shim(exe)
    res = subprocess.run([exe, "200", "6", "5"], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and "TABLE_IO_SHIM OK" in res.stdout, res.stdout[-2000:] + res.stderr[-2000:]
    assert "5: 200 Transforms" in res.stdout
