"""The plugin's light-visibility frame without Rust: tests/light_shim.c keeps Bevy-native archetype tables (casters and
non-casters, NoFrustumCulling, VisibilityRange, a ShadowLodOrigin among the range views), runs the cull and then the
light step of b200_check_light_visibility through the C ABI -- items, set_shadow_items, run_shadow_culling, the second
WB_SET_VISIBLE, sink growth and b200vis_emit_shadow_entities, the component fills and the CascadesVisibleEntities
bookkeeping -- and checks every list, every ViewVisibility byte and its change tick against the CPU oracle every frame."""
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
           os.path.join(ROOT, "tests", "light_shim.c"), "-o", out,
           "-L" + os.path.join(ROOT, "bevy_b200"), "-lb200vis", "-L" + os.path.join(ROOT, "oracle"), "-lbevy_oracle", "-lm",
           "-Wl,-rpath," + os.path.join(ROOT, "bevy_b200"), "-Wl,-rpath," + os.path.join(ROOT, "oracle")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr


def test_light_layouts(tmp_path):
    """No GPU needed: the shim compiles as C11 with -Wall -Wextra -Werror, links against libb200vis.so, and
    b200vis_shadow_item and b200vis_shadow_entities_sink have the layouts abi declares."""
    exe = str(tmp_path / "light_shim")
    build_shim(exe)
    res = subprocess.run([exe, "--sizeof"], capture_output=True, text=True, timeout=60)
    assert res.returncode == 0, res.stderr
    lay = json.loads(res.stdout)
    for key, struct in (("shadow_item", abi.ShadowItem), ("shadow_entities_sink", abi.ShadowEntitiesSink)):
        assert lay[key]["sizeof"] == C.sizeof(struct), key
        for name, _ in struct._fields_:
            assert lay[key][name] == getattr(struct, name).offset, (key, name)


def run_shim(tmp_path, args, timeout):
    exe = str(tmp_path / "light_shim")
    build_shim(exe)
    res = subprocess.run([exe] + [str(a) for a in args], capture_output=True, text=True, timeout=timeout)
    assert res.returncode == 0 and "LIGHT_SHIM OK" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]
    print(res.stdout)
    return json.loads([line for line in res.stdout.splitlines() if line.startswith("{")][-1])


@pytest.mark.gpu
def test_light_shim_small_world_matches_the_oracle(tmp_path):
    stats = run_shim(tmp_path, [60, 6, 6, 6, 4], 600)
    # the scenario reaches what it claims: the sink grew through the emit, an inactive light kept its lists
    assert stats["grown"] >= 2 and stats["inactive_kept"] > 0 and stats["entries"] > 0


@pytest.mark.gpu
def test_light_shim_bench_world_matches_the_oracle(tmp_path):
    """3922 trees of 255, 16 point lights, 8 spot lights, one directional light x 2 views x 4 cascades."""
    stats = run_shim(tmp_path, [3922, 8, 3, 16, 8], 900)
    assert stats["entities"] == 3922 * 255 + 24 and stats["grown"] >= 1
