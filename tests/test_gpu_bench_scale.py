"""Parity at the sizes the headline numbers are quoted on (BASELINE.json configs #3, #4 and one rank's share of #5), once per
tile-kernel variant.  The variant switches (B200VIS_TILE_KERNEL, B200VIS_TILES_PER_CTA, ...) are read once per process, so
every case runs in its own interpreter.  Same bit-exact comparison against the CPU oracle as the small tests
(tests/parity.py): GlobalTransform bits, both change-flag columns, ViewVisibility bytes, sorted visible lists, cluster
offsets / indices / farthest_z / index counts, over several animated frames with the cluster feedback loop closed."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

VARIANTS = {
    "default": {},                                                                  # kernel 1b: TMA-staged tiles, 4 persistent CTAs per SM
    "lean": {"B200VIS_TILE_KERNEL": "lean"},                                        # kernel 1L: 1b on an instruction diet
    "default_serial": {"B200VIS_PIPELINE": "0"},
    "lean_top_through_loop": {"B200VIS_TILE_KERNEL": "lean", "B200VIS_LEAN_PROBE": "4"},                           # A/B switch: top levels through the level loop instead of registers
    "lean_sphere_reject": {"B200VIS_TILE_KERNEL": "lean", "B200VIS_LEAN_PROBE": "8"},                              # A/B switch: sphere instead of box in the warp-level view rejection
    "lean_pipe": {"B200VIS_TILE_KERNEL": "lean", "B200VIS_LEAN_PIPE": "1"},                                        # the CTA's warps drift up to a tile apart (no closing barrier)
    "lean_5ctas": {"B200VIS_TILE_KERNEL": "lean", "B200VIS_LEAN_CTAS": "5"},                                       # Transform out of the staged window, 48 registers
    "lean_6ctas": {"B200VIS_TILE_KERNEL": "lean", "B200VIS_LEAN_CTAS": "6"},
    "lean_static_handout": {"B200VIS_TILE_KERNEL": "lean", "B200VIS_TILE_HANDOUT": "static"},
    "lean_2_tiles": {"B200VIS_TILE_KERNEL": "lean", "B200VIS_TILES_PER_CTA": "2"},
    "tma": {"B200VIS_TILE_KERNEL": "tma"},                                          # kernel 1b selected explicitly
    "scout": {"B200VIS_TILE_KERNEL": "scout"},                                      # TMA-staged tiles + a scout warp one tile ahead
    "scout_2ctas": {"B200VIS_TILE_KERNEL": "scout", "B200VIS_SCOUT_CTAS_PER_SM": "2"},
    "scout_2_tiles": {"B200VIS_TILE_KERNEL": "scout", "B200VIS_SCOUT_TILES_PER_CTA": "2"},
    "warp": {"B200VIS_TILE_KERNEL": "warp", "B200VIS_WARP_VARIANT": "2p"},          # one warp per tile
    "warp_dynamic": {"B200VIS_TILE_KERNEL": "warp", "B200VIS_WARP_DYNAMIC": "1", "B200VIS_WARP_VARIANT": "4n"},
    "tma_2_tiles": {"B200VIS_TILE_KERNEL": "tma", "B200VIS_TILES_PER_CTA": "2"},
    "tma_4_tiles": {"B200VIS_TILE_KERNEL": "tma", "B200VIS_TILES_PER_CTA": "4"},
    "classic": {"B200VIS_TILE_KERNEL": "classic"},
    "flow": {"B200VIS_TILE_KERNEL": "flow"},                                        # no CTA barrier between tiles, named level barriers
    "flow_cta_levels": {"B200VIS_TILE_KERNEL": "flow", "B200VIS_LEVEL_SYNC": "cta"},
}


def run_case(code, env, timeout=240):
    e = dict(os.environ)
    for k in [k for k in e if k.startswith("B200VIS_")]:
        del e[k]
    e.update(env)
    prog = (f"import sys; sys.path.insert(0, {ROOT!r}); sys.path.insert(0, {HERE!r})\n"
            "from bevy_b200 import scenes\nfrom parity import run_parity\n" + code)
    res = subprocess.run([sys.executable, "-c", prog], env=e, capture_output=True, text=True, timeout=timeout)
    assert res.returncode == 0, f"{env}\n{res.stdout[-2000:]}\n{res.stderr[-4000:]}"


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_config3_bench_workload_1m_entities_256_lights_4_views(variant):
    # bench.py's workload: 3922 complete binary trees x 255 nodes (BFS) + 256 point lights, 4 views, every root moves
    run_case("run_parity(scenes.forest(3922, 8, 256), frames=3)", VARIANTS[variant])


@pytest.mark.parametrize("variant", ["default", "lean", "lean_pipe", "tma", "scout", "warp", "tma_2_tiles", "flow"])
def test_config3_static_frames_and_static_optimizations_off(variant):
    run_case("run_parity(scenes.forest(3922, 8, 256), frames=3, animate=False)\n"
             "run_parity(scenes.forest(1500, 8, 64, seed=5), frames=3, static_opt=False)", VARIANTS[variant])


@pytest.mark.parametrize("variant", ["default", "lean", "lean_pipe", "tma", "scout", "warp"])
def test_config4_many_lights_100k_meshes_1024_lights(variant):
    # 1024 lights = 32 mask words per cluster; range 0.3 as in many_lights.rs:48-86, and a wider range for denser clusters
    run_case("run_parity(scenes.many_cubes(100_000, n_lights=1024, light_range=(0.3, 0.3)), frames=3)\n"
             "run_parity(scenes.many_cubes(100_000, n_lights=1024, light_range=(0.3, 12.0), seed=3), frames=3)", VARIANTS[variant])


@pytest.mark.parametrize("variant", ["default", "lean", "lean_pipe", "tma", "scout"])
def test_config5_one_ranks_share_1_25m_rows_512_lights(variant):
    # config #5 on 8 GPUs: 39,220 trees / 8 = 4,903 trees (1,250,265 rows) + 4096 / 8 = 512 lights per rank
    run_case("run_parity(scenes.forest(4903, 8, 512, seed=11), frames=2)", VARIANTS[variant])
