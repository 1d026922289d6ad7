"""No GPU needed: include/b200vis.h's b200vis_shadow_entities_sink, compiled as C11 with -Wall -Wextra -Werror, has the
size and field offsets abi.ShadowEntitiesSink declares, and the two new entry points are declared with the argument
types the Python signatures pass."""
import ctypes as C
import json
import os
import subprocess

from bevy_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r"""
#include <stddef.h>
#include <stdio.h>
#include "b200vis.h"
int main(void) {
    int32_t (*sink_fn)(b200vis_ctx *, const b200vis_shadow_entities_sink *) = b200vis_set_shadow_entities_sink;
    int32_t (*caster_fn)(b200vis_ctx *, uint32_t, const uint8_t *) = b200vis_set_table_shadow_casters;
    (void)sink_fn; (void)caster_fn;
    printf("{\"sizeof\": %zu, \"entities\": %zu, \"capacity\": %zu, \"max_items\": %zu, \"offsets\": %zu, \"active\": %zu}\n",
           sizeof(b200vis_shadow_entities_sink), offsetof(b200vis_shadow_entities_sink, entities),
           offsetof(b200vis_shadow_entities_sink, capacity), offsetof(b200vis_shadow_entities_sink, max_items),
           offsetof(b200vis_shadow_entities_sink, offsets), offsetof(b200vis_shadow_entities_sink, active));
    return 0;
}
"""


def test_shadow_entities_sink_layout_matches_ctypes(tmp_path):
    src, exe = tmp_path / "layout.c", str(tmp_path / "layout")
    src.write_text(SRC)
    cmd = ["gcc", "-O2", "-std=gnu11", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    lay = json.loads(subprocess.run([exe], capture_output=True, text=True, check=True).stdout)
    assert lay["sizeof"] == C.sizeof(abi.ShadowEntitiesSink)
    for name, _ in abi.ShadowEntitiesSink._fields_:
        assert lay[name] == getattr(abi.ShadowEntitiesSink, name).offset, name
    assert "b200vis_set_shadow_entities_sink" in abi.EXPORTED_SYMBOLS
    assert "b200vis_set_table_shadow_casters" in abi.EXPORTED_SYMBOLS
