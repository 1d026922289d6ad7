"""No GPU needed: include/b200vis.h declares b200vis_emit_shadow_entities with the argument types the Python signature
passes (compiled as C11 with -Wall -Wextra -Werror), and the built library exports it."""
import os
import subprocess

from bevy_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r"""
#include "b200vis.h"
int main(void) {
    int32_t (*emit_fn)(b200vis_ctx *) = b200vis_emit_shadow_entities;
    return emit_fn == 0;
}
"""


def test_emit_shadow_entities_is_declared_and_exported(tmp_path):
    src = tmp_path / "decl.c"
    src.write_text(SRC)
    cmd = ["gcc", "-std=gnu11", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(src)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    assert "b200vis_emit_shadow_entities" in abi.EXPORTED_SYMBOLS
    assert hasattr(abi.load_library(), "b200vis_emit_shadow_entities")
    assert hasattr(abi.Context, "emit_shadow_entities")
