"""No GPU needed: include/b200vis.h's b200vis_view_diff_sink, compiled as C11 with -Wall -Wextra -Werror, has the size and
field offsets abi.ViewDiffSink declares, the two new entry points are declared with the argument types the Python
signatures pass, B200VIS_VIEW_NO_SLOT is abi.VIEW_NO_SLOT, and the built library exports both symbols."""
import ctypes as C
import json
import os
import subprocess

import pytest

from bevy_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r"""
#include <stddef.h>
#include <stdio.h>
#include "b200vis.h"
#define OFF(f) offsetof(b200vis_view_diff_sink, f)
int main(void) {
    int32_t (*sink_fn)(b200vis_ctx *, const b200vis_view_diff_sink *) = b200vis_set_view_diff_sink;
    int32_t (*slots_fn)(b200vis_ctx *, uint32_t, const uint32_t *) = b200vis_set_view_diff_slots;
    (void)sink_fn; (void)slots_fn;
    printf("{\"sizeof\": %zu, \"added\": %zu, \"added_capacity\": %zu, \"removed\": %zu, \"removed_capacity\": %zu, "
           "\"added_offsets\": %zu, \"removed_offsets\": %zu, \"max_slots\": %zu, \"no_slot\": %u}\n",
           sizeof(b200vis_view_diff_sink), OFF(added), OFF(added_capacity), OFF(removed), OFF(removed_capacity),
           OFF(added_offsets), OFF(removed_offsets), OFF(max_slots), (unsigned)B200VIS_VIEW_NO_SLOT);
    return 0;
}
"""


def test_view_diff_sink_layout_matches_ctypes(tmp_path):
    src, exe = tmp_path / "layout.c", str(tmp_path / "layout")
    src.write_text(SRC)
    cmd = ["gcc", "-O2", "-std=c11", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    lay = json.loads(subprocess.run([exe], capture_output=True, text=True, check=True).stdout)
    assert lay["sizeof"] == C.sizeof(abi.ViewDiffSink)
    for name, _ in abi.ViewDiffSink._fields_:
        assert lay[name] == getattr(abi.ViewDiffSink, name).offset, name
    assert lay["no_slot"] == abi.VIEW_NO_SLOT


def test_view_diff_symbols_are_exported():
    for name in ("b200vis_set_view_diff_sink", "b200vis_set_view_diff_slots"):
        assert name in abi.EXPORTED_SYMBOLS
    lib = os.path.join(ROOT, "bevy_b200", "libb200vis.so")
    if not os.path.exists(lib):
        pytest.skip("libb200vis.so is not built")
    syms = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True, check=True).stdout.split()
    assert "b200vis_set_view_diff_sink" in syms and "b200vis_set_view_diff_slots" in syms
