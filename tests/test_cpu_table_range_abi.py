"""No GPU needed: include/b200vis.h's b200vis_visibility_range_layout and b200vis_table_visibility_ranges, compiled as C11
with -Wall -Wextra -Werror, have the sizes and field offsets abi.py declares, and b200vis_set_table_visibility_ranges is
declared with the argument types the Python signature passes."""
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
    int32_t (*fn)(b200vis_ctx *, uint32_t, const b200vis_table_visibility_ranges *, const b200vis_visibility_range_layout *) =
        b200vis_set_table_visibility_ranges;
    (void)fn;
    printf("{\"layout\": {\"sizeof\": %zu, \"stride\": %zu, \"start\": %zu, \"end\": %zu, \"use_aabb\": %zu}, "
           "\"table\": {\"sizeof\": %zu, \"ranges\": %zu, \"changed_ticks\": %zu}}\n",
           sizeof(b200vis_visibility_range_layout), offsetof(b200vis_visibility_range_layout, stride),
           offsetof(b200vis_visibility_range_layout, start), offsetof(b200vis_visibility_range_layout, end),
           offsetof(b200vis_visibility_range_layout, use_aabb), sizeof(b200vis_table_visibility_ranges),
           offsetof(b200vis_table_visibility_ranges, ranges), offsetof(b200vis_table_visibility_ranges, changed_ticks));
    return 0;
}
"""


def test_visibility_range_structs_match_ctypes(tmp_path):
    src, exe = tmp_path / "layout.c", str(tmp_path / "layout")
    src.write_text(SRC)
    cmd = ["gcc", "-O2", "-std=c11", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    lay = json.loads(subprocess.run([exe], capture_output=True, text=True, check=True).stdout)
    for key, cls in (("layout", abi.VisibilityRangeLayout), ("table", abi.TableVisibilityRanges)):
        assert lay[key]["sizeof"] == C.sizeof(cls), key
        for name, _ in cls._fields_:
            assert lay[key][name] == getattr(cls, name).offset, (key, name)


def test_signature_and_layout_guess():
    res, args = abi._SIGNATURES["b200vis_set_table_visibility_ranges"]
    assert res is C.c_int32
    assert args[1] is C.c_uint32 and args[3] is C.POINTER(abi.VisibilityRangeLayout)
    assert "b200vis_set_table_visibility_ranges" in abi.EXPORTED_SYMBOLS
    # the guess is a valid layout: 4-byte floats inside the stride, the bool byte apart from both
    stride, start, end, ua = abi.BEVY_VISIBILITY_RANGE_LAYOUT
    assert stride % 4 == 0 and start % 4 == 0 and end % 4 == 0
    assert max(start, end) + 4 <= stride and ua < stride
    assert abs(start - end) >= 4 and not start <= ua < start + 4 and not end <= ua < end + 4
