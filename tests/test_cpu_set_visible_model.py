"""The numpy model of the CPU-owned ViewVisibility that the B200VIS_WB_SET_VISIBLE table write-back is checked against
(tests/set_visible_model.py) reproduces the reference's view_visibility_lifecycle, and mutants of it do not."""
import numpy as np
import pytest

import set_visible_model as m


def test_the_model_reproduces_view_visibility_lifecycle():
    assert m.run_lifecycle() == [(b, ch) for _, b, ch in m.LIFECYCLE]


def _tick_when_visible_last_frame(vv, ticks, slots, tick):
    slots = np.asarray(slots, np.int64)
    b = vv[slots]
    need = (b & 1) == 0
    vv[slots[need]] = b[need] | 1
    ticks[slots[need][(b[need] & 2) != 0]] = tick


def _write_without_reading(vv, ticks, slots, tick):
    slots = np.asarray(slots, np.int64)
    vv[slots] = 1                                   # the byte inferred from the device state
    ticks[slots] = tick


def _tick_on_every_call(vv, ticks, slots, tick):
    slots = np.asarray(slots, np.int64)
    b = vv[slots]
    vv[slots] = b | 1
    ticks[slots[(b & 2) == 0]] = tick


@pytest.mark.parametrize("mutant", [_tick_when_visible_last_frame, _write_without_reading])
def test_mutants_of_set_visible_fail_the_lifecycle(mutant):
    assert m.run_lifecycle(mutant) != [(b, ch) for _, b, ch in m.LIFECYCLE]


def test_a_slot_another_system_already_set_is_not_ticked_again():
    """set_visible() twice in one frame (another CheckVisibility system first): one write, one tick."""
    vv = np.array([0b00, 0b10, 0b00, 0b10], np.uint8)   # after reset: hidden / visible last frame
    ticks = np.zeros(4, np.uint32)
    m.set_visible(vv, ticks, [0, 1], 5)                # the other system
    m.set_visible(vv, ticks, [0, 1, 2, 3], 6)          # the cull
    assert vv.tolist() == [0b01, 0b11, 0b01, 0b11]
    assert ticks.tolist() == [5, 0, 6, 0]
    # a mutant that does not read the byte stamps the second call's tick over the first
    vv2, t2 = np.array([0b00, 0b10, 0b00, 0b10], np.uint8), np.zeros(4, np.uint32)
    _tick_on_every_call(vv2, t2, [0, 1], 5)
    _tick_on_every_call(vv2, t2, [0, 1, 2, 3], 6)
    assert t2.tolist() != ticks.tolist()
