"""A numpy model of ViewVisibility as the CPU owns it (a build whose ViewVisibility column the device does not own):
reset_view_visibility, SetViewVisibility::set_visible and mark_newly_hidden_entities_invisible
(crates/bevy_camera/src/visibility/mod.rs:226-306, 733-737, 908-919), each over a byte column and its changed_ticks
column.  A tick is stamped exactly where the reference's Mut<ViewVisibility> would mark the component changed."""
import numpy as np


def reset(vv):
    """reset_view_visibility: bit 0 moves to bit 1 through bypass_change_detection (no tick)."""
    vv[:] = (vv & 1) << 1


def set_visible(vv, ticks, slots, tick):
    """set_visible() on every slot of `slots`: only a byte without bit 0 is written; the tick is stamped only when bit 1
    was clear too (hidden last frame -> visible now)."""
    slots = np.asarray(slots, np.int64)
    b = vv[slots]
    need = (b & 1) == 0
    s = slots[need]
    vv[s] = b[need] | 1
    if ticks is not None:
        ticks[s[(b[need] & 2) == 0]] = tick


def mark_hidden(vv, ticks, tick):
    """mark_newly_hidden_entities_invisible: visible last frame, not now -> HIDDEN through DerefMut (ticked)."""
    sel = (vv & 3) == 2
    vv[sel] = 0
    if ticks is not None:
        ticks[sel] = tick


def frame(vv, ticks, visible_slots, tick, set_visible_fn=set_visible):
    """One CheckVisibility pass: reset, set_visible over the visible slots, mark the newly hidden ones."""
    reset(vv)
    set_visible_fn(vv, ticks, visible_slots, tick)
    mark_hidden(vv, ticks, tick)


# view_visibility_lifecycle (visibility/mod.rs:1314-1448): one entity spawned HIDDEN, then frames 1-5 with the manual
# set_visible() on or off.  Per frame: (set_visible called, ViewVisibility byte after the frame, Changed<ViewVisibility>
# observed after MarkNewlyHiddenEntitiesInvisible).  The assertions there check bit 0 and the Changed flag; the bytes
# follow from reset / set_visible / mark_newly_hidden.
LIFECYCLE = (
    (False, 0b00, False),   # frame 1: do nothing
    (True, 0b01, True),     # frame 2: set visible
    (True, 0b11, False),    # frame 3: still visible
    (False, 0b00, True),    # frame 4: becomes hidden
    (False, 0b00, False),   # frame 5: do nothing
)


def run_lifecycle(set_visible_fn=set_visible):
    """[(byte, changed)] over LIFECYCLE's frames; ticks are the frame numbers (the spawn frame's tick is 0)."""
    vv = np.zeros(1, np.uint8)
    ticks = np.zeros(1, np.uint32)
    out = []
    for f, (mark, _, _) in enumerate(LIFECYCLE, start=1):
        frame(vv, ticks, [0] if mark else [], f, set_visible_fn)
        out.append((int(vv[0]), bool(ticks[0] == f)))
    return out
