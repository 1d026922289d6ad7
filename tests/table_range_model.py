"""What b200vis_read_tables(RD_CULL_INPUTS) must give each row's VisibilityRange parameters while
b200vis_set_table_visibility_ranges is attached, slot by slot, stated without any knowledge of the kernel.

A row's range state is what b200vis_upload_visibility_ranges gives it: (start_margin.start, end_margin.end) as two f32
and the use_aabb byte, taken as 0 or 1.  A table is read when it has a range column.  A slot of such a table is
considered when it is below len and mapped to a row.  It is read in full when its "fresh" mark is set (the slot was
(re)mapped, its table's range entry changed, or the ranges were attached after none, since the last cull read);
otherwise it is read only where its range tick is newer by Tick::is_newer_than (strict, with the MAX_CHANGE_AGE clamp).
The read clears the fresh marks of the slots below len.

`read` returns the state after the read.  With `mutant` set it follows one wrong rule instead, so that tests can show
that a scenario's inputs tell each wrong rule apart from the right one in the model's state.  That is a check of the
scenarios, not of the kernel: the device is held to the right rule by the GPU twins' comparisons of the masks, the
visible lists and the shadow lists against the oracle.  Each mutant here changes a row's parameters as
range_mask_of reads them (use_aabb only as a bool), so a kernel with that fault would show in those comparisons wherever
the distance test's outcome changes."""
import numpy as np

from table_read_model import UNMAPPED, is_newer

# VisibilityRange as bytes: the four floats of start_margin / end_margin and the use_aabb byte.  ABI layout =
# (stride, start_margin.start, end_margin.end, use_aabb).
STRUCTS = {
    "bevy": dict(stride=20, s0=0, s1=4, e0=8, e1=12, ua=16),      # the field order (abi.BEVY_VISIBILITY_RANGE_LAYOUT)
    "ua_first": dict(stride=20, ua=0, s0=4, s1=8, e0=12, e1=16),  # use_aabb before the floats
    "reversed": dict(stride=24, e0=0, e1=4, ua=8, s0=12, s1=16),  # end_margin first, use_aabb between, tail padding
}


def abi_layout(name):
    s = STRUCTS[name]
    return (s["stride"], s["s0"], s["e1"], s["ua"])


MUTANTS = (
    "end_margin_start",  # reads end_margin.start instead of end_margin.end
    "equal_tick_newer",  # a tick equal to last_run counts as newer
    "ignore_fresh",      # a fresh slot is read only by its tick
    "use_aabb_bit0",     # use_aabb taken as bit 0 of the byte, not as != 0
)


class RangeTable:
    """One registered table as the reader sees it.  ranges: uint8 [capacity, stride] or None (no VisibilityRange
    column); ticks: uint32 [capacity]; rows: the slot -> row map; fresh: bool [capacity], the "read in full" marks."""

    def __init__(self, length, capacity, rows, fresh, ranges=None, ticks=None):
        self.len, self.capacity = int(length), int(capacity)
        self.rows = np.asarray(rows, np.uint32)
        self.fresh = fresh
        self.ranges, self.ticks = ranges, ticks


def newer(ticks, last_run, this_run, mutant=None):
    right = is_newer(ticks, last_run, this_run)
    if mutant == "equal_tick_newer":
        return right | (np.asarray(ticks, np.uint64) == np.uint64(last_run & 0xFFFFFFFF))
    return right


def read(tables, struct, last_run, this_run, se, ua, mutant=None):
    """se [N, 2] uint32 (the f32 bits), ua [N] uint8: the device state before the read.  Returns (se, ua, fresh): the
    state after it, and each table's fresh marks after it (the inputs are not changed)."""
    st = STRUCTS[struct] if isinstance(struct, str) else struct
    se, ua = se.copy(), ua.copy()
    fresh_out = []
    for tb in tables:
        fresh = tb.fresh.copy()
        fresh_out.append(fresh)
        if tb.ranges is None or not tb.len:
            continue
        end = tb.len
        rows = tb.rows[:end]
        live = rows != UNMAPPED
        full = fresh[:end] & (mutant != "ignore_fresh")
        sel = live & (full | newer(tb.ticks[:end], last_run, this_run, mutant))
        b = tb.ranges[:end]
        eo = st["e0"] if mutant == "end_margin_start" else st["e1"]
        vals = np.stack([np.ascontiguousarray(b[:, st["s0"]:st["s0"] + 4]).view(np.uint32)[:, 0],
                         np.ascontiguousarray(b[:, eo:eo + 4]).view(np.uint32)[:, 0]], 1)
        byte = b[:, st["ua"]]
        se[rows[sel]] = vals[sel]
        ua[rows[sel]] = (byte[sel] & 1 if mutant == "use_aabb_bit0" else byte[sel] != 0).astype(np.uint8)
        fresh[:end] = False
    return se, ua, fresh_out


def same(a, b):
    """Two read results leave the same device state."""
    return (a[0] == b[0]).all() and (a[1] == b[1]).all()


def put(col, struct, slots, start, end, use_aabb, margins=None):
    """Write VisibilityRange values into the slots' bytes.  margins: [k, 2] (start_margin.end, end_margin.start); by
    default the midpoint of start and end, so that a wrong float read shows."""
    st = STRUCTS[struct] if isinstance(struct, str) else struct
    slots = np.asarray(slots, np.int64)
    start, end = np.asarray(start, np.float32).reshape(-1), np.asarray(end, np.float32).reshape(-1)
    if margins is None:
        mid = ((start + end) * np.float32(0.5)).astype(np.float32)
        margins = np.stack([mid, mid], 1)
    margins = np.asarray(margins, np.float32).reshape(-1, 2)
    for key, v in (("s0", start), ("s1", margins[:, 0]), ("e0", margins[:, 1]), ("e1", end)):
        col[slots, st[key]:st[key] + 4] = np.ascontiguousarray(v, np.float32).reshape(-1, 1).view(np.uint8)
    col[slots, st["ua"]] = np.asarray(use_aabb, np.uint8)


def game(tables, struct, rng, L, R, n_edits=8, past_len=True):
    """The other systems between two cull runs.  Every slot's VisibilityRange bytes are overwritten with values that
    would change the masks, with ticks at or before L (bypass_change_detection; some exactly at L); then n_edits live
    slots get new values with ticks in (L, R].  Slots at and past len get newer ticks (never read).  Returns the stamped
    (table, slot) pairs."""
    stamped = []
    for tb in tables:
        if tb.ranges is None or not tb.capacity:
            continue
        cap = tb.capacity
        s = rng.uniform(0, 400, cap).astype(np.float32)
        put(tb.ranges, struct, np.arange(cap), s, s + rng.uniform(0, 5, cap).astype(np.float32), rng.integers(0, 256, cap))
        tb.ticks[:] = ((L - rng.integers(0, 40, cap)) & 0xFFFFFFFF).astype(np.uint32)
        tb.ticks[rng.random(cap) < 0.25] = L & 0xFFFFFFFF
        if past_len and tb.len < cap:
            tb.ticks[tb.len:] = (R - 1) & 0xFFFFFFFF
    live = [(t, s) for t, tb in enumerate(tables) if tb.ranges is not None for s in np.nonzero(tb.rows[:tb.len] != UNMAPPED)[0]]
    for k in (rng.choice(len(live), size=min(n_edits, len(live)), replace=False) if live else []):
        t, s = live[k]
        a = np.float32(rng.uniform(0, 60))
        put(tables[t].ranges, struct, [s], [a], [a + np.float32(rng.uniform(10, 150))], [rng.choice([0, 1, 2, 255])])
        tables[t].ticks[s] = (R - int(rng.integers(0, min((R - L) & 0xFFFFFFFF, 16)))) & 0xFFFFFFFF
        stamped.append((t, int(s)))
    return stamped
