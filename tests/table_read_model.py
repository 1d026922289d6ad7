"""What b200vis_read_tables must read, slot by slot, stated without any knowledge of the kernel.

A table is read at slot s when s < len, the slot maps to a row, and the slot's tick is newer than the reading system's
last run by Bevy's Tick::is_newer_than (crates/bevy_ecs/src/change_detection/tick.rs): both ages are wrapping u32
differences from this_run, each clamped to MAX_CHANGE_AGE, and the comparison is strict.
- RD_TRANSFORM reads the table's Transform column at the layout's byte offsets: the row gets the packed 10 floats of
  b200vis_upload_transforms_scattered (translation.xyz, rotation.xyzw, scale.xyz) as bits, and Changed<Transform>.
- RD_GLOBAL_TRANSFORM reads the table's global_transforms column where it has gt_changed_ticks: the row gets lanes 0-2 of
  the four Vec3A (x_axis, y_axis, z_axis, translation), the 12 floats of b200vis_write_global_transforms_scattered.

`read` returns those two sets.  With `mutant` set it follows one wrong rule instead, so that tests can show that some
scenario tells each wrong rule apart from the right one."""
import numpy as np

CHECK_TICK_THRESHOLD = 518_400_000
MAX_CHANGE_AGE = 0xFFFFFFFF - (2 * CHECK_TICK_THRESHOLD - 1)
UNMAPPED = 0xFFFFFFFF
RD_TRANSFORM, RD_GLOBAL_TRANSFORM = 0x1, 0x2

MUTANTS = (
    "plain_compare",     # tick > last_run, no wrapping arithmetic
    "no_clamp",          # the ages are not clamped to MAX_CHANGE_AGE
    "ge",                # >= for >: a tick equal to last_run counts as newer
    "capacity",          # slots up to capacity are read instead of up to len
    "unmapped",          # an unmapped slot is read into the row it held before it was unmapped
    "packed_layout",     # the layout's offsets ignored: translation @ 0, rotation @ 12, scale @ 28
    "gt_without_ticks",  # a table with global_transforms but no gt_changed_ticks is read in full
)


def is_newer(tick, last_run, this_run, mutant=None):
    """Tick::is_newer_than on u32 values (scalars or arrays)."""
    tick, last_run, this_run = (np.asarray(x, np.uint64) for x in (tick, last_run, this_run))
    if mutant == "plain_compare":
        return tick > last_run
    m = np.uint64(0xFFFFFFFF)
    since_insert = (this_run - tick) & m
    since_system = (this_run - last_run) & m
    if mutant != "no_clamp":
        since_insert = np.minimum(since_insert, MAX_CHANGE_AGE)
        since_system = np.minimum(since_system, MAX_CHANGE_AGE)
    return since_system >= since_insert if mutant == "ge" else since_system > since_insert


class ModelTable:
    """One registered table as the reader sees it.  trs: uint8 [capacity, stride] or None; trs_ticks: uint32 [capacity]
    or None; gt: float32 [capacity, 16] or None; gt_ticks: uint32 [capacity] or None; rows: the slot -> row map
    (UNMAPPED = unmapped); held: the row each slot held before it was last unmapped (for the "unmapped" mutant)."""

    def __init__(self, length, capacity, rows, trs=None, trs_ticks=None, gt=None, gt_ticks=None, held=None):
        self.len, self.capacity = int(length), int(capacity)
        self.rows = np.asarray(rows, np.uint32)
        self.held = self.rows if held is None else np.asarray(held, np.uint32)
        self.trs, self.trs_ticks, self.gt, self.gt_ticks = trs, trs_ticks, gt, gt_ticks


def transform_bits(trs_bytes, layout, mutant=None):
    """[k, stride] bytes -> [k, 10] uint32: translation.xyz, rotation.xyzw, scale.xyz at the layout's offsets."""
    _, t, r, s = (12, 0, 12, 28) if mutant == "packed_layout" else layout
    b = np.ascontiguousarray(trs_bytes, np.uint8)
    parts = [np.ascontiguousarray(b[:, o:o + 4 * k]).view(np.uint32) for o, k in ((t, 3), (r, 4), (s, 3))]
    return np.concatenate(parts, axis=1)


def gt_bits(affine16):
    """[k, 16] float32 Affine3A -> [k, 12] uint32: lanes 0-2 of x_axis, y_axis, z_axis, translation."""
    a = np.ascontiguousarray(affine16, np.float32).view(np.uint32).reshape(-1, 4, 4)
    return a[:, :, :3].reshape(-1, 12)


def read(tables, layout, which, last_run, this_run, mutant=None):
    """Returns ({row: [10] uint32}, {row: [12] uint32}): what RD_TRANSFORM and RD_GLOBAL_TRANSFORM give each row."""
    trs_out, gt_out = {}, {}
    for tb in tables:
        end = tb.capacity if mutant == "capacity" else tb.len
        slots = np.arange(end)
        rows = tb.rows[:end].copy()
        if mutant == "unmapped":
            rows = np.where(rows == UNMAPPED, tb.held[:end], rows)
        live = rows != UNMAPPED
        if which & RD_TRANSFORM and tb.trs is not None and end:
            sel = live & is_newer(tb.trs_ticks[:end], last_run, this_run, mutant)
            for s, v in zip(slots[sel], transform_bits(tb.trs[slots[sel]], layout, mutant)):
                trs_out[int(rows[s])] = v
        if which & RD_GLOBAL_TRANSFORM and tb.gt is not None and end:
            if tb.gt_ticks is not None:
                sel = live & is_newer(tb.gt_ticks[:end], last_run, this_run, mutant)
            elif mutant == "gt_without_ticks":
                sel = live
            else:
                continue
            for s, v in zip(slots[sel], gt_bits(tb.gt[slots[sel]])):
                gt_out[int(rows[s])] = v
    return trs_out, gt_out


def as_uploads(trs_out, gt_out):
    """The two sets as the scattered uploads take them: (rows, trs [k, 10] float32), (rows, gt [k, 12] float32)."""
    def pack(d, width):
        rows = np.array(sorted(d), np.uint32)
        vals = np.array([d[int(r)] for r in rows], np.uint32).reshape(-1, width).view(np.float32)
        return rows, vals
    return pack(trs_out, 10), pack(gt_out, 12)


def same(a, b):
    """Two read results are the same sets with the same bits."""
    return all(x.keys() == y.keys() and all((x[k] == y[k]).all() for k in x) for x, y in zip(a, b))
