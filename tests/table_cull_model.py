"""What b200vis_read_tables(RD_CULL_INPUTS) must give each row, slot by slot, stated without any knowledge of the kernel.

The device state of a row is the one b200vis_upload_bounds gives it: six bounds floats and a flag byte (plus F_TCHANGED,
0x80, which the propagate owns).  A table is read when its entry of b200vis_set_table_cull_inputs has a column or flags.
A slot of a read table is considered when it is below len and mapped to a row.  It is read in full when its "fresh" mark
is set (the slot was (re)mapped, or its table (re)attached, since the last cull read); otherwise each column is read only
where its tick is newer by Tick::is_newer_than (tests/table_read_model.py).
- Full read: flags = the table's flags | HAS_AABB (the table has Aabb) or HAS_SPHERE (Sphere and no Aabb) |
  INHERITED_VISIBLE (the byte is nonzero), the row's F_TCHANGED kept; bounds from the Aabb or else the Sphere column.
- Aabb (newer tick): bounds = center.xyz, half_extents.xyz.  Sphere (table without Aabb, newer tick): center.xyz,
  radius, 0, 0.  InheritedVisibility (newer tick): bit 0 of the flags only.
- The read clears the fresh marks of the slots below len of every read table.

`read` returns the state after the read.  With `mutant` set it follows one wrong rule instead, so that tests can show
that some scenario tells each wrong rule apart from the right one.  `game` is the "other systems" of a frame, shared by
the CPU and GPU tests: it overwrites every column without a tick (bypass writes that would flip visibility if read) and
stamps a few slots with newer ticks."""
import numpy as np

from table_read_model import UNMAPPED, is_newer

F_INHERITED, F_AABB, F_SPHERE, F_NO_FRUSTUM = 0x01, 0x02, 0x04, 0x08
F_RANGE, F_NO_CPU, F_SPHERE_FROM_GT, F_TCHANGED = 0x10, 0x20, 0x40, 0x80
BEVY_LAYOUT = (32, 0, 16, 32, 0, 16)
PERMUTED_LAYOUT = (48, 28, 8, 40, 20, 4)    # half_extents before center; radius before center
PACKED_LAYOUT = (24, 0, 12, 16, 0, 12)

MUTANTS = (
    "fresh_by_ticks",    # a fresh slot is read only by its ticks
    "sphere_over_aabb",  # a table with both takes the Sphere
    "capacity",          # slots up to capacity are considered instead of up to len
    "unmapped",          # an unmapped slot is read into the row it held before it was unmapped
    "packed_layout",     # the layout's offsets ignored: fields back to back from 0
    "drop_tchanged",     # a full read clears the row's F_TCHANGED
    "iv_by_aabb_tick",   # InheritedVisibility is read where the Aabb tick is newer
)

# the archetype tables of the GPU scenarios: which columns each has, and its per-archetype flags
ARCHETYPES = (
    dict(has=("aabb", "iv"), flags=0),
    dict(has=("aabb", "iv"), flags=F_NO_FRUSTUM),
    dict(has=("sphere", "iv"), flags=0),
    dict(has=("aabb", "sphere", "iv"), flags=F_RANGE),
    dict(has=("aabb",), flags=F_NO_CPU),
    dict(has=("sphere", "iv"), flags=F_SPHERE_FROM_GT),
    dict(has=("iv",), flags=0),                      # Visibility without bounds (a camera, a plain parent): bounds kept
    dict(has=(), flags=F_NO_CPU),                     # outside the visibility query: flags only
)


class CullTable:
    """One registered table as the reader sees it.  aabb / sphere: uint8 [capacity, stride] or None; iv: uint8
    [capacity] or None; *_ticks: uint32 [capacity]; rows: the slot -> row map; held: the row each slot held before it
    was last unmapped (for the "unmapped" mutant); fresh: bool [capacity], the "read in full" marks."""

    def __init__(self, length, capacity, rows, fresh, aabb=None, aabb_ticks=None, sphere=None, sphere_ticks=None,
                 iv=None, iv_ticks=None, flags=0, held=None):
        self.len, self.capacity = int(length), int(capacity)
        self.rows = np.asarray(rows, np.uint32)
        self.held = self.rows if held is None else np.asarray(held, np.uint32)
        self.fresh = fresh
        self.aabb, self.aabb_ticks, self.sphere, self.sphere_ticks = aabb, aabb_ticks, sphere, sphere_ticks
        self.iv, self.iv_ticks, self.flags = iv, iv_ticks, int(flags)

    @property
    def read(self):
        return self.aabb is not None or self.sphere is not None or self.iv is not None or self.flags != 0


def floats(col, slots, fields):
    """[k, sum(n)] uint32 bits of the f32 fields (offset, n) of the slots' bytes."""
    b = np.ascontiguousarray(col[slots], np.uint8)
    return np.concatenate([np.ascontiguousarray(b[:, o:o + 4 * n]).view(np.uint32) for o, n in fields], axis=1)


def bounds_bits(tb, slots, layout, mutant=None):
    """(kind, [k, 6] uint32): the bounds upload_bounds takes for the slots, from the Aabb or else the Sphere column."""
    lay = PACKED_LAYOUT if mutant == "packed_layout" else layout
    if tb.aabb is not None and not (mutant == "sphere_over_aabb" and tb.sphere is not None):
        return "aabb", floats(tb.aabb, slots, ((lay[1], 3), (lay[2], 3)))
    if tb.sphere is not None:
        v = floats(tb.sphere, slots, ((lay[4], 3), (lay[5], 1)))
        return "sphere", np.concatenate([v, np.zeros((len(v), 2), np.uint32)], axis=1)
    return None, None


def read(tables, layout, last_run, this_run, bounds, flags, mutant=None):
    """bounds [N, 6] uint32, flags [N] uint8: the device state before the read.  Returns (bounds, flags, fresh): the state
    after it, and each table's fresh marks after it (the inputs are not changed)."""
    bounds, flags = bounds.copy(), flags.copy()
    fresh_out = []
    for tb in tables:
        fresh = tb.fresh.copy()
        fresh_out.append(fresh)
        if not tb.read:
            continue
        end = tb.capacity if mutant == "capacity" else tb.len
        if not end:
            continue
        slots = np.arange(end)
        rows = tb.rows[:end].copy()
        if mutant == "unmapped":
            rows = np.where(rows == UNMAPPED, tb.held[:end], rows)
        live = rows != UNMAPPED
        full = fresh[:end] & (mutant != "fresh_by_ticks")
        kind, vals = bounds_bits(tb, slots, layout, mutant)
        tflags = tb.flags | (F_AABB if kind == "aabb" else F_SPHERE if kind == "sphere" else 0)
        if kind is not None:
            ticks = tb.aabb_ticks if kind == "aabb" else tb.sphere_ticks
            sel = live & (full | is_newer(ticks[:end], last_run, this_run))
            bounds[rows[sel]] = vals[sel]
        ivbit = np.zeros(end, np.uint8) if tb.iv is None else (tb.iv[:end] != 0).astype(np.uint8)
        newer_iv = np.zeros(end, bool)
        if tb.iv is not None:
            ticks = tb.aabb_ticks if mutant == "iv_by_aabb_tick" and tb.aabb is not None else tb.iv_ticks
            newer_iv = is_newer(ticks[:end], last_run, this_run)
        sel = live & full
        keep = 0 if mutant == "drop_tchanged" else F_TCHANGED
        flags[rows[sel]] = (tflags | ivbit[sel] | (flags[rows[sel]] & keep)).astype(np.uint8)
        sel = live & newer_iv & ~full
        flags[rows[sel]] = ((flags[rows[sel]] & (0xFF ^ F_INHERITED)) | ivbit[sel]).astype(np.uint8)
        fresh[:end] = False
    return bounds, flags, fresh_out


def same(a, b):
    """Two read results leave the same device state."""
    return (a[0] == b[0]).all() and (a[1] == b[1]).all()


def put(col, slots, fields):
    """Write f32 fields (offset, values [k, n]) into the slots' bytes."""
    slots = np.asarray(slots, np.int64)
    for off, vals in fields:
        v = np.ascontiguousarray(vals, np.float32).reshape(len(slots), -1)
        col[slots, off:off + 4 * v.shape[1]] = v.view(np.uint8)


def newer_tick(rng, L, R):
    """A tick in (L, R] within 16 of R."""
    return (R - int(rng.integers(0, min((R - L) & 0xFFFFFFFF, 16)))) & 0xFFFFFFFF


def game(tables, layout, rng, L, R, n_bounds=8, n_iv=4, past_len=True):
    """The other systems between two cull runs.  Every slot's Aabb, Sphere and InheritedVisibility bytes are overwritten
    with values that would change visibility, with ticks at or before L (bypass_change_detection); then n_bounds live
    slots get new bounds and n_iv live slots a toggled InheritedVisibility, with ticks in (L, R].  Slots at and past len
    get newer ticks (never read).  Returns the stamped (table, slot) pairs."""
    stamped = []
    for t, tb in enumerate(tables):
        cap = tb.capacity
        if not cap:
            continue
        old = lambda: ((L - rng.integers(0, 40, cap)) & 0xFFFFFFFF).astype(np.uint32)
        if tb.aabb is not None:
            put(tb.aabb, np.arange(cap), ((layout[1], rng.uniform(-400, 400, (cap, 3))), (layout[2], rng.uniform(0, 0.01, (cap, 3)))))
            tb.aabb_ticks[:] = old()
        if tb.sphere is not None:
            put(tb.sphere, np.arange(cap), ((layout[4], rng.uniform(-400, 400, (cap, 3))), (layout[5], rng.uniform(0, 0.01, (cap, 1)))))
            tb.sphere_ticks[:] = old()
        if tb.iv is not None:
            tb.iv[:] = rng.integers(0, 2, cap)
            tb.iv_ticks[:] = old()
        if past_len and tb.len < cap:
            for ticks in (tb.aabb_ticks, tb.sphere_ticks, tb.iv_ticks):
                if ticks is not None:
                    ticks[tb.len:] = newer_tick(rng, L, R)
    live = [(t, s) for t, tb in enumerate(tables) for s in np.nonzero(tb.rows[:tb.len] != UNMAPPED)[0]]
    if not live:
        return stamped
    for k in rng.choice(len(live), size=min(n_bounds, len(live)), replace=False):
        t, s = live[k]
        tb = tables[t]
        if tb.aabb is not None:
            put(tb.aabb, [s], ((layout[1], rng.uniform(-30, 30, (1, 3))), (layout[2], rng.uniform(0.2, 2.0, (1, 3)))))
            tb.aabb_ticks[s] = newer_tick(rng, L, R)
        if tb.sphere is not None:
            put(tb.sphere, [s], ((layout[4], rng.uniform(-30, 30, (1, 3))), (layout[5], rng.uniform(0.2, 2.0, (1, 1)))))
            tb.sphere_ticks[s] = newer_tick(rng, L, R)
        stamped.append((t, int(s)))
    ivs = [x for x in live if tables[x[0]].iv is not None]
    for k in rng.choice(len(ivs), size=min(n_iv, len(ivs)), replace=False) if ivs else []:
        t, s = ivs[k]
        tables[t].iv[s] = rng.integers(0, 2)
        tables[t].iv_ticks[s] = newer_tick(rng, L, R)
        stamped.append((t, int(s)))
    return stamped
