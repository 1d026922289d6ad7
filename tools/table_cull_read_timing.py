"""Cost of b200vis_read_tables(RD_CULL_INPUTS) on the bench world (config #3: 3922 trees x 255 nodes + 256 lights =
1,000,366 rows).

The rows are split into five archetype tables (roots, inner nodes, seven eighths of the leaves: Aabb +
InheritedVisibility; lights: Sphere + InheritedVisibility with SPHERE_FROM_GT; the other eighth of the leaves:
InheritedVisibility only, as for an entity with Visibility and no mesh), each in a shuffled slot order, over plain numpy
memory that the library registers, in Bevy's layouts (32 B per Aabb and per Sphere).  Three kinds of read:
  none       no slot newer
  8_subtrees every node of 8 roots' subtrees in an Aabb table has a newer Aabb tick
  fresh      every slot (re)mapped since the last cull read (the first frame after a remap): read in full
Per kind this times, with CUDA events on the context's stream and alternating inside each round:
  read       b200vis_read_tables(RD_CULL_INPUTS) (for `fresh`: the maps are sent again and flushed before each timed read)
  h2d        a pinned host-to-device copy of the bytes the read needs, in the same run (the PCIe reference)
  host       a host-side stand-in for the shim loop the read replaces (not Bevy, and without its per-entity hash lookups):
             numpy tick scans of both columns of every table, five full-length host arrays, the repack of the changed
             rows, one b200vis_upload_bounds per contiguous run of rows and a synchronize, timed with a host clock
The bytes a read needs are 4 B per slot per tick column, plus 24 B per newer Aabb, or for a full read the fields of the
slot's columns (24 B of Aabb or 16 B of Sphere, and the InheritedVisibility byte).  Finally the tile pass (PROPAGATE | CULL) is timed right after
a cull read with nothing newer and after no read.  Prints one JSON line with the card and its power limit.
Run from the repository root: python tools/table_cull_read_timing.py [--reps 20] [--rounds 5]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from table_read_timing import card  # noqa: E402


def spread(v):
    return [round(float(min(v)), 4), round(float(max(v)), 4)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    import bevy_b200 as bb
    from bevy_b200 import abi, scenes
    import table_read_model as M
    assert torch.cuda.is_available(), "this tool measures the GPU: no CUDA device"
    sc = scenes.forest(3922, 8, 256)
    pipe = bb.VisibilityPipeline(sc)
    c = pipe.ctx
    stream = torch.cuda.Stream()                              # the context's stream: the events are recorded on it
    c.set_stream(stream.cuda_stream)
    n = sc.n
    rng = np.random.default_rng(0)
    kids = np.zeros(n, np.int64)
    real = sc.parent < n
    np.add.at(kids, sc.parent[real].astype(np.int64), 1)
    light = np.zeros(n, bool); light[sc.light_row] = True
    leaves = np.nonzero(real & (kids == 0))[0]
    # the fifth table: an eighth of the leaves without bounds (Visibility on an entity without a mesh)
    groups = [np.nonzero(~real & (kids > 0))[0], np.nonzero(real & (kids > 0))[0], leaves[len(leaves) // 8:],
              np.nonzero(light)[0], leaves[:len(leaves) // 8]]
    assert sum(len(g) for g in groups) == n
    T0 = 1000
    caps = [len(g) for g in groups]
    tabs, buf = abi.host_tables(caps, tick_fill=T0)
    culls, cbuf = abi.host_table_cull_inputs(caps, tick_fill=T0)
    maps = [rng.permutation(g).astype(np.uint32) for g in groups]
    c.set_tables(tabs)
    for t, m in enumerate(maps):
        cu = culls[t]
        if t == 3:
            cu.has, cu.flags = ("sphere", "iv"), abi.F_SPHERE_FROM_GT
            cu.put_sphere(np.arange(len(m)), sc.bounds[m, 0:3], sc.bounds[m, 3])
        elif t == 4:
            cu.has, cu.flags = ("iv",), 0
        else:
            cu.has, cu.flags = ("aabb", "iv"), 0
            cu.put_aabb(np.arange(len(m)), sc.bounds[m, 0:3], sc.bounds[m, 3:6])
        cu.iv[:] = 1
    c.set_table_cull_inputs(culls)

    def send_maps():
        for t, m in enumerate(maps):
            c.set_table_rows(t, 0, np.full(len(m), abi.UNMAPPED, np.uint32))
            c.set_table_rows(t, 0, m)
        c.read_tables(0, T0, T0)                              # flushes the queued map changes, reads nothing
    send_maps()
    pipe.update_views()
    c.read_tables(abi.RD_CULL_INPUTS, T0, T0 + 1)
    c.run(abi.STAGE_PROPAGATE | abi.STAGE_CULL)
    c.synchronize()
    # the subtrees of 8 roots (their rows), and where each row sits
    slot = np.zeros(n, np.int64); table = np.zeros(n, np.int64)
    for t, m in enumerate(maps):
        slot[m] = np.arange(len(m)); table[m] = t
    parent = sc.parent.astype(np.int64)
    roots = rng.choice(groups[0], 8, replace=False)
    top = np.arange(n)
    for _ in range(10):                                       # every row's root (levels <= 8)
        up = parent[top]
        top = np.where(up < n, up, top)
    sub = np.nonzero(np.isin(top, roots))[0]

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(call, reps, before=None):
        tot = 0.0
        for _ in range(reps):
            if before:
                before()
            e0.record(stream)
            call()
            e1.record(stream)
            e1.synchronize()
            tot += e0.elapsed_time(e1)
        return tot / reps

    out = {"card": None, "power_limit": None, "rows": n, "tables": caps}
    last, this = T0 + 10, T0 + 20
    for kind in ("none", "8_subtrees", "fresh"):
        for cu in culls:
            cu.aabb_ticks[:] = last; cu.sphere_ticks[:] = last
            cu.iv_ticks[:] = last
        k = 0
        if kind == "8_subtrees":
            for t in range(3):
                s = slot[sub[table[sub] == t]]
                culls[t].aabb_ticks[s] = this - 1
                k += len(s)
        full = kind == "fresh"
        n_aabb, n_sph, n_none = sum(caps[:3]), caps[3], caps[4]
        ticks_bytes = 4 * n + 4 * (n_aabb + n_sph)
        nbytes = ticks_bytes + ((24 + 1) * n_aabb + (16 + 1) * n_sph + n_none if full else 24 * k)
        dev = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        host = torch.empty(nbytes, dtype=torch.uint8).pin_memory()

        def h2d():
            with torch.cuda.stream(stream):
                dev.copy_(host, non_blocking=True)

        def stand_in():
            t0 = time.perf_counter()
            bounds = np.zeros((n, 6), np.float32); flags = np.zeros(n, np.uint8); cls = np.zeros(n, np.uint8)
            layer = np.ones(n, np.uint64); rmask = np.zeros(n, np.uint32)
            dirty = []
            for t, cu in enumerate(culls):
                sph, box = "sphere" in cu.has, "aabb" in cu.has
                newer = M.is_newer(cu.iv_ticks, last, this)
                if sph or box:
                    newer |= M.is_newer(cu.sphere_ticks if sph else cu.aabb_ticks, last, this)
                ch = np.nonzero(newer)[0]
                rows = maps[t][ch]
                if sph:
                    bounds[rows, 0:4] = cu.get_sphere(ch)
                elif box:
                    bounds[rows] = cu.get_aabb(ch)
                flags[rows] = (cu.iv[ch] != 0) | (abi.F_HAS_SPHERE | abi.F_SPHERE_FROM_GT if sph else abi.F_HAS_AABB if box else 0)
                cls[rows] = 1
                dirty.append(rows)
            d = np.sort(np.concatenate(dirty))
            if len(d):
                cut = np.nonzero(np.diff(d) != 1)[0] + 1
                for run in np.split(d, cut):
                    f, m = int(run[0]), len(run)
                    c.upload_bounds(f, bounds[f:f + m], flags[f:f + m], cls[f:f + m], layer[f:f + m], None)
            c.synchronize()
            return (time.perf_counter() - t0) * 1e3
        res = {"read_ms": [], "h2d_ms": [], "host_ms": []}
        for _ in range(args.rounds):
            res["read_ms"].append(timed(lambda: c.read_tables(abi.RD_CULL_INPUTS, last, this), args.reps,
                                        send_maps if full else None))
            res["h2d_ms"].append(timed(h2d, args.reps))
            res["host_ms"].append(float(np.median([stand_in() for _ in range(3)])))
        med = {k2: float(np.median(v)) for k2, v in res.items()}
        out[kind] = {"newer_slots": n if full else k, "bytes": nbytes, **{k2: round(v, 4) for k2, v in med.items()},
                     "read_GBps": round(nbytes / med["read_ms"] / 1e6, 2), "h2d_GBps": round(nbytes / med["h2d_ms"] / 1e6, 2),
                     "spread_read_ms": spread(res["read_ms"]), "spread_host_ms": spread(res["host_ms"])}
        out[kind]["read_over_h2d"] = round(out[kind]["read_GBps"] / out[kind]["h2d_GBps"], 3)
        del dev, host
    # the tile pass after a cull read with nothing newer, against after no read
    for cu in culls:
        cu.aabb_ticks[:] = last; cu.sphere_ticks[:] = last
        cu.iv_ticks[:] = last
    tile = {"after_read_ms": [], "after_no_read_ms": []}
    for _ in range(args.rounds):
        for key, read in (("after_read_ms", True), ("after_no_read_ms", False)):
            before = (lambda: c.read_tables(abi.RD_CULL_INPUTS, last, this)) if read else None
            tile[key].append(timed(lambda: c.run(abi.STAGE_PROPAGATE | abi.STAGE_CULL), args.reps, before))
    out["tile_pass"] = {k2: round(float(np.median(v)), 4) for k2, v in tile.items()}
    out["tile_pass"].update({"spread_" + k2: spread(v) for k2, v in tile.items()})
    c.set_tables([])
    pipe.close()
    out["card"], out["power_limit"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
