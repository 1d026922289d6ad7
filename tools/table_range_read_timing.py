"""Cost of reading VisibilityRange from the archetype tables (b200vis_set_table_visibility_ranges) on the bench world
(config #3: 3922 trees x 255 nodes + 256 lights = 1,000,366 rows).

The rows are split into the five tables of tools/table_cull_read_timing.py (roots, inner nodes, seven eighths of the
leaves with Aabb + InheritedVisibility; lights with Sphere; an eighth of the leaves with InheritedVisibility only), each
in a shuffled slot order.  The inner-node and leaf tables (933,436 rows) also carry VisibilityRange (20 B, use_aabb at
16) and HAS_VIS_RANGE.  Times, with CUDA events on the context's stream, the cases alternated inside each round:
  read     b200vis_read_tables(RD_CULL_INPUTS), with the ranges attached and detached, when no slot is newer and when
           every slot is fresh (the maps sent again and flushed before each timed read)
  tile     the tile pass (PROPAGATE | CULL, static frame) of a context whose range columns are resident (the cull
           evaluates check_visibility_ranges; the non-SIMPLE instantiation) against a twin context with none
  host     a host stand-in for the per-frame loop the read replaces (not Bevy, and without its per-entity hash lookups):
           the repack of bounds, flags, class, layers and a range mask for every ranged row, one b200vis_upload_bounds per
           contiguous run of those rows and a synchronize, with a host clock
Prints one JSON line with the card and its power limit.
Run from the repository root: python tools/table_range_read_timing.py [--reps 20] [--rounds 5]"""
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

RANGED = (1, 2)


def spread(v):
    return [round(float(min(v)), 4), round(float(max(v)), 4)]


def world(sc, rng, ranged):
    """A context over the bench world in five tables, cull inputs attached, and VisibilityRange on `ranged` tables."""
    import bevy_b200 as bb
    from bevy_b200 import abi
    n = sc.n
    pipe = bb.VisibilityPipeline(sc)
    c = pipe.ctx
    kids = np.zeros(n, np.int64)
    real = sc.parent < n
    np.add.at(kids, sc.parent[real].astype(np.int64), 1)
    light = np.zeros(n, bool); light[sc.light_row] = True
    leaves = np.nonzero(real & (kids == 0) & ~light)[0]
    groups = [np.nonzero(~real & (kids > 0))[0], np.nonzero(real & (kids > 0))[0], leaves[len(leaves) // 8:],
              np.nonzero(light)[0], leaves[:len(leaves) // 8]]
    assert sum(len(g) for g in groups) == n
    T0 = 1000
    caps = [len(g) for g in groups]
    tabs, buf = abi.host_tables(caps, tick_fill=T0)
    culls, cbuf = abi.host_table_cull_inputs(caps, tick_fill=T0)
    rgs, rbuf = abi.host_table_ranges(caps, tick_fill=T0)
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
            cu.has, cu.flags = ("aabb", "iv"), abi.F_HAS_VIS_RANGE if t in ranged else 0
            cu.put_aabb(np.arange(len(m)), sc.bounds[m, 0:3], sc.bounds[m, 3:6])
        cu.iv[:] = 1
        if t in RANGED:
            start = rng.uniform(0, 40, len(m)).astype(np.float32)
            rgs[t].put(np.arange(len(m)), np.stack([start, start + 400], 1), rng.integers(0, 2, len(m)))
    c.set_table_cull_inputs(culls)
    if ranged:
        c.set_table_visibility_ranges([rgs[t] if t in ranged else None for t in range(5)])
        c.set_visibility_range_views(np.stack([np.asarray(cam.gt, np.float32)[9:12] for cam in sc.cameras]))
        sc.view_range_index = list(range(len(sc.cameras)))

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
    return dict(pipe=pipe, c=c, culls=culls, rgs=rgs, maps=maps, send_maps=send_maps, keep=(buf, cbuf, rbuf, tabs))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    from bevy_b200 import abi, scenes
    assert torch.cuda.is_available(), "this tool measures the GPU: no CUDA device"
    rng = np.random.default_rng(0)
    sc = scenes.forest(3922, 8, 256)
    sc_plain = scenes.forest(3922, 8, 256)
    W = world(sc, rng, RANGED)
    P = world(sc_plain, np.random.default_rng(0), ())
    stream = torch.cuda.Stream()                              # both contexts' stream: the events are recorded on it
    for w in (W, P):
        w["c"].set_stream(stream.cuda_stream)
    c = W["c"]
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

    n = sc.n
    out = {"card": None, "power_limit": None, "rows": n, "ranged_rows": int(sum(len(W["maps"][t]) for t in RANGED))}
    last, this = 1000 + 10, 1000 + 20
    for w in (W,):
        for cu in w["culls"]:
            cu.aabb_ticks[:] = last; cu.sphere_ticks[:] = last; cu.iv_ticks[:] = last
        for r in w["rgs"]:
            r.ticks[:] = last
    attach = lambda: c.set_table_visibility_ranges([W["rgs"][t] if t in RANGED else None for t in range(5)])
    for kind in ("none", "fresh"):
        res = {"with_ranges_ms": [], "without_ranges_ms": []}
        for _ in range(args.rounds):
            attach()                                          # an attach after none: every ranged slot marked fresh,
            c.read_tables(abi.RD_CULL_INPUTS, last, this)     # so one untimed read consumes the marks
            res["with_ranges_ms"].append(timed(lambda: c.read_tables(abi.RD_CULL_INPUTS, last, this), args.reps,
                                               W["send_maps"] if kind == "fresh" else None))
            c.set_table_visibility_ranges(None)
            res["without_ranges_ms"].append(timed(lambda: c.read_tables(abi.RD_CULL_INPUTS, last, this), args.reps,
                                                  W["send_maps"] if kind == "fresh" else None))
        out[kind] = {k: round(float(np.median(v)), 4) for k, v in res.items()}
        out[kind].update({"spread_" + k: spread(v) for k, v in res.items()})
    attach()
    # the tile pass with the range columns resident against none
    tile = {"ranges_resident_ms": [], "no_ranges_ms": []}
    for _ in range(args.rounds):
        for key, w in (("ranges_resident_ms", W), ("no_ranges_ms", P)):
            tile[key].append(timed(lambda: w["c"].run(abi.STAGE_PROPAGATE | abi.STAGE_CULL), args.reps))
    out["tile_pass"] = {k: round(float(np.median(v)), 4) for k, v in tile.items()}
    out["tile_pass"].update({"spread_" + k: spread(v) for k, v in tile.items()})
    # the host stand-in for the removed loop: every ranged row repacked and uploaded as contiguous runs, every frame
    ranged_rows = np.sort(np.concatenate([W["maps"][t] for t in RANGED])).astype(np.int64)
    bounds_all, flags_all = sc.bounds, sc.flags

    def stand_in():
        t0 = time.perf_counter()
        d = ranged_rows
        bounds = bounds_all[d].copy(); flags = (flags_all[d] | abi.F_HAS_VIS_RANGE).astype(np.uint8)
        cls = np.ones(len(d), np.uint8); layer = np.ones(len(d), np.uint64); rmask = np.zeros(len(d), np.uint32)
        cut = np.nonzero(np.diff(d) != 1)[0] + 1
        i = 0
        for run in np.split(d, cut):
            f, m = int(run[0]), len(run)
            c.upload_bounds(f, bounds[i:i + m], flags[i:i + m], cls[i:i + m], layer[i:i + m], rmask[i:i + m])
            i += m
        c.synchronize()
        return (time.perf_counter() - t0) * 1e3, len(cut) + 1
    hs = [stand_in() for _ in range(args.rounds)]
    out["host_stand_in_ms"] = round(float(np.median([h[0] for h in hs])), 3)
    out["host_stand_in_spread_ms"] = spread([h[0] for h in hs])
    out["host_stand_in_uploads"] = hs[0][1]
    for w in (W, P):
        w["c"].set_tables([])
        w["pipe"].close()
    out["card"], out["power_limit"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
