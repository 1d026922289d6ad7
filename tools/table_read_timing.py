"""Cost of b200vis_read_tables on the bench world (config #3: 3922 trees x 255 nodes + 256 lights = 1,000,366 rows).

The rows are split into four archetype tables (roots, inner nodes, leaves, lights), each in a shuffled slot order, over
plain numpy memory that the library registers, every table with a Transform column in Bevy's layout (48 B per slot) and
its ticks.  Three kinds of frame: no slot newer, 8 roots newer, all 3,922 roots newer (their Transform and, for the
GlobalTransform read, their GlobalTransform).  Per kind, alternating inside each round, this times:
  read_t     b200vis_read_tables(RD_TRANSFORM), CUDA events on the context's stream
  read_tg    b200vis_read_tables(RD_TRANSFORM | RD_GLOBAL_TRANSFORM)
  h2d        a pinned host-to-device copy of the bytes read_tg needs, in the same run (the PCIe reference)
  host       a host-side stand-in for the loops the read replaces (not Bevy): a numpy tick scan of every Transform tick,
             the gather and repack of the newer slots into 10 floats, b200vis_upload_transforms_scattered, and a
             synchronize, timed with a host clock
The bytes a read needs are 4 B per slot per tick column plus 40 B per newer Transform and 48 B per newer
GlobalTransform (the kernel loads each Affine3A as four 16-byte lanes, 64 B).  Finally the tile pass (PROPAGATE | CULL)
is timed right after an RD_GLOBAL_TRANSFORM read with nothing newer (kernel 1b's marked instantiation) and after an
RD_TRANSFORM read (the unmarked one).  Prints one JSON line with the card and its power limit.
Run from the repository root: python tools/table_read_timing.py [--reps 20] [--rounds 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [x.strip() for x in out.split(",")]
        return name, limit
    except Exception:
        return "unknown", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
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
    groups = [np.nonzero(~real & (kids > 0))[0], np.nonzero(real & (kids > 0))[0], np.nonzero(real & (kids == 0))[0],
              np.nonzero(light)[0]]
    assert sum(len(g) for g in groups) == n
    T0 = 1000
    caps = [len(g) for g in groups]
    tabs, buf = abi.host_tables(caps, tick_fill=T0)
    ins, ibuf = abi.host_table_inputs(caps, tick_fill=T0)
    maps = [rng.permutation(g).astype(np.uint32) for g in groups]
    c.set_tables_ex(tabs, ins, abi.BEVY_TRANSFORM_LAYOUT)
    for t, m in enumerate(maps):
        c.set_table_rows(t, 0, m)
        ins[t].put(np.arange(len(m)), sc.trs[m])
    slot_of_root = {int(r): s for s, r in enumerate(maps[0])}
    pipe.update_views()
    c.run(abi.STAGE_PROPAGATE | abi.STAGE_CULL)
    c.synchronize()

    def timed(call, reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        call(); torch.cuda.synchronize()
        e0.record(stream)
        for _ in range(reps):
            call()
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / reps

    last, this = T0, T0 + 10
    sizes = {"none": 0, "8_roots": 8, "all_roots": len(groups[0])}
    out = {"card": None, "power_limit": None, "rows": n, "tables": caps}
    for kind, k in sizes.items():
        for t in range(4):
            ins[t].ticks[:] = last
            tabs[t].gt_ticks[:] = last
        slots = np.sort(rng.choice(len(groups[0]), k, replace=False)) if k < len(groups[0]) else np.arange(k)
        ins[0].ticks[slots] = this - 1
        tabs[0].gt_ticks[slots] = this - 1
        tabs[0].gt[slots] = np.tile(np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 5, 5, 5, 0], np.float32), (k, 1))
        bytes_t = 4 * n + 40 * k
        bytes_tg = bytes_t + 4 * n + 48 * k
        dev = torch.empty(bytes_tg, dtype=torch.uint8, device="cuda")
        host = torch.empty(bytes_tg, dtype=torch.uint8).pin_memory()

        def h2d():
            with torch.cuda.stream(stream):
                dev.copy_(host, non_blocking=True)

        def stand_in():
            t0 = time.perf_counter()
            rows_l, trs_l = [], []
            for t in range(4):
                newer = np.nonzero(M.is_newer(ins[t].ticks, last, this))[0]
                rows_l.append(maps[t][newer])
                trs_l.append(ins[t].get(newer))
            rows = np.concatenate(rows_l)
            trs = np.ascontiguousarray(np.concatenate(trs_l), np.float32)
            c.upload_transforms_scattered(rows, trs)
            c.synchronize()
            return (time.perf_counter() - t0) * 1e3
        res = {"read_t_ms": [], "read_tg_ms": [], "h2d_ms": [], "host_ms": []}
        for _ in range(args.rounds):
            res["read_t_ms"].append(timed(lambda: c.read_tables(abi.RD_TRANSFORM, last, this), args.reps))
            res["read_tg_ms"].append(timed(lambda: c.read_tables(abi.RD_TRANSFORM | abi.RD_GLOBAL_TRANSFORM, last, this), args.reps))
            res["h2d_ms"].append(timed(h2d, args.reps))
            res["host_ms"].append(float(np.median([stand_in() for _ in range(3)])))
            c.run(abi.STAGE_PROPAGATE | abi.STAGE_CULL)          # consume the marks the GlobalTransform reads left
            c.synchronize()
        med = {k2: float(np.median(v)) for k2, v in res.items()}
        out[kind] = {"newer_slots": k, "bytes_t": bytes_t, "bytes_tg": bytes_tg, **{k2: round(v, 4) for k2, v in med.items()},
                     "read_t_GBps": round(bytes_t / med["read_t_ms"] / 1e6, 2),
                     "read_tg_GBps": round(bytes_tg / med["read_tg_ms"] / 1e6, 2),
                     "h2d_GBps": round(bytes_tg / med["h2d_ms"] / 1e6, 2),
                     "spread_read_tg_ms": [round(min(res["read_tg_ms"]), 4), round(max(res["read_tg_ms"]), 4)]}
        out[kind]["read_tg_over_h2d"] = round(out[kind]["read_tg_GBps"] / out[kind]["h2d_GBps"], 3)
        del dev, host
    # the tile pass after a GlobalTransform read with nothing newer (marked instantiation) against after a Transform read
    for t in range(4):
        ins[t].ticks[:] = last
        tabs[t].gt_ticks[:] = last
    tile = {"marked_ms": [], "unmarked_ms": []}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for key, which in (("marked_ms", abi.RD_GLOBAL_TRANSFORM), ("unmarked_ms", abi.RD_TRANSFORM)):
            tot = 0.0
            for _ in range(args.reps):
                c.read_tables(which, last, this)
                e0.record(stream)
                c.run(abi.STAGE_PROPAGATE | abi.STAGE_CULL)
                e1.record(stream)
                e1.synchronize()
                tot += e0.elapsed_time(e1)
            tile[key].append(tot / args.reps)
    out["tile_pass"] = {k2: round(float(np.median(v)), 4) for k2, v in tile.items()}
    out["tile_pass"]["spread_marked_ms"] = [round(min(tile["marked_ms"]), 4), round(max(tile["marked_ms"]), 4)]
    out["tile_pass"]["spread_unmarked_ms"] = [round(min(tile["unmarked_ms"]), 4), round(max(tile["unmarked_ms"]), 4)]
    c.set_tables([])
    pipe.close()
    out["card"], out["power_limit"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
