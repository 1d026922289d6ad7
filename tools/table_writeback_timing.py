"""Cost of the table write-back on the bench world (config #3: 3922 trees x 255 nodes + 256 lights = 1,000,366 rows).

The rows are split into four archetype tables (roots, inner nodes, leaves, lights), each in a shuffled slot order, over plain
numpy memory that the library registers.  After one frame of the given pattern -- dense: every root moves, so every row's
GlobalTransform changes; sparse: 8 roots move (2,040 rows) -- this times, with CUDA events on the context's stream:
  tables   b200vis_writeback_tables(GlobalTransform only): 64 B matrix + 4 B tick per changed row, in slot order
  columns  b200vis_writeback_columns_ex(GlobalTransform only), stride 16: 64 B per changed row + the change bit set, on
           its zero-copy scatter path (B200VIS_WRITEBACK_DENSE=0: row-order stores, no device repack + copy engine)
  d2h      a plain pinned device-to-host copy of 64 MB (cudaMemcpyAsync through torch), the PCIe reference of the same run
and the host wall time of b200vis_set_tables registering one new 64 MB table (the cost of a table reallocation).
Rates are the bytes the write-back must deliver over its time.  Prints one JSON line with the card and its power limit.
Run from the repository root: python tools/table_writeback_timing.py [--reps 20] [--rounds 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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
    os.environ["B200VIS_WRITEBACK_DENSE"] = "0"                 # read once, at the first column write-back
    import torch
    import bevy_b200 as bb
    from bevy_b200 import abi, scenes
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
    tabs, buf = abi.host_tables([len(g) for g in groups])
    c.set_tables(tabs)
    for t, g in enumerate(groups):
        c.set_table_rows(t, 0, rng.permutation(g).astype(np.uint32))
    col_gt = np.zeros((n, 16), np.float32)
    col_bits = np.zeros((n + 31) // 32, np.uint32)
    c.set_column_sinks(col_gt, col_bits, None, None)

    def frame(pattern, f):
        scenes.advance_cameras(sc, 0.02)
        if pattern == "dense":
            rows, trs = scenes.mutate_roots(sc, f)
        else:
            rows = np.sort(rng.choice(sc.roots, 8, replace=False)).astype(np.uint32)
            trs = sc.trs[rows].copy(); trs[:, 0] += 0.01
            sc.trs[rows] = trs
        c.upload_transforms_scattered(rows, trs)
        pipe.update_views()
        c.run(abi.STAGE_PROPAGATE | abi.STAGE_CULL)
        c.writeback_tables(abi.WB_VIEW_VISIBILITY, 0, f)       # ViewVisibility bytes settle: not part of the timed window
        c.synchronize()
        return int(pipe.read_feedback().gt_changed_count)

    def timed(call, reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        call(); torch.cuda.synchronize()
        e0.record(stream)
        for _ in range(reps):
            call()
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / reps

    dev = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")

    def d2h():
        with torch.cuda.stream(stream):
            host.copy_(dev, non_blocking=True)
    host = torch.empty(64 << 20, dtype=torch.uint8).pin_memory()
    out = {"card": None, "power_limit": None, "rows": n, "tables": [len(g) for g in groups]}
    f = 0
    for pattern in ("dense", "sparse"):
        res = {"tables_ms": [], "columns_ms": [], "d2h_ms": []}
        for _ in range(args.rounds):
            f += 1
            changed = frame(pattern, f)
            for _ in range(2):                                   # alternate the paths inside one round
                res["tables_ms"].append(timed(lambda: c.writeback_tables(abi.WB_GLOBAL_TRANSFORM, f, 0), args.reps))
                res["columns_ms"].append(timed(lambda: c.writeback_columns(abi.WB_GLOBAL_TRANSFORM), args.reps))
                res["d2h_ms"].append(timed(d2h, args.reps))
        med = {k: float(np.median(v)) for k, v in res.items()}
        out[pattern] = {"gt_changed_rows": changed, **{k: round(v, 4) for k, v in med.items()},
                        "tables_GBps": round(changed * 68 / med["tables_ms"] / 1e6, 2),
                        "columns_GBps": round((changed * 64 + (n + 31) // 32 * 4) / med["columns_ms"] / 1e6, 2),
                        "d2h_GBps": round((64 << 20) / med["d2h_ms"] / 1e6, 2),
                        "spread_tables_ms": [round(min(res["tables_ms"]), 4), round(max(res["tables_ms"]), 4)]}
        out[pattern]["tables_over_d2h"] = round(out[pattern]["tables_GBps"] / out[pattern]["d2h_GBps"], 3)
    # re-registration: a newly allocated 1M-slot table (64 MB of GlobalTransform + ticks and ViewVisibility)
    reg = []
    for _ in range(args.rounds):
        (big,), big_buf = abi.host_tables([1 << 20])
        t0 = time.perf_counter()
        c.set_tables(tabs + [big])
        reg.append((time.perf_counter() - t0) * 1e3)
        c.set_tables(tabs)
        del big, big_buf
    out["set_tables_new_64MB_ms"] = [round(x, 2) for x in reg]
    c.set_column_sinks()
    c.set_tables([])
    pipe.close()
    out["card"], out["power_limit"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
