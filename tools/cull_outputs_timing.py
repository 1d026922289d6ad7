"""Cost of the cull system's device-written outputs on the bench world (config #3: 1,000,366 rows, 4 views).

  entities   the Entity emission of b200vis_set_visible_entities_sink (k_count_visible_classes + k_emit_visible_entities):
             CUDA events around a pipelined STAGE_ALL frame with and without the sink registered, joined on the tail; the
             difference is how much the emission lengthens the frame.  The scene's class masks are used as they are.
  set_vis    b200vis_writeback_tables(WB_SET_VISIBLE) on four shuffled tables (roots, inner nodes, leaves, lights) over plain
             numpy memory, CUDA events around it, for three device states: nothing visible, the bench frame's visible set
             and everything visible.  The table bytes are reset by numpy before each call (reset_view_visibility).
  host       numpy stand-ins for the two host loops the device work replaces, timed with a host clock after a synchronise:
             a gather of every view's sorted visible rows into per-class Entity arrays, and the scan of a 1 MB
             ViewVisibility column that applies set_visible() to every visible row (vectorised numpy, so a lower bound
             on a per-entity loop).
Prints one JSON line with the card and its power limit.
Run from the repository root: python tools/cull_outputs_timing.py [--reps 20]"""
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
    args = ap.parse_args()
    import torch
    import bevy_b200 as bb
    from bevy_b200 import abi, scenes
    assert torch.cuda.is_available(), "this tool measures the GPU: no CUDA device"
    sc = scenes.forest(3922, 8, 256)
    pipe = bb.VisibilityPipeline(sc)
    c = pipe.ctx
    stream = torch.cuda.Stream()
    c.set_stream(stream.cuda_stream)
    n, V = sc.n, len(sc.cameras)
    ev = lambda: torch.cuda.Event(enable_timing=True)

    def frames_ms(reps):
        a, b = ev(), ev()
        a.record(stream)
        for _ in range(reps):
            pipe.update_views()
            c.run(abi.STAGE_ALL)
        c.join()
        b.record(stream)
        b.synchronize()
        return a.elapsed_time(b) / reps

    for _ in range(5):
        frames_ms(1)
    ent = torch.zeros((V, n), dtype=torch.int64).pin_memory().numpy().view(np.uint64)
    off = torch.zeros((V, 9), dtype=torch.int32).pin_memory().numpy().view(np.uint32)
    res = {"metric": "cull_outputs_timing", "card": card()[0], "power_limit": card()[1], "rows": n, "views": V}
    without, with_sink = [], []
    for _ in range(3):                                        # alternate the two configurations
        c.set_visible_entities_sink(None, None)
        without.append(frames_ms(args.reps))
        c.set_visible_entities_sink(ent, off)
        frames_ms(2)
        with_sink.append(frames_ms(args.reps))
    res["frame_ms_without_entities_sink"] = [round(x, 4) for x in without]
    res["frame_ms_with_entities_sink"] = [round(x, 4) for x in with_sink]
    c.synchronize()
    res["entities_per_view"] = [int(off[v, 8]) for v in range(V)]
    # the emission kernels' own device time, in a profiled run of its own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            pipe.update_views()
            c.run(abi.STAGE_ALL)
        c.synchronize()
    k_us = {}
    for e in prof.key_averages():
        if "visible_classes" in e.key or "emit_visible_entities" in e.key or "expand_visible" in e.key:
            k_us[e.key.split("(")[0].split("::")[-1]] = round(e.device_time_total / max(e.count, 1), 2)
    res["kernel_us_per_frame"] = k_us
    c.set_visible_entities_sink(None, None)

    # ---- WB_SET_VISIBLE on four shuffled tables ----
    real = sc.parent < n
    kids = np.zeros(n, np.int64); np.add.at(kids, sc.parent[real].astype(np.int64), 1)
    light = np.zeros(n, bool); light[sc.light_row] = True
    groups = [np.nonzero(~real & (kids > 0) & ~light)[0], np.nonzero(real & (kids > 0))[0],
              np.nonzero(real & (kids == 0) & ~light)[0], np.nonzero(light)[0]]
    groups = [g for g in groups if len(g)]
    groups[-1] = np.union1d(groups[-1], np.setdiff1d(np.arange(n), np.concatenate(groups)))
    assert sum(len(g) for g in groups) == n
    tabs, buf = abi.host_tables([len(g) for g in groups])
    c.set_tables(tabs)
    rng = np.random.default_rng(0)
    for t, g in enumerate(groups):
        c.set_table_rows(t, 0, rng.permutation(g.astype(np.uint32)))
    vv0, _ = c.download_view_visibility(0, n)

    def set_visible_ms(reps):
        ts = []
        for _ in range(reps):
            for tab in tabs:
                tab.vv[:] = (tab.vv & 1) << 1                 # reset_view_visibility
            c.synchronize()
            a, b = ev(), ev()
            a.record(stream)
            c.writeback_tables(abi.WB_SET_VISIBLE, 0, 7)
            b.record(stream)
            b.synchronize()
            ts.append(a.elapsed_time(b))
        return round(float(np.median(ts)), 4)

    out = {}
    for name, state in (("none_visible", np.zeros(n, np.uint8)), ("bench_visible", vv0), ("all_visible", np.full(n, 3, np.uint8))):
        c.upload_view_visibility(0, state)
        set_visible_ms(3)
        out[name] = set_visible_ms(args.reps)
        out[name + "_rows"] = int((state & 1).sum())
    res["set_visible_ms"] = out

    # ---- numpy stand-ins for the host loops ----
    c.upload_view_visibility(0, vv0)
    pipe.update_views(); c.run(abi.STAGE_ALL); c.synchronize()
    lists = [c.download_visible(v) for v in range(V)]
    cls = sc.class_mask
    bits = sc.entity_bits
    t0 = time.perf_counter()
    for v in range(V):                                        # row -> Entity, one gather per class bit
        rows = lists[v].astype(np.int64)
        m = cls[rows]
        per_class = [bits[rows[(m >> k) & 1 == 1]] for k in range(8)]
    host_lists_ms = (time.perf_counter() - t0) * 1e3
    col = vv0.copy()
    t0 = time.perf_counter()
    vis = np.nonzero(col & 1)[0]                              # the unforked loop: set_visible() on every visible row
    b = col[vis]
    col[vis[(b & 1) == 0]] |= 1
    touched = len(vis)
    host_vv_ms = (time.perf_counter() - t0) * 1e3
    res["host_standin_ms"] = {"visible_entities_push": round(host_lists_ms, 3), "view_visibility_scan": round(host_vv_ms, 3),
                              "visible_rows": [len(l) for l in lists], "set_visible_rows": touched}
    del buf
    pipe.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
