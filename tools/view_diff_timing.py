"""Cost of the per-class camera diff (b200vis_set_view_diff_sink) on the bench world (config #3: 1,000,366 rows, 4 views).
The class masks are split into meshes (class 0) and lights (class 1), and every seventh row is in both, so a view has
three non-empty class lists.  Every view has its own diff slot.

  frame      one STAGE_ALL frame (b200vis_run, then b200vis_join so the pipelined tail is inside the window), CUDA events
             around it, with and without the sink, the two setups alternated.  Static frames (nothing moves, cameras
             still) and moving frames (each --move-share: that share of the trees translated every frame)
  kernels    per-kernel device time per frame with the sink on the largest moving share, from a torch.profiler run of
             its own
  host_bytes what the sink writes into host memory per frame (entries x 8 + both offset arrays)
  cpu_path   the host path the sink replaces, on two moving frames: each view's row list and class masks downloaded,
             mapped to Entity bits and split by class, then the oracle's single-threaded update_cpu_culled_entities per
             (view, class) against the previous frame's lists, host clock
Prints one JSON line with the card and its power limit.
Run from the repository root: python tools/view_diff_timing.py [--reps 20] [--move-share 0.05,0.5]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from cull_outputs_timing import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--move-share", default="0.05,0.5", help="shares of the trees moved on every moving frame, comma-separated")
    args = ap.parse_args()
    import torch
    import bevy_b200 as bb
    import oracle as orc
    from bevy_b200 import abi, scenes
    assert torch.cuda.is_available(), "this tool measures the GPU: no CUDA device"
    name, limit = card()
    sc = scenes.forest()
    n, V = sc.n, len(sc.cameras)
    sc.class_mask = np.where(np.arange(n) % 7 == 0, 3, 1).astype(np.uint8)
    sc.class_mask[sc.light_row] = 2
    pipe = bb.VisibilityPipeline(sc)
    c = pipe.ctx
    stream = torch.cuda.Stream()
    c.set_stream(stream.cuda_stream)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    n_lists = V * 8
    pin = lambda k, dt, tdt: torch.zeros(k, dtype=tdt).pin_memory().numpy().view(dt)
    add, rem = pin(2 * n, np.uint64, torch.int64), pin(2 * n, np.uint64, torch.int64)
    aoff, roff = pin(n_lists + 1, np.uint32, torch.int32), pin(n_lists + 1, np.uint32, torch.int32)

    def setup(kind):
        c.set_view_diff_sink(None, None, None, None)
        if kind == "diff":
            c.set_view_diff_sink(add, rem, aoff, roff, V)
            c.set_view_diff_slots(np.arange(V))

    rng = np.random.default_rng(0)
    roots = np.asarray(sc.roots, np.int64)
    shares = [float(x) for x in args.move_share.split(",")]
    n_moves = {sh: max(1, int(round(sh * len(roots)))) for sh in shares}

    def frame_ms(n_move):
        if n_move:
            rows = np.sort(rng.choice(roots, n_move, replace=False)).astype(np.uint32)
            sc.trs[rows, 0:3] += rng.uniform(-1.0, 1.0, (len(rows), 3)).astype(np.float32)
            c.upload_transforms_scattered(rows, sc.trs[rows])
        pipe.update_views()
        a, b = ev(), ev()
        a.record(stream)
        c.run(abi.STAGE_ALL)
        c.join()
        b.record(stream)
        b.synchronize()
        pipe.read_feedback()
        return a.elapsed_time(b)

    kinds = ("none", "diff")
    modes = [("static", 0)] + [(f"moving_{sh}", n_moves[sh]) for sh in shares]
    runs = {f"{k}:{m}": [] for k in kinds for m, _ in modes}
    nbytes, changes = {}, {}
    for _ in range(3):                                        # alternate the two setups
        for k in kinds:
            setup(k)
            for _ in range(3):
                frame_ms(0)                                   # warm up; the slots fill on the first frame
            for m, nm in modes:
                ts = []
                for _ in range(args.reps):
                    ts.append(frame_ms(nm))
                    if k == "diff":
                        nbytes.setdefault(m, []).append((int(aoff[n_lists]) + int(roff[n_lists])) * 8 + 2 * (n_lists + 1) * 4)
                runs[f"{k}:{m}"].append(round(float(np.median(ts)), 4))
                if k == "diff":
                    changes[f"{m}_added_removed"] = [int(aoff[n_lists]), int(roff[n_lists])]
    res = {"metric": "view_diff_timing", "card": name, "power_limit": limit, "rows": n, "views": V, "lists": n_lists,
           "trees": len(roots), "trees_moved_per_frame": {str(sh): n_moves[sh] for sh in shares},
           "frame_ms_median": runs, "host_bytes_per_frame_median": {m: int(np.median(b)) for m, b in nbytes.items()}, **changes}

    from torch.profiler import ProfilerActivity, profile
    k_us = {}
    big = n_moves[max(shares)]
    setup("diff")
    for _ in range(3):
        frame_ms(big)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            frame_ms(big)
        c.synchronize()
    for e in prof.key_averages():
        if "view_diff" in e.key or "k_expand_visible" in e.key:
            k_us[e.key.split("(")[0].split("::")[-1]] = round(e.device_time_total / max(e.count, 1), 2)
    res["kernel_us_per_frame_moving_" + str(max(shares))] = k_us

    # ---- the host path the sink replaces: lists and class masks downloaded, mapped, split, diffed per (view, class) ----
    setup("none")

    def host_lists():
        out = {}
        for v in range(V):
            for k, r in c.download_visible_by_class(v).items():
                out[(v, k)] = sc.entity_bits[r]
        return out
    frame_ms(big); c.synchronize()
    old = host_lists()
    host, entries = [], 0
    for _ in range(3):
        frame_ms(big); c.synchronize()
        t0 = time.perf_counter()
        new = host_lists()
        for key in set(old) | set(new):
            o_, n_ = old.get(key, np.zeros(0, np.uint64)), new.get(key, np.zeros(0, np.uint64))
            orc.update_cpu_culled_entities(o_, o_, n_, n_)
        host.append(round((time.perf_counter() - t0) * 1e3, 3))
        entries = int(sum(len(x) for x in new.values()))
        old = new
    res["cpu_path_ms"] = host
    res["cpu_threads"] = 1
    res["cpu_path_entries"] = entries
    pipe.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
