"""Cost of the shadow-list diff (b200vis_set_shadow_diff_sink) on the bench world (config #3: 1,000,366 rows, 4 views), with
the items of tools/shadow_outputs_timing.py: 16 point lights, 8 spot lights and one directional light x 4 views x 4
cascades (40 shadow items, 240 lists), every item with its own diff slot.  The items stay fixed across frames.

  run        b200vis_run_shadow_culling, CUDA events around it, for three setups alternated in one run: the entity sink
             only, the diff sink only, both (row lists of one row in all three).  Each on static frames (nothing moves,
             cameras still) and on moving frames (each --move-share: that share of the trees translated every frame)
  kernels    per-kernel device time per run of each setup on moving frames, from a torch.profiler run of its own
  host_bytes what each setup writes into host memory per run (entries x 8 + offsets + active flags), static and moving
  cpu_diff   the render world's work the diff replaces: the oracle's single-threaded orc_update_cpu_culled_entities over
             the same 240 lists (last frame's and this frame's entity-sink lists), host clock
Prints one JSON line with the card and its power limit.
Run from the repository root: python tools/shadow_diff_timing.py [--reps 20] [--move-share 0.05,0.5]"""
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

IDENT9 = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1], np.float32)


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
    pipe = bb.VisibilityPipeline(sc)
    c = pipe.ctx
    stream = torch.cuda.Stream()
    c.set_stream(stream.cuda_stream)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    caster = np.ones(n, np.uint8); caster[sc.light_row] = 0
    c.upload_shadow_casters(0, caster)
    for _ in range(3):
        pipe.update_views(); c.run(abi.STAGE_ALL)
    c.synchronize()
    gt, _ = c.download_global_transforms(0, n)
    listed = set(np.concatenate([c.download_visible(v) for v in range(V)]).tolist())
    on = [o for o in range(len(sc.light_row)) if int(sc.light_row[o]) in listed]
    assert len(on) >= 24, f"only {len(on)} lights are in some view's VisibleEntities"
    items = []
    for k, o in enumerate(on[:24]):
        row = int(sc.light_row[o])
        fr = abi.host_point_light_frusta(gt[row], float(sc.light_range[o]))
        kind = 0 if k < 16 else 1
        items.append(dict(kind=kind, light_row=row, range=float(sc.light_range[o]), range_view_index=0, frusta=fr if kind == 0 else fr[k % 6]))
    for v in range(V):
        for cc, rr in enumerate((10.0, 30.0, 90.0, 270.0)):
            centre = np.asarray(sc.cameras[v].gt[9:12], np.float32)
            fr = abi.host_point_light_frusta(np.concatenate([IDENT9, centre]).astype(np.float32), rr)[(v + cc) % 6]
            items.append(dict(kind=2, range_view_index=-1, layer_mask=1, frusta=fr))
    n_items, n_lists = len(items), len(items) * 6
    slots = np.arange(n_items, dtype=np.uint32)
    pin = lambda k, dt, tdt: torch.zeros(k, dtype=tdt).pin_memory().numpy().view(dt)
    ent, off, act = pin(4 * n, np.uint64, torch.int64), pin(n_lists + 1, np.uint32, torch.int32), pin(n_items, np.uint8, torch.uint8)
    add, rem = pin(4 * n, np.uint64, torch.int64), pin(4 * n, np.uint64, torch.int64)
    aoff, roff = pin(n_lists + 1, np.uint32, torch.int32), pin(n_lists + 1, np.uint32, torch.int32)

    def setup(kind):
        c.set_shadow_entities_sink(None, None, None)
        c.set_shadow_diff_sink(None, None, None, None)
        if kind in ("entity", "both"):
            c.set_shadow_entities_sink(ent, off, act)
        if kind in ("diff", "both"):
            c.set_shadow_diff_sink(add, rem, aoff, roff, n_items)
        c.set_shadow_items(items, 1, diff_slots=None if kind == "entity" else slots)

    rng = np.random.default_rng(0)
    roots = np.asarray(sc.roots, np.int64)
    shares = [float(x) for x in args.move_share.split(",")]
    n_moves = {sh: max(1, int(round(sh * len(roots)))) for sh in shares}

    def frame_ms(n_move):
        """One frame's CULL stage (untimed), then run_shadow_culling under CUDA events.  n_move trees move first."""
        if n_move:
            rows = np.sort(rng.choice(roots, n_move, replace=False)).astype(np.uint32)
            sc.trs[rows, 0:3] += rng.uniform(-1.0, 1.0, (len(rows), 3)).astype(np.float32)
            c.upload_transforms_scattered(rows, sc.trs[rows])
        pipe.update_views(); c.run(abi.STAGE_ALL)
        a, b = ev(), ev()
        a.record(stream)
        c.run_shadow_culling()
        b.record(stream)
        b.synchronize()
        pipe.read_feedback()
        return a.elapsed_time(b)

    def host_bytes(kind):
        by = 0
        if kind in ("entity", "both"):
            by += int(off[n_lists]) * 8 + (n_lists + 1) * 4 + n_items
        if kind in ("diff", "both"):
            by += (int(aoff[n_lists]) + int(roff[n_lists])) * 8 + 2 * (n_lists + 1) * 4
        return by

    kinds = ("entity", "diff", "both")
    modes = [("static", 0)] + [(f"moving_{sh}", n_moves[sh]) for sh in shares]
    runs = {f"{k}:{m}": [] for k in kinds for m, _ in modes}
    nbytes, changes = {}, {}
    for _ in range(3):                                        # alternate the three setups
        for k in kinds:
            setup(k)
            for _ in range(3):
                frame_ms(0)                                   # warm up; the diff's slots fill on the first run
            for m, nm in modes:
                ts = [frame_ms(nm) for _ in range(args.reps)]
                runs[f"{k}:{m}"].append(round(float(np.median(ts)), 4))
                nbytes[f"{k}:{m}"] = host_bytes(k)
                if k == "diff":
                    changes[f"{m}_added_removed"] = [int(aoff[n_lists]), int(roff[n_lists])]
    res = {"metric": "shadow_diff_timing", "card": name, "power_limit": limit, "rows": n, "views": V, "items": n_items,
           "lists": n_lists, "trees": len(roots), "trees_moved_per_frame": {str(sh): n_moves[sh] for sh in shares},
           "run_shadow_culling_ms_median": runs, "host_bytes_per_run": nbytes, "entries": int(off[n_lists]), **changes}

    from torch.profiler import ProfilerActivity, profile
    k_us = {}
    big = n_moves[max(shares)]
    for k in kinds:
        setup(k)
        for _ in range(3):
            frame_ms(big)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                frame_ms(big)
            c.synchronize()
        for e in prof.key_averages():
            if "k_shadow" in e.key or "k_expand_shadow" in e.key or "k_emit_shadow_diff" in e.key:
                k_us[k + ":" + e.key.split("(")[0].split("::")[-1]] = round(e.device_time_total / max(e.count, 1), 2)
    res["kernel_us_per_run_moving_" + str(max(shares))] = k_us

    # ---- the render world's diff on the host: update_cpu_culled_entities over the 240 lists of two moving frames ----
    setup("entity")
    frame_ms(big); c.synchronize()
    old = [ent[off[l]:off[l + 1]].copy() for l in range(n_lists)]
    frame_ms(big); c.synchronize()
    new = [ent[off[l]:off[l + 1]].copy() for l in range(n_lists)]
    host = []
    for _ in range(3):
        t0 = time.perf_counter()
        for o_, n_ in zip(old, new):
            orc.update_cpu_culled_entities(o_, o_, n_, n_)
        host.append(round((time.perf_counter() - t0) * 1e3, 3))
    res["cpu_update_cpu_culled_entities_ms"] = host
    res["cpu_threads"] = 1
    res["cpu_entries_old_new"] = [int(sum(len(x) for x in old)), int(sum(len(x) for x in new))]
    pipe.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
