"""Tile-pass time with GlobalTransforms written by other systems pending (b200vis_write_global_transforms_scattered), on
the bench world (config #3: 3922 trees x 255 nodes + 256 lights = 1,000,366 rows, 4 views, every root moves each frame).

Cases, alternated round by round in one process so that clock and thermal drift hit all of them alike:
  none      no writes: the frame runs kernel 1b as it is without the feature;
  one       one row with children (a tree's first child) written every frame: the marked instantiation of kernel 1b;
  percent1  1 % of the rows (10,003, random, fixed) written every frame.
The tile pass is what b200vis_set_profiling brackets (the tile kernel launches of b200vis_run; the write itself is not
in it).  Prints one JSON line with the card and its power limit.
Run from the repository root: python tools/external_gt_timing.py [--rounds 5] [--frames 40]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bevy_b200 as bb  # noqa: E402
from bevy_b200 import scenes  # noqa: E402


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
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=40)
    args = ap.parse_args()
    sc = scenes.forest(3922, 8, 256)
    pipe = bb.VisibilityPipeline(sc)
    c = pipe.ctx
    rng = np.random.default_rng(1)
    one = np.array([int(sc.roots[0]) + 1], np.uint32)                  # the first child of the first tree
    pct = np.sort(rng.choice(sc.n, size=sc.n // 100, replace=False)).astype(np.uint32)
    for _ in range(3):                                                 # warm-up: first-touch launches, converged state
        pipe.run_frame()
    c.synchronize()
    gt, _ = c.download_global_transforms(0, sc.n, want_changed=False)
    cases = {"none": None, "one": one, "percent1": pct}
    per = {k: [] for k in cases}
    f = 0
    for _ in range(args.rounds):
        for name, rows in cases.items():
            c.set_profiling(True)
            for _ in range(args.frames):
                f += 1
                scenes.advance_cameras(sc, 0.02)
                r, t = scenes.mutate_roots(sc, f)
                c.upload_transforms_scattered(r, t)
                if rows is not None:
                    c.write_global_transforms_scattered(rows, gt[rows])
                pipe.update_views()
                pipe.run_frame()
                pipe.read_feedback()
            c.synchronize()
            tile, _, _, k = c.collect_stage_times_ms()
            c.set_profiling(False)
            per[name].append(tile / max(k, 1) * 1e3)
    name, limit = card()
    out = {"what": "tile pass per frame, us (median over rounds; every round's value listed)", "rows": sc.n,
           "frames_per_round": args.frames, "card": name, "power_limit": limit}
    for k, v in per.items():
        out[k] = {"median_us": float(np.median(v)), "rounds_us": [round(x, 2) for x in v]}
    print(json.dumps(out))
    pipe.close()


if __name__ == "__main__":
    main()
