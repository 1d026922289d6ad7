"""Cost of views past the eighth on the bench world (config #3: 3922 trees x 255 nodes + 256 lights = 1,000,366 rows, every
root moves each frame), for 4, 8, 9, 16, 24 and 32 cameras at the origin, yaw 2 pi k / V.

Views 0..7 are culled inside the tile pass; every further group of up to eight views is one extra k_cull pass (MERGE
instantiation) behind it.  Per camera count this prints, in microseconds per frame:
  tile_groups  the profiled tile window (tile pass + group passes + light snapshot; b200vis_set_profiling)
  groups       tile_groups minus tile_groups of the 8-camera world (the group passes alone, by difference)
  expand, clusters   the profiled tail stages
  e2e          wall time per frame with profiling off (update_views + run_frame + read_feedback)
with the frames pipelined (default) and serial (B200VIS_PIPELINE=0, in its own interpreter: the switch is read once).
Profiled and end-to-end runs are separate.  Prints one JSON line per mode with the card and its power limit.
Run from the repository root: python tools/view_group_timing.py [--frames 40] [--rounds 3]"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

COUNTS = (4, 8, 9, 16, 24, 32)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [x.strip() for x in out.split(",")]
        return name, limit
    except Exception:
        return "unknown", "unknown"


def measure(frames, rounds):
    import bevy_b200 as bb
    from bevy_b200 import scenes
    res = {}
    for V in COUNTS:
        sc = scenes.forest(3922, 8, 256)
        sc.cameras = [scenes._camera(2.0 * math.pi * k / V) for k in range(V)]
        pipe = bb.VisibilityPipeline(sc)
        c = pipe.ctx
        f = 0

        def frame():
            nonlocal f
            f += 1
            scenes.advance_cameras(sc, 0.02)
            r, t = scenes.mutate_roots(sc, f)
            c.upload_transforms_scattered(r, t)
            pipe.update_views()
            pipe.run_frame()
            pipe.read_feedback()
        for _ in range(5):
            frame()
        prof, e2e = [], []
        for _ in range(rounds):
            c.set_profiling(True)
            for _ in range(frames):
                frame()
            c.synchronize()
            tile, expand, clus, k = c.collect_stage_times_ms()
            c.set_profiling(False)
            prof.append((tile / k * 1e3, expand / k * 1e3, clus / k * 1e3))
            c.synchronize()
            t0 = time.perf_counter()
            for _ in range(frames):
                frame()
            c.synchronize()
            e2e.append((time.perf_counter() - t0) / frames * 1e6)
        p = np.median(np.array(prof), 0)
        res[V] = {"tile_groups": round(float(p[0]), 1), "expand": round(float(p[1]), 1), "clusters": round(float(p[2]), 1),
                  "e2e": round(float(np.median(e2e)), 1)}
        pipe.close()
    for V in COUNTS:
        res[V]["groups"] = round(res[V]["tile_groups"] - res[8]["tile_groups"], 1) if V > 8 else 0.0
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--child", action="store_true")
    args = ap.parse_args()
    if args.child:
        print(json.dumps(measure(args.frames, args.rounds)))
        return
    name, limit = card()
    for mode, env in (("pipelined", {}), ("serial", {"B200VIS_PIPELINE": "0"})):
        e = {k: v for k, v in os.environ.items() if not k.startswith("B200VIS_")}
        e.update(env)
        out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--frames", str(args.frames), "--rounds",
                              str(args.rounds)], env=e, capture_output=True, text=True, check=True).stdout.strip().splitlines()[-1]
        print(json.dumps({"mode": mode, "rows": 1000366, "unit": "us per frame", "card": name, "power_limit": limit,
                          "by_cameras": json.loads(out)}))


if __name__ == "__main__":
    main()
