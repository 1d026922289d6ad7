"""Fixed (B200VIS_SWEEP_ORDER=fixed) against alternating sweep order (the default), all in one process tree on one card.

1. bench.py --steps 2000 --no-cpu-baseline --no-next-rows, --runs times per arm, the arms alternated run by run: value,
   roofline.kernel_ms / expand_ms / cluster_ms, parity_checked, clocks and device of every run, and the median value per arm.
2. Mechanism control on the bench world (config #3): the profiled tile window (b200vis_set_profiling) per frame for both
   orders, every frame behind a device synchronise, once as is and once with a scratch write of 2x the L2 size between
   frames.  If the alternating order gains by finding the previous pass's rows in L2, the flush should take the gain away.
3. tools/view_group_timing.py's measurement at 8, 9, 16 and 32 cameras for both orders (groups = tile window minus the
   8-camera one: the k_cull group passes alone).
Prints one JSON line (and writes it to --out when given).  Run from the repository root:
  python tools/sweep_order_timing.py [--runs 4] [--steps 2000] [--out FILE]"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

ARMS = (("fixed", {"B200VIS_SWEEP_ORDER": "fixed"}), ("alternating", {}))


def env_of(extra):
    e = {k: v for k, v in os.environ.items() if not k.startswith("B200VIS_")}
    e.update(extra)
    return e


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [x.strip() for x in out.split(",")]
    except Exception:
        return ["unknown", "unknown", "unknown"]


def bench_run(extra, steps):
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps), "--no-cpu-baseline", "--no-next-rows"]
    r = subprocess.run(cmd, env=env_of(extra), capture_output=True, text=True, cwd=ROOT)
    if r.returncode != 0:
        raise RuntimeError(r.stderr[-3000:])
    line = [l for l in r.stdout.strip().splitlines() if l.startswith("{")][-1]
    j = json.loads(line)
    rf = j.get("roofline", {})
    return {"value": j["value"], "kernel_ms": rf.get("kernel_ms"), "expand_ms": rf.get("expand_ms"),
            "cluster_ms": rf.get("cluster_ms"), "parity_checked": j.get("parity_checked"), "clocks": j.get("clocks"),
            "device": j.get("device")}


def child_tile(frames, rounds):
    """Profiled tile window (µs per frame) on the bench world, every frame behind a device synchronise, without and with a
    2x-L2 scratch write between frames."""
    import torch
    import bevy_b200 as bb
    from bevy_b200 import scenes
    l2 = torch.cuda.get_device_properties(0).L2_cache_size
    scratch = torch.empty(2 * l2 // 4, dtype=torch.float32, device="cuda")
    sc = scenes.forest(3922, 8, 256)
    pipe = bb.VisibilityPipeline(sc)
    c = pipe.ctx
    f = 0

    def frame(flush):
        nonlocal f
        f += 1
        scenes.advance_cameras(sc, 0.02)
        r, t = scenes.mutate_roots(sc, f)
        c.upload_transforms_scattered(r, t)
        pipe.update_views()
        c.synchronize()
        if flush:
            scratch.fill_(float(f))
        torch.cuda.synchronize()
        pipe.run_frame()
        pipe.read_feedback()
    out = {"l2_bytes": l2}
    for flush in (False, True):
        for _ in range(6):
            frame(flush)
        per = []
        for _ in range(rounds):
            c.set_profiling(True)
            for _ in range(frames):
                frame(flush)
            c.synchronize()
            tile, _, _, k = c.collect_stage_times_ms()
            c.set_profiling(False)
            per.append(tile / k * 1e3)
        out["flushed" if flush else "warm"] = round(float(np.median(per)), 2)
    pipe.close()
    return out


def child_groups(frames, rounds):
    import view_group_timing as vgt
    vgt.COUNTS = (8, 9, 16, 32)
    return vgt.measure(frames, rounds)


def run_child(kind, extra, frames, rounds):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", kind, "--frames", str(frames), "--rounds", str(rounds)],
                       env=env_of(extra), capture_output=True, text=True, cwd=ROOT)
    if r.returncode != 0:
        raise RuntimeError(r.stderr[-3000:])
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=4)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip", default="", help="comma list of parts to skip: bench, control, groups")
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", default=None)
    args = ap.parse_args()
    if args.child == "tile":
        print(json.dumps(child_tile(args.frames, args.rounds)))
        return
    if args.child == "groups":
        print(json.dumps(child_groups(args.frames, args.rounds)))
        return
    skip = set(args.skip.split(","))
    name, limit, max_sm = card()
    res = {"card": name, "power_limit": limit, "clocks_max_sm": max_sm}
    t0 = time.time()
    if "bench" not in skip:
        runs = {a: [] for a, _ in ARMS}
        for i in range(args.runs):
            for arm, extra in (ARMS if i % 2 == 0 else ARMS[::-1]):
                runs[arm].append(bench_run(extra, args.steps))
        res["bench"] = runs
        med = {a: float(np.median([r["value"] for r in runs[a]])) for a in runs}
        res["value_median"] = med
        res["value_spread"] = {a: (max(r["value"] for r in runs[a]) - min(r["value"] for r in runs[a])) / med[a] for a in runs}
        res["gain"] = med["alternating"] / med["fixed"] - 1.0
        res["kernel_ms_median"] = {a: float(np.median([r["kernel_ms"] for r in runs[a]])) for a in runs}
    if "control" not in skip:
        res["tile_us_control"] = {arm: run_child("tile", extra, args.frames, args.rounds) for arm, extra in ARMS}
    if "groups" not in skip:
        res["view_groups_us"] = {arm: run_child("groups", extra, args.frames, args.rounds) for arm, extra in ARMS}
    res["seconds"] = round(time.time() - t0, 1)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
