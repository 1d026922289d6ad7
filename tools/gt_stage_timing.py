"""Full staging (B200VIS_GT_STAGE=full) against row-0 staging of the old GlobalTransform in kernel 1b (the default), in one
process tree on one card.

1. bench.py --steps 2000 --no-cpu-baseline --no-next-rows, --runs times per arm, the arms alternated run by run: value,
   roofline.kernel_ms / expand_ms / cluster_ms, parity_checked, clocks and device of every run, and the median value per arm.
2. The profiled tile window (b200vis_set_profiling), µs per frame, on the bench world (config #3) under four motions:
   bench (every root moves, as bench.py), sparse8 (8 roots move, the e2e_sparse pattern), static (nothing moves) and
   adversarial (roots rotate about x and move in y/z only, so no row 0 ever changes and every row falls back to rows 1-2);
   pipelined (frames back to back) and serial (every frame behind a device synchronise).
Prints one JSON line (and writes it to --out when given).  Run from the repository root:
  python tools/gt_stage_timing.py [--runs 4] [--steps 2000] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ARMS = (("full", {"B200VIS_GT_STAGE": "full"}), ("row0", {}))
MOTIONS = ("bench", "sparse8", "static", "adversarial")


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


def quat_x(a):
    return np.stack([np.sin(a / 2), np.zeros_like(a), np.zeros_like(a), np.cos(a / 2)], axis=-1).astype(np.float32)


def child_tile(frames, rounds):
    """Profiled tile window (µs per frame, median over rounds) per motion, pipelined and serial."""
    import bevy_b200 as bb
    from bevy_b200 import scenes
    out = {}
    for motion in MOTIONS:
        sc = scenes.forest(3922, 8, 256)
        roots = sc.roots.astype(np.int64)
        ang = np.arange(len(roots)) * 0.37
        if motion == "adversarial":
            sc.trs[roots, 3:7] = quat_x(ang)
        pipe = bb.VisibilityPipeline(sc)
        c = pipe.ctx
        f = 0

        def frame(serial):
            nonlocal f
            f += 1
            scenes.advance_cameras(sc, 0.02)
            if motion == "bench":
                r, t = scenes.mutate_roots(sc, f)
                c.upload_transforms_scattered(r, t)
            elif motion == "sparse8":
                r = roots[:8]
                sc.trs[r, 2] += np.float32(0.01)
                c.upload_transforms_scattered(r, sc.trs[r])
            elif motion == "adversarial":
                sc.trs[roots, 3:7] = quat_x(ang + 0.001 * f)
                sc.trs[roots, 1] += np.float32(0.01)
                sc.trs[roots, 2] -= np.float32(0.01)
                c.upload_transforms_scattered(roots, sc.trs[roots])
            pipe.update_views()
            if serial:
                c.synchronize()
            pipe.run_frame()
            pipe.read_feedback()
        res = {}
        for serial in (False, True):
            for _ in range(6):
                frame(serial)
            per = []
            for _ in range(rounds):
                c.synchronize()
                c.set_profiling(True)
                for _ in range(frames):
                    frame(serial)
                c.synchronize()
                tile, _, _, k = c.collect_stage_times_ms()
                c.set_profiling(False)
                per.append(tile / k * 1e3)
            res["serial" if serial else "pipelined"] = round(float(np.median(per)), 2)
        pipe.close()
        out[motion] = res
    return out


def run_child(extra, frames, rounds):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--frames", str(frames), "--rounds", str(rounds)],
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
    ap.add_argument("--skip", default="", help="comma list of parts to skip: bench, shapes")
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", action="store_true")
    args = ap.parse_args()
    if args.child:
        print(json.dumps(child_tile(args.frames, args.rounds)))
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
        res["gain"] = med["row0"] / med["full"] - 1.0
        res["row0_min_above_full_max"] = min(r["value"] for r in runs["row0"]) > max(r["value"] for r in runs["full"])
        res["kernel_ms_median"] = {a: float(np.median([r["kernel_ms"] for r in runs[a]])) for a in runs}
        res["all_parity_checked"] = all(r["parity_checked"] is True for a in runs for r in runs[a])
    if "shapes" not in skip:
        res["tile_us"] = {arm: run_child(extra, args.frames, args.rounds) for arm, extra in ARMS}
    res["seconds"] = round(time.time() - t0, 1)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
