"""How much of the next tile pass the pipelined frame tail displaces (debug build, not the product library).

    cd bevy_b200/csrc && nvcc <the flags of bevy_b200/build.py> -DB200VIS_TILE_TIMING \
        -o ../../build/libb200vis_timing.so kernels.cu api.cu host_view.cpp
    B200VIS_LIB=build/libb200vis_timing.so python tools/tail_displacement.py [--frames N] [--json out.json]

In pipelined frames the tail of frame f (visible-list expansion, cluster kernel) runs on high-priority streams beside the
tile pass of frame f+1, and its CTAs hold registers the tile pass's persistent grid needs.  The timing build logs, for
every CTA of kernel 1b, of k_expand_visible and of k_cluster_fused, the %globaltimer when it starts (kernel 1b: when it may
start its first tile) and when it exits.  Over the bench's device-resident loop (bench.py's Rig: the 1M-entity world,
recorded frame constants, frames back to back) this prints:

  * per tile-pass launch, how late each kernel-1b CTA starts after the launch's first CTA: the histogram, and the share
    of CTAs more than 5 us late;
  * the tail's SM-us per frame: CTA lifetime x the share of an SM's registers the CTA holds (threads x registers / 64 K),
    in all and inside the next tile pass's window;
  * the tile-window time (collect_stage_times_ms) of the pipelined loop, and of the same loop with B200VIS_PIPELINE=0
    (a child process: the switch is read when a context is created), where no tail runs beside the tile pass.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

REC = np.dtype([("t0", "<u8"), ("t1", "<u8"), ("kind", "<u4"), ("tag", "<u4"), ("blk", "<u4"), ("threads", "<u4")])
# registers per thread (-Xptxas -v, sm_90a, allocated in steps of 8) by (kind, CTA threads): the 1024-thread expand of
# earlier builds used 32, every other shape runs at its 64-register launch bound
REGS = {(1, 1024): 32}
BINS_US = [0, 1, 2, 5, 10, 15, 20, 30, 50, 1e9]


def make_rig():
    import torch
    import bench                      # bench.py keeps the real stdout aside for its JSON line: give it back
    os.dup2(bench.REAL_STDOUT, 1)
    sys.stdout = sys.__stdout__
    import bevy_b200 as bb
    from bevy_b200 import parallel, scenes
    saved, sys.argv = sys.argv, [sys.argv[0]]       # bench.py's defaults: the bench world
    args = bench.parse_args()
    sys.argv = saved
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    rig = bench.Rig(args, torch, None, bb, scenes, parallel, "strong", 1, 0, 0, dev, stream)
    rig.ctx.run(bb.STAGE_ALL)
    rig.pipe.read_feedback()
    rig.value_setup()
    return torch, rig


def stage_times(rig, frames):
    rig.ctx.set_profiling(True)
    for i in range(frames):
        rig.value_step(i)
    t, e, c, nf = rig.ctx.collect_stage_times_ms()
    rig.ctx.set_profiling(False)
    return {"tile_us": 1e3 * t / nf, "expand_us": 1e3 * e / nf, "cluster_us": 1e3 * c / nf, "frames": nf}


def window_only(frames):
    torch, rig = make_rig()
    for i in range(50):
        rig.value_step(i)
    torch.cuda.synchronize()
    out = stage_times(rig, frames)
    rig.close()
    return out


def sm_share(recs):
    """Share of one SM's 64 K registers each record's CTA holds."""
    return np.array([int(n) * REGS.get((int(k), int(n)), 64) / 65536 for k, n in zip(recs["kind"], recs["threads"])])


def analyse(recs, frames):
    tile = recs[recs["kind"] == 0]
    tail = recs[recs["kind"] != 0]
    delays, launches = [], []
    overlap_sm_us = 0.0
    for tag in np.unique(tile["tag"]):
        g = tile[tile["tag"] == tag]
        t_begin, t_end = int(g["t0"].min()), int(g["t1"].max())
        d = (g["t0"].astype(np.int64) - t_begin) / 1e3
        delays.append(d)
        lo = np.maximum(tail["t0"].astype(np.int64), t_begin)
        hi = np.minimum(tail["t1"].astype(np.int64), t_end)
        share = sm_share(tail)
        ov = float((np.clip(hi - lo, 0, None) * share).sum()) / 1e3
        overlap_sm_us += ov
        launches.append({"ctas": int(len(g)), "window_us": (t_end - t_begin) / 1e3, "late_5us": float((d > 5).mean()),
                         "tail_sm_us_inside": ov})
    d = np.concatenate(delays) if delays else np.zeros(0)
    hist = np.histogram(d, bins=BINS_US)[0]
    life = (tail["t1"].astype(np.int64) - tail["t0"].astype(np.int64)) / 1e3
    share_all = sm_share(tail)
    per_kind = {}
    for k, name in ((1, "expand"), (2, "clusters")):
        m = tail["kind"] == k
        per_kind[name] = {"ctas_per_frame": float(m.sum()) / frames, "threads": sorted({int(x) for x in tail["threads"][m]}),
                          "cta_lifetime_us_mean": float(life[m].mean()) if m.any() else 0.0,
                          "sm_us_per_frame": float((life[m] * share_all[m]).sum()) / frames}
    n_launch = max(len(launches), 1)
    return {
        "tile_launches": len(launches),
        "tile_ctas": int(len(d)),
        "start_delay_hist_us": {f"{BINS_US[i]:g}-{BINS_US[i + 1]:g}": int(hist[i]) for i in range(len(hist))},
        "start_delay_us_p50_p90_p99_max": [float(np.percentile(d, q)) for q in (50, 90, 99, 100)] if len(d) else [],
        "share_late_over_5us": float((d > 5).mean()) if len(d) else 0.0,
        "tail": per_kind,
        "tail_sm_us_per_frame": sum(v["sm_us_per_frame"] for v in per_kind.values()),
        "tail_sm_us_inside_tile_window_per_launch": overlap_sm_us / n_launch,
        "tile_window_us_probe_mean": float(np.mean([x["window_us"] for x in launches])) if launches else 0.0,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--json", default=None, help="also write the numbers here")
    ap.add_argument("--window-only", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.window_only:
        print("WINDOW " + json.dumps(window_only(args.frames)), flush=True)
        return
    torch, rig = make_rig()
    from bevy_b200 import abi
    lib = abi.load_library()
    if not hasattr(lib, "b200vis_debug_probe"):
        raise SystemExit("the library has no residency log: build it with -DB200VIS_TILE_TIMING and point B200VIS_LIB at it")
    lib.b200vis_debug_probe.restype = ctypes.c_longlong
    lib.b200vis_debug_probe.argtypes = [ctypes.c_void_p, ctypes.c_uint]
    for i in range(50):
        rig.value_step(i)
    rig.ctx.join(); torch.cuda.synchronize()
    assert lib.b200vis_debug_probe(None, 0) >= 0
    F = args.frames
    for i in range(50, 50 + F):
        rig.value_step(i)
    rig.ctx.join(); torch.cuda.synchronize()
    buf = np.zeros(1 << 18, REC)
    n = lib.b200vis_debug_probe(ctypes.c_void_p(buf.ctypes.data), len(buf))
    assert 0 <= n <= len(buf), n
    res = analyse(buf[:n], F)
    res["frames"] = F
    res["pipelined"] = stage_times(rig, F)
    rig.close()
    env = dict(os.environ, B200VIS_PIPELINE="0")
    p = subprocess.run([sys.executable, os.path.abspath(__file__), "--window-only", "--frames", str(F)], env=env,
                       capture_output=True, text=True, cwd=ROOT)
    line = [x for x in p.stdout.splitlines() if x.startswith("WINDOW ")]
    if p.returncode != 0 or not line:
        sys.stderr.write(p.stdout[-2000:] + p.stderr[-4000:])
        raise SystemExit("the B200VIS_PIPELINE=0 run failed")
    res["serial"] = json.loads(line[0][7:])
    print(json.dumps(res, indent=1))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
