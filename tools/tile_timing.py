"""Where a kernel-1b CTA spends its time (debug build, not the product library).

    cd bevy_b200/csrc && nvcc <the flags of bevy_b200/build.py> -DB200VIS_TILE_TIMING \
        -o ../../build/libb200vis_timing.so kernels.cu api.cu host_view.cpp
    B200VIS_LIB=build/libb200vis_timing.so python tools/tile_timing.py [--json out.json]

Thread 0 of every CTA of k_propagate_cull_tma sums the clock64 cycles it spends in each phase of a tile over all the CTA's
tiles (and, separately, over its tiles after the first).  Printed, for the last tile-pass launch of a bench-sized frame: the
mean cycles per tile of each phase over every tile of the launch, the same over the tiles after each CTA's first (steady
state), and the spread over CTAs of their own per-tile means.  Thread 0's warp walks the tile's top levels, which every
later level waits for, so its load wait and closing barrier are what the tile's critical path pays for loads and stragglers.
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bevy_b200 as bb  # noqa: E402
from bevy_b200 import abi, scenes  # noqa: E402

PHASES = [
    (1, "descriptor load issued"),
    (2, "load wait (TMA mbarrier)"),
    (3, "dirty phase (opening barrier)"),
    (4, "local affine + level 0"),
    (5, "levels 1.. (walk done)"),
    (6, "ticket, descriptor, next TMA"),
    (7, "cull"),
    (8, "closing barrier"),
    (9, "store issue / loop back"),
]
OVERHEAD = (1, 2, 6, 8)      # descriptor, load wait, ticket + next TMA, closing barrier


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None, help="also write the numbers here")
    args = ap.parse_args()
    sc = scenes.forest(3922, 8, 256)
    pipe = bb.VisibilityPipeline(sc)
    ctx = pipe.ctx
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)
    for f in range(30):
        scenes.advance_cameras(sc)
        rows, trs = scenes.mutate_roots(sc, f + 1)
        ctx.upload_transforms_scattered(rows, trs)
        pipe.update_views_fast()
        ctx.run(bb.STAGE_ALL)
    ctx.join(); torch.cuda.synchronize()
    lib = abi.load_library()
    n = 8192
    buf = np.zeros((n, 32), np.uint64)
    rc = lib.b200vis_debug_tile_phases(ctypes.c_void_p(buf.ctypes.data), n)
    assert rc == 0, rc
    t = buf.astype(np.float64)
    ctas = t[:, 0] > 0
    print(f"CTAs with tiles: {int(ctas.sum())}, tiles: {int(t[:, 0].sum())}, tiles after a CTA's first: {int(t[:, 16].sum())}")
    out = {"ctas": int(ctas.sum()), "tiles": int(t[:, 0].sum()), "all": {}, "steady": {}}
    for key, base in (("all", 0), ("steady", 16)):
        m = t[:, base] > 0
        cnt = t[m, base]
        total = t[m, base + 1:base + 10].sum(axis=1)
        mean_total = total.sum() / cnt.sum()
        label = "every tile" if key == "all" else "tiles after each CTA's first"
        print(f"\n{label}: thread 0, clock64 cycles per tile -- mean over tiles, share, per-CTA mean p10 / p90")
        for ph, name in PHASES:
            x = t[m, base + ph]
            mean = x.sum() / cnt.sum()
            per_cta = x / cnt
            print(f"  {name:38s} {mean:9.0f}  {100 * mean / mean_total:5.1f} %   "
                  f"({np.percentile(per_cta, 10):8.0f} / {np.percentile(per_cta, 90):8.0f})")
            out[key][name] = mean
        ov = sum(t[m, base + ph].sum() for ph in OVERHEAD) / cnt.sum()
        print(f"  {'tile total':38s} {mean_total:9.0f}")
        print(f"  descriptor + load wait + ticket/TMA + closing barrier: {ov:.0f} cycles = {100 * ov / mean_total:.1f} % of a tile")
        out[key]["tile total"] = mean_total
        out[key]["overhead share"] = ov / mean_total
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)
    pipe.close()


if __name__ == "__main__":
    main()
