"""Cost of b200vis_compact_topology on the bench world (config #3, 1,000,366 rows), against today's fallback.

The world is churned until 1 % and then 10 % of its rows are tombstones, with children spawned under existing trees so
that the plan has grown a second pass.  At each level it reports, as one JSON line:
  - the compaction: host clock around the (synchronised) call, split by B200VIS_COMPACT_TRACE into host planning and the
    device part, and the permutation kernel's achieved bandwidth (2 x resident bytes per row x rows) against the H100
    SXM data-sheet 3.35 TB/s;
  - the fallback: b200vis_set_topology plus re-uploading every column (host clock, synchronised);
  - the tile-pass time per frame before and after the compaction (b200vis_set_profiling), and after b200vis_set_topology
    of the compacted world's own row order;
  - the card and its power limit.
Run from the repository root: python tools/compact_timing.py [--frames 20]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["B200VIS_COMPACT_TRACE"] = "1"

import bevy_b200 as bb  # noqa: E402
from bevy_b200 import scenes  # noqa: E402

NO_PARENT = 0xFFFFFFFF
PEAK_TBS = 3.35


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [x.strip() for x in out.split(",")]
        return name, limit
    except Exception:
        return "unknown", "unknown"


def tile_ms(pipe, frames):
    c = pipe.ctx
    c.set_profiling(True)
    for _ in range(frames):
        pipe.update_views()
        pipe.run_frame()
    c.synchronize()
    t, _, _, k = c.collect_stage_times_ms()
    c.set_profiling(False)
    return t / max(k, 1)


def captured_stderr(fn):
    """fn() with file descriptor 2 captured (the library's trace line)."""
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+b") as f:
        os.dup2(f.fileno(), 2)
        try:
            out = fn()
        finally:
            sys.stderr.flush()
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        return out, f.read().decode()


def parse_trace(line):
    w = line.split()
    get = lambda key, off: float(w[w.index(key) + off])
    return dict(host_plan_ms=get("plan", 1), device_part_ms=get("part", 1), row_bytes=int(w[w.index("permute:") + 1]),
                gather_ms=float(w[w.index("gather") + 1]), copy_back_ms=float(w[w.index("copy-back") + 1]))


class World:
    def __init__(self, headroom):
        self.sc = scenes.forest(3922, 8, 256)
        self.pipe = bb.VisibilityPipeline(self.sc, max_entities=self.sc.n + headroom)
        self.pipe.enable_visible_diff()
        self.rng = np.random.default_rng(1)
        self.alive = np.ones(self.sc.n, bool)
        self.parent = self.sc.parent.astype(np.int64).copy()
        self.bits = self.sc.entity_bits.copy()
        self.next_bits = int(self.bits.max()) + 1

    def churn_to(self, dead_fraction, kids=64):
        """Despawns leaves (never a light) until dead_fraction of the rows are tombstones; spawns as many rows, a few of
        them children of existing rows (appended tiles with an external parent: a second pass)."""
        c, n = self.pipe.ctx, len(self.parent)
        want = int(dead_fraction * n) - int((~self.alive).sum())
        if want <= 0:
            return
        has_kids = np.zeros(n, bool); has_kids[self.parent[self.parent < n]] = True
        lights = np.zeros(n, bool); lights[self.sc.light_row] = True
        leaves = np.nonzero(self.alive & ~has_kids & ~lights)[0]
        despawn = np.sort(self.rng.choice(leaves, size=min(want, len(leaves)), replace=False)).astype(np.uint32)
        k = len(despawn)
        parents = np.full(k, NO_PARENT, np.int64)
        parents[:kids] = self.rng.choice(np.nonzero(self.alive & has_kids & ~lights)[0], size=kids)
        bits = np.arange(self.next_bits, self.next_bits + k, dtype=np.uint64)
        self.next_bits += k
        c.edit_topology(despawn=despawn, spawn_parent=parents.astype(np.uint32), spawn_entity_bits=bits)
        trs = np.zeros((k, 10), np.float32); trs[:, 3:7] = (0, 0, 0, 1); trs[:, 7:10] = 1.0
        trs[:, 0:3] = self.rng.uniform(-100, 100, (k, 3))
        bounds = np.zeros((k, 6), np.float32); bounds[:, 3:6] = 0.5
        c.upload_transforms(n, trs)
        c.upload_global_transforms(n, np.tile(np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], np.float32), (k, 1)))
        c.upload_bounds(n, bounds, np.full(k, scenes.F_INHERITED_VISIBLE | scenes.F_HAS_AABB, np.uint8), np.ones(k, np.uint8))
        self.alive[despawn] = False
        self.parent[despawn] = 0xFFFFFFFE
        self.parent = np.concatenate([self.parent, parents])
        self.bits = np.concatenate([self.bits, bits])
        self.alive = np.concatenate([self.alive, np.ones(k, bool)])

    def compact(self):
        c = self.pipe.ctx
        c.synchronize()
        t0 = time.perf_counter()
        o2n, err = captured_stderr(lambda: c.compact_topology())
        wall = (time.perf_counter() - t0) * 1e3
        o2n = o2n.astype(np.int64)
        keep = np.nonzero(o2n != 0xFFFFFFFF)[0]
        p = self.parent.copy(); real = p < len(p); p[real] = o2n[p[real]]
        parent = np.zeros(len(keep), np.int64); parent[o2n[keep]] = p[keep]
        bits = np.zeros(len(keep), np.uint64); bits[o2n[keep]] = self.bits[keep]
        alive = np.zeros(len(keep), bool); alive[o2n[keep]] = self.alive[keep]
        self.parent, self.bits, self.alive = parent, bits, alive
        self.sc.light_row = o2n[self.sc.light_row].astype(np.uint32)
        self.sc.roots = o2n[self.sc.roots].astype(np.uint32)
        trace = [l for l in err.splitlines() if l.startswith("[b200vis_compact]")][-1]
        return wall, parse_trace(trace)

    def fallback_ms(self):
        """set_topology plus every column uploaded again, on the compacted world (host arrays prepared beforehand)."""
        c, n = self.pipe.ctx, len(self.parent)
        gt, _ = c.download_global_transforms(0, n)
        vv, _ = c.download_view_visibility(0, n)
        trs = np.zeros((n, 10), np.float32); trs[:, 3:7] = (0, 0, 0, 1); trs[:, 7:10] = 1.0
        bounds = np.zeros((n, 6), np.float32); bounds[:, 3:6] = 0.5
        flags = np.full(n, scenes.F_INHERITED_VISIBLE | scenes.F_HAS_AABB, np.uint8); cls = np.ones(n, np.uint8)
        parent = self.parent.astype(np.uint32)
        c.synchronize()
        t0 = time.perf_counter()
        c.set_topology(parent, self.bits)
        c.upload_transforms(0, trs)
        c.upload_global_transforms(0, gt)
        c.upload_bounds(0, bounds, flags, cls)
        c.upload_view_visibility(0, vv)
        c.set_lights(self.sc.light_row, self.sc.light_range, self.sc.light_layers)
        c.synchronize()
        return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=20)
    args = ap.parse_args()
    name, limit = card()
    w = World(headroom=120_000)
    for f in range(3):
        w.pipe.update_views(); w.pipe.run_frame()
    base = tile_ms(w.pipe, args.frames)
    for frac in (0.01, 0.10):
        w.churn_to(frac)
        for _ in range(3):                                   # two frames after the despawns: no held result names them
            w.pipe.update_views(); w.pipe.run_frame()
        rows, live, tiles, passes = w.pipe.ctx.topology_summary()
        before = tile_ms(w.pipe, args.frames)
        wall, tr = w.compact()
        rows2, live2, tiles2, passes2 = w.pipe.ctx.topology_summary()
        after = tile_ms(w.pipe, args.frames)
        alg = 2.0 * tr["row_bytes"] * rows2
        print(json.dumps(dict(
            card=name, power_limit=limit, tombstones=round(1 - live / rows, 4), rows_before=rows, rows_after=rows2,
            passes_before=passes, passes_after=passes2, tiles_before=tiles, tiles_after=tiles2,
            compact_wall_ms=round(wall, 3), host_plan_ms=tr["host_plan_ms"], device_part_ms=tr["device_part_ms"],
            permute_bytes_per_row=tr["row_bytes"], permute_gather_ms=tr["gather_ms"], permute_copy_back_ms=tr["copy_back_ms"],
            permute_gather_tb_s=round(alg / (tr["gather_ms"] * 1e-3) / 1e12, 3),
            permute_gather_fraction_of_peak=round(alg / (tr["gather_ms"] * 1e-3) / 1e12 / PEAK_TBS, 3),
            tile_pass_ms_fresh_world=round(base, 4), tile_pass_ms_before=round(before, 4), tile_pass_ms_after=round(after, 4))),
            flush=True)
    for _ in range(2):
        w.pipe.update_views(); w.pipe.run_frame()
    # set_topology of the compacted world's own order and keys, columns left as they are: the tile pass a fresh plan of
    # the same rows gives (the columns' contents are those of the compacted world)
    w.pipe.ctx.set_topology(w.parent.astype(np.uint32), w.bits)
    for _ in range(3):
        w.pipe.update_views(); w.pipe.run_frame()
    same_order = tile_ms(w.pipe, args.frames)
    print(json.dumps(dict(card=name, power_limit=limit, tile_pass_ms_set_topology_same_order=round(same_order, 4),
                          fallback_set_topology_and_uploads_ms=round(w.fallback_ms(), 3))), flush=True)
    w.pipe.close()


if __name__ == "__main__":
    main()
