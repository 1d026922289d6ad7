"""Cost of RenderLayers blocks 1..3 on lights and shadow items, on the bench world (config #3: 1,000,366 rows, 256 point
lights, 4 views).

  clusters   the cluster stage of STAGE_ALL frames (b200vis_set_profiling's cluster interval, per frame), without light
             blocks (every light on layer 0) and with half of the lights on layer 70 only (block 0 empty, so the kernel
             reads their blocks 1..3 for every view); the views hold layers 0 and 70, the light rows too, so both
             configurations cluster the same lights the same way
  shadows    b200vis_run_shadow_culling with the 40-item set of tools/shadow_outputs_timing.py (16 point, 8 spot,
             4 views x 4 cascades), CUDA events around it: item blocks off (k_shadow_cull<false>) against half of the items
             on layer 70 only (k_shadow_cull<true>, every row's blocks loaded); every row holds layers 0 and 70, so the lists
             are the same
The two configurations alternate, three rounds of --reps runs each (medians).  Prints one JSON line with the card and its
power limit.  Run from the repository root: python tools/light_layers_timing.py [--reps 20]"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from cull_outputs_timing import card  # noqa: E402

IDENT9 = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1], np.float32)
L70 = np.array([0, 1 << 6, 0], np.uint64)          # layer 70 = block 1, bit 6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import torch
    import bevy_b200 as bb
    from bevy_b200 import abi, scenes
    assert torch.cuda.is_available(), "this tool measures the GPU: no CUDA device"
    name, power = card()
    sc = scenes.forest()
    n, V, L = sc.n, len(sc.cameras), len(sc.light_row)
    pipe = bb.VisibilityPipeline(sc)
    c = pipe.ctx
    stream = torch.cuda.Stream()
    c.set_stream(stream.cuda_stream)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    res = {"metric": "light_layers_timing", "card": name, "power_limit": power, "rows": n, "lights": L, "views": V}

    # every row and view: layers 0 and 70
    c.upload_render_layers_ext(0, np.tile(L70, (n, 1)))
    half = np.arange(L) % 2 == 1
    l0_with = np.where(half, 0, 1).astype(np.uint64)
    ext_with = np.where(half[:, None], L70[None], 0).astype(np.uint64)

    def frame():
        pipe.update_views()
        for v in range(V):
            c.set_view_render_layers_ext(v, L70)
        c.run(abi.STAGE_ALL)

    def lights(with_blocks):
        if with_blocks:
            c.set_lights(sc.light_row, sc.light_range, l0_with)
            c.set_light_render_layers_ext(ext_with)
        else:
            c.set_lights(sc.light_row, sc.light_range, np.ones(L, np.uint64))

    def cluster_ms(reps):
        c.set_profiling(True)
        c.collect_stage_times_ms()
        for _ in range(reps):
            frame()
            pipe.read_feedback()
        _, _, cl, frames = c.collect_stage_times_ms()
        c.set_profiling(False)
        return round(cl / max(frames, 1), 4)

    runs = {"without_blocks": [], "with_blocks": []}
    counts = {}
    for _ in range(3):
        for key, wb in (("without_blocks", False), ("with_blocks", True)):
            lights(wb)
            for _ in range(3):
                frame(); pipe.read_feedback()
            runs[key].append(cluster_ms(args.reps))
            st = pipe.read_feedback()
            counts[key] = [int(st.cluster_index_count[v]) for v in range(V)]
    res["cluster_stage_ms_per_frame"] = runs
    res["cluster_index_counts"] = counts
    assert counts["without_blocks"] == counts["with_blocks"], counts

    # ---- shadows: the 40 items ----
    caster = np.ones(n, np.uint8); caster[sc.light_row] = 0
    c.upload_shadow_casters(0, caster)
    lights(False)
    for _ in range(3):
        frame()
    c.synchronize()
    gt, _ = c.download_global_transforms(0, n)
    listed = set(np.concatenate([c.download_visible(v) for v in range(V)]).tolist())
    on = [o for o in range(L) if int(sc.light_row[o]) in listed]
    assert len(on) >= 24, f"only {len(on)} lights are in some view's VisibleEntities"
    items = []
    for k, o in enumerate(on[:24]):
        row = int(sc.light_row[o])
        fr = abi.host_point_light_frusta(gt[row], float(sc.light_range[o]))
        kind = 0 if k < 16 else 1
        items.append(dict(kind=kind, light_row=row, range=float(sc.light_range[o]), range_view_index=0,
                          frusta=fr if kind == 0 else fr[k % 6]))
    for v in range(V):
        for cc, rr in enumerate((10.0, 30.0, 90.0, 270.0)):
            centre = np.asarray(sc.cameras[v].gt[9:12], np.float32)
            fr = abi.host_point_light_frusta(np.concatenate([IDENT9, centre]).astype(np.float32), rr)[(v + cc) % 6]
            items.append(dict(kind=2, range_view_index=-1, layer_mask=1, frusta=fr))
    ni = len(items)
    ihalf = np.arange(ni) % 2 == 1
    items_with = [dict(it, layer_mask=0 if ihalf[i] else 1) for i, it in enumerate(items)]
    iext = np.where(ihalf[:, None], L70[None], 0).astype(np.uint64)

    def shadow_ms(reps):
        ts = []
        for _ in range(reps):
            a, b = ev(), ev()
            a.record(stream)
            c.run_shadow_culling()
            b.record(stream)
            b.synchronize()
            ts.append(a.elapsed_time(b))
        return round(float(np.median(ts)), 4)

    def entries():
        return sum(len(c.download_shadow_visible(i, f)) for i in range(ni) for f in range(6))

    sruns = {"without_blocks": [], "with_blocks": []}
    totals = {}
    for _ in range(3):
        c.set_shadow_items(items)
        shadow_ms(3); sruns["without_blocks"].append(shadow_ms(args.reps))
        totals["without_blocks"] = entries()
        c.set_shadow_items(items_with)
        c.set_shadow_item_render_layers_ext(iext)
        shadow_ms(3); sruns["with_blocks"].append(shadow_ms(args.reps))
        totals["with_blocks"] = entries()
    res["run_shadow_culling_ms_median"] = sruns
    res["shadow_entries"] = totals
    assert totals["without_blocks"] == totals["with_blocks"], totals
    res["shadow_items"] = {"point": 16, "spot": 8, "cascades": 4 * V}
    pipe.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
