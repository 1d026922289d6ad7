"""Cost of the light-visibility systems' device-written outputs on the bench world (config #3: 1,000,366 rows, 4 views),
with 16 point lights, 8 spot lights and one directional light x 4 views x 4 cascades (40 shadow items).

  run        b200vis_run_shadow_culling, CUDA events around it, without the sink (row lists of max_entities rows) and with
             b200vis_set_shadow_entities_sink (row lists of one row), alternated in one run
  emission   k_shadow_offsets + k_expand_shadow<true> against k_expand_shadow<false>, from a torch.profiler run of its own
  set_vis    the second b200vis_writeback_tables(WB_SET_VISIBLE) after the shadow stage, on one shuffled table over plain
             numpy memory, CUDA events around it (the table bytes as the camera pass left them)
  replaced   what the sink replaces: all 6 x items b200vis_download_shadow_visible calls plus a numpy row -> Entity map,
             host clock
  cpu        the oracle's single-threaded C restatement of check_dir_light_mesh_visibility and
             check_point_light_mesh_visibility over the same world and items, host clock.  A CPU restatement, not Bevy.
Prints one JSON line with the card and its power limit.
Run from the repository root: python tools/shadow_outputs_timing.py [--reps 20]"""
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
    args = ap.parse_args()
    import torch
    import bevy_b200 as bb
    import oracle as orc
    from bevy_b200 import abi, scenes
    assert torch.cuda.is_available(), "this tool measures the GPU: no CUDA device"
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
    items, dir_items = [], []
    for k, o in enumerate(on[:24]):
        row = int(sc.light_row[o])
        fr = abi.host_point_light_frusta(gt[row], float(sc.light_range[o]))
        kind = 0 if k < 16 else 1
        items.append(dict(kind=kind, light_row=row, range=float(sc.light_range[o]), range_view_index=0, frusta=fr if kind == 0 else fr[k % 6]))
    for v in range(V):
        frs = []
        for cc, rr in enumerate((10.0, 30.0, 90.0, 270.0)):
            centre = np.asarray(sc.cameras[v].gt[9:12], np.float32)
            fr = abi.host_point_light_frusta(np.concatenate([IDENT9, centre]).astype(np.float32), rr)[(v + cc) % 6]
            items.append(dict(kind=2, range_view_index=-1, layer_mask=1, frusta=fr)); frs.append(fr)
        dir_items.append((np.stack(frs), 1, -1))
    n_items = len(items)
    res = {"metric": "shadow_outputs_timing", "card": card()[0], "power_limit": card()[1], "rows": n, "views": V,
           "items": {"point": 16, "spot": 8, "cascades": 4 * V}}
    ent = torch.zeros(16 * n, dtype=torch.int64).pin_memory().numpy().view(np.uint64)
    off = torch.zeros(n_items * 6 + 1, dtype=torch.int32).pin_memory().numpy().view(np.uint32)
    act = torch.zeros(n_items, dtype=torch.uint8).pin_memory().numpy()

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

    def without():
        c.set_shadow_entities_sink(None, None, None)
        c.set_shadow_items(items, 0)

    def with_sink():
        c.set_shadow_entities_sink(ent, off, act)
        c.set_shadow_items(items, 1)

    runs = {"without_sink": [], "with_sink": []}
    for _ in range(3):                                        # alternate the two configurations
        without(); shadow_ms(3); runs["without_sink"].append(shadow_ms(args.reps))
        with_sink(); shadow_ms(3); runs["with_sink"].append(shadow_ms(args.reps))
    res["run_shadow_culling_ms_median"] = runs
    c.synchronize()
    res["entries"] = int(off[n_items * 6])
    assert res["entries"] <= len(ent)

    from torch.profiler import ProfilerActivity, profile
    k_us = {}
    for name, setup in (("without_sink", without), ("with_sink", with_sink)):
        setup()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                c.run_shadow_culling()
            c.synchronize()
        for e in prof.key_averages():
            if "k_shadow" in e.key or "k_expand_shadow" in e.key:
                k_us[name + ":" + e.key.split("(")[0].split("::")[-1]] = round(e.device_time_total / max(e.count, 1), 2)
    res["kernel_us_per_run"] = k_us

    # ---- the second WB_SET_VISIBLE, behind the shadow stage ----
    tabs, buf = abi.host_tables([n])
    c.set_tables(tabs)
    c.set_table_rows(0, 0, np.random.default_rng(0).permutation(n).astype(np.uint32))
    with_sink()
    ts = []
    for r in range(args.reps + 3):
        pipe.update_views(); c.run(abi.STAGE_ALL)
        c.writeback_tables(abi.WB_SET_VISIBLE, 0, 2 * r)     # the camera pass
        c.run_shadow_culling()
        a, b = ev(), ev()
        a.record(stream)
        c.writeback_tables(abi.WB_SET_VISIBLE, 0, 2 * r + 1)
        b.record(stream)
        b.synchronize()
        pipe.read_feedback()
        if r >= 3:
            ts.append(a.elapsed_time(b))
        tabs[0].vv[:] = (tabs[0].vv & 1) << 1               # reset_view_visibility for the next frame
    res["second_set_visible_ms_median"] = round(float(np.median(ts)), 4)
    vv, _ = c.download_view_visibility(0, n)
    res["rows_visible_after_lights"] = int((vv & 1).sum())

    # ---- the path the sink replaces: every list downloaded, rows mapped to Entity ----
    without()
    c.run_shadow_culling(); c.synchronize()
    host = []
    for _ in range(3):
        t0 = time.perf_counter()
        out = []
        for i in range(n_items):
            for face in range(6):
                out.append(sc.entity_bits[c.download_shadow_visible(i, face)])
        host.append((time.perf_counter() - t0) * 1e3)
    res["download_and_map_ms"] = [round(x, 3) for x in host]
    res["download_entries"] = int(sum(len(x) for x in out))

    # ---- the oracle's C restatement on the host, single-threaded ----
    gt, _ = c.download_global_transforms(0, n)
    vv0 = np.zeros(n, np.uint8); vch = np.zeros(n, np.uint8)
    t0 = time.perf_counter()
    orc.check_dir_light_mesh_visibility(gt, sc.bounds, sc.flags, caster, sc.entity_bits, vv0, vch, dir_items,
                                        layer_mask=sc.layer_mask, range_mask=sc.range_mask)
    for it in items[:24]:
        row = it["light_row"]
        sphere = np.concatenate([gt[row, 9:12], [it["range"]]]).astype(np.float32)[None]
        fr = np.asarray(it["frusta"], np.float32)
        if it["kind"] == 0:
            orc.check_point_light_mesh_visibility(gt, sc.bounds, sc.flags, caster, sc.entity_bits, vv0, vch, sphere, fr[None],
                                                  layer_mask=sc.layer_mask, range_mask=sc.range_mask)
        else:
            orc.check_spot_light_mesh_visibility(gt, sc.bounds, sc.flags, caster, sc.entity_bits, vv0, vch, sphere, fr[None],
                                                 layer_mask=sc.layer_mask, range_mask=sc.range_mask)
    res["cpu_restatement_ms"] = round((time.perf_counter() - t0) * 1e3, 2)
    res["cpu_restatement_threads"] = 1
    del buf
    pipe.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
