#!/usr/bin/env python
"""Turns ncu artefacts into small text summaries.

  python tools/ncu_summary.py launches <launches.csv> > rNN_launches.txt
  python tools/ncu_summary.py kernel <prof.ncu-rep>   > rNN_<kernel>_full.txt
"""
import csv
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "launch__occupancy_limit_registers",
        "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_warps", "smsp__inst_executed.sum",
        "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct", "sm__cycles_elapsed.avg",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"]


def launches(path):
    rows = list(csv.reader(open(path)))
    hi = [i for i, r in enumerate(rows) if r and r[0] == "ID"][0]
    hdr = rows[hi]
    kn, mv, mu = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    agg = {}
    for r in rows[hi + 1:]:
        if len(r) <= mv:
            continue
        try:
            v = float(r[mv].replace(",", ""))
        except ValueError:
            continue
        agg.setdefault(r[kn].split("(")[0], []).append(v)
    unit = rows[hi + 1][mu]
    tot = sum(sum(v) for v in agg.values())
    print(f"# ncu --metrics gpu__time_duration.sum --clock-control none  ({path}); cold-cache, serialised: compare SHARES")
    for k, v in sorted(agg.items(), key=lambda kv: -sum(kv[1])):
        print(f"{k[:70]:70s} n={len(v):4d} avg={sum(v) / len(v):10.1f} {unit} share={100 * sum(v) / tot:5.1f}%")


def kernel(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    r = list(csv.reader(out.splitlines()))
    hdr, units, rows = r[0], r[1], r[2:]
    print(f"# ncu --set full --clock-control none ({path}), {len(rows)} launches")
    print("kernel:", rows[0][hdr.index("Kernel Name")][:120])
    for k in KEYS:
        if k in hdr:
            i = hdr.index(k)
            print(f"{k:70s} {units[i]:12s} {[row[i] for row in rows]}")
    stalls = []
    for i, h in enumerate(hdr):
        if "pcsamp_warps_issue_stalled" in h and "not_issued" not in h:
            try:
                stalls.append((float(rows[0][i]), h))
            except ValueError:
                pass
    tot = sum(v for v, _ in stalls) or 1.0
    print("warp stall samples (launch 0):")
    for v, h in sorted(stalls, reverse=True)[:8]:
        print(f"  {100 * v / tot:5.1f}%  {h.replace('smsp__pcsamp_warps_issue_stalled_', '')}")


if __name__ == "__main__":
    {"launches": launches, "kernel": kernel}[sys.argv[1]](sys.argv[2])
