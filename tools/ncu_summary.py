#!/usr/bin/env python
"""Summarise ncu captures brought back in gpurun_out/ into profiles/ (tracked).

  python tools/ncu_summary.py launches gpurun_out/launches.csv profiles/r01_launches.md
  python tools/ncu_summary.py report   gpurun_out/prof_raster.ncu-rep profiles/r01_raster.md [--traffic-key raster]
"""
import collections
import csv
import json
import os
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size",
    "launch__block_size", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
    "smsp__inst_executed.sum", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio",
]


def launches(src, dst):
    rows = [r for r in csv.reader(open(src)) if len(r) > 5]
    hdr, data = None, []
    for r in rows:
        if r[0] == "ID":
            hdr = r
            continue
        if hdr and len(r) == len(hdr):
            data.append(dict(zip(hdr, r)))
    agg = collections.OrderedDict()
    for d in data:
        agg.setdefault(d["Kernel Name"].split("(")[0], []).append(float(d["Metric Value"].replace(",", "")) / 1000.0)
    ours = {k: v for k, v in agg.items() if ("gs::" in k or "k_" in k) and "at::" not in k}
    per_frame = sum(sum(v) / len(v) for v in ours.values())
    with open(dst, "w") as f:
        f.write(f"# ncu launch list ({os.path.basename(src)}): gpu__time_duration.sum per launch, --clock-control none\n\n")
        f.write("Per-launch times are cold-cache and serialised: compare SHARES, not absolutes.\n\n")
        f.write("| kernel | launches | mean us | share of frame |\n|---|---|---|---|\n")
        for k, v in agg.items():
            m = sum(v) / len(v)
            share = f"{100 * m / per_frame:.1f} %" if k in ours and "k_pack" not in k else "-"
            f.write(f"| `{k}` | {len(v)} | {m:.1f} | {share} |\n")
        f.write(f"\nSum of our per-frame kernels (mean): {per_frame:.1f} us\n")
    print(open(dst).read())


def report(src, dst, traffic_key=None):
    out = subprocess.run(["ncu", "-i", src, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    with open(dst, "w") as f:
        f.write(f"# ncu --set full summary of {os.path.basename(src)} (--clock-control none)\n")
        for r in rows[2:]:
            name = r[hdr.index("Kernel Name")]
            f.write(f"\n## {name[:110]}\n\n| metric | value | unit |\n|---|---|---|\n")
            vals = {}
            for k in KEYS:
                if k in hdr:
                    i = hdr.index(k)
                    vals[k] = (r[i], units[i])
                    f.write(f"| {k} | {r[i]} | {units[i]} |\n")
            if traffic_key and "dram__bytes_read.sum" in vals:
                def to_bytes(v, u):
                    mult = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}[u]
                    return float(v.replace(",", "")) * mult
                t = to_bytes(*vals["dram__bytes_read.sum"]) + to_bytes(*vals["dram__bytes_write.sum"])
                tp = os.path.join(os.path.dirname(dst), "traffic.json")
                cur = json.load(open(tp)) if os.path.exists(tp) else {}
                cur[traffic_key] = t
                json.dump(cur, open(tp, "w"), indent=1)
                f.write(f"\nDRAM traffic per launch (read + write): {t/1e6:.1f} MB -> profiles/traffic.json['{traffic_key}']\n")
    print(open(dst).read())


def stage_traffic(src, key, pattern, dst_dir):
    """Sum of mean DRAM bytes (read + write) per launch over the kernels whose name matches `pattern`
    (one frame's worth of a multi-kernel stage) -> profiles/traffic.json[key]."""
    import re
    out = subprocess.run(["ncu", "-i", src, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    ik, ir, iw = hdr.index("Kernel Name"), hdr.index("dram__bytes_read.sum"), hdr.index("dram__bytes_write.sum")
    mult = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
    per = collections.OrderedDict()
    for r in rows[2:]:
        name = r[ik].split("(")[0].strip()
        if not re.search(pattern, name):
            continue
        b = float(r[ir].replace(",", "")) * mult[units[ir]] + float(r[iw].replace(",", "")) * mult[units[iw]]
        per.setdefault(name, []).append(b)
    total = sum(sum(v) / len(v) for v in per.values())
    tp = os.path.join(dst_dir, "traffic.json")
    cur = json.load(open(tp)) if os.path.exists(tp) else {}
    cur[key] = total
    json.dump(cur, open(tp, "w"), indent=1)
    for k, v in per.items():
        print(f"{k:40s} {sum(v)/len(v)/1e6:8.1f} MB x{len(v)}")
    print(f"{key}: {total/1e6:.1f} MB per frame")


if __name__ == "__main__":
    if sys.argv[1] == "launches":
        launches(sys.argv[2], sys.argv[3])
    elif sys.argv[1] == "stage":
        stage_traffic(sys.argv[2], sys.argv[3], sys.argv[4], sys.argv[5])
    else:
        tk = sys.argv[sys.argv.index("--traffic-key") + 1] if "--traffic-key" in sys.argv else None
        report(sys.argv[2], sys.argv[3], tk)
