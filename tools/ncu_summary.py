#!/usr/bin/env python
"""Turns ncu outputs into small text summaries (and the profiles/*_traffic.json that bench.py reads).

  python tools/ncu_summary.py launches out/launches.csv          > profiles/rNN_launches.txt
  python tools/ncu_summary.py full     out/prof.ncu-rep          > profiles/rNN_full.txt
"""
import collections
import csv
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "smsp__inst_executed.sum", "smsp__thread_inst_executed_per_inst_executed.ratio",
    "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic", "launch__shared_mem_per_block_static",
    "launch__grid_size", "launch__block_size", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_tensor.sum", "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "lts__t_sector_hit_rate.pct",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
]


def launches(path):
    rows = list(csv.reader(open(path)))
    hdr = [i for i, r in enumerate(rows) if r and r[0] == "ID"][0]
    h = rows[hdr]
    ki, vi = h.index("Kernel Name"), h.index("Metric Value")
    acc = collections.OrderedDict()
    for r in rows[hdr + 2:]:
        if len(r) <= vi:
            continue
        a = acc.setdefault(r[ki].split("(")[0], [0, 0.0])
        a[0] += 1
        a[1] += float(r[vi].replace(",", ""))
    tot = sum(a[1] for a in acc.values())
    print(f"# ncu --metrics gpu__time_duration.sum --clock-control none (cold-cache, serialised: compare SHARES)")
    print(f"{'kernel':28s} {'launches':>8s} {'total_ms':>10s} {'avg_us':>10s} {'share':>7s}")
    for n, (c, t) in sorted(acc.items(), key=lambda kv: -kv[1][1]):
        print(f"{n:28s} {c:8d} {t / 1e6:10.3f} {t / c / 1e3:10.1f} {t / tot:7.3f}")


def full(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    h, units = rows[0], rows[1]
    for r in rows[2:]:
        print("=" * 100)
        print(r[h.index("Kernel Name")])
        for k in KEYS:
            if k in h:
                print(f"  {k:88s} {r[h.index(k)]:>16s} {units[h.index(k)]}")


def traffic(path):
    """JSON for bench.py's `roofline.traffic` / `roofline.issue`: per kernel (bench.py's short names) the DRAM
    bytes and warp instructions of ONE launch (mean over the captured launches) from an `ncu --set full` report."""
    import json
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    h = rows[0]
    acc = collections.OrderedDict()
    alias = {"k_tc_pass<0>": "k_tc_top2", "k_tc_pass<1>": "k_tc_filter",
             "k_mb_blur_tma<6>": "k_mb_blur", "k_mb_blur_tma<9>": "k_mb_blur"}
    for r in rows[2:]:
        name = r[h.index("Kernel Name")].split("(")[0].replace("void ", "").strip()
        name = alias.get(name, name)
        a = acc.setdefault(name, {"n": 0, "dram": 0.0, "inst": 0.0, "ns": 0.0, "sm_hz": 0.0})
        f = lambda k: float(r[h.index(k)].replace(",", "")) if k in h and r[h.index(k)] not in ("", "n/a") else 0.0
        unit = lambda k: rows[1][h.index(k)] if k in h else ""
        scale = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
        a["n"] += 1
        a["dram"] += f("dram__bytes_read.sum") * scale.get(unit("dram__bytes_read.sum"), 1.0) + \
            f("dram__bytes_write.sum") * scale.get(unit("dram__bytes_write.sum"), 1.0)
        a["inst"] += f("smsp__inst_executed.sum")
        a["ns"] += f("gpu__time_duration.sum") * {"ns": 1.0, "us": 1e3, "ms": 1e6, "s": 1e9}.get(unit("gpu__time_duration.sum"), 1.0)
        a["sm_hz"] += f("sm__cycles_elapsed.avg.per_second") * {"Hz": 1.0, "Khz": 1e3, "Mhz": 1e6, "Ghz": 1e9}.get(unit("sm__cycles_elapsed.avg.per_second"), 1.0)
    res = {k: {"dram_bytes_per_launch": v["dram"] / v["n"], "warp_instructions_per_launch": v["inst"] / v["n"],
               "ncu_duration_ms": v["ns"] / v["n"] / 1e6, "ncu_sm_hz": v["sm_hz"] / v["n"]} for k, v in acc.items()}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    {"launches": launches, "full": full, "traffic": traffic}[sys.argv[1]](sys.argv[2])
