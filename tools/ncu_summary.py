#!/usr/bin/env python
"""tools/ncu_summary.py REPORT.ncu-rep [--kernel REGEX] [--capture TEXT] [--workload TEXT] [--alg-bytes N] [--note K=V ...]

Reads an `ncu --set full` report (here, no GPU needed: `ncu -i ... --page raw --csv`) and prints the JSON summary that is
that bench.py can read for `roofline.traffic` / `roofline.issue_frac`."""
import argparse
import csv
import io
import json
import re
import subprocess
import sys

KEYS = {
    "gpu_time_us": "gpu__time_duration.sum",
    "dram_bytes_read": "dram__bytes_read.sum",
    "dram_bytes_write": "dram__bytes_write.sum",
    "registers_per_thread": "launch__registers_per_thread",
    "issue_active_pct": "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "warp_instructions": "smsp__inst_executed.sum",
    "pipe_alu_pct": "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
    "pipe_fma_pct": "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
    "pipe_fmaheavy_pct": "sm__inst_executed_pipe_fmaheavy.avg.pct_of_peak_sustained_active",
    "pipe_lsu_pct": "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
    "pipe_xu_pct": "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
    "pipe_tmem_pct": "sm__inst_executed_pipe_tmem.avg.pct_of_peak_sustained_active",
    "shared_wavefronts": "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
    "shared_bank_conflicts": "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
    "warps_active_pct": "sm__warps_active.avg.pct_of_peak_sustained_active",
    "sm_cycles_active_avg": "sm__cycles_active.avg",
    "sm_cycles_elapsed_avg": "sm__cycles_elapsed.avg",
    "dram_throughput_pct": "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "l2_throughput_pct": "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm_throughput_pct": "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "achieved_occupancy_pct": "sm__warps_active.avg.pct_of_peak_sustained_active",
    "shared_mem_per_block": "launch__shared_mem_per_block_dynamic",
}
UNIT = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1, "ms": 1e3, "us": 1, "ns": 1e-3, "s": 1e6}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("report")
    ap.add_argument("--kernel", default=".")
    ap.add_argument("--capture", default="")
    ap.add_argument("--workload", default="")
    ap.add_argument("--alg-bytes", type=float, default=0)
    ap.add_argument("--note", action="append", default=[])
    ap.add_argument("--all", action="store_true", help="one summary per matching launch (a list)")
    a = ap.parse_args()
    raw = subprocess.run(["ncu", "-i", a.report, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units, body = rows[0], rows[1], rows[2:]
    col = {h: i for i, h in enumerate(hdr)}
    outs = []
    for r in body:
        name = r[col["Kernel Name"]]
        if not re.search(a.kernel, name):
            continue

        def val(metric):
            if metric not in col or r[col[metric]] in ("", "n/a"):
                return None
            v = float(r[col[metric]].replace(",", ""))
            u = units[col[metric]]
            return v * UNIT[u] if u in UNIT and ("byte" in u or metric.startswith("gpu__time")) else v
        o = {"capture": a.capture, "kernel": name, "grid": r[col["Grid Size"]] if "Grid Size" in col else None,
             "block": r[col["Block Size"]] if "Block Size" in col else None, "workload": a.workload}
        for k, m in KEYS.items():
            o[k] = val(m)
        if o["dram_bytes_read"] is not None and o["dram_bytes_write"] is not None:
            o["dram_bytes_total"] = o["dram_bytes_read"] + o["dram_bytes_write"]
        if a.alg_bytes:
            o["algorithmic_bytes_per_launch"] = a.alg_bytes
        o["stalls_per_issue"] = {m.group(1): float(r[i]) for h, i in col.items()
                                 for m in [re.match(r"smsp__average_warps_issue_stalled_(\w+)_per_issue_active.ratio", h)] if m and r[i] not in ("", "n/a")}
        for kv in a.note:
            k, _, v = kv.partition("=")
            o[k] = v
        outs.append(o)
        if not a.all:
            break
    if not outs:
        sys.exit("no launch matches " + a.kernel)
    print(json.dumps(outs if a.all else outs[0], indent=1))


if __name__ == "__main__":
    main()
