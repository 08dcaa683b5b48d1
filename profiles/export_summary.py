"""Turns an ncu --set full report into two summaries (profiles/out/ is kept out of git):
    python profiles/export_summary.py <report>.ncu-rep <tag>
 -> profiles/out/<tag>_ncu_full_summary.csv  (one column per kernel)
 -> profiles/out/<tag>_traffic.json (DRAM bytes per launch)"""
import csv
import json
import os
import re
import subprocess
import sys

rep, tag = sys.argv[1], sys.argv[2]
HERE = os.path.dirname(os.path.abspath(__file__))
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout.splitlines()
rows = list(csv.reader(raw))
hdr, units, data = rows[0], rows[1], rows[2:]
KEEP = ["Grid Size", "Block Size", "gpu__time_duration.sum", "smsp__inst_executed.sum", "sm__inst_executed.avg.per_cycle_active",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "smsp__thread_inst_executed_per_inst_executed.ratio", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "dram__throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_bytes.sum", "l1tex__t_bytes.sum",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
        "launch__shared_mem_per_block_static", "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_registers",
        "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_warps", "sm__maximum_warps_per_active_cycle_pct",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_drain_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio"]
idx = {h: i for i, h in enumerate(hdr)}
names = []
for r in data:
    n = re.sub(r"\(.*", "", r[idx["Kernel Name"]]).replace("void ", "").replace("<unnamed>::", "").strip()
    names.append(n)
OUT = os.path.join(HERE, "out")
os.makedirs(OUT, exist_ok=True)
with open(os.path.join(OUT, tag + "_ncu_full_summary.csv"), "w", newline="") as f:
    w = csv.writer(f)
    w.writerow(["metric", "unit"] + names)
    for k in KEEP:
        if k in idx:
            w.writerow([k, units[idx[k]]] + [r[idx[k]] for r in data])
traffic = {"workload": "7680x4320 RGB q75 rst36 S-photo",
           "source": "ncu --set full --clock-control none, profiles/run_step.py 8k photo, report %s (kept out of git)" % os.path.basename(rep),
           "kernels": {}}
for n, r in zip(names, data):
    def val(k):
        v, u = float(r[idx[k]]), units[idx[k]]
        return v * {"Mbyte": 1e6, "Kbyte": 1e3, "Gbyte": 1e9, "byte": 1.0}.get(u, 1.0)
    dur, du = float(r[idx["gpu__time_duration.sum"]]), units[idx["gpu__time_duration.sum"]]
    traffic["kernels"][n] = {"dram_bytes_read": val("dram__bytes_read.sum"), "dram_bytes_write": val("dram__bytes_write.sum"),
                             "duration_us_under_ncu": dur * {"us": 1.0, "ns": 1e-3, "ms": 1e3}.get(du, 1.0)}
json.dump(traffic, open(os.path.join(OUT, tag + "_traffic.json"), "w"), indent=1)
print(json.dumps(traffic["kernels"], indent=1))
