#!/usr/bin/env python
"""Pull the judged metrics of one kernel launch out of .ncu-rep captures into a small JSON.

usage: ncu_extract.py label=path.ncu-rep [label=path.ncu-rep ...] > summary.json     (takes the LAST captured launch)"""
import csv, io, json, subprocess, sys

KEEP = ["dram__bytes_read.sum", "dram__bytes_write.sum", "dram__cycles_active.avg",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "gpu__time_duration.sum", "launch__block_size",
        "launch__cluster_dim_x", "launch__grid_size", "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic",
        "sm__cycles_active.avg", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
        "smsp__issue_active.avg.pct_of_peak_sustained_active"]

out = {}
for arg in sys.argv[1:]:
    label, path = arg.split("=", 1)
    txt = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(txt)))
    head, units, last = rows[0], rows[1], rows[-1]
    d = {}
    for name, unit, val in zip(head, units, last):
        if name in KEEP:
            d[name] = f"{val} {unit}".strip()
    d["kernel"] = last[head.index("Kernel Name")] if "Kernel Name" in head else ""
    out[label] = d
print(json.dumps(out, indent=1, sort_keys=True))
