#!/usr/bin/env python
"""Turn an ncu report (`ncu --set full ... -o X`) into a small per-kernel summary.
Usage: python profiles/summarize.py prof.ncu-rep > kernels.md"""
import csv
import io
import subprocess
import sys

rep = sys.argv[1]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units = rows[0], rows[1]
idx = {h: i for i, h in enumerate(hdr)}
base = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__t_sector_hit_rate.pct", "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
        "launch__shared_mem_per_block_dynamic", "sm__inst_executed_pipe_tensor.sum", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"]
stalls = [h for h in hdr if h.startswith("smsp__average_warps_issue_stalled_") and h.endswith("_per_issue_active.ratio")]
print(f"# ncu summary of `{rep}` (`--set full --clock-control none`, cold cache, serialised launches)\n")
for r in rows[2:]:
    print(f"## {r[idx['Kernel Name']]}\n")
    print("| metric | value | unit |\n|---|---|---|")
    for m in base:
        if m in idx and r[idx[m]] != "":
            print(f"| {m} | {r[idx[m]]} | {units[idx[m]]} |")
    st = sorted(((float(r[idx[h]] or 0), h[len("smsp__average_warps_issue_stalled_"):-len("_per_issue_active.ratio")]) for h in stalls), reverse=True)[:6]
    print("\nwarps stalled per issue (top): " + ", ".join(f"{n} {v:.2f}" for v, n in st) + "\n")

# dram traffic per launch of every captured kernel -> profiles/traffic.json (bench.py reads it for `roofline.traffic`)
import json
import os
tj = os.path.join(os.path.dirname(os.path.abspath(__file__)), "traffic.json")
try:
    traffic = json.load(open(tj))
except Exception:
    traffic = {}
def _bytes(v, u):
    v = float(v.replace(",", ""))
    return v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(u, 1)
for r in rows[2:]:
    name = r[idx["Kernel Name"]].split("<")[0].split("(")[0].strip().split("::")[-1].replace("void ", "")
    if "dram__bytes_read.sum" in idx and r[idx["dram__bytes_read.sum"]] != "":
        rd = _bytes(r[idx["dram__bytes_read.sum"]], units[idx["dram__bytes_read.sum"]])
        wr = _bytes(r[idx["dram__bytes_write.sum"]], units[idx["dram__bytes_write.sum"]])
        traffic[name] = {"dram_bytes_per_launch": int(rd + wr), "dram_bytes_read": int(rd), "dram_bytes_write": int(wr), "source": os.path.basename(rep)}
json.dump(traffic, open(tj, "w"), indent=1)
