#!/usr/bin/env python3
"""Summarise an .ncu-rep (ncu --set full capture) as markdown: python tools/ncu_summary.py file.ncu-rep > summary.md"""
import csv, subprocess, sys
rep = sys.argv[1]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units, vals = rows[0], rows[1], rows[-1]
m = {h: (v, u) for h, v, u in zip(hdr, vals, units)}
keys = [
    ("Kernel Name", "kernel"), ("gpu__time_duration.sum", "duration"), ("launch__grid_size", "grid"), ("launch__block_size", "block"),
    ("launch__registers_per_thread", "registers/thread"), ("launch__shared_mem_per_block_static", "static smem/block"),
    ("launch__shared_mem_per_block_dynamic", "dynamic smem/block"), ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy %"),
    ("dram__bytes_read.sum", "DRAM read"), ("dram__bytes_write.sum", "DRAM write"),
    ("dram__throughput.avg.pct_of_peak_sustained_elapsed", "DRAM throughput % of peak"), ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "DRAM throughput % of peak"),
    ("lts__t_bytes.sum", "L2 bytes"), ("l1tex__t_sector_hit_rate.pct", "L1 hit %"), ("lts__t_sector_hit_rate.pct", "L2 hit %"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM throughput % of peak"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots busy %"), ("smsp__inst_executed.sum", "warp instructions"),
    ("smsp__thread_inst_executed_per_inst_executed.ratio", "active threads / instruction"),
    ("sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "ALU pipe %"), ("sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "LSU pipe %"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe % (expected 0)"),
]
print(f"# ncu --set full: `{rep.split('/')[-1]}`\n")
print("| metric | value |\n|---|---|")
seen = set()
for k, name in keys:
    if k in m and name not in seen:
        seen.add(name); v, u = m[k]
        print(f"| {name} | {v} {u} |")
stalls = sorted(((float(v[0]), k) for k, v in m.items() if k.startswith("smsp__average_warps_issue_stalled_") and k.endswith("_per_issue_active.ratio") and v[0]), reverse=True)[:6]
if not stalls:
    stalls = sorted(((float(v[0]), k) for k, v in m.items() if "issue_stalled" in k and k.endswith(".pct") and v[0].replace('.', '', 1).isdigit()), reverse=True)[:6]
print("\nTop warp stall reasons:\n")
for v, k in stalls:
    print(f"* `{k}` = {v:.2f}")
