#!/usr/bin/env python
"""`ncu -i X.ncu-rep --page raw --csv` -> a compact markdown table (one row per captured launch) of the metrics the roofline
discussion uses.  Usage: python tools/ncu_extract.py raw.csv [--title T] > ncu_full.md"""
import csv
import sys

WANT = [("gpu__time_duration.sum", "time"), ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe active %"),
        ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM throughput %"),
        ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "DRAM throughput %"),
        ("dram__bytes_read.sum", "DRAM read"), ("dram__bytes_write.sum", "DRAM write"),
        ("lts__t_sector_hit_rate.pct", "L2 hit %"), ("l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "smem wavefronts"),
        ("launch__registers_per_thread", "regs"), ("launch__shared_mem_per_block_dynamic", "dyn smem"),
        ("sm__cycles_active.avg", "SM active cycles"), ("smsp__cycles_active.avg.pct_of_peak_sustained_elapsed", "SMSP active %")]
path = sys.argv[1]
title = sys.argv[sys.argv.index("--title") + 1] if "--title" in sys.argv else path
rows = list(csv.reader(l for l in open(path, newline="") if l.startswith('"')))
head, units, data = rows[0], rows[1], rows[2:]
cols = [(head.index(m), lab) for m, lab in WANT if m in head]
ki, gi = head.index("Kernel Name"), head.index("Grid Size")
print(f"# {title}\n")
print("| kernel | grid | " + " | ".join(f"{lab} [{units[i]}]" if units[i] else lab for i, lab in cols) + " |")
print("|---|---|" + "---:|" * len(cols))
for r in data:
    name = r[ki].replace("void ", "").replace("s3r::", "").split("(")[0][:60]
    vals = []
    for i, _ in cols:
        try:
            vals.append(f"{float(r[i].replace(',', '')):.4g}")
        except ValueError:
            vals.append(r[i])
    print(f"| `{name}` | {r[gi]} | " + " | ".join(vals) + " |")
