#!/usr/bin/env python
"""Summarise an .ncu-rep: per kernel, the DRAM, L2 and issue metrics."""
import csv, io, subprocess, sys

rep = sys.argv[1]
want = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_bytes.sum", "lts__t_sector_hit_rate.pct",
        "l1tex__t_sector_hit_rate.pct", "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
        "launch__grid_size", "launch__block_size", "launch__occupancy_limit_registers", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
        "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum", "sm__cycles_elapsed.avg",
        "smsp__cycles_active.avg", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum", "l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum",
        "smsp__average_warp_latency_issue_stalled_long_scoreboard.ratio", "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        ]
out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(out)))
hdr = rows[0]
units = rows[1]
for r in rows[2:]:
    d = dict(zip(hdr, r))
    print("=" * 100)
    print(d.get("Kernel Name", "?")[:110])
    for k in hdr:
        if any(k == w for w in want) or "warp_issue_stalled" in k and k.endswith("_per_warp_active.pct"):
            v = d[k]
            u = units[hdr.index(k)]
            try:
                if float(v.replace(",", "")) == 0 and "stalled" in k:
                    continue
            except ValueError:
                pass
            print(f"  {k:95s} {v:>18s} {u}")
