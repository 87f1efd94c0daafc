"""Summarise one kernel of an .ncu-rep into the text kept under profiles/:
    python tools/ncu_summary.py x.ncu-rep "header line" > profiles/rNN_x.txt
(ncu --set full --clock-control none capture)"""
import csv, subprocess, sys

KEEP = ("gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct",
        "launch__registers_per_thread", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
        "launch__waves_per_multiprocessor", "launch__grid_size", "launch__block_size",
        "sm__cycles_active.avg", "sm__cycles_elapsed.avg", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fp64.sum.pct_of_peak_sustained_active",
        "smsp__inst_executed.sum", "smsp__thread_inst_executed.sum", "smsp__thread_inst_executed_per_inst_executed.ratio",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__warps_eligible.avg.per_cycle_active",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum")
PREFIX = ("smsp__average_warps_issue_stalled_",)

rep, title = sys.argv[1], (sys.argv[2] if len(sys.argv) > 2 else "")
rows = list(csv.reader(subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout.splitlines()))
hdr, units, vals = rows[0], rows[1], rows[2]
print(f"# {title}")
print(f"# kernel: {vals[hdr.index('Kernel Name')]}")
for i, h in enumerate(hdr):
    if h in KEEP or (h.startswith(PREFIX) and h.endswith("per_issue_active.ratio")):
        print(f"{h:90s} {units[i]:15s} {vals[i]}")
