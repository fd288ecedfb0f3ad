"""Dev tool: condense an .ncu-rep (ncu --set full) into per-kernel metrics.
usage: python tools/ncu_summary.py report.ncu-rep > <name>.txt"""
import csv, subprocess, sys
KEEP = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
    "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
    "sm__inst_executed_pipe_alu.sum.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_fma.sum.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_lsu.sum.pct_of_peak_sustained_active",
    "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio",
]
out = subprocess.run(["ncu", "-i", sys.argv[1], "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(out.splitlines()))
hdr, units = rows[0], rows[1]
for r in rows[2:]:
    d = dict(zip(hdr, r))
    print("Kernel Name\t\t" + d.get("Kernel Name", "?"))
    for k in KEEP:
        if k in d:
            print("%s\t%s\t%s" % (k, units[hdr.index(k)], d[k]))
    print()
