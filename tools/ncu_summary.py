"""Selected columns of an ncu report (`ncu -i X.ncu-rep --page raw --csv`) as a small CSV.
    python tools/ncu_summary.py gpurun_out/X.ncu-rep > profiles/rNN_X_summary.csv"""
import csv
import subprocess
import sys

WANT = ["Kernel Name", "Grid Size", "Block Size", "gpu__time_duration.sum", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
        "smsp__issue_active.avg.pct", "smsp__warps_eligible.avg.per_cycle_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct",
        "launch__registers_per_thread", "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_registers", "launch__cluster_max_active",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smsp__pcsamp_warps_issue_stalled_wait", "smsp__pcsamp_warps_issue_stalled_short_scoreboard",
        "smsp__pcsamp_warps_issue_stalled_long_scoreboard", "smsp__pcsamp_warps_issue_stalled_barrier", "smsp__pcsamp_warps_issue_stalled_math_pipe_throttle",
        "smsp__pcsamp_warps_issue_stalled_mio_throttle", "smsp__pcsamp_warps_issue_stalled_sleeping", "smsp__pcsamp_warps_issue_stalled_membar"]
raw = subprocess.run(["ncu", "-i", sys.argv[1], "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units = rows[0], rows[1]
cols = [hdr.index(w) for w in WANT if w in hdr]
out = csv.writer(sys.stdout)
out.writerow([hdr[c] for c in cols])
out.writerow([units[c] for c in cols])
for r in rows[2:]:
    out.writerow([r[c] for c in cols])
