#!/usr/bin/env python
"""Condense an .ncu-rep (read here, no GPU needed) into the few numbers the roofline needs.

    python tools/ncu_summary.py report.ncu-rep > ncu_summary.txt
"""
import csv
import io
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_bytes.sum",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__inst_executed_pipe_fma.sum", "sm__inst_executed_pipe_alu.sum", "sm__inst_executed.sum",
    "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
    "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_dynamic",
    "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
    "smsp__cycles_active.avg", "sm__cycles_elapsed.max",
]


def main(path):
    raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr = rows[0]
    units = rows[1]
    name_col = hdr.index("Kernel Name")
    for row in rows[2:]:
        print("== %s  (id %s)" % (row[name_col][:90], row[0]))
        for k in KEYS:
            if k in hdr:
                i = hdr.index(k)
                print("   %-82s %s %s" % (k, row[i], units[i]))
        print()


if __name__ == "__main__":
    main(sys.argv[1])
