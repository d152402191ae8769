#!/usr/bin/env python
"""Summarise an .ncu-rep (from `ncu --set full`) into the handful of numbers DESIGN.md / bench.py quote.
usage: python profiles/ncu_summary.py prof.ncu-rep > prof_summary.txt"""
import csv
import subprocess
import sys

KEYS = [
    ("gpu__time_duration.sum", "duration"),
    ("dram__bytes_read.sum", "dram read"),
    ("dram__bytes_write.sum", "dram write"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram % of peak"),
    ("launch__registers_per_thread", "regs/thread"),
    ("launch__occupancy_limit_registers", "occ limit regs (CTAs)"),
    ("launch__occupancy_limit_shared_mem", "occ limit smem (CTAs)"),
    ("launch__waves_per_multiprocessor", "waves/SM"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps active %"),
    ("smsp__inst_executed.sum", "warp instructions"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots busy %"),
    ("sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "pipe alu %"),
    ("sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "pipe fma %"),
    ("sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "pipe lsu %"),
    ("sm__inst_executed_pipe_tma.avg.pct_of_peak_sustained_active", "pipe tma %"),
    ("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smem bank conflicts"),
    ("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "stall long_scoreboard"),
    ("smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "stall short_scoreboard"),
    ("smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "stall wait"),
    ("smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio", "stall math_pipe_throttle"),
    ("smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio", "stall not_selected"),
    ("smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio", "stall branch_resolving"),
    ("smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "stall barrier"),
    ("smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio", "stall no_instruction"),
    ("smsp__average_warps_issue_stalled_sleeping_per_issue_active.ratio", "stall sleeping"),
    ("smsp__average_warps_issue_stalled_membar_per_issue_active.ratio", "stall membar"),
]


def main():
    rep = sys.argv[1]
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], stdout=subprocess.PIPE, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units, data = rows[0], rows[1], rows[2:]
    col = {h: i for i, h in enumerate(hdr)}
    for r in data:
        name = r[col["Kernel Name"]].split("(")[0]
        print("== %s  grid %s block %s" % (name, r[col["Grid Size"]], r[col["Block Size"]]))
        for key, label in KEYS:
            if key in col:
                print("   %-28s %s %s" % (label, r[col[key]], units[col[key]]))


if __name__ == "__main__":
    main()
