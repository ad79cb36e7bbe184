#!/usr/bin/env python
"""Condense an .ncu-rep (ncu --set full) into a CSV of the key metrics:
  python tools/ncu_summary.py x.ncu-rep > x_summary.csv"""
import csv
import subprocess
import sys

KEEP = ["Kernel Name", "gpu__time_duration", "launch__", "smsp__inst_executed.sum", "smsp__issue_active",
        "smsp__average_warps_issue_stalled", "l1tex__data_pipe_lsu_wavefronts", "l1tex__data_bank_conflicts",
        "l1tex__throughput", "l1tex__t_sector_hit_rate", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "dram__throughput", "sm__throughput", "sm__warps_active", "lts__t_sector_hit_rate", "lts__throughput",
        "lts__t_sectors_op", "smsp__warps_eligible", "sm__inst_executed_pipe_alu", "sm__inst_executed_pipe_lsu",
        "smsp__thread_inst_executed_per_inst_executed", "sm__cycles_active.avg", "smsp__inst_executed_op"]


def main():
    raw = subprocess.run(["ncu", "-i", sys.argv[1], "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    w = csv.writer(sys.stdout)
    w.writerow(["launch", "metric", "unit", "value"])
    for n, r in enumerate(rows[2:]):
        for i, h in enumerate(hdr):
            if any(k in h for k in KEEP) and "not_issued" not in h:
                w.writerow([n, h, units[i], r[i]])


if __name__ == "__main__":
    main()
