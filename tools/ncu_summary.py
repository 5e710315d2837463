#!/usr/bin/env python
"""One line per kernel launch of an .ncu-rep: duration, DRAM bytes, occupancy, issue activity.
usage: python tools/ncu_summary.py <file.ncu-rep>"""
import csv
import io
import subprocess
import sys


def main():
    txt = subprocess.run(["ncu", "-i", sys.argv[1], "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(txt)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    want = [("Kernel Name", "kernel"), ("launch__grid_size", "grid"), ("launch__block_size", "block"), ("launch__registers_per_thread", "regs"),
            ("gpu__time_duration.sum", "dur"), ("dram__bytes_read.sum", "dram_rd"), ("dram__bytes_write.sum", "dram_wr"),
            ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps_act%"), ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue%"),
            ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm_thr%"), ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram_thr%"),
            ("lts__t_sector_hit_rate.pct", "l2_hit%")]
    idx = [(n, hdr.index(k)) for k, n in want if k in hdr]
    print(" | ".join("%s[%s]" % (n, units[i]) for n, i in idx))
    for r in data:
        print(" | ".join((r[i].split("(")[0] if n == "kernel" else r[i])[:26] for n, i in idx))


if __name__ == "__main__":
    main()
