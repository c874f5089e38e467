#!/usr/bin/env python
"""Pivot an `ncu --csv --metrics ...` log (one row per launch x metric) into one row per launch, labelled with the
engine's launch names (gpurun_out/launch_names.txt written by tools/profile_forward.py).
usage: python tools/condense_ncu.py raw.csv launch_names.txt > ncu_metrics_<tag>.csv"""
import csv
import sys

COLS = [("duration_ns", "gpu__time_duration.sum"),
        ("tensor_pipe_pct", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"),
        ("dram_read_B", "dram__bytes_read.sum"), ("dram_write_B", "dram__bytes_write.sum"),
        ("l2_bytes", "lts__t_bytes.sum"), ("l2_pct", "lts__throughput.avg.pct_of_peak_sustained_elapsed"),
        ("dram_pct", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed"),
        ("warps_active_pct", "sm__warps_active.avg.pct_of_peak_sustained_active"),
        ("regs", "launch__registers_per_thread"), ("waves", "launch__waves_per_multiprocessor")]
UNIT = {"Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "byte": 1.0, "usecond": 1e3, "msecond": 1e6, "nsecond": 1.0, "second": 1e9}


def main():
    raw, names_path = sys.argv[1], sys.argv[2]
    lines = open(raw, newline="").read().splitlines()
    start = next(i for i, l in enumerate(lines) if l.startswith('"ID"'))
    rows = list(csv.DictReader(lines[start:]))
    per = {}
    for r in rows:
        v = r["Metric Value"].replace(",", "")
        try:
            v = float(v) * UNIT.get(r["Metric Unit"], 1.0)
        except ValueError:
            continue
        per.setdefault(int(r["ID"]), {})[r["Metric Name"]] = v
    names = [l.strip() for l in open(names_path) if l.strip()]
    ids = sorted(per)
    w = csv.writer(sys.stdout)
    w.writerow(["launch"] + [c for c, _ in COLS])
    for k, i in enumerate(ids):
        name = names[k % len(names)] if names else str(i)
        w.writerow([name] + [("%g" % per[i][m]) if m in per[i] else "" for _, m in COLS])


if __name__ == "__main__":
    main()
