#!/usr/bin/env python
"""Per-kernel roofline table from a condensed ncu metrics file (tools/condense_ncu.py) and the layer FLOPs of the graph:
the three numbers SURVEY.md 8(d) asks for -- tensor-pipe % per kernel with the FLOP-weighted network average, achieved
DRAM GB/s per kernel, and the end-to-end rate against the PCIe ceiling.
usage: python tools/roofline_table.py ncu_metrics.csv [bench.json] > roofline.md"""
import csv
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tensorrt_laboratory_b200 import graph, weights  # noqa: E402

PEAK_TF = float(os.environ.get("PEAK_TFLOPS", "989"))  # sustained tensor peak of the GPU; default: H100 SXM data sheet, dense fp16
PEAK_HBM = 6587.7    # GB/s, measured copy bandwidth
BATCH = 8


def main():
    rows = list(csv.DictReader(open(sys.argv[1])))
    bench = json.load(open(sys.argv[2])) if len(sys.argv) > 2 else None
    net = graph.resnet_caffe(50)
    low = graph.lower(net, weights.random_weights(net, 0))
    T = low["tensors"]
    flops = {}
    for op in low["ops"]:
        if op["type"] == "conv":
            _, ho, wo = T[op["output"]]
            flops[op["name"]] = 2.0 * BATCH * ho * wo * op["cout"] * op["cin"] * op["k"] ** 2
        elif op["type"] == "fc":
            flops[op["name"]] = 2.0 * BATCH * op["cout"] * op["cin"] if "cin" in op else 2.0 * BATCH * 1000 * 2048
    print("| launch | tactic | µs (ncu, cold, serialised) | GFLOP | TFLOP/s | % of 1429 | tensor pipe % (active) | DRAM GB/s | % of 6588 | L2→SM MB |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    tot_t = tot_f = wsum = 0.0
    for r in rows:
        kind, _, rest = r["launch"].partition(":")
        name = rest.split(" ")[0]
        tactic = " ".join(x for x in rest.split(" ")[1:] if not x.startswith(("grid", "kblk")))
        t = float(r["duration_ns"]) * 1e-3
        f = flops.get(name, 0.0)
        dram = (float(r["dram_read_B"] or 0) + float(r["dram_write_B"] or 0))
        tp = float(r["tensor_pipe_pct"] or 0)
        tot_t += t
        tot_f += f
        wsum += tp * f
        tfs = f / (t * 1e-6) / 1e12 if f else 0.0
        print(f"| {kind}:{name} | {tactic} | {t:.1f} | {f / 1e9:.2f} | {tfs:.0f} | {100 * tfs / PEAK_TF:.1f} | {tp:.1f} | "
              f"{dram / (t * 1e-6) / 1e9:.0f} | {100 * dram / (t * 1e-6) / 1e9 / PEAK_HBM:.1f} | {float(r['l2_bytes'] or 0) / 1e6:.1f} |")
    print()
    print(f"Serialised total {tot_t:.0f} µs for {tot_f / 1e9:.2f} GFLOP → {tot_f / (tot_t * 1e-6) / 1e12:.0f} TFLOP/s; "
          f"FLOP-weighted tensor-pipe activity {wsum / tot_f:.1f} % (of the cycles the issuing SMs are active).")
    if bench:
        v, e = bench["value"], bench["e2e"]["value"]
        pcie = 53.2e9 / (BATCH * 3 * 224 * 224 * 4) * BATCH  # img/s one H2D engine can feed (measured 53.2 GB/s pinned)
        print(f"\nIn the timed benchmark (4 contexts overlapping): {v:.0f} img/s device-resident = "
              f"{bench['roofline']['achieved']:.0f} TFLOP/s on the conv stack ({100 * bench['roofline']['frac']:.1f} % of {PEAK_TF:.0f}); "
              f"end to end {e:.0f} img/s = {100 * e / pcie:.0f} % of the PCIe ceiling for fp32 inputs ({pcie:.0f} img/s at 53.2 GB/s).")


if __name__ == "__main__":
    main()
