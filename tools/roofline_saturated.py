#!/usr/bin/env python
"""Per-layer roofline in the SERVING regime, from the load-time tuner's dump (tools/gpu_tune_dump.py, B2_TUNE_VERBOSE):
time per launch of each convolution's winning tactic with N concurrent copies of the layer, against BOTH roofs --
  tensor:  2*M*N*K / the sustained fp16 tensor peak (TFLOP/s, measured on the same GPU)
  memory:  algorithmic bytes (activations in + weights + residual + output, fp16) / the L2 bandwidth tools/micro/l2_stream.cu
           measures for unique streaming data, separately for reads and writes (TB/s)
and names the roof that binds each layer.  The sum of the winners is the forward pass's cost in that regime.
usage: python tools/roofline_saturated.py TUNE_DUMP PEAK_TFLOPS L2_READ_TBS L2_WRITE_TBS [step_us]"""
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tensorrt_laboratory_b200 import graph, roofs, weights  # noqa: E402

BATCH = 8


def main():
    best = {}
    pat = re.compile(r"\[b2 tune\] (\S+) b=(\d+) M=(\d+) N=(\d+) K=(\d+) best bn=(\d+) st=(\d+) sp=(\d+) sps=(\d+) ws=(\d+) cn=(\d+) halo=(\d+) : ([\d.]+) us/launch \((\d+) streams\)")
    for line in open(sys.argv[1]):
        m = pat.match(line)
        if m:
            best[m.group(1)] = dict(M=int(m.group(3)), N=int(m.group(4)), K=int(m.group(5)), bn=int(m.group(6)), st=int(m.group(7)),
                                    sps=int(m.group(9)), ws=int(m.group(10)), us=float(m.group(13)), streams=int(m.group(14)))
    peak_tf, l2_read, l2_write = float(sys.argv[2]), float(sys.argv[3]) * 1e12, float(sys.argv[4]) * 1e12
    step_us = float(sys.argv[5]) if len(sys.argv) > 5 else None
    net = graph.resnet_caffe(50)
    low = graph.lower(net, weights.random_weights(net, 0))
    floors = {f["name"]: f for f in roofs.conv_floors(low, BATCH, peak_tf, l2_read, l2_write)}
    print("| layer | GEMM M×N×K | tactic | µs per launch (saturated) | TFLOP/s | tensor floor µs | bytes MB (rd / wr) | memory floor µs | binding roof | floor / measured |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    tot = tot_tensor = tot_mem = tot_floor = flops_all = 0.0
    by_roof = {"tensor": [0.0, 0.0], "memory": [0.0, 0.0]}
    for op in low["ops"]:
        if op["type"] != "conv" or op["name"] not in best:
            continue
        b, f = best[op["name"]], floors[op["name"]]
        tot += b["us"]; tot_tensor += f["tensor_floor_us"]; tot_mem += f["memory_floor_us"]; tot_floor += f["floor_us"]; flops_all += f["flops"]
        by_roof[f["roof"]][0] += b["us"]; by_roof[f["roof"]][1] += f["floor_us"]
        tactic = f"bn={b['bn']} st={b['st']}x{b['sps']}" + (f" ws={b['ws']}" if b["ws"] else "")
        print(f"| {op['name']} | {b['M']}×{b['N']}×{b['K']} | {tactic} | {b['us']:.2f} | {f['flops'] / b['us'] * 1e-6:.0f} | {f['tensor_floor_us']:.2f} | "
              f"{f['read_bytes'] / 1e6:.1f} / {f['write_bytes'] / 1e6:.1f} | {f['memory_floor_us']:.2f} | {f['roof']} | {f['floor_us'] / b['us']:.2f} |")
    print()
    print(f"Sum of the {len(best)} winners: **{tot:.1f} µs** per forward pass" + (f" (measured step of the whole network: {step_us:.0f} µs)" if step_us else "")
          + f"; {flops_all / tot * 1e-6:.0f} TFLOP/s = {flops_all / tot * 1e-6 / peak_tf:.2f} of the sustained tensor peak.")
    print(f"Floors: tensor {tot_tensor:.1f} µs, memory (L2 stream) {tot_mem:.1f} µs, per-layer max of the two {tot_floor:.1f} µs "
          f"= {tot_floor / tot:.2f} of the measured sum.")
    for roof, (us, fl) in by_roof.items():
        print(f"Layers bound by the {roof} roof: {us:.1f} µs measured against {fl:.1f} µs of floor ({fl / max(us, 1e-9):.2f}).")


if __name__ == "__main__":
    main()
