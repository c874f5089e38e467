#!/usr/bin/env python
"""DenseNet-121 (fp16) against ResNet-50 (fp16), timed alternately in one process.

Two device-resident workloads: batch 8 with 4 contexts per plan (bench.py's headline shape) and batch 32 with 8 contexts.
Each plan is tuned for its context count first; then --rounds windows of --steps steps each, the two plans in turn.  Per
workload one JSON line: images/s of each plan (median of the windows and their range), DenseNet-121's algorithmic TFLOP/s
from the lowered shapes (graph.conv_flops), and the card name, power limit and sampled SM clock.  Then one line for the
end-to-end path: DenseNet-121 through InferenceManager at batch 8 with pinned fp32 input, its rate and p50 / p99 latency;
and one line with the per-op device times of one serialised Session.profile pass of the batch-8 plan, grouped into the
stem (conv1 and pool1), the prologue 1x1s, the 3x3 slice writers, the transitions (prologue pool + 1x1) and the tail
(BatchNorm-ReLU global pool, fc, softmax); the prologue 1x1s and 3x3s also per dense block.

  python tools/bench_densenet.py [--steps 200] [--rounds 5] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler  # noqa: E402
from tensorrt_laboratory_b200 import builder, capi, graph  # noqa: E402

WORKLOADS = [(8, 4), (32, 8)]  # (batch, contexts)


class Runner:
    def __init__(self, blob, x, contexts):
        self.batch = x.shape[0]
        self.eng = capi.Engine(blob)
        self.eng.tune(contexts)
        self.sessions = [capi.Session(self.eng) for _ in range(contexts)]
        for s in self.sessions:
            s.host_array(0, self.batch)[...] = x
            s.h2d(self.batch)
            s.prepare(self.batch)

    def window(self, lib, steps: int) -> float:
        capi.check(lib.b2_device_sync())
        t0 = time.perf_counter()
        for i in range(steps):
            self.sessions[i % len(self.sessions)].enqueue(self.batch)
        capi.check(lib.b2_device_sync())
        return steps * self.batch / (time.perf_counter() - t0)

    def profile(self) -> list:
        for _ in range(3):  # the last of three serialised passes
            prof = self.sessions[0].profile(self.batch)
        return prof

    def close(self):
        for s in self.sessions:
            s.close()
        self.eng.destroy()


def op_group(name: str) -> str:
    kind, rest = name.split(":", 1)
    op = rest.split(" ")[0]
    if op in ("conv1", "pool1") or kind == "input_cast":
        return "stem"
    if op.endswith("_blk") or (kind == "avgpool_bnrelu" and op != "pool5"):
        return "transitions"
    if op.endswith("/x1"):
        return "prologue_1x1"
    if op.endswith("/x2"):
        return "slice_3x3"
    return "tail"


def block_of(name: str) -> str:
    op = name.split(":", 1)[1].split(" ")[0]
    return op.split("_")[0].replace("conv", "block") if op.endswith(("/x1", "/x2")) else ""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="steps per timed window")
    ap.add_argument("--rounds", type=int, default=5, help="alternating windows per plan")
    ap.add_argument("--warmup", type=int, default=40)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--out", help="also append the JSON lines to this file")
    a = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("bench_densenet.py: no CUDA device visible and there is no CPU fallback")
    lib = capi.load()
    capi.check(lib.b2_device_set(a.device))
    try:  # the card's power limit is part of the number
        power_limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(a.device)],
                                     capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power_limit = None
    device = capi.device_info(a.device)
    gflop = graph.conv_flops(graph.lower(graph.densenet_caffe(121))) / 1e9
    lines = []
    prof = None
    for batch, contexts in WORKLOADS:
        x = np.random.default_rng(7).standard_normal((batch, 3, 224, 224)).astype(np.float32)
        runners = {"densenet121": Runner(builder.build_densenet_plan(121, max_batch=batch), x, contexts),
                   "resnet50": Runner(builder.build_resnet_plan(50, builder.PREC_FP16, batch), x, contexts)}
        for r in runners.values():
            r.window(lib, max(a.warmup, contexts))
        sampler = ClockSampler(a.device)
        sampler.start()
        rates = {k: [] for k in runners}
        for _ in range(a.rounds):
            for k, r in runners.items():
                rates[k].append(r.window(lib, a.steps))
        clocks = sampler.stop()
        if batch == 8:
            prof = runners["densenet121"].profile()
        for r in runners.values():
            r.close()
        med = {k: float(np.median(v)) for k, v in rates.items()}
        lines.append({
            "metric": f"DenseNet-121 vs ResNet-50 fp16 b={batch}, {contexts} contexts: images/s",
            "images_per_s": med, "range": {k: [float(min(v)), float(max(v))] for k, v in rates.items()},
            "densenet121_tflops": med["densenet121"] * gflop / 1e3, "densenet121_gflop_per_image": gflop,
            "densenet121_over_resnet50": med["densenet121"] / med["resnet50"],
            "workload": f"synthetic weights and N(0, 1) images, batch {batch}, {contexts} device-resident contexts per plan, each "
                        f"plan tuned for {contexts} streams, {a.rounds} alternating windows of {a.steps} steps",
            "device": device, "power_limit": power_limit, "clocks": clocks,
        })
    # end to end: pinned fp32 input through the InferenceManager pipeline (H2D, forward, D2H per request)
    blob = builder.build_densenet_plan(121, max_batch=8)
    m = capi.InferenceManager(4, 8)  # 4 executions, 8 pinned Buffers (bench.py's end-to-end shape)
    try:
        m.register_model("densenet121", blob)
        m.update_resources()
        m.prefill_inputs("densenet121", np.random.default_rng(9).standard_normal((8, 3, 224, 224)).astype(np.float32))
        m.bench("densenet121", 8, seconds=600.0, max_batches=max(a.warmup, 32), want_latencies=False)
        sampler = ClockSampler(a.device)
        sampler.start()
        res, lat = m.bench("densenet121", 8, seconds=600.0, max_batches=a.steps, want_latencies=True)
        clocks = sampler.stop()
    finally:
        m.close()
    lines.append({
        "metric": "DenseNet-121 fp16 b=8 end to end through InferenceManager (4 executions, pinned fp32 input)",
        "images_per_s": a.steps * 8 / res["kWalltime"], "p50_ms": float(np.percentile(lat, 50) * 1e3),
        "p99_ms": float(np.percentile(lat, 99) * 1e3), "requests": a.steps,
        "h2d_bytes_per_image": 3 * 224 * 224 * 4, "device": device, "power_limit": power_limit, "clocks": clocks,
    })
    groups, blocks = {}, {}
    for p in prof:
        g = op_group(p["name"])
        groups[g] = groups.get(g, 0.0) + p["ms"]
        b = block_of(p["name"])
        if b:
            blocks[f"{b} {g}"] = blocks.get(f"{b} {g}", 0.0) + p["ms"]
    total = sum(groups.values())
    lines.append({
        "metric": "DenseNet-121 fp16 b=8: device ms per op group, one serialised pass (Session.profile)",
        "ms": {k: round(v, 4) for k, v in groups.items()}, "share": {k: round(v / total, 4) for k, v in groups.items()},
        "dense_layers_ms": {k: round(v, 4) for k, v in sorted(blocks.items())}, "total_ms": total, "launches": len(prof),
        "device": device, "power_limit": power_limit,
    })
    for line in lines:
        print(json.dumps(line), flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
