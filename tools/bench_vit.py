#!/usr/bin/env python
"""ViT-B/16 (fp16) against ResNet-50 (fp16), timed alternately in one process.

Two device-resident workloads: batch 8 with 4 contexts per plan (bench.py's headline shape) and batch 32 with 8 contexts.
Each plan is tuned for its context count first; then --rounds windows of --steps steps each, the two plans in turn.  Per
workload one JSON line: images/s of each plan (median of the windows and their range), ViT's algorithmic TFLOP/s from the
shapes (vit_gflop), and the card name, power limit and sampled SM clock.  Then one line for the end-to-end path: ViT-B/16
through InferenceManager at batch 8 with pinned fp32 input (602 KB per image host to device), its rate and p50 / p99
latency; and one line with the per-op device times of one serialised Session.profile pass of the batch-8 plan, grouped
into patchify, patch GEMM, tokens, LayerNorm, encoder GEMMs, attention, head and softmax.

  python tools/bench_vit.py [--steps 200] [--rounds 5] [--out FILE]
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
from tensorrt_laboratory_b200 import builder, capi, vit  # noqa: E402

WORKLOADS = [(8, 4), (32, 8)]  # (batch, contexts)


def vit_gflop(cfg) -> float:
    """algorithmic GFLOP per image from the shapes: the patch GEMM, per layer the QKV, output and two FFN GEMMs and the two
    attention products (Q K^T and P V over all L tokens), and the classifier.  ViT-B/16: 35.1."""
    H, F, P, L = cfg.hidden, cfg.ffn, cfg.patches, cfg.tokens
    layer = 2 * L * H * (3 * H + H + 2 * F) + 4 * L * L * H
    return (2 * P * H * 3 * cfg.patch ** 2 + cfg.layers * layer + 2 * H * cfg.classes) / 1e9


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
    kind, op = name.split(":", 1)
    op = op.split(" ")[0]
    if kind.startswith("conv_tcgen05"):
        return "patch_gemm" if op == "patch_embed" else "encoder_gemms"
    if kind.startswith("attention"):
        return "attention"
    return {"patchify": "patchify", "tokens": "tokens", "layernorm": "layernorm", "cls_head": "head", "softmax": "softmax"}.get(kind, kind)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="steps per timed window")
    ap.add_argument("--rounds", type=int, default=5, help="alternating windows per plan")
    ap.add_argument("--warmup", type=int, default=40)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--out", help="also append the JSON lines to this file")
    a = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("bench_vit.py: no CUDA device visible and there is no CPU fallback")
    lib = capi.load()
    capi.check(lib.b2_device_set(a.device))
    try:  # the card's power limit is part of the number
        power_limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(a.device)],
                                     capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power_limit = None
    device = capi.device_info(a.device)
    cfg = vit.VIT_B16
    gflop = vit_gflop(cfg)
    lines = []
    prof = None
    for batch, contexts in WORKLOADS:
        x = np.random.default_rng(7).standard_normal((batch, 3, 224, 224)).astype(np.float32)
        runners = {"vit_b16": Runner(builder.build_vit_plan(cfg, max_batch=batch), x, contexts),
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
            prof = runners["vit_b16"].profile()
        for r in runners.values():
            r.close()
        med = {k: float(np.median(v)) for k, v in rates.items()}
        lines.append({
            "metric": f"ViT-B/16 vs ResNet-50 fp16 b={batch}, {contexts} contexts: images/s",
            "images_per_s": med, "range": {k: [float(min(v)), float(max(v))] for k, v in rates.items()},
            "vit_tflops": med["vit_b16"] * gflop / 1e3, "vit_gflop_per_image": gflop,
            "vit_over_resnet50": med["vit_b16"] / med["resnet50"],
            "workload": f"synthetic weights and N(0, 1) images, batch {batch}, {contexts} device-resident contexts per plan, each "
                        f"plan tuned for {contexts} streams, {a.rounds} alternating windows of {a.steps} steps",
            "device": device, "power_limit": power_limit, "clocks": clocks,
        })
    # end to end: pinned fp32 input through the InferenceManager pipeline (H2D, forward, D2H per request)
    blob = builder.build_vit_plan(cfg, max_batch=8)
    m = capi.InferenceManager(4, 8)  # 4 executions, 8 pinned Buffers (bench.py's end-to-end shape)
    try:
        m.register_model("vit", blob)
        m.update_resources()
        m.prefill_inputs("vit", np.random.default_rng(9).standard_normal((8, 3, 224, 224)).astype(np.float32))
        m.bench("vit", 8, seconds=600.0, max_batches=max(a.warmup, 32), want_latencies=False)
        sampler = ClockSampler(a.device)
        sampler.start()
        res, lat = m.bench("vit", 8, seconds=600.0, max_batches=a.steps, want_latencies=True)
        clocks = sampler.stop()
    finally:
        m.close()
    lines.append({
        "metric": "ViT-B/16 fp16 b=8 end to end through InferenceManager (4 executions, pinned fp32 input)",
        "images_per_s": a.steps * 8 / res["kWalltime"], "p50_ms": float(np.percentile(lat, 50) * 1e3),
        "p99_ms": float(np.percentile(lat, 99) * 1e3), "requests": a.steps,
        "h2d_bytes_per_image": 3 * 224 * 224 * 4, "device": device, "power_limit": power_limit, "clocks": clocks,
    })
    groups = {}
    for p in prof:
        g = op_group(p["name"])
        groups[g] = groups.get(g, 0.0) + p["ms"]
    total = sum(groups.values())
    lines.append({
        "metric": "ViT-B/16 fp16 b=8: device ms per op group, one serialised pass (Session.profile)",
        "ms": {k: round(v, 4) for k, v in groups.items()}, "share": {k: round(v / total, 4) for k, v in groups.items()},
        "total_ms": total, "device": device, "power_limit": power_limit,
    })
    for line in lines:
        print(json.dumps(line), flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
