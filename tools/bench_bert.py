#!/usr/bin/env python
"""BERT-base fp16, batch 16, S = 128 by default (seeded weights, random tokens with ragged padding): device-resident
sequences/s of 4 concurrent contexts with tactics tuned at load, end-to-end requests through the C++ InferenceManager
(p50 / p99), the whole-program FLOP rate from the algorithmic FLOPs of the shapes, and the attention launches' share of
one serialised forward pass (per-launch CUDA events), as one JSON line.  The SM clock and the power limit are read in the
same run.

  python tools/bench_bert.py --steps 500 --warmup 20 [--seq 128] [--batch 16] [--dump-outputs DIR]
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
from tensorrt_laboratory_b200 import bert, builder, capi  # noqa: E402

CONTEXTS = 4


def algorithmic_flops_per_sequence(cfg: bert.BertConfig) -> dict:
    """2 x MACs of every GEMM (QKV, attention output, FFN1, FFN2, pooler) and of Q K^T and P V, from the shapes."""
    S, H, F = cfg.seq, cfg.hidden, cfg.ffn
    gemm = cfg.layers * 2 * S * H * (3 * H + H + F + F) + 2 * H * H
    attention = cfg.layers * 2 * 2 * S * S * H
    return {"gemm": gemm, "attention": attention, "total": gemm + attention}


def inputs(cfg: bert.BertConfig, n: int, seed: int = 1) -> dict:
    rng = np.random.default_rng(seed)
    mask = np.ones((n, cfg.seq), np.int32)
    for i in range(n):
        mask[i, cfg.seq - int(rng.integers(0, cfg.seq // 2)):] = 0
    return dict(input_ids=rng.integers(0, cfg.vocab, (n, cfg.seq)).astype(np.int32),
                segment_ids=rng.integers(0, cfg.types, (n, cfg.seq)).astype(np.int32), input_mask=mask)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq", type=int, default=128, help="sequence length S (64, 128, 256, 384 or 512)")
    ap.add_argument("--batch", type=int, default=16, help="sequences per step and per request")
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--requests", type=int, default=200, help="end-to-end InferenceManager requests")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the outputs of the last timed step as DIR/bert_*.npy")
    a = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("bench_bert.py: no CUDA device visible and there is no CPU fallback")
    lib = capi.load()
    capi.check(lib.b2_device_set(a.device))
    cfg = bert.BertConfig(seq=a.seq)
    batch = a.batch
    blob = builder.build_bert_plan(cfg, max_batch=batch, seed=0)
    eng = capi.Engine(blob)
    eng.tune(CONTEXTS)  # tactics timed in the regime of the run, ahead of the timed window
    tuned = builder.attach_tactics(blob, eng.tactics())
    x = inputs(cfg, batch)
    sessions = [capi.Session(eng) for _ in range(CONTEXTS)]
    for s in sessions:
        for i, b in enumerate(eng.bindings):
            if b["is_input"]:
                s.host_array(i, batch)[...] = x[b["name"]]
        s.h2d(batch)
        s.prepare(batch)
    sampler = ClockSampler(a.device)
    for i in range(max(a.warmup, CONTEXTS)):
        sessions[i % CONTEXTS].enqueue(batch)
    capi.check(lib.b2_device_sync())
    sampler.start()
    t0 = time.perf_counter()
    for i in range(a.steps):
        sessions[i % CONTEXTS].enqueue(batch)
    capi.check(lib.b2_device_sync())
    dt = time.perf_counter() - t0
    clocks = sampler.stop()
    if a.dump_outputs:
        last = sessions[(a.steps - 1) % CONTEXTS]
        last.d2h(batch)
        last.stream.sync()
        os.makedirs(a.dump_outputs, exist_ok=True)
        for i, b in enumerate(eng.bindings):
            if not b["is_input"]:
                np.save(os.path.join(a.dump_outputs, f"bert_{b['name']}.npy"), last.host_array(i, batch).copy())
    for _ in range(3):  # the last of three serialised passes
        prof = sessions[0].profile(batch)
    attn = [p for p in prof if p["name"].startswith("attention_f16_wgmma")]
    attn_ms, pass_ms = sum(p["ms"] for p in attn), sum(p["ms"] for p in prof)
    for s in sessions:
        s.close()
    eng.destroy()

    m = capi.InferenceManager(max_exec_concurrency=CONTEXTS)
    m.register_model("bert", tuned)
    m.update_resources()
    for _ in range(10):
        m.infer_bindings("bert", x)
    lat = []
    t1 = time.perf_counter()
    for _ in range(a.requests):
        r0 = time.perf_counter()
        m.infer_bindings("bert", x)
        lat.append(time.perf_counter() - r0)
    e2e = time.perf_counter() - t1
    m.close()
    try:  # the card's power limit is part of the number
        power_limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(a.device)],
                                     capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power_limit = None
    fl = algorithmic_flops_per_sequence(cfg)
    seq_s = a.steps * batch / dt
    print(json.dumps({
        "metric": f"BERT-base fp16 b={batch} S={cfg.seq} sequences/sec", "value": seq_s, "unit": "sequences/s",
        "workload": f"BERT-base (12 layers, hidden 768) fp16, batch={batch}, S={cfg.seq}, {CONTEXTS} concurrent contexts, "
                    "tuned tactics, token bindings resident in HBM",
        "ms_per_step": dt * 1e3 / a.steps, "steps": a.steps,
        "algorithmic_gflop_per_sequence": {k: v / 1e9 for k, v in fl.items()},
        "whole_program_tflops": fl["total"] * seq_s / 1e12,
        "attention_profile": {"kernel": attn[0]["name"].split(":")[0], "launches": len(attn), "ms": attn_ms,
                              "share_of_forward_pass": attn_ms / pass_ms, "forward_pass_ms": pass_ms,
                              "tflops": sum(p["flops"] for p in attn) / (attn_ms * 1e-3) / 1e12,
                              "note": "one serialised forward pass, per-launch CUDA events"},
        "e2e_inference_manager": {"requests": a.requests, "batch": batch, "sequences_per_s": a.requests * batch / e2e,
                                  "p50_ms": float(np.percentile(lat, 50) * 1e3), "p99_ms": float(np.percentile(lat, 99) * 1e3),
                                  "note": "one request in flight at a time"},
        "device": capi.device_info(a.device), "power_limit": power_limit, "clocks": clocks,
    }), flush=True)


if __name__ == "__main__":
    main()
