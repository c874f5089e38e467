#!/usr/bin/env python
"""Padded against packed (``--remove-padding``) BERT-base fp16 plans of one seed, batch 16, at S = 128 and S = 384, for
four mask fills: every token valid, tools/bench_bert.py's distribution (0 ... S/2 - 1 trailing tokens masked per
sequence), half and a quarter of the tokens valid (right padding).  Both plans run with the same tuned tactic table, 4
device-resident contexts each, timed alternately in one process (--rounds windows of --steps steps per plan).  Per
point: sequences/s of both plans (median of the windows and the spread), the valid-token algorithmic FLOP rate (the
GEMM and attention FLOPs of each sequence's valid tokens, from the mask on the host), the attention launches' share of
one serialised pass of each plan, and whether the packed plan's valid rows matched the padded plan's bit for bit.  The
card name, power limit and SM clock are read in the same run; one JSON line per point.

  python tools/bench_bert_packed.py [--steps 100] [--rounds 5] [--seq 128 384] [--out FILE]
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
BATCH = 16


def lengths(S: int, fill: str, rng) -> np.ndarray:
    if fill == "bench_bert":  # tools/bench_bert.py: 0 ... S/2 - 1 trailing tokens masked
        return S - rng.integers(0, S // 2, BATCH)
    return np.full(BATCH, max(1, int(round(float(fill) * S))))


def valid_token_flops(cfg: bert.BertConfig, mask: np.ndarray) -> float:
    """GEMMs over the valid tokens of each sequence, Q K^T and P V over valid x valid, and the pooler"""
    H, F = cfg.hidden, cfg.ffn
    total = 0.0
    for L in (mask != 0).sum(1):
        total += cfg.layers * (2.0 * L * H * (3 * H + H + 2 * F) + 4.0 * L * L * H) + 2.0 * H * H
    return total


class Runner:
    def __init__(self, blob, x):
        self.eng = capi.Engine(blob)
        self.sessions = [capi.Session(self.eng) for _ in range(CONTEXTS)]
        for s in self.sessions:
            for i, b in enumerate(self.eng.bindings):
                if b["is_input"]:
                    s.host_array(i, BATCH)[...] = x[b["name"]]
            s.h2d(BATCH)
            s.prepare(BATCH)

    def window(self, lib, steps: int) -> float:
        capi.check(lib.b2_device_sync())
        t0 = time.perf_counter()
        for i in range(steps):
            self.sessions[i % CONTEXTS].enqueue(BATCH)
        capi.check(lib.b2_device_sync())
        return steps * BATCH / (time.perf_counter() - t0)

    def outputs(self) -> dict:
        s = self.sessions[0]
        s.enqueue(BATCH)
        s.d2h(BATCH)
        s.stream.sync()
        return {b["name"]: s.host_array(i, BATCH).copy() for i, b in enumerate(self.eng.bindings) if not b["is_input"]}

    def attention_share(self) -> dict:
        for _ in range(3):  # the last of three serialised passes
            prof = self.sessions[0].profile(BATCH)
        attn = sum(p["ms"] for p in prof if p["name"].startswith("attention_f16_wgmma"))
        total = sum(p["ms"] for p in prof)
        return {"attention_ms": attn, "forward_pass_ms": total, "share": attn / total}

    def close(self):
        for s in self.sessions:
            s.close()
        self.eng.destroy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq", type=int, nargs="+", default=[128, 384])
    ap.add_argument("--fills", nargs="+", default=["1.0", "bench_bert", "0.5", "0.25"])
    ap.add_argument("--steps", type=int, default=100, help="steps per timed window")
    ap.add_argument("--rounds", type=int, default=5, help="alternating windows per plan")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--out", help="also append the JSON lines to this file")
    a = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("bench_bert_packed.py: no CUDA device visible and there is no CPU fallback")
    lib = capi.load()
    capi.check(lib.b2_device_set(a.device))
    try:  # the card's power limit is part of the number
        power_limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(a.device)],
                                     capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power_limit = None
    for S in a.seq:
        cfg = bert.BertConfig(seq=S)
        W = bert.random_weights(cfg, 0)
        padded_blob = builder.build_bert_plan(cfg, W, max_batch=BATCH)
        eng = capi.Engine(padded_blob)
        eng.tune(CONTEXTS)
        tactics = eng.tactics()
        eng.destroy()
        blobs = {"padded": builder.attach_tactics(padded_blob, tactics),
                 "packed": builder.attach_tactics(builder.build_bert_plan(cfg, W, max_batch=BATCH, remove_padding=True), tactics)}
        for fill in a.fills:
            rng = np.random.default_rng(1)
            mask = np.zeros((BATCH, S), np.int32)
            for n, L in enumerate(lengths(S, fill, rng)):
                mask[n, :L] = 1
            x = dict(input_ids=rng.integers(0, cfg.vocab, (BATCH, S)).astype(np.int32),
                     segment_ids=rng.integers(0, cfg.types, (BATCH, S)).astype(np.int32), input_mask=mask)
            runners = {k: Runner(b, x) for k, b in blobs.items()}
            for r in runners.values():
                r.window(lib, max(a.warmup, CONTEXTS))
            sampler = ClockSampler(a.device)
            sampler.start()
            rates = {k: [] for k in runners}
            for _ in range(a.rounds):
                for k, r in runners.items():
                    rates[k].append(r.window(lib, a.steps))
            clocks = sampler.stop()
            outs = {k: r.outputs() for k, r in runners.items()}
            valid = mask != 0
            bit_identical = bool(np.array_equal(outs["packed"]["last_hidden_state"][valid], outs["padded"]["last_hidden_state"][valid])
                                 and np.array_equal(outs["packed"]["pooled_output"], outs["padded"]["pooled_output"])
                                 and not outs["packed"]["last_hidden_state"][~valid].any())
            shares = {k: r.attention_share() for k, r in runners.items()}
            for r in runners.values():
                r.close()
            fl = valid_token_flops(cfg, mask)
            med = {k: float(np.median(v)) for k, v in rates.items()}
            line = {
                "metric": f"BERT-base fp16 b={BATCH} S={S} fill={fill}: padded vs packed sequences/s",
                "seq": S, "fill": fill, "valid_token_fraction": float(valid.mean()),
                "sequences_per_s": med, "spread": {k: [float(min(v)), float(max(v))] for k, v in rates.items()},
                "packed_over_padded": med["packed"] / med["padded"],
                "valid_token_tflops": {k: fl / BATCH * med[k] / 1e12 for k in med},
                "attention_share_of_one_pass": shares,
                "valid_rows_bit_identical": bit_identical,
                "workload": f"BERT-base (12 layers, hidden 768) fp16, batch {BATCH}, {CONTEXTS} contexts per plan, same tuned "
                            f"tactic table, {a.rounds} alternating windows of {a.steps} steps, token bindings resident in HBM",
                "device": capi.device_info(a.device), "power_limit": power_limit, "clocks": clocks,
            }
            print(json.dumps(line), flush=True)
            if a.out:
                with open(a.out, "a") as f:
                    f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
