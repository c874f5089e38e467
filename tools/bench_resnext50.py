#!/usr/bin/env python
"""ResNeXt-50 32x4d fp16, batch 8: device-resident inferences/s of 4 concurrent contexts with tactics tuned at load,
measured like the headline of bench.py (same ring of synthetic inputs, same clock sampling), as one JSON line.

  python tools/bench_resnext50.py --steps 2000 --warmup 50
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import BATCH, CONTEXTS, UNIT, ClockSampler, build_inputs  # noqa: E402
from tensorrt_laboratory_b200 import builder, capi  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("bench_resnext50.py: no CUDA device visible and there is no CPU fallback")
    capi.check(capi.load().b2_device_set(a.device))
    blob = builder.build_resnext_plan(50, builder.PREC_FP16, BATCH, seed=0)
    ring = build_inputs()
    sampler = ClockSampler(a.device)
    sampler.start()
    ms, launches = capi.device_throughput(blob, CONTEXTS, BATCH, a.steps, max(a.warmup, 3), ring)  # tunes at load
    clocks = sampler.stop()
    try:  # the card's power limit is part of the number
        power_limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(a.device)],
                                     capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power_limit = None
    flops = capi.Engine(blob, inspect_only=True).flops(BATCH)  # algorithmic: Cin/groups inputs per output channel
    print(json.dumps({
        "metric": "ResNeXt-50 32x4d fp16 b=8 inferences/sec", "value": a.steps * BATCH / (ms * 1e-3), "unit": UNIT,
        "workload": f"ResNeXt-50 32x4d fp16 batch={BATCH}, {CONTEXTS} concurrent ExecutionContexts/streams, tuned tactics, "
                    "synthetic 3x224x224 inputs resident in HBM",
        "ms_per_step": ms / a.steps, "steps": a.steps, "gpu_launches": launches * a.steps,
        "algorithmic_tflops": flops * a.steps / (ms * 1e-3) / 1e12, "device": capi.device_info(a.device), "power_limit": power_limit, "clocks": clocks,
    }), flush=True)


if __name__ == "__main__":
    main()
