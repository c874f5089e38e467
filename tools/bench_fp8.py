#!/usr/bin/env python
"""fp16 against INT8 against FP8 (E4M3) ResNet plans of one seed, timed alternately in one process.

Two workloads: ResNet-50 at batch 8 with 4 device-resident contexts per plan (bench.py's headline shape) and ResNet-152
at batch 32 with 8 contexts.  Each plan is tuned for its context count first and runs with that tactic table; then
--rounds windows of --steps steps each, the three plans in turn.  Per workload, one JSON line: images/s of each plan
(median of the windows and the spread), the per-layer device times of one serialised pass of the INT8 and FP8 plans
(Session.profile) with the FP8 / INT8 ratio of every 1-byte convolution, whether the plans' top-1 classes agree, and the
card name, power limit and sampled SM clock.

--model resnext50: the same comparison for ResNeXt-50 32x4d at batch 8 / 4 contexts and batch 32 / 8 contexts, whose 16
grouped 3x3 convolutions run on the grouped 1-byte kernels in the INT8 and FP8 plans.  Its lines add the per-layer device
times of those 16 layers in all three precisions.

  python tools/bench_fp8.py [--model resnext50] [--steps 200] [--rounds 5] [--out FILE]
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
from tensorrt_laboratory_b200 import builder, capi, weights  # noqa: E402

WORKLOADS = [(50, 8, 4), (152, 32, 8)]  # (depth, batch, contexts)
RESNEXT_WORKLOADS = [(50, 8, 4), (50, 32, 8)]
PRECISIONS = {"fp16": builder.PREC_FP16, "int8": builder.PREC_INT8, "fp8": builder.PREC_FP8}


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

    def top1(self) -> np.ndarray:
        s = self.sessions[0]
        s.enqueue(self.batch)
        s.d2h(self.batch)
        s.stream.sync()
        return s.host_array(1, self.batch).argmax(1)

    def layer_ms(self) -> list:
        for _ in range(3):  # the last of three serialised passes
            prof = self.sessions[0].profile(self.batch)
        return prof

    def close(self):
        for s in self.sessions:
            s.close()
        self.eng.destroy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="steps per timed window")
    ap.add_argument("--rounds", type=int, default=5, help="alternating windows per plan")
    ap.add_argument("--warmup", type=int, default=40)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--out", help="also append the JSON lines to this file")
    ap.add_argument("--model", choices=["resnet", "resnext50"], default="resnet",
                    help="resnet: ResNet-50 and ResNet-152 (default); resnext50: ResNeXt-50 32x4d at batch 8 and 32")
    a = ap.parse_args()
    resnext = a.model == "resnext50"
    build = builder.build_resnext_plan if resnext else builder.build_resnet_plan
    if capi.device_count() < 1:
        raise SystemExit("bench_fp8.py: no CUDA device visible and there is no CPU fallback")
    lib = capi.load()
    capi.check(lib.b2_device_set(a.device))
    try:  # the card's power limit is part of the number
        power_limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(a.device)],
                                     capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power_limit = None
    for depth, batch, contexts in RESNEXT_WORKLOADS if resnext else WORKLOADS:
        x = weights.synthetic_input(batch, seed=7)
        runners = {k: Runner(build(depth, p, batch), x, contexts) for k, p in PRECISIONS.items()}
        for r in runners.values():
            r.window(lib, max(a.warmup, contexts))
        sampler = ClockSampler(a.device)
        sampler.start()
        rates = {k: [] for k in runners}
        for _ in range(a.rounds):
            for k, r in runners.items():
                rates[k].append(r.window(lib, a.steps))
        clocks = sampler.stop()
        top1 = {k: r.top1() for k, r in runners.items()}
        prof = {k: runners[k].layer_ms() for k in (("fp16", "int8", "fp8") if resnext else ("int8", "fp8"))}
        for r in runners.values():
            r.close()
        conv = {k: [(p["name"].split(":", 1)[1].split(" ")[0], p["ms"]) for p in v if p["name"].startswith(f"conv_{k[0]}8_tcgen05")]
                for k, v in prof.items() if k != "fp16"}
        assert [n for n, _ in conv["int8"]] == [n for n, _ in conv["fp8"]]
        ratio = np.array([f / i for (_, i), (_, f) in zip(conv["int8"], conv["fp8"])])
        med = {k: float(np.median(v)) for k, v in rates.items()}
        model = f"ResNeXt-{depth}" if resnext else f"ResNet-{depth}"
        line = {
            "metric": f"{model} b={batch}, {contexts} contexts: fp16 vs INT8 vs FP8 images/s",
            "images_per_s": med, "spread": {k: [float(min(v)), float(max(v))] for k, v in rates.items()},
            "fp8_over_int8": med["fp8"] / med["int8"], "fp8_over_fp16": med["fp8"] / med["fp16"],
            "one_pass_ms": {k: float(sum(p["ms"] for p in v)) for k, v in prof.items() if k != "fp16"},
            "one_byte_conv_ms": {k: float(sum(ms for _, ms in v)) for k, v in conv.items()},
            "per_layer_fp8_over_int8": {"median": float(np.median(ratio)), "min": float(ratio.min()), "max": float(ratio.max()),
                                        "layers": {n: [round(i * 1e3, 2), round(f * 1e3, 2)]  # us: [int8, fp8]
                                                   for (n, i), (_, f) in zip(conv["int8"], conv["fp8"])}},
            "top1_agreement": {k: float((top1[k] == top1["fp16"]).mean()) for k in ("int8", "fp8")},
            "workload": f"{model} (synthetic weights), batch {batch}, {contexts} device-resident contexts per plan, each "
                        f"plan tuned for {contexts} streams, {a.rounds} alternating windows of {a.steps} steps",
            "device": capi.device_info(a.device), "power_limit": power_limit, "clocks": clocks,
        }
        if resnext:  # the 16 grouped layers, us per pass: [fp16, int8, fp8]
            grouped = {k: {p["name"].split(":", 1)[1].split(" ")[0]: p["ms"] for p in v if " span=" in p["name"]} for k, v in prof.items()}
            assert all(len(g) == 16 for g in grouped.values()), {k: len(g) for k, g in grouped.items()}
            line["grouped_layers_us"] = {n: [round(grouped[k][n] * 1e3, 2) for k in ("fp16", "int8", "fp8")] for n in grouped["fp16"]}
            line["grouped_ms"] = {k: float(sum(g.values())) for k, g in grouped.items()}
        print(json.dumps(line), flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
