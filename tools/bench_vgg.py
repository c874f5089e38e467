#!/usr/bin/env python
"""VGG-16 (fp16) against ResNet-50 (fp16), timed alternately in one process, and its FC layers against HBM.

Two device-resident workloads: batch 8 with 4 contexts per plan and batch 32 with 8 contexts.  Each plan is tuned for its
context count first; then --rounds windows of --steps steps each, the two plans in turn.  Per workload one JSON line:
images/s of each plan (median of the windows and their range), VGG-16's algorithmic TFLOP/s from the lowered shapes
(graph.conv_flops), and the card name, power limit and sampled SM clock.  Then:
  * VGG-16 end to end through InferenceManager at batch 8 with pinned fp32 input: its rate and p50 / p99 latency;
  * per batch size, the device time of each op group of one serialised Session.profile pass (convolutions per block, max
    pools, each FC layer, the rest) and, for each FC layer, its weight bytes over its kernel time against the H100 SXM
    data-sheet HBM3 bandwidth of 3.35 TB/s (a data-sheet figure, not a measured peak);
  * fc6 alone (25088 -> 4096) on one stream at batch 8 and 32: the streaming kernel (fc6 + ReLU, a single-FC plan whose FC
    carries kFcStream) against the same single-FC plan without the flag, which runs fc_kernel<__half>.

  python tools/bench_vgg.py [--steps 100] [--rounds 5] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler  # noqa: E402
from tensorrt_laboratory_b200 import builder, capi, graph, weights  # noqa: E402
from tools.bench_densenet import Runner  # noqa: E402

WORKLOADS = [(8, 4), (32, 8)]  # (batch, contexts)
HBM_TBPS = 3.35  # H100 SXM data sheet, HBM3


def op_group(name: str) -> str:
    kind, rest = name.split(":", 1)
    op = rest.split(" ")[0]
    if kind.startswith("conv"):
        return "conv_block" + op[4]
    if kind == "fc_stream_f16_wgmma" or kind == "fc":
        return op
    return "pool" if kind == "maxpool" else "other"


def fc_lines(prof, low, batch):
    fcs = {o["name"]: o for o in low["ops"] if o["type"] == graph.OP_FC}
    out = {}
    for p in prof:
        op = p["name"].split(":", 1)[1].split(" ")[0]
        if op in fcs:
            o = fcs[op]
            wbytes = 2.0 * ((o["cout"] + 127) // 128 * 128) * o["cin"]
            out[op] = {"launch": p["name"], "us": round(p["ms"] * 1e3, 2), "weight_MB": round(wbytes / 1e6, 1),
                       "TB_per_s": round(wbytes / (p["ms"] * 1e-3) / 1e12, 3),
                       "of_datasheet_hbm": round(wbytes / (p["ms"] * 1e-3) / 1e12 / HBM_TBPS, 3), "batch": batch}
    return out


def profile_median(s, batch, passes=7):
    profs = [s.profile(batch) for _ in range(passes)]
    return [dict(profs[0][i], ms=float(np.median([p[i]["ms"] for p in profs]))) for i in range(len(profs[0]))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100, help="steps per timed window")
    ap.add_argument("--rounds", type=int, default=5, help="alternating windows per plan")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--out", help="also append the JSON lines to this file")
    a = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("bench_vgg.py: no CUDA device visible and there is no CPU fallback")
    lib = capi.load()
    capi.check(lib.b2_device_set(a.device))
    try:  # the card's power limit is part of the number
        power_limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(a.device)],
                                     capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power_limit = None
    device = capi.device_info(a.device)
    net = graph.vgg_caffe(16)
    wts = weights.random_weights(net, 0)
    low = graph.lower(net, wts)
    gflop = graph.conv_flops(low) / 1e9
    lines = []
    for batch, contexts in WORKLOADS:
        x = np.random.default_rng(7).standard_normal((batch, 3, 224, 224)).astype(np.float32)
        vgg_blob = builder.build_plan(low, builder.PREC_FP16, batch)
        runners = {"vgg16": Runner(vgg_blob, x, contexts),
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
        prof = profile_median(runners["vgg16"].sessions[0], batch)
        for r in runners.values():
            r.close()
        med = {k: float(np.median(v)) for k, v in rates.items()}
        lines.append({
            "metric": f"VGG-16 vs ResNet-50 fp16 b={batch}, {contexts} contexts: images/s",
            "images_per_s": med, "range": {k: [float(min(v)), float(max(v))] for k, v in rates.items()},
            "vgg16_tflops": med["vgg16"] * gflop / 1e3, "vgg16_gflop_per_image": gflop,
            "workload": f"seeded weights and N(0, 1) images, batch {batch}, {contexts} device-resident contexts per plan, each "
                        f"plan tuned for {contexts} streams, {a.rounds} alternating windows of {a.steps} steps",
            "device": device, "power_limit": power_limit, "clocks": clocks,
        })
        groups = {}
        for p in prof:
            g = op_group(p["name"])
            groups[g] = groups.get(g, 0.0) + p["ms"]
        total = sum(groups.values())
        lines.append({
            "metric": f"VGG-16 fp16 b={batch}: device ms per op group, one serialised pass (Session.profile, median of 7)",
            "ms": {k: round(v, 4) for k, v in groups.items()}, "share": {k: round(v / total, 4) for k, v in groups.items()},
            "total_ms": total, "fc": fc_lines(prof, low, batch), "device": device, "power_limit": power_limit,
        })
    # end to end: pinned fp32 input through the InferenceManager pipeline (H2D, forward, D2H per request)
    m = capi.InferenceManager(4, 8)
    try:
        m.register_model("vgg16", builder.build_plan(low, builder.PREC_FP16, 8))
        m.update_resources()
        m.prefill_inputs("vgg16", np.random.default_rng(9).standard_normal((8, 3, 224, 224)).astype(np.float32))
        m.bench("vgg16", 8, seconds=600.0, max_batches=max(a.warmup, 32), want_latencies=False)
        sampler = ClockSampler(a.device)
        sampler.start()
        res, lat = m.bench("vgg16", 8, seconds=600.0, max_batches=a.steps, want_latencies=True)
        clocks = sampler.stop()
    finally:
        m.close()
    lines.append({
        "metric": "VGG-16 fp16 b=8 end to end through InferenceManager (4 executions, pinned fp32 input)",
        "images_per_s": a.steps * 8 / res["kWalltime"], "p50_ms": float(np.percentile(lat, 50) * 1e3),
        "p99_ms": float(np.percentile(lat, 99) * 1e3), "requests": a.steps, "device": device, "power_limit": power_limit,
        "clocks": clocks,
    })
    # fc6 alone on one stream: streaming kernel against the unflagged single-FC plan (fc_kernel<__half>)
    fc6 = {"name": "fc6_alone", "input": "data", "input_dims": [1, 512, 7, 7], "layers": [
        dict(name="fc6", type="InnerProduct", bottoms=["data"], tops=["fc6"], num_output=4096, bias_term=True)]}
    relu = dict(fc6, layers=fc6["layers"] + [dict(name="relu6", type="ReLU", bottoms=["fc6"], tops=["fc6"])])
    w6 = {"fc6": wts["fc6"]}
    for batch in (8, 32):
        x = np.random.default_rng(3).standard_normal((batch, 512, 7, 7)).astype(np.float32)
        res = {}
        for tag, n in (("stream", relu), ("fc_kernel", fc6)):
            flow = graph.lower(n, w6)
            eng = capi.Engine(builder.build_plan(flow, builder.PREC_FP16, batch))
            s = capi.Session(eng)
            try:
                s.infer(x)
                prof = profile_median(s, batch, passes=21)
            finally:
                s.close()
                eng.destroy()
            res[tag] = fc_lines(prof, flow, batch)["fc6"]
        lines.append({
            "metric": f"fc6 alone (25088 -> 4096) b={batch}, one stream: streaming wgmma kernel vs fc_kernel<__half>",
            "stream": res["stream"], "fc_kernel": res["fc_kernel"], "speedup": round(res["fc_kernel"]["us"] / res["stream"]["us"], 2),
            "device": device, "power_limit": power_limit,
        })
    for line in lines:
        print(json.dumps(line), flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
