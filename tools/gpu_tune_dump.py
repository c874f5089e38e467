#!/usr/bin/env python
"""Dump the tuner's view of every convolution of a ResNet at one batch size: time per launch of every candidate tactic
with `streams` concurrent copies of the layer (B2_TUNE_VERBOSE=2).  The sum over layers of the winners is the forward
pass's cost if nothing but the per-layer saturated throughput mattered.
  TUNE_DEPTH=50 TUNE_BATCH=8 TUNE_STREAMS=4 python tools/gpu_tune_dump.py > tune_dump.log 2>&1
  TUNE_MODEL=resnext50 ... : ResNeXt-50 32x4d (fp16) instead of a ResNet
  TUNE_MODEL=bert TUNE_BATCH=16 ... : BERT-base fp16 at S = 128 (its six GEMMs per layer are 1x1 convolutions)"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("B2_TUNE_VERBOSE", "2")
from tensorrt_laboratory_b200 import builder, capi  # noqa: E402

depth = int(os.environ.get("TUNE_DEPTH", "50"))
batch = int(os.environ.get("TUNE_BATCH", "8"))
streams = int(os.environ.get("TUNE_STREAMS", "4"))
prec = {"fp16": builder.PREC_FP16, "int8": builder.PREC_INT8}[os.environ.get("TUNE_PREC", "fp16")]
if os.environ.get("TUNE_MODEL") == "bert":
    eng = capi.Engine(builder.build_bert_plan(max_batch=batch))
elif os.environ.get("TUNE_MODEL") == "resnext50":
    eng = capi.Engine(builder.build_resnext_plan(50, builder.PREC_FP16, batch))
else:
    eng = capi.Engine(builder.build_resnet_plan(depth, prec, batch))
n = eng.tune(streams=streams)
print(f"tuned {n} tactics, depth {depth}, batch {batch}, streams {streams}", file=sys.stderr)
