"""Device-resident throughput of the persistent network kernel against the per-layer kernels (4 contexts, RN50 b=8)."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tensorrt_laboratory_b200 import builder, capi, weights  # noqa: E402

BATCH = int(os.environ.get("SWEEP_BATCH", "8"))
steps = int(os.environ.get("SWEEP_STEPS", "400"))
PREC = {"fp16": builder.PREC_FP16, "int8": builder.PREC_INT8}[os.environ.get("SWEEP_PREC", "fp16")]
blob = builder.build_resnet_plan(int(os.environ.get("SWEEP_DEPTH", "50")), PREC, BATCH, seed=0)
ring = weights.synthetic_input(BATCH, seed=1234, ring=32)
settings = sys.argv[1:] or ["net=0", "net=1,ctas=37", "net=1,ctas=48", "net=1,ctas=74", "net=1,ctas=148", "net=1,ctas=37,bn=64",
                            "ctx=1,net=0", "ctx=1,net=1,ctas=148", "ctx=1,net=1,ctas=74", "ctx=2,net=1,ctas=74", "ctx=8,net=1,ctas=18",
                            "ctx=8,net=1,ctas=37"]
for st in settings:
    kv = dict(x.split("=") for x in st.split(","))
    os.environ["B2_NET"] = kv.get("net", "0")
    os.environ.pop("B2_NET_CTAS", None)
    os.environ.pop("B2_NET_BN", None)
    if "ctas" in kv:
        os.environ["B2_NET_CTAS"] = kv["ctas"]
    if "bn" in kv:
        os.environ["B2_NET_BN"] = kv["bn"]
    for k in ("B2_FUSE_TAIL", "B2_GRAPH", "B2_AUTOTUNE", "B2_ARENA_SLACK", "B2_TAIL_CTAS", "B2_TAIL_PDL", "B2_I8_BN", "B2_I8_STAGES"):
        os.environ.pop(k, None)
    if "tail" in kv:
        os.environ["B2_FUSE_TAIL"] = kv["tail"]
    if "graph" in kv:
        os.environ["B2_GRAPH"] = kv["graph"]
    if "i8st" in kv:
        os.environ["B2_I8_STAGES"] = kv["i8st"]
    if "i8bn" in kv:
        os.environ["B2_I8_BN"] = kv["i8bn"]
    if "tctas" in kv:
        os.environ["B2_TAIL_CTAS"] = kv["tctas"]
    if "tpdl" in kv:
        os.environ["B2_TAIL_PDL"] = kv["tpdl"]
    if "slack" in kv:
        os.environ["B2_ARENA_SLACK"] = kv["slack"]
    if "tune" in kv:
        os.environ["B2_AUTOTUNE"] = kv["tune"]
    ctx = int(kv.get("ctx", "4"))
    try:
        ms, nl = capi.device_throughput(blob, ctx, BATCH, steps, 40, ring)
        print(json.dumps({"setting": st, "img_per_s": steps * BATCH / (ms * 1e-3), "ms_per_step": ms / steps, "launches": nl}), flush=True)
    except Exception as ex:  # keep sweeping
        print(json.dumps({"setting": st, "error": str(ex)}), flush=True)
