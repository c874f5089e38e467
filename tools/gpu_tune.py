#!/usr/bin/env python
"""Time ResNet-50 fp16 b=8 forward passes under different engine options in one process.
usage: python tools/gpu_tune.py [opt=val,opt=val ...]   (each argument = one configuration; "-" = defaults)
Prints one JSON line per configuration: single-stream graph replay ms, direct-launch ms, 4-context throughput."""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tensorrt_laboratory_b200 import builder, capi, weights  # noqa: E402


def parse(arg):
    if arg == "-":
        return {}
    return {kv.split("=")[0]: int(kv.split("=")[1]) for kv in arg.split(",")}


def time_session(sess, iters=100):
    ev0, ev1 = capi.Event(), capi.Event()
    for _ in range(10):
        sess.enqueue(8)
    sess.stream.sync()
    ev0.record(sess.stream)
    for _ in range(iters):
        sess.enqueue(8)
    ev1.record(sess.stream)
    sess.stream.sync()
    return ev0.elapsed_ms(ev1) / iters


def main():
    configs = [parse(a) for a in sys.argv[1:]] or [{}]
    multi = os.environ.get("TUNE_MULTI", "1") != "0"
    from tensorrt_laboratory_b200 import graph
    net = graph.resnet_caffe(50)
    low = graph.lower(net, weights.random_weights(net, 0))
    pack = os.environ.get("TUNE_PACK", "1") != "0"
    blob = builder.build_plan(low, builder.PREC_FP16, 8, pack_weights=pack)
    eng = capi.Engine(blob)
    x = weights.synthetic_input(8)
    ring = weights.synthetic_input(8, ring=8)
    env_keys = {"bn": "B2_FORCE_BN", "stages": "B2_FORCE_STAGES", "splits": "B2_FORCE_SPLITS", "pdl": "B2_PDL",
                "pdl_trigger": "B2_PDL_TRIGGER", "graph": "B2_GRAPH", "autotune": "B2_AUTOTUNE", "sps": "B2_FORCE_SPS", "ws": "B2_FORCE_WS", "halo": "B2_FORCE_HALO", "cn": "B2_FORCE_CN"}
    for cfg in configs:
        sess = capi.Session(eng, cfg)
        sess.infer(x)
        rec = {"cfg": cfg, "graph_ms": time_session(sess)}
        if os.environ.get("TUNE_NAMES"):
            n = sess.nb_launches(8)
            rec["names"] = [capi.load().b2_context_launch_name(sess.ctx, 8, i).decode() for i in range(n)]
        sess.set_option("graph", 0)
        rec["direct_ms"] = time_session(sess, 50)
        sess.close()
        if multi:
            for k, v in env_keys.items():
                os.environ.pop(v, None)
            for k, v in cfg.items():
                os.environ[env_keys[k]] = str(v)
            ms, _ = capi.device_throughput(blob, 4, 8, 400, 20, ring)
            rec["ctx4_img_s"] = 400 * 8 / (ms * 1e-3)
            ms, _ = capi.device_throughput(blob, 8, 8, 400, 20, ring)
            rec["ctx8_img_s"] = 400 * 8 / (ms * 1e-3)
        print(json.dumps(rec), flush=True)
    capi.check(capi.load().b2_context_set_option(capi.Session(eng).ctx, b"pdl", 1))


if __name__ == "__main__":
    main()
