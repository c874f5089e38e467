"""FP8 (E4M3) path on the GPU: conv_f8_tcgen05 and its SIMT helpers against the FP8 oracle (oracle/fp8_forward.py).

The tensor core's FP8 accumulation is not reproducible on the CPU (quantize.py), so a convolution's output codes are held
to an interval: with the exact accumulator A and P = sum |Wq * q| from the oracle, every code must lie between
e4m3(t(A - eps * P)) and e4m3(t(A + eps * P)), t being the epilogue.  eps = ceil(K / 32) * 2^-W: one rounding of at most
2^-W of the magnitude sum per 32-deep MMA step, W bits kept by the accumulation.  W below 12 would mean a broken kernel.

Measured on an H100 80GB HBM3 over the 19 ResNet bottleneck shapes at batch 3 (printed by the shape test): 98.6 % (the
512-channel 3x3, K = 4608) to 99.9 % (64-channel 1x1s) of the output codes equal the exact-accumulation oracle's; every
code lies inside the W = 12 interval.

The quantize, average-pool and output-cast kernels have no accumulation to speak of: they are bit-exact."""
import math

import numpy as np
import pytest

from oracle import fp8_forward as O8
from oracle.caffe_forward import caffe_forward
from tensorrt_laboratory_b200 import builder, capi, graph, quantize, weights
from tests import helpers
from tests.test_int8 import RN_SHAPES

pytestmark = pytest.mark.gpu

W_BITS = 12  # accumulation width the bound assumes (at least 12)


def _conv_graph(cin, h, cout, k, stride, relu=True, residual=False, seed=0):
    net = builder.single_conv_net(cin, h, h, cout, k, stride, k // 2, relu=relu, residual=residual)
    return graph.lower(net, weights.random_weights(net, seed))


def _fp16_exact(x):
    return x.astype(np.float16).astype(np.float32)


def _codes(y, s):
    """Output-cast values y = fl(value(q) * s) -> the codes q (exact: E4M3 neighbours differ by far more than fp32 ulps)."""
    q = O8.e4m3((np.asarray(y, np.float32) / np.float32(s)).astype(np.float32))
    np.testing.assert_array_equal((O8.value(q) * np.float32(s)).astype(np.float32), y)  # y has the output cast's form
    return q


def _within(op, q_in, got, res=None):
    """-> share of codes equal to the exact oracle; asserts every code within the accumulation interval."""
    A, P = O8.conv_fp8(q_in, op)
    K = op["Wq"].shape[1] * op["Wq"].shape[2] * op["Wq"].shape[3]
    eps = math.ceil(K / 32) * 2.0 ** -W_BITS
    lo = O8.value(O8.requant(A - eps * P, op, res))
    hi = O8.value(O8.requant(A + eps * P, op, res))
    v = O8.value(got)
    bad = ~((lo <= v) & (v <= hi))
    assert not bad.any(), f"{int(bad.sum())} codes outside the W={W_BITS} interval, e.g. {v[bad][:5]} vs [{lo[bad][:5]}, {hi[bad][:5]}]"
    return float((got == O8.requant(A, op, res)).mean())


def _run(lq, x, outputs, options=None):
    out = helpers.run_engine(lq, x, builder.PREC_FP8, options=options, outputs=outputs)
    s = lq["tensor_scales"]
    return {k: (_codes(v, s[k]).reshape(x.shape[0], -1, *v.shape[2:]) if k in s else v) for k, v in out.items()}


@pytest.mark.parametrize("cin,h,cout,k,stride", RN_SHAPES)
def test_fp8_conv_within_the_accumulation_bound(gpu, cin, h, cout, k, stride):
    low = _conv_graph(cin, h, cout, k, stride, relu=True, seed=cin + cout + k)
    x = _fp16_exact(np.random.default_rng(cin * 7 + h).standard_normal((3, cin, h, h)).astype(np.float32))  # ragged last M tile
    lq = quantize.quantize_lowered(low, x, fmt="e4m3")
    qop, cop = lq["ops"]
    got = _run(lq, x, [qop["output"], cop["output"]])
    assert any(n.startswith("conv_f8_tcgen05") for n in helpers.LAST_LAUNCH_NAMES), helpers.LAST_LAUNCH_NAMES
    assert any(n.startswith("quantize_f8") for n in helpers.LAST_LAUNCH_NAMES), helpers.LAST_LAUNCH_NAMES
    _, snap = O8.fp8_forward(lq, x, keep=[qop["output"]])
    np.testing.assert_array_equal(got[qop["output"]], snap[qop["output"]])  # the quantize kernel: bit-exact
    share = _within(cop, got[qop["output"]], got[cop["output"]])
    print(f"[fp8] {cin}x{h} -> {cout} k{k}/s{stride}: {share:.4f} of codes equal the exact oracle")


@pytest.mark.parametrize("cin,h,cout,k,stride,bn", [(64, 56, 256, 1, 1, 256), (256, 14, 256, 3, 1, 256), (512, 7, 2048, 1, 1, 256),
                                                    (128, 28, 128, 3, 1, 128), (64, 56, 64, 3, 1, 128)])
@pytest.mark.parametrize("relu", [True, False])
def test_fp8_conv_fused_residual_both_tiles(gpu, cin, h, cout, k, stride, bn, relu):
    """y = [relu](conv_b(x) + conv_a(x)): the fused residual reads the E4M3 residual tile with its own scale."""
    low = _conv_graph(cin, h, cout, k, stride, relu=relu, residual=True, seed=3 + relu)
    x = _fp16_exact(np.random.default_rng(5).standard_normal((2, cin, h, h)).astype(np.float32))
    lq = quantize.quantize_lowered(low, x, fmt="e4m3")
    qop, short, conv = lq["ops"]
    assert conv["residual"] == short["output"]
    got = _run(lq, x, [qop["output"], short["output"], conv["output"]], options={"i8_bn": bn})
    assert sum(f" bn={bn}" in n for n in helpers.LAST_LAUNCH_NAMES if n.startswith("conv_f8")) == 2
    _within(short, got[qop["output"]], got[short["output"]])
    _within(conv, got[qop["output"]], got[conv["output"]], res=got[short["output"]])
    if not relu:
        assert (O8.value(got[conv["output"]]) < 0).any()


def test_fp8_avgpool_and_output_cast_bit_exact(gpu):
    net = {"name": "conv_pool", "input": "data", "input_dims": [1, 64, 7, 7], "layers": [
        dict(name="conv", type="Convolution", bottoms=["data"], tops=["conv"], num_output=256, kernel_size=1, pad=0, stride=1, bias_term=True),
        dict(name="pool", type="Pooling", bottoms=["conv"], tops=["pool"], pool="AVE", kernel_size=7, stride=1, pad=0)]}
    low = graph.lower(net, weights.random_weights(net, 1))
    x = _fp16_exact(np.random.default_rng(2).standard_normal((5, 64, 7, 7)).astype(np.float32))
    lq = quantize.quantize_lowered(low, x, fmt="e4m3")
    got = _run(lq, x, ["conv", "pool"])  # _codes() checks the output cast's form
    names = helpers.LAST_LAUNCH_NAMES
    assert any(n.startswith("avgpool_f8") for n in names) and any(n.startswith("output_cast_f8") for n in names), names
    pool_op = next(o for o in lq["ops"] if o["type"] == "avgpool")
    want = O8.avgpool_fp8(got["conv"], pool_op["k_scale"])
    np.testing.assert_array_equal(got["pool"].reshape(5, -1), want.reshape(5, -1).astype(np.float32))


def test_fp8_tactics_give_the_same_bits(gpu):
    """Every (N tile, ring depth) adds the same products in the same order: the same codes.  A tuned engine runs what the
    tuner chose and gives the untuned engine's codes."""
    for cin, h, cout, k, stride in [(256, 14, 256, 3, 1), (512, 28, 1024, 1, 2), (64, 56, 256, 1, 1)]:
        low = _conv_graph(cin, h, cout, k, stride, relu=False, residual=True, seed=9)
        x = _fp16_exact(np.random.default_rng(3).standard_normal((3, cin, h, h)).astype(np.float32))
        lq = quantize.quantize_lowered(low, x, fmt="e4m3")
        blob = builder.build_plan(lq, builder.PREC_FP8, 3)
        eng = capi.Engine(blob)
        try:
            ref = None
            for bn in (128, 256):
                for st in (1, 2, 3, 4):
                    if bn == 256 and st == 4:
                        continue
                    sess = capi.Session(eng, {"i8_bn": bn, "i8_stages": st, "autotune": 0})
                    try:
                        out = list(sess.infer(x).values())[0]
                        n = sess.nb_launches(3)
                        names = [capi.load().b2_context_launch_name(sess.ctx, 3, i).decode() for i in range(n)]
                    finally:
                        sess.close()
                    assert any(f"bn={bn} st={st}" in nm for nm in names if nm.startswith("conv_f8")), names
                    if ref is None:
                        ref = out
                    np.testing.assert_array_equal(out, ref, err_msg=f"bn={bn} st={st}")
            assert eng.tune(streams=4) > 0
            sess = capi.Session(eng)
            try:
                np.testing.assert_array_equal(list(sess.infer(x).values())[0], ref)
            finally:
                sess.close()
        finally:
            eng.destroy()


def _full_net_check(depth, batch, max_batch, seed):
    net = graph.resnet_caffe(depth)
    wts = weights.random_weights(net, 0)
    low = graph.lower(net, wts)
    lq = quantize.quantize_lowered(low, weights.synthetic_input(8, seed=4321), fmt="e4m3")
    x = weights.synthetic_input(batch, seed=seed)
    blob = builder.build_plan(lq, builder.PREC_FP8, max_batch, outputs=["pool1", "prob"])
    eng = capi.Engine(blob)
    sess = capi.Session(eng)
    try:
        out = sess.infer(x)
        names = [capi.load().b2_context_launch_name(sess.ctx, batch, i).decode() for i in range(sess.nb_launches(batch))]
    finally:
        sess.close()
        eng.destroy()
    assert sum(n.startswith("conv_f8_tcgen05") for n in names) == sum(1 for o in lq["ops"] if o.get("fp8"))
    assert not any(n.startswith("conv_i8") for n in names)
    # 1. the fp16 stem within fp16 tolerance of the oracle's own stem
    _, snaps = O8.fp8_forward(lq, x, keep=["pool1"])
    assert helpers.rel_err(out["pool1"], snaps["pool1"]) <= 4e-3
    oracle = O8.fp8_forward(lq, x, start_from={"pool1": out["pool1"].astype(np.float64)})
    # 2. no further from the FP8 oracle than the FP8 oracle is from the fp32 model (+ 1e-3)
    ref = caffe_forward(net, wts, x)
    gap, dist = helpers.rel_err(oracle, ref), helpers.rel_err(out["prob"], oracle)
    assert dist <= gap + 1e-3, (dist, gap)
    # 3. downstream of the GPU's pool1: the FP8 oracle's top-1 wherever the oracle's two leading classes are further apart
    #    than twice that distance.  ResNet-152's synthetic softmax has two classes near p = 0.5 on most images (see
    #    test_int8.py), and there the 1 % of codes that the tensor core's accumulation moves by one step can swap them: the
    #    class must then still be one of the oracle's top two.
    top2 = np.sort(oracle, axis=1)[:, -2:]
    clear = top2[:, 1] - top2[:, 0] > 2 * dist * oracle.max()
    got, want = out["prob"].argmax(1), oracle.argmax(1)
    print(f"[fp8] ResNet-{depth} b={batch}: top-1 equal on {int((got == want).sum())} of {batch} images, {int(clear.sum())} with a "
          f"clear margin; distance {dist:.2e}, oracle vs fp32 {gap:.2e}")
    assert (got[clear] == want[clear]).all()
    assert all(g in t for g, t in zip(got, np.argsort(-oracle, axis=1)[:, :2]))
    if depth == 50:
        assert (got == want).all()


def test_fp8_resnet50_full_network(gpu):
    _full_net_check(50, 8, 8, seed=1234)
    _full_net_check(50, 3, 8, seed=5)  # partial batch through a max-batch-8 plan


def test_fp8_resnet152_batch32_full_network(gpu):
    _full_net_check(152, 32, 32, seed=11)


def test_fp8_resnet152_behind_the_dynamic_batcher(gpu):
    """Single-image requests -> BatchedInferRunner -> FP8 engine: every image's result is the direct batched result."""
    blob = builder.build_resnet_plan(152, builder.PREC_FP8, 32)
    x = weights.synthetic_input(40, seed=21)
    eng = capi.Engine(blob)
    sess = capi.Session(eng)
    try:
        direct = np.concatenate([sess.infer(x[:32])["prob"], sess.infer(x[32:])["prob"]], 0)
    finally:
        sess.close()
        eng.destroy()
    mgr = capi.InferenceManager(max_exec_concurrency=2, max_copy_concurrency=4)
    try:
        mgr.register_model("rn152f8", blob)
        mgr.update_resources()
        got, batches = mgr.infer_batched("rn152f8", x, window_us=20000)
        assert batches == 2
        np.testing.assert_array_equal(got, direct)
    finally:
        mgr.close()
