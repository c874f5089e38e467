"""Grouped INT8 / FP8 convolutions on the GPU: conv_i8_grouped_tcgen05 / conv_f8_grouped_tcgen05 against the CPU oracles.

INT8 is bit-exact against the integer oracle.  FP8 is held to the accumulation interval of test_gpu_fp8.py, with eps =
steps * 2^-12 where steps counts the 32-deep MMAs the kernel issues per output: taps * ceil(cpg / 32) in the diagonal
modes (each K-slice only meets its own output columns) and taps * cpg / 32 in the dense mode.  Grouped layers reach the
oracles as their dense block-diagonal expansion (tests/grouped_1byte_ref.py), which gives the same exact sums.

Measured on an H100 80GB HBM3 (printed by the FP8 shape test): 99.0 % (cpg 256, dense mode) to 99.99 % (cpg 1) of the
FP8 codes equal the exact-accumulation oracle's, 99.7-99.9 % on the seven ResNeXt-50 shapes; every code lies inside the
interval.  FP8 ResNeXt-50 is 1.7e-2 (batch 8) and 2.1e-2 (batch 3) from the FP8 oracle, which is 4.1e-2 and 4.5e-2 from
fp32, and gives the oracle's top-1 on every image.

Every case checks the launch name: the grouped kernel ran, with the expected span and MMA mode (32: one m64n32k32 per
K-slice, 64: m64n64k32, dense: the n128 / n256 sequence over the tile's span), and no SIMT or fp16 convolution ran."""
import math

import numpy as np
import pytest

from oracle import fp8_forward as O8
from oracle.caffe_forward import caffe_forward
from oracle.int8_forward import _requant, int8_forward
from tensorrt_laboratory_b200 import builder, capi, graph, quantize, weights
from tests import grouped_1byte_ref as G1
from tests import helpers
from tests.grouped_oracle import dense_net

pytestmark = pytest.mark.gpu

W_BITS = 12
PREC = {"int8": builder.PREC_INT8, "e4m3": builder.PREC_FP8}
KERNEL = {"int8": "conv_i8_tcgen05", "e4m3": "conv_f8_tcgen05"}


def _resnext50_grouped_shapes():
    """(C, H_in, stride) of the seven distinct grouped convolutions of ResNeXt-50 32x4d (cpg 4 ... 32)."""
    low = graph.lower(graph.resnext_caffe(50))
    seen = []
    for op in low["ops"]:
        if op.get("groups", 1) != 1:
            s = (op["cin"], low["tensors"][op["input"]][1], op["stride"])
            if s not in seen:
                seen.append(s)
    return seen


RX_SHAPES = _resnext50_grouped_shapes()
assert len(RX_SHAPES) == 7
# (C, groups, H_in, stride, relu, residual, batch)
CASES = [(c, 32, h, s, True, False, 3) for c, h, s in RX_SHAPES] + [
    (128, 128, 10, 1, True, False, 3),   # cpg 1 (depthwise)
    (256, 128, 10, 2, True, False, 3),   # cpg 2
    (128, 16, 10, 1, True, False, 3),    # cpg 8
    (256, 16, 9, 2, True, False, 3),     # cpg 16
    (256, 8, 10, 1, True, False, 3),     # cpg 32, two tiles
    (256, 4, 10, 1, True, False, 3),     # cpg 64
    (256, 2, 10, 1, True, False, 3),     # cpg 128: dense mode, span 128
    (512, 2, 8, 1, True, False, 3),      # cpg 256: dense mode, span 256, BN 256 admitted
    (64, 2, 10, 1, True, False, 3),      # a 64-channel input: one padded row, 2 real slices
    (96, 3, 10, 1, True, False, 3),      # Cin 96, cpg 32: 3 real slices
    (192, 6, 10, 1, True, False, 3),     # tile 0 has 4 real slices, tile 1 has 2
    (320, 10, 10, 2, True, False, 3),    # tiles of 4, 4 and 2 real slices
    (128, 32, 10, 1, False, False, 3),   # ReLU off
    (256, 4, 10, 1, False, False, 3),    # ReLU off, cpg 64
    (128, 32, 10, 1, True, True, 3),     # fused residual (dense 1-byte shortcut)
    (256, 4, 10, 1, False, True, 3),     # fused residual, cpg 64, no ReLU
    (512, 2, 8, 1, True, True, 3),       # fused residual, dense mode
    (128, 32, 10, 1, True, False, 1),    # batch 1
    (256, 16, 9, 2, True, False, 1),
]


def _ids(case):
    c, g, h, s, relu, res, b = case
    return f"c{c}g{g}h{h}s{s}" + ("" if relu else "-norelu") + ("-res" if res else "") + f"-b{b}"


def _mode(cpg):
    return "32" if cpg <= 32 else "64" if cpg == 64 else "dense"


def _steps(cpg, taps=9):
    return taps * math.ceil(cpg / 32) if cpg <= 64 else taps * cpg // 32


def _case(c, groups, h, stride, relu, residual, batch, fmt, seed=0):
    net = builder.single_conv_net(c, h, h, c, 3, stride, 1, relu=relu, residual=residual, group=groups)
    low = graph.lower(net, weights.random_weights(net, seed + c + groups))
    x = np.random.default_rng(seed + c * 7 + h).standard_normal((batch, c, h, h)).astype(np.float16).astype(np.float32)
    lq = quantize.quantize_lowered(low, x, fmt=fmt, grouped=True)
    return lq, x


def _values(y, s, fmt):
    """Output-cast values y = fl(value(q) * s) -> the 1-byte values q (int8 as int32, E4M3 as codes)."""
    if fmt == "int8":
        q = np.rint(np.asarray(y, np.float64) / np.float32(s)).astype(np.int32)
        np.testing.assert_array_equal((q.astype(np.float32) * np.float32(s)).astype(np.float32), y)
        return q
    q = O8.e4m3((np.asarray(y, np.float32) / np.float32(s)).astype(np.float32))
    np.testing.assert_array_equal((O8.value(q) * np.float32(s)).astype(np.float32), y)
    return q


def _run(lq, x, fmt, options=None, max_batch=None):
    """-> ({tensor: values}, launch names): every tensor of the graph but the fp16 input, as the 1-byte values."""
    s = lq["tensor_scales"]
    outs = [o["output"] for o in lq["ops"]]
    got = helpers.run_engine(lq, x, PREC[fmt], options=options, outputs=outs, max_batch=max_batch)
    return {k: _values(v, s[k], fmt).reshape(x.shape[0], -1, *v.shape[2:]) for k, v in got.items()}, list(helpers.LAST_LAUNCH_NAMES)


def _check_names(names, fmt, span, cpg, n_grouped=1):
    grouped = [n for n in names if n.startswith(KERNEL[fmt]) and " span=" in n]
    assert len(grouped) == n_grouped, names
    assert all(f" span={span} mode={_mode(cpg)}" in n for n in grouped), grouped
    assert not any(n.startswith(("conv_simt", "conv_tcgen05")) for n in names), names


def _within(op, q_in, got, res, steps):
    """-> share of codes equal to the exact oracle; asserts every code within the accumulation interval."""
    A, P = G1.conv_fp8_grouped(q_in, op)
    eps = steps * 2.0 ** -W_BITS
    lo = O8.value(O8.requant(A - eps * P, op, res))
    hi = O8.value(O8.requant(A + eps * P, op, res))
    v = O8.value(got)
    bad = ~((lo <= v) & (v <= hi))
    assert not bad.any(), f"{int(bad.sum())} codes outside the interval, e.g. {v[bad][:5]} vs [{lo[bad][:5]}, {hi[bad][:5]}]"
    return float((got == O8.requant(A, op, res)).mean())


def _ops(lq):
    conv = next(o for o in lq["ops"] if o.get("groups", 1) != 1)
    short = next((o for o in lq["ops"] if o["type"] == "conv" and o.get("groups", 1) == 1), None)
    q = next(o for o in lq["ops"] if o["type"] == "quantize")
    return q, short, conv


@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_int8_grouped_conv_bit_exact(gpu, case):
    c, groups, h, stride, relu, residual, batch = case
    lq, x = _case(*case, "int8")
    got, names = _run(lq, x, "int8")
    q, short, conv = _ops(lq)
    _check_names(names, "int8", max(c // groups, 128), c // groups)
    _, snap = int8_forward(G1.dense_quantized(lq), x, keep=[q["output"]])
    np.testing.assert_array_equal(got[q["output"]], snap[q["output"]])
    res = None
    if short is not None:
        assert conv["residual"] == short["output"]
        res = got[short["output"]]
    want = _requant(G1.conv_int8_grouped(got[q["output"]], conv), conv, res)
    np.testing.assert_array_equal(got[conv["output"]], want)
    if not relu:
        assert want.min() < 0


@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_fp8_grouped_conv_within_the_accumulation_bound(gpu, case):
    c, groups, h, stride, relu, residual, batch = case
    lq, x = _case(*case, "e4m3")
    got, names = _run(lq, x, "e4m3")
    q, short, conv = _ops(lq)
    cpg = c // groups
    _check_names(names, "e4m3", max(cpg, 128), cpg)
    _, snap = O8.fp8_forward(G1.dense_quantized(lq), x, keep=[q["output"]])
    np.testing.assert_array_equal(got[q["output"]], snap[q["output"]])
    res = got[short["output"]] if short is not None else None
    share = _within(conv, got[q["output"]], got[conv["output"]], res, _steps(cpg))
    print(f"[fp8 grouped] {_ids(case)} mode {_mode(cpg)}: {share:.4f} of codes equal the exact oracle")


@pytest.mark.parametrize("fmt", ["int8", "e4m3"])
def test_grouped_tactics_give_the_same_bits(gpu, fmt):
    """Every admitted (N tile, ring depth) gives the same bits; a forced 256-wide N tile on a span-128 layer falls back to
    128; a tuned engine gives the untuned engine's bits."""
    for c, groups in [(256, 64), (256, 4), (512, 2)]:  # cpg 4, 64, 256
        span = max(c // groups, 128)
        lq, x = _case(c, groups, 10, 1, False, True, 3, fmt, seed=9)
        blob = builder.build_plan(lq, PREC[fmt], 3)
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
                        names = [capi.load().b2_context_launch_name(sess.ctx, 3, i).decode() for i in range(sess.nb_launches(3))]
                    finally:
                        sess.close()
                    grouped = [n for n in names if " span=" in n]
                    assert len(grouped) == 1, names
                    want_bn = bn if span % bn == 0 else 128
                    assert f"bn={want_bn} st={st}" in grouped[0], (bn, st, grouped)
                    if ref is None:
                        ref = out
                    np.testing.assert_array_equal(out, ref, err_msg=f"c={c} g={groups} bn={bn} st={st}")
            assert eng.tune(streams=4) > 0
            sess = capi.Session(eng)
            try:
                np.testing.assert_array_equal(list(sess.infer(x).values())[0], ref)
            finally:
                sess.close()
        finally:
            eng.destroy()


def _resnext(fmt):
    net = graph.resnext_caffe(50)
    wts = weights.random_weights(net, 0)
    low = graph.lower(net, wts)
    lq = quantize.quantize_lowered(low, weights.synthetic_input(8, seed=4321), fmt=fmt, grouped=True)
    return net, wts, lq


def _infer(lq, fmt, x, max_batch, outputs):
    blob = builder.build_plan(lq, PREC[fmt], max_batch, outputs=outputs)
    eng = capi.Engine(blob)
    sess = capi.Session(eng)
    try:
        out = sess.infer(x)
        b = x.shape[0]
        names = [capi.load().b2_context_launch_name(sess.ctx, b, i).decode() for i in range(sess.nb_launches(b))]
    finally:
        sess.close()
        eng.destroy()
    return out, names


def _check_resnext_launches(lq, names, fmt):
    mark = "fp8" if fmt == "e4m3" else "int8"
    assert sum(n.startswith(KERNEL[fmt]) for n in names) == sum(1 for o in lq["ops"] if o.get(mark)) == 52
    grouped = [n for n in names if n.startswith(KERNEL[fmt]) and " span=128 mode=32" in n]
    assert len(grouped) == 16, names
    assert not any(n.startswith("conv_simt") for n in names)


def test_int8_resnext50_full_network(gpu):
    """ResNeXt-50 INT8 at batch 8, and a partial batch of 3 through the same max-batch-8 plan: the fp16 stem within fp16
    tolerance; downstream of the GPU's pool1 every INT8 tensor and the pooled features bit for bit, the classifier within
    1e-3 with the oracle's class; each image's result independent of its batch position."""
    net, wts, lq = _resnext("int8")
    last = [o for o in lq["ops"] if o.get("int8")][-1]["output"]
    outputs = ["pool1", last, "pool5", "prob"]
    x8 = weights.synthetic_input(8, seed=1234)
    results = {}
    for x in (x8, x8[5:]):
        b = x.shape[0]
        out, names = _infer(lq, "int8", x, 8, outputs)
        _check_resnext_launches(lq, names, "int8")
        dq = G1.dense_quantized(lq)
        _, snaps = int8_forward(dq, x, keep=["pool1"])
        assert helpers.rel_err(out["pool1"], snaps["pool1"]) <= 4e-3
        full, snaps = int8_forward(dq, x, keep=[last, "pool5"], start_from={"pool1": out["pool1"].astype(np.float64)})
        np.testing.assert_array_equal(out[last], snaps[last].astype(np.float32) * np.float32(lq["tensor_scales"][last]))
        np.testing.assert_array_equal(out["pool5"].reshape(b, -1), snaps["pool5"].reshape(b, -1).astype(np.float32))
        assert (out["prob"].argmax(1) == full.argmax(1)).all()
        assert (np.abs(out["prob"] - full) / full.max(1, keepdims=True)).max() <= 1e-3
        results[b] = out
    for k in ("pool1", last, "pool5", "prob"):  # batch-position invariance: images 5..7 alone give the batch-8 rows
        np.testing.assert_array_equal(results[3][k], results[8][k][5:])
    ref = caffe_forward(*dense_net(net, wts), x8)
    assert (results[8]["prob"].argmax(1) == ref.argmax(1)).all()


def _fp8_full_net_check(net, wts, lq, batch, max_batch, seed):
    """test_gpu_fp8.py's three whole-network rules on ResNeXt-50."""
    x = weights.synthetic_input(batch, seed=seed)
    out, names = _infer(lq, "e4m3", x, max_batch, ["pool1", "prob"])
    _check_resnext_launches(lq, names, "e4m3")
    dq = G1.dense_quantized(lq)
    _, snaps = O8.fp8_forward(dq, x, keep=["pool1"])
    assert helpers.rel_err(out["pool1"], snaps["pool1"]) <= 4e-3
    oracle = O8.fp8_forward(dq, x, start_from={"pool1": out["pool1"].astype(np.float64)})
    ref = caffe_forward(*dense_net(net, wts), x)
    gap, dist = helpers.rel_err(oracle, ref), helpers.rel_err(out["prob"], oracle)
    assert dist <= gap + 1e-3, (dist, gap)
    top2 = np.sort(oracle, axis=1)[:, -2:]
    clear = top2[:, 1] - top2[:, 0] > 2 * dist * oracle.max()
    got, want = out["prob"].argmax(1), oracle.argmax(1)
    print(f"[fp8] ResNeXt-50 b={batch}: top-1 equal on {int((got == want).sum())} of {batch} images, {int(clear.sum())} with a "
          f"clear margin; distance {dist:.2e}, oracle vs fp32 {gap:.2e}")
    assert (got[clear] == want[clear]).all()
    assert all(g in t for g, t in zip(got, np.argsort(-oracle, axis=1)[:, :2]))


def test_fp8_resnext50_full_network(gpu):
    net, wts, lq = _resnext("e4m3")
    _fp8_full_net_check(net, wts, lq, 8, 8, seed=1234)
    _fp8_full_net_check(net, wts, lq, 3, 8, seed=5)  # partial batch through a max-batch-8 plan


@pytest.mark.parametrize("prec", [builder.PREC_INT8, builder.PREC_FP8])
def test_resnext50_1byte_serving_with_tuned_tactics(gpu, prec):
    """A plan carrying tuned tactics, served by InferenceManager's batcher, gives the direct session's results."""
    blob = builder.build_resnext_plan(50, prec, 8)
    x = weights.synthetic_input(12, seed=21)
    eng = capi.Engine(blob)
    try:
        assert eng.tune(streams=2) > 0
        blob = builder.attach_tactics(blob, eng.tactics())
    finally:
        eng.destroy()
    eng = capi.Engine(blob)
    sess = capi.Session(eng)
    try:
        direct = np.concatenate([sess.infer(x[:8])["prob"], sess.infer(x[8:])["prob"]], 0)
    finally:
        sess.close()
        eng.destroy()
    mgr = capi.InferenceManager(max_exec_concurrency=2, max_copy_concurrency=4)
    try:
        mgr.register_model("rx50", blob)
        mgr.update_resources()
        got, batches = mgr.infer_batched("rx50", x, window_us=20000)
        assert batches == 2
        np.testing.assert_array_equal(got, direct)
    finally:
        mgr.close()
