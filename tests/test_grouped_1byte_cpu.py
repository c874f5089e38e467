"""CPU: grouped INT8 / FP8 convolutions through the host layers -- the quantizer's opt-in and its refusals, the version-2
plan's block-diagonal 1-byte weight layout, the engine's plan validation, the oracles' grouped evaluation, and the accuracy
of the scheme on ResNeXt-50 32x4d."""
import struct

import numpy as np
import pytest

from oracle import fp8_forward as O8
from oracle.caffe_forward import caffe_forward
from oracle.int8_forward import conv_int8, int8_forward
from tensorrt_laboratory_b200 import builder, capi, graph, quantize, weights
from tests import grouped_1byte_ref as G1
from tests.grouped_oracle import dense_net

FMTS = {"int8": builder.PREC_INT8, "e4m3": builder.PREC_FP8}
# op-record and tensor-record field offsets (plan_format.h OpRec / OpRecV2, TensorRec)
IN, TAPS_PHYS, W_BYTES, GROUPS = 68, 124, 136, 176


def _grouped_case(c, h, k, stride, groups, cout=None, seed=0, relu=True):
    net = builder.single_conv_net(c, h, h, cout or c, k, stride, k // 2, relu=relu, group=groups)
    return graph.lower(net, weights.random_weights(net, seed))


def _quantized_case(c, h, groups, fmt, k=3, stride=1, seed=0):
    low = _grouped_case(c, h, k, stride, groups, seed=seed)
    x = np.random.default_rng(seed).standard_normal((2, c, h, h)).astype(np.float32)
    return quantize.quantize_lowered(low, x, fmt=fmt, grouped=True)


@pytest.fixture(scope="module")
def resnext50():
    net = graph.resnext_caffe(50)
    wts = weights.random_weights(net, 0)
    return net, wts, graph.lower(net, wts)


@pytest.fixture(scope="module")
def resnext50_q(resnext50):
    """{fmt: ResNeXt-50 quantized with grouped=True, calibrated like build_resnext_plan}"""
    calib = weights.synthetic_input(8, seed=4321)
    amax = quantize.calibrate(resnext50[2], calib)
    return {fmt: quantize.quantize_lowered(resnext50[2], calib, amax=amax, fmt=fmt, grouped=True) for fmt in FMTS}


def _half_step_e4m3(v):
    """Half the distance between neighbouring E4M3 values around |v| (subnormal step 2^-9)."""
    e = np.floor(np.log2(np.maximum(np.abs(v), 2.0 ** -6)))
    return 0.5 * 2.0 ** (e - 3)


@pytest.mark.parametrize("fmt", sorted(FMTS))
def test_resnext50_quantizes_its_grouped_convolutions(resnext50_q, fmt):
    lq = resnext50_q[fmt]
    mark = "fp8" if fmt == "e4m3" else "int8"
    grouped = [o for o in lq["ops"] if o["type"] == "conv" and o.get("groups", 1) != 1]
    assert len(grouped) == 16 and all(o.get(mark) and o["groups"] == 32 for o in grouped)
    assert {o["cin"] // 32 for o in grouped} == {4, 8, 16, 32}
    scales = lq["tensor_scales"]
    one_byte = [o for o in lq["ops"] if o.get(mark)]
    assert len(one_byte) == 52  # every convolution but the 3-channel stem
    for o in one_byte:
        for t in (o["input"], o["output"], o["residual"]):
            assert t is None or (t in scales and np.float32(scales[t]) == scales[t] and scales[t] > 0), (o["name"], t)
    for o in grouped:
        W = np.asarray(o["W"], np.float64)
        assert o["Wq"].shape == W.shape == (o["cout"], 3, 3, o["cin"] // 32)
        s = o["w_scale"][:, None, None, None]
        if fmt == "int8":
            assert np.abs(o["Wq"]).max() <= 127
            assert (np.abs(o["Wq"].astype(np.float64) * s - W) <= 0.5 * s * (1 + 1e-9)).all(), o["name"]
        else:
            v = W / s
            assert (np.abs(O8.value(o["Wq"]) - v) <= _half_step_e4m3(v) * (1 + 1e-6)).all(), o["name"]


@pytest.mark.parametrize("fmt,name", [("int8", "INT8"), ("e4m3", "FP8")])
@pytest.mark.parametrize("c,groups,cout", [(64, 2, 128),   # Cin/g != Cout/g
                                           (96, 2, None),  # cpg 48
                                           (192, 2, None)])  # cpg 96
def test_geometries_outside_the_rule_are_refused_before_calibration(fmt, name, c, groups, cout):
    low = _grouped_case(c, 4, 3, 1, groups, cout=cout)
    with pytest.raises(ValueError, match=rf"conv conv: {name} grouped convolution needs Cin/g == Cout/g dividing 128"):
        quantize.quantize_lowered(low, None, fmt=fmt, grouped=True)  # no calibration input: refused before calibrating


def test_default_still_refuses_grouped_graphs():
    low = _grouped_case(128, 4, 3, 1, 32)
    with pytest.raises(ValueError, match="conv conv: INT8 grouped convolution is not supported"):
        quantize.quantize_lowered(low, None)


def test_calibration_of_dense_graphs_is_unchanged():
    """calibrate() passes groups= to the convolution; a dense graph gives the same amax and plan as without grouped=True."""
    blob = builder.build_resnet_plan(50, builder.PREC_INT8, 2)
    net = graph.resnet_caffe(50)
    low = quantize.quantize_lowered(graph.lower(net, weights.random_weights(net, 0)), weights.synthetic_input(8, seed=4321),
                                    grouped=True)
    assert builder.build_plan(low, builder.PREC_INT8, 2) == blob


def _plan_tables(blob):
    hdr = struct.unpack_from("<8sIIIIIIQQ", blob, 0)
    version, prec, n_t, n_o, payload = hdr[1], hdr[2], hdr[4], hdr[5], hdr[7]
    rec = {1: 176, 2: 192, 3: 224}[version]
    op0 = 128 + n_t * 96
    return version, prec, payload, [op0 + i * rec for i in range(n_o)]


def _conv_offset(blob):
    _, _, _, offs = _plan_tables(blob)
    return next(o for o in offs if struct.unpack_from("<I", blob, o + 64)[0] == builder.OP_CONV)


def _unpack_sw128_i8(flat, cout_phys, K):
    """Inverse of builder.pack_weights_sw128_i8, written out element by element."""
    blk = flat.reshape(K // 128, cout_phys // 32, 32, 8, 16)
    W = np.zeros((cout_phys, K), flat.dtype)
    for kb in range(K // 128):
        for nb in range(cout_phys // 32):
            for r in range(32):
                for j in range(8):
                    W[nb * 32 + r, kb * 128 + j * 16:kb * 128 + j * 16 + 16] = blk[kb, nb, r, j ^ (r % 8)]
    return W


@pytest.mark.parametrize("fmt", sorted(FMTS))
@pytest.mark.parametrize("c,groups", [(128, 128), (128, 32), (192, 6), (128, 2), (512, 2)])  # cpg 1, 4, 32, 64, 256
def test_packed_payload_is_the_block_diagonal_expansion(lib, fmt, c, groups):
    lq = _quantized_case(c, 4, groups, fmt)
    op = next(o for o in lq["ops"] if o["type"] == "conv")
    cpg, span, taps = c // groups, max(c // groups, 128), 9
    blob = builder.build_plan(lq, FMTS[fmt], 2)
    version, prec, payload, _ = _plan_tables(blob)
    assert version == builder.VERSION_GROUPED and prec == FMTS[fmt]
    off = _conv_offset(blob)
    cout_phys = struct.unpack_from("<I", blob, off + 116)[0]
    w_off, w_bytes = struct.unpack_from("<QQ", blob, off + 128)
    assert cout_phys == -(-c // 128) * 128 and w_bytes == cout_phys * taps * span
    assert struct.unpack_from("<I", blob, off + GROUPS)[0] == groups
    got = _unpack_sw128_i8(np.frombuffer(blob, np.int8, w_bytes, payload + w_off), cout_phys, taps * span)
    got = got.reshape(cout_phys, taps, span)
    Wq = op["Wq"].view(np.int8).reshape(c, taps, cpg)
    want = np.zeros((cout_phys, taps, span), np.int8)
    for o in range(c):  # row o reads input channels (o // span) * span + j; only its own group's are non-zero
        for j in range(span):
            ci = (o // span) * span + j
            if ci // cpg == o // cpg:
                want[o, :, j] = Wq[o, :, ci % cpg]
    np.testing.assert_array_equal(got, want)
    eng = capi.Engine(blob, inspect_only=True)
    try:
        assert eng.precision == FMTS[fmt]
        assert eng.flops(3) == 3 * 2.0 * 4 * 4 * c * cpg * taps  # algorithmic: Cin/g per output
    finally:
        eng.destroy()


def _mutated(blob, offset, fmt, value):
    bad = bytearray(blob)
    struct.pack_into(fmt, bad, offset, value)
    return bytes(bad)


@pytest.mark.parametrize("fmt,name", [("int8", "INT8"), ("e4m3", "FP8")])
def test_malformed_grouped_1byte_records_are_refused(lib, fmt, name):
    lq = _quantized_case(192, 4, 6, fmt)  # cpg 32
    blob = builder.build_plan(lq, FMTS[fmt], 2)
    capi.Engine(blob, inspect_only=True).destroy()
    off = _conv_offset(blob)
    w_bytes = struct.unpack_from("<Q", blob, off + W_BYTES)[0]
    cases = {
        "weight bytes": (_mutated(blob, off + W_BYTES, "<Q", w_bytes // 2), "grouped conv conv weight / requantisation size"),
        "cpg 48": (_mutated(blob, off + GROUPS, "<I", 4), f"{name} grouped convolution needs"),
        "fp16 input": (_mutated(blob, off + IN, "<i", 0), f"{name} grouped convolution needs"),  # tensor 0: the fp16 input
        "taps_phys != taps": (_mutated(blob, off + TAPS_PHYS, "<I", 10), f"{name} grouped convolution needs"),
    }
    for case, (bad, msg) in cases.items():
        with pytest.raises(capi.B2Error) as ei:
            capi.Engine(bad, inspect_only=True)
        assert ei.value.code == 1 and msg in str(ei.value), (case, str(ei.value))


def test_resnext50_1byte_plans(lib):
    """build_resnext_plan in INT8 and FP8: version 2, 16 grouped 1-byte records, algorithmic flops equal to fp16's."""
    fp16 = capi.Engine(builder.build_resnext_plan(50, builder.PREC_FP16, 2), inspect_only=True)
    try:
        for prec in (builder.PREC_INT8, builder.PREC_FP8):
            blob = builder.build_resnext_plan(50, prec, 2)
            version, p, _, offs = _plan_tables(blob)
            assert version == 2 and p == prec
            g = [o for o in offs if struct.unpack_from("<I", blob, o + 64)[0] == builder.OP_CONV and
                 struct.unpack_from("<I", blob, o + GROUPS)[0] == 32]
            assert len(g) == 16 and all(struct.unpack_from("<I", blob, o + 96)[0] & builder.CONV_INT8 for o in g)
            eng = capi.Engine(blob, inspect_only=True)
            try:
                assert eng.flops(2) == fp16.flops(2)
            finally:
                eng.destroy()
    finally:
        fp16.destroy()


def _random_codes(rng, shape, fmt):
    if fmt == "int8":
        return rng.integers(-127, 128, size=shape).astype(np.int32)
    q = rng.integers(0, 256, size=shape).astype(np.uint8)
    return np.where((q & 0x7F) == 0x7F, q & 0xF0, q).astype(np.uint8)  # no NaN codes


@pytest.mark.parametrize("fmt", sorted(FMTS))
def test_grouped_oracle_equals_the_dense_expansion(resnext50_q, fmt):
    """Each grouped ResNeXt-50 convolution evaluated with groups= gives, bit for bit, what the oracles compute on its dense
    block-diagonal expansion: the integer accumulator (INT8), and A and P (FP8)."""
    lq = resnext50_q[fmt]
    dense = {o["name"]: o for o in G1.dense_quantized(lq)["ops"]}
    rng = np.random.default_rng(7)
    seen = set()
    for op in lq["ops"]:
        if op.get("groups", 1) == 1 or (op["cin"], op["stride"]) in seen:
            continue
        seen.add((op["cin"], op["stride"]))
        q = _random_codes(rng, (2, op["cin"], 9, 9), fmt)
        d = dense[op["name"]]
        assert d["groups"] == 1 and d["Wq"].shape == (op["cout"], 3, 3, op["cin"])
        if fmt == "int8":
            np.testing.assert_array_equal(G1.conv_int8_grouped(q, op), conv_int8(q, d))
        else:
            A, P = G1.conv_fp8_grouped(q, op)
            A2, P2 = O8.conv_fp8(q, d)
            np.testing.assert_array_equal(A, A2)
            np.testing.assert_array_equal(P, P2)
    assert len(seen) == 7  # the seven grouped shapes: cpg 4 ... 32, strides 1 and 2


def test_resnext50_1byte_accuracy(resnext50, resnext50_q):
    """INT8 and FP8 ResNeXt-50 (oracle, exact accumulation) against the fp32 model on 8 synthetic images.

    Measured: both give the fp32 model's top-1 on 8 of 8 images, whose lead over the second class is 0.60 to 0.85 in
    probability; the largest difference from fp32, relative to each row's maximum, is 1.6e-2 for INT8 and 4.4e-2 for FP8."""
    net, wts, _ = resnext50
    x = weights.synthetic_input(8)
    ref = caffe_forward(*dense_net(net, wts), x)
    for fmt, run, bound in (("int8", int8_forward, 0.03), ("e4m3", O8.fp8_forward, 0.08)):
        out = run(G1.dense_quantized(resnext50_q[fmt]), x)
        gap = float((np.abs(out - ref) / ref.max(1, keepdims=True)).max())
        print(f"[{fmt}] ResNeXt-50: top-1 equal on {int((out.argmax(1) == ref.argmax(1)).sum())} of 8, largest gap {gap:.2e}")
        assert (out.argmax(1) == ref.argmax(1)).all(), fmt
        assert gap <= bound, (fmt, gap)
