"""FP8 (E4M3) precision on the CPU: the quantizer, the E4M3 rounding and epilogue contract of the oracle, the plan layout,
the engine's validation of FP8 plans, and the accuracy of the scheme against the fp32 oracle."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from oracle import fp8_forward as O8
from oracle.caffe_forward import caffe_forward
from tensorrt_laboratory_b200 import builder, capi, graph, quantize, weights

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _conv_graph(cin, h, cout, k, stride, relu=True, residual=False, seed=0):
    net = builder.single_conv_net(cin, h, h, cout, k, stride, k // 2, relu=relu, residual=residual)
    return graph.lower(net, weights.random_weights(net, seed))


def _fp16_exact(x):
    return x.astype(np.float16).astype(np.float32)


def _e4m3_bits(x: np.ndarray) -> np.ndarray:
    """Independent bit-level E4M3 (e4m3fn) encoder: fp32 -> code, round to nearest even, saturating to +-448, NaN -> 0x7F
    (with the sign bit).  Exponent bias 7, 3 mantissa bits, subnormals k * 2^-9."""
    x = np.asarray(x, np.float32)
    bits = x.view(np.uint32)
    sign = ((bits >> 31) & 1).astype(np.uint8) << 7
    with np.errstate(invalid="ignore"):
        a = np.abs(x).astype(np.float64)
    code = np.zeros(x.shape, np.int64)
    sub = a < 2.0 ** -6
    code[sub] = np.rint(a[sub] * 2.0 ** 9).astype(np.int64)          # exact scaling; rint = round half to even
    norm = ~sub & (a < 448.0) & np.isfinite(a)
    e = np.floor(np.log2(a[norm])).astype(np.int64)
    e += (a[norm] >= 2.0 ** (e + 1)).astype(np.int64)                 # guard log2 rounding at powers of two
    e -= (a[norm] < 2.0 ** e).astype(np.int64)
    n = np.rint(a[norm] / 2.0 ** (e - 3)).astype(np.int64)           # 8 .. 16 units of the exponent's ulp
    code[norm] = ((e + 7) << 3) + (n - 8)                             # n = 16 carries into the next exponent
    code[(a >= 448.0) & ~np.isnan(a)] = 0x7E                          # saturate (inf included)
    code[np.isnan(a)] = 0x7F
    return (code.astype(np.uint8) | sign).astype(np.uint8)


# ------------------------------------------------------------------------------------------------------------------
# E4M3 rounding and the epilogue contract
# ------------------------------------------------------------------------------------------------------------------
def test_e4m3_matches_a_bit_level_encoder():
    """The oracle's e4m3 (torch's cast behind a clamp) against the independent encoder: every fp16 value, every E4M3 value,
    the exact ties between neighbours and one fp32 ulp either side of them, the subnormal range and its edge, and values
    around the saturation point."""
    f16 = np.arange(65536, dtype=np.uint32).astype(np.uint16).view(np.float16).astype(np.float32)
    vals = O8.E4M3_VALUES[np.isfinite(O8.E4M3_VALUES)]
    pos = np.unique(vals[vals >= 0]).astype(np.float64)
    ties = ((pos[:-1] + pos[1:]) / 2).astype(np.float32)                # exact in fp32
    assert np.array_equal(ties.astype(np.float64), (pos[:-1] + pos[1:]) / 2)
    near = np.concatenate([np.nextafter(ties, np.float32(0)), np.nextafter(ties, np.float32(np.inf))])
    sat = np.array([447.0, 448.0, 455.9, 456.0, 463.99, 464.0, 470.0, 479.0, 480.0, 1e6, 3.4e38, np.inf], np.float32)
    sub = np.linspace(0, 2.0 ** -5, 4097).astype(np.float32)
    rng = np.random.default_rng(0)
    rnd = (rng.standard_normal(200000) * np.exp2(rng.uniform(-14, 10, 200000))).astype(np.float32)
    x = np.concatenate([f16, vals, ties, near, sat, sub, rnd])
    x = np.concatenate([x, -x])
    want = _e4m3_bits(x)
    got = O8.e4m3(x)
    nan = np.isnan(x)
    assert np.array_equal(got[~nan], want[~nan])
    assert np.all((got[nan] & 0x7F) == 0x7F)
    assert np.array_equal(quantize.e4m3(x[~nan]), got[~nan])            # the quantizer's weight conversion is the same
    # spot values: ties to even, saturation instead of NaN, the smallest subnormal, signed zero
    np.testing.assert_array_equal(O8.e4m3(np.array([1.0625, 1.1875, 470.0, -1e9, 2.0 ** -9, 2.0 ** -10, -0.0], np.float32)),
                                  [0x38, 0x3A, 0x7E, 0xFE, 0x01, 0x00, 0x80])


def test_epilogue_contract_on_chosen_accumulators():
    """t = fma(fl32(acc), m, b); t = fma(value(q_res), r, t); t = fmax(t, 0) under ReLU; q = e4m3(t): ties, saturation,
    ReLU, the residual, accumulators above 2^24 (rounded to fp32 before the multiply-add), and NaN."""
    f = np.float32
    op = dict(m=np.array([1.0, 1.0, 1.0, 2.0 ** -20, 1.0], f), b=np.array([0.0, 0.0, -1000.0, 0.0, 0.0], f), r=f(0.5), relu=False)
    #           1.0625 (tie -> 1.0), 1.1875 (tie -> 1.25), saturates at -448, 2^25 + 1 -> fp32 2^25 -> 32, 500 -> 448
    acc = np.array([1.0625, 1.1875, 0.0, 2.0 ** 25 + 1, 500.0]).reshape(1, 5, 1, 1)
    np.testing.assert_array_equal(O8.value(O8.requant(acc, op, None)).ravel(), [1.0, 1.25, -448.0, 32.0, 448.0])
    res = O8.e4m3(np.array([0.125, 0.125, 4.0, 0.0, -8.0], f)).reshape(1, 5, 1, 1)  # + 0.5 * value
    np.testing.assert_array_equal(O8.value(O8.requant(acc, op, res)).ravel(), [1.125, 1.25, -448.0, 32.0, 448.0])
    op["relu"] = True
    np.testing.assert_array_equal(O8.value(O8.requant(-acc, op, None)).ravel(), [0.0, 0.0, 0.0, 0.0, 0.0])
    np.testing.assert_array_equal(O8.value(O8.requant(-acc, op, res)).ravel(), [0.0, 0.0, 0.0, 0.0, 0.0])
    # NaN: kept without ReLU (a NaN code), 0 with it (fmaxf takes the number)
    nan = np.full((1, 5, 1, 1), np.nan)
    op["relu"] = False
    assert (O8.requant(nan, op, None) & 0x7F == 0x7F).all() and (O8.requant(nan, op, res) & 0x7F == 0x7F).all()
    op["relu"] = True
    np.testing.assert_array_equal(O8.value(O8.requant(nan, op, None)).ravel(), [0.0] * 5)
    np.testing.assert_array_equal(O8.value(O8.requant(nan, op, res)).ravel(), [0.0] * 5)


def test_avgpool_contract():
    q = O8.e4m3(np.array([448.0, 448.0, 2.0 ** -9, -1.5] * 12 + [0.25], np.float32)).reshape(1, 1, 7, 7)
    k = np.float32(0.5 / 49)
    s = float(np.float32(448.0 * 2 * 12 + 2.0 ** -9 * 12 - 1.5 * 12 + 0.25))  # exact fp32 sum of the 49 values
    assert O8.avgpool_fp8(q, k).item() == float(np.float16(np.float32(s) * k))


# ------------------------------------------------------------------------------------------------------------------
# quantizer and plan
# ------------------------------------------------------------------------------------------------------------------
def test_quantizer_scales_weights_and_structure():
    low = _conv_graph(64, 14, 128, 3, 1, residual=True, seed=2)
    x = _fp16_exact(np.random.default_rng(0).standard_normal((4, 64, 14, 14)).astype(np.float32))
    lq = quantize.quantize_lowered(low, x, fmt="e4m3")
    li = quantize.quantize_lowered(low, x)
    assert lq["fp8"] and "int8" not in lq and not any(o.get("int8") for o in lq["ops"])
    # same graph as INT8: the same ops, tensors and quantize points
    assert [(o["type"], o["name"], o["input"], o["output"], o.get("residual")) for o in lq["ops"]] == \
           [(o["type"], o["name"], o["input"], o["output"], o.get("residual")) for o in li["ops"]]
    assert sorted(lq["tensor_scales"]) == sorted(li["tensor_scales"])
    for op in lq["ops"][1:]:
        assert op["fp8"] and op["Wq"].dtype == np.uint8
        v = O8.value(op["Wq"])
        # the per-channel maximum maps to +-448
        np.testing.assert_array_equal(np.abs(v).reshape(v.shape[0], -1).max(axis=1), 448.0)
        w_scaled = (np.asarray(op["W"], np.float64) / op["w_scale"][:, None, None, None]).astype(np.float32)
        np.testing.assert_array_equal(op["Wq"], _e4m3_bits(np.clip(w_scaled, -448, 448)))
        assert op["m"].dtype == np.float32 and op["b"].dtype == np.float32
    s = lq["tensor_scales"]
    assert all(np.float32(v) == v for v in s.values())  # scales are fp32 numbers: what the plan stores
    assert s["data_q"] == float(np.float32(np.abs(x).max() / 448.0))
    out_q = O8.fp8_forward(lq, x)
    from oracle.caffe_forward import lowered_forward_f16emu
    ref = lowered_forward_f16emu(low, x, round16=False)
    assert float(np.abs(out_q - ref).max() / np.abs(ref).max()) < 0.08


def test_grouped_graph_refused_before_calibration():
    net = graph.resnext_caffe(50)
    low = graph.lower(net, weights.random_weights(net, 0))
    with pytest.raises(ValueError, match=r"conv \S+: FP8 grouped convolution is not supported"):
        quantize.quantize_lowered(low, None, fmt="e4m3")  # no calibration input: refused before calibrating
    with pytest.raises(ValueError, match="fmt"):
        quantize.quantize_lowered(low, None, fmt="e5m2")


def test_fp8_plan_layout():
    blob = builder.build_resnet_plan(50, builder.PREC_FP8, 4)
    eng = capi.Engine(blob, inspect_only=True)
    assert eng.precision == builder.PREC_FP8 == 3 and eng.precision_name == "fp8" and eng.max_batch == 4
    assert [b["name"] for b in eng.bindings] == ["data", "prob"] and all(b["dtype"] == 0 for b in eng.bindings)
    fp16_blob = builder.build_resnet_plan(50, builder.PREC_FP16, 4)
    i8_blob = builder.build_resnet_plan(50, builder.PREC_INT8, 4)
    assert len(blob) < 0.62 * len(fp16_blob) and len(blob) == len(i8_blob)  # 1-byte weights: half the bytes of the conv stack
    low = graph.lower(graph.resnet_caffe(50), weights.random_weights(graph.resnet_caffe(50), 0))
    with pytest.raises(ValueError, match="PREC_FP8"):
        builder.build_plan(low, builder.PREC_FP8, 4)
    lq = quantize.quantize_lowered(low, weights.synthetic_input(8, seed=4321), fmt="e4m3")
    with pytest.raises(ValueError, match="PREC_INT8"):
        builder.build_plan(lq, builder.PREC_INT8, 4)
    with pytest.raises(ValueError, match="FP8 BERT"):
        builder.build_bert_plan(precision=builder.PREC_FP8)


def _fp16_then_fp8_plan():
    """An fp16 3x3 convolution (3 -> 64 channels) feeding an FP8 1x1 one (64 -> 128)."""
    net = {"name": "fp16_then_fp8", "input": "data", "input_dims": [1, 3, 8, 8], "layers": [
        dict(name="a", type="Convolution", bottoms=["data"], tops=["a"], num_output=64, kernel_size=3, pad=1, stride=1, bias_term=True),
        dict(name="relu_a", type="ReLU", bottoms=["a"], tops=["a"]),
        dict(name="b", type="Convolution", bottoms=["a"], tops=["b"], num_output=128, kernel_size=1, pad=0, stride=1, bias_term=True)]}
    low = graph.lower(net, weights.random_weights(net, 0))
    x = _fp16_exact(np.random.default_rng(1).standard_normal((2, 3, 8, 8)).astype(np.float32))
    return builder.build_plan(quantize.quantize_lowered(low, x, fmt="e4m3"), builder.PREC_FP8, 2)


def _tables(blob):
    hdr = builder._HEADER.unpack_from(blob, 0)
    n_t, n_o, n_b, payload_off = hdr[4], hdr[5], hdr[6], hdr[7]
    t0 = builder._HEADER.size
    o0 = t0 + n_t * builder._TENSOR.size
    tensors = [builder._TENSOR.unpack_from(blob, t0 + i * builder._TENSOR.size) for i in range(n_t)]
    ops = [builder._OP.unpack_from(blob, o0 + i * builder._OP.size) for i in range(n_o)]
    return hdr, tensors, ops, o0, n_b, payload_off


def _op_index(ops, name):
    return next(i for i, o in enumerate(ops) if o[0].rstrip(b"\0").decode() == name)


def test_engine_refuses_malformed_fp8_plans():
    blob = _fp16_then_fp8_plan()
    hdr, tensors, ops, o0, n_b, payload_off = _tables(blob)
    assert hdr[2] == builder.PREC_FP8
    capi.Engine(blob, inspect_only=True).destroy()
    a, b = _op_index(ops, "a"), _op_index(ops, "b")
    assert ops[b][9] & builder.CONV_INT8 and not ops[a][9] & builder.CONV_INT8  # relu bit 2: the 1-byte (here E4M3) conv

    def mutated(offset, fmt, *vals):
        bad = bytearray(blob)
        struct.pack_into(fmt, bad, offset, *vals)
        return bytes(bad)

    def grouped():
        """The same plan as version 2, with the FP8 convolution split into two groups."""
        recs = b"".join(builder._OP_V2.pack(*o, 2 if i == b else 1) for i, o in enumerate(ops))
        n_t = len(tensors)
        tables = builder._HEADER.size + n_t * builder._TENSOR.size + len(recs) + n_b * builder._BINDING.size
        new_off = (tables + 255) // 256 * 256
        h = list(hdr)
        h[1], h[7] = builder.VERSION_GROUPED, new_off
        out = builder._HEADER.pack(*h) + blob[builder._HEADER.size:o0] + recs
        out += blob[o0 + len(ops) * builder._OP.size:o0 + len(ops) * builder._OP.size + n_b * builder._BINDING.size]
        return out + bytes(new_off - len(out)) + blob[payload_off:]

    W_BYTES, OUT = 136, 76
    t_b = ops[b][4]
    cases = {
        "grouped fp8 conv": (grouped(), "FP8 grouped convolution"),
        "weight bytes": (mutated(o0 + b * builder._OP.size + W_BYTES, "<Q", ops[b][18] - 128), "fp8 conv b weight / requantisation size"),
        "fp16 conv writes an fp8 tensor": (mutated(o0 + a * builder._OP.size + OUT, "<i", t_b), "fp16 conv a touches an fp8 tensor"),
    }
    for name, (bad, msg) in cases.items():
        with pytest.raises(capi.B2Error) as ei:
            capi.Engine(bad, inspect_only=True)
        assert ei.value.code == 1 and msg in str(ei.value), (name, str(ei.value))
    # precision 4 does not exist
    with pytest.raises(capi.B2Error) as ei:
        capi.Engine(mutated(12, "<I", 4), inspect_only=True)
    assert ei.value.code == 1 and "unknown precision" in str(ei.value)


def test_build_engine_tool_writes_the_builder_bytes(tmp_path):
    out = tmp_path / "rn50_fp8.plan"
    subprocess.run([sys.executable, os.path.join(ROOT, "tools", "build_engine.py"), "--model", "resnet50", "--precision", "fp8",
                    "--batch", "2", "-o", str(out)], check=True, capture_output=True, cwd=str(tmp_path))
    assert out.read_bytes() == builder.build_resnet_plan(50, builder.PREC_FP8, 2)


# ------------------------------------------------------------------------------------------------------------------
# accuracy of the scheme
# ------------------------------------------------------------------------------------------------------------------
def test_fp8_resnet50_agrees_with_the_fp32_oracle():
    """Same top-1 class as the fp32 oracle on every synthetic image (oracle with exact accumulation)."""
    net = graph.resnet_caffe(50)
    wts = weights.random_weights(net, 0)
    low = graph.lower(net, wts)
    lq = quantize.quantize_lowered(low, weights.synthetic_input(8, seed=4321), fmt="e4m3")
    x = weights.synthetic_input(6, seed=77)
    q = O8.fp8_forward(lq, x)
    ref = caffe_forward(net, wts, x)
    assert (q.argmax(1) == ref.argmax(1)).all()
    assert len(lq["tensor_scales"]) == 53  # pool1_q + the 52 bottleneck convolution outputs
