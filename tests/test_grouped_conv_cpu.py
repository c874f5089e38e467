"""CPU: grouped convolutions through every host layer -- prototxt / generator / ONNX / caffemodel front ends, the oracles,
the version-2 plan format and its weight layouts, the engine's plan validation, and the INT8 refusal."""
import struct

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import numpy_ops
from oracle.caffe_forward import caffe_forward, lowered_forward_f16emu
from tests import grouped_oracle
from tensorrt_laboratory_b200 import builder, caffemodel, capi, graph, onnx_import, onnx_lite, quantize, weights
from tests import helpers

# op-record field offsets (plan_format.h OpRec / OpRecV2)
RELU, CIN, W_OFF, W_BYTES, GROUPS = 96, 104, 128, 136, 176


def _grouped_case(c, h, k, stride, groups, cout=None, seed=0):
    net = builder.single_conv_net(c, h, h, cout or c, k, stride, k // 2, group=groups)
    wts = weights.random_weights(net, seed)
    return net, wts, graph.lower(net, wts)


def _plan_ops(blob):
    hdr = struct.unpack_from("<8sIIIIIIQQ", blob, 0)
    version, n_t, n_o, payload = hdr[1], hdr[4], hdr[5], hdr[7]
    rec = 192 if version == 2 else 176
    op0 = 128 + n_t * 96
    return version, payload, [op0 + i * rec for i in range(n_o)]


def _conv_record(blob):
    version, payload, offs = _plan_ops(blob)
    off = next(o for o in offs if struct.unpack_from("<I", blob, o + 64)[0] == builder.OP_CONV)
    return version, payload, off


def _unpack_sw128(flat, cout_phys, K):
    """Inverse of builder.pack_weights_sw128, written out element by element."""
    blk = flat.reshape(K // 64, cout_phys // 32, 32, 8, 8)
    W = np.zeros((cout_phys, K), flat.dtype)
    for kb in range(K // 64):
        for nb in range(cout_phys // 32):
            for r in range(32):
                for j in range(8):
                    W[nb * 32 + r, kb * 64 + j * 8:kb * 64 + j * 8 + 8] = blk[kb, nb, r, j ^ (r % 8)]
    return W


def test_group_field_parses_from_prototxt():
    txt = '''name: "g" input: "data" input_dim: 1 input_dim: 8 input_dim: 6 input_dim: 6
    layer { bottom: "data" top: "c" name: "c" type: "Convolution"
            convolution_param { num_output: 16 kernel_size: 3 pad: 1 stride: 1 group: 4 bias_term: false } }
    layer { bottom: "c" top: "d" name: "d" type: "Convolution" convolution_param { num_output: 16 kernel_size: 1 } }'''
    net = graph.parse_prototxt(txt)
    assert net["layers"][0]["group"] == 4 and net["layers"][1].get("group", 1) == 1
    low = graph.lower(net, weights.random_weights(net, 0))
    assert low["ops"][0]["groups"] == 4 and low["ops"][0]["W"].shape == (16, 3, 3, 2)  # OHWI, I = Cin / groups
    assert low["ops"][1]["groups"] == 1


def test_group_that_does_not_divide_is_rejected():
    net = builder.single_conv_net(12, 4, 4, 12, 3, 1, 1, group=5)
    with pytest.raises(ValueError, match="groups"):
        graph.lower(net)


def test_resnext50_census_and_flops():
    net = graph.resnext_caffe(50)
    assert net["name"] == "ResNeXt-50-32x4d"
    convs = [L for L in net["layers"] if L["type"] == "Convolution"]
    grouped = [L for L in convs if L.get("group", 1) != 1]
    assert len(convs) == 53 and len(grouped) == 16 and all(L["group"] == 32 and L["kernel_size"] == 3 for L in grouped)
    # same layer list and names as ResNet-50; only widths, groups and stride placement differ
    rn = graph.resnet_caffe(50)
    assert [L["name"] for L in net["layers"]] == [L["name"] for L in rn["layers"]]
    by = {L["name"]: L for L in net["layers"]}
    for tag, width in (("2a", 128), ("3a", 256), ("4a", 512), ("5a", 1024)):
        s = 1 if tag == "2a" else 2
        assert by[f"res{tag}_branch2b"]["num_output"] == width and by[f"res{tag}_branch2b"]["stride"] == s
        assert by[f"res{tag}_branch2a"]["stride"] == 1 and by[f"res{tag}_branch1"]["stride"] == s
    shapes = graph.infer_shapes(net)
    assert shapes["res2c"] == (256, 56, 56) and shapes["res3a_branch2b"] == (256, 28, 28)
    assert shapes["res5c"] == (2048, 7, 7) and shapes["prob"] == (1000, 1, 1)
    low = graph.lower(net)
    assert sum(o["type"] == "conv" for o in low["ops"]) == 53
    assert sorted({(o["cin"] // o["groups"]) for o in low["ops"] if o["type"] == "conv" and o["groups"] > 1}) == [4, 8, 16, 32]
    gflops = graph.conv_flops(low) / 1e9
    assert round(gflops, 2) == 8.46, gflops
    # grouped weights are [Cout, Cin/g, k, k] with He std over Cin/g * k * k
    w = weights.random_weights(net, 0)
    assert w["res2a_branch2b"]["W"].shape == (128, 4, 3, 3)
    assert 0.9 < np.std(w["res4a_branch2b"]["W"]) / np.sqrt(2.0 / (16 * 9)) < 1.1


def test_dense_weight_draws_are_unchanged():
    # group = 1 draws exactly what the He rule over Cin * k * k always drew, so every existing seed keeps its weights
    net = graph.resnet_caffe(50)
    a = weights.random_weights(net, 0)
    rng = np.random.default_rng(0)
    np.testing.assert_array_equal(a["conv1"]["W"], (rng.standard_normal((64, 3, 7, 7)) * np.sqrt(2.0 / (3 * 49))).astype(np.float32))
    np.testing.assert_array_equal(a["conv1"]["b"], (rng.standard_normal(64) * 0.01).astype(np.float32))


def test_onnx_round_trip_with_groups():
    net, wts, _ = _grouped_case(32, 6, 3, 2, 8)
    model = onnx_lite.parse_model(onnx_import.export_onnx(net, wts))
    conv = next(n for n in model["nodes"] if n["op"] == "Conv")
    assert int(conv["attrs"]["group"]) == 8
    net2, wts2 = onnx_import.import_onnx(model)
    c2 = next(L for L in net2["layers"] if L["type"] == "Convolution")
    assert c2["group"] == 8 and c2["stride"] == 2
    np.testing.assert_array_equal(wts2[c2["name"]]["W"], wts["conv"]["W"])
    x = np.random.default_rng(1).standard_normal((2, 32, 6, 6), dtype=np.float32)
    np.testing.assert_allclose(caffe_forward(*grouped_oracle.dense_net(net2, wts2), x, dtype=torch.float64),
                               caffe_forward(*grouped_oracle.dense_net(net, wts), x, dtype=torch.float64), rtol=0, atol=1e-12)


def test_onnx_import_still_rejects_dilation():
    net, wts, _ = _grouped_case(8, 6, 3, 1, 2)
    model = onnx_lite.parse_model(onnx_import.export_onnx(net, wts))
    next(n for n in model["nodes"] if n["op"] == "Conv")["attrs"]["dilations"] = [2, 2]
    with pytest.raises(ValueError, match="dilated"):
        onnx_import.import_onnx(model)


def test_caffemodel_round_trip_with_groups():
    net, wts, _ = _grouped_case(64, 5, 3, 1, 16)
    back = caffemodel.load_caffemodel(caffemodel.save_caffemodel(net, wts), net)
    assert back["conv"]["W"].shape == (64, 4, 3, 3)
    np.testing.assert_array_equal(back["conv"]["W"], wts["conv"]["W"])
    bad = dict(wts, conv=dict(wts["conv"], W=np.zeros((64, 8, 3, 3), np.float32)))  # Cin/g of 8 groups, file says 16
    with pytest.raises(ValueError, match="groups"):
        caffemodel.load_caffemodel(caffemodel.save_caffemodel(net, bad), net)


@pytest.mark.parametrize("c,cout,groups,k,stride", [(32, 32, 8, 3, 1), (64, 64, 64, 3, 2), (12, 24, 3, 1, 1), (48, 96, 2, 3, 2)])
def test_numpy_grouped_conv_equals_torch(c, cout, groups, k, stride):
    """Both ways the oracles see a grouped convolution -- group by group (numpy witness) and as the dense block-diagonal
    convolution -- equal torch's own grouped convolution."""
    rng = np.random.default_rng(7)
    x = rng.standard_normal((2, c, 7, 7))
    w = rng.standard_normal((cout, c // groups, k, k))
    b = rng.standard_normal(cout)
    ref = F.conv2d(torch.from_numpy(x), torch.from_numpy(w), torch.from_numpy(b), stride=stride, padding=k // 2, groups=groups).numpy()
    np.testing.assert_allclose(grouped_oracle.numpy_conv2d(x, w, b, stride, k // 2, groups), ref, rtol=0, atol=1e-10)
    dense = grouped_oracle.dense_weight(w, groups)
    assert dense.shape == (cout, c, k, k) and np.count_nonzero(dense) == np.count_nonzero(w)
    np.testing.assert_allclose(numpy_ops.conv2d(x, dense, b, stride, k // 2), ref, rtol=0, atol=1e-10)


def test_oracles_agree_on_a_grouped_network():
    net, wts, low = _grouped_case(32, 6, 3, 1, 8)
    x = np.random.default_rng(2).standard_normal((2, 32, 6, 6), dtype=np.float32)
    dnet, dwts = grouped_oracle.dense_net(net, wts)
    assert "group" in net["layers"][0] and "group" not in dnet["layers"][0]  # the input net is left as it was
    a = caffe_forward(dnet, dwts, x, dtype=torch.float64)
    np.testing.assert_allclose(numpy_ops.forward(dnet, dwts, x), a, rtol=0, atol=1e-10)
    # the folded, lowered graph (BN/Scale folded per output channel into the grouped weights) says the same
    np.testing.assert_allclose(lowered_forward_f16emu(grouped_oracle.dense_lowered(low), x, round16=False), a, rtol=0, atol=1e-10)
    # the group-by-group numpy witness (conv + bias + ReLU is the whole net)
    y = grouped_oracle.numpy_conv2d(x.astype(np.float64), wts["conv"]["W"], wts["conv"]["b"], 1, 1, 8)
    np.testing.assert_allclose(np.maximum(y, 0).reshape(2, -1), a, rtol=0, atol=1e-10)


@pytest.mark.parametrize("c,groups,span", [(128, 32, 64), (256, 2, 128)])  # cpg = 4 and cpg = 128
def test_builder_writes_block_diagonal_packed_weights(c, groups, span):
    _, _, low = _grouped_case(c, 4, 3, 1, groups)
    blob = builder.build_plan(low, builder.PREC_FP16, 2)
    version, payload, off = _conv_record(blob)
    assert version == 2
    relu, w_off, w_bytes, g = (struct.unpack_from("<I", blob, off + RELU)[0], struct.unpack_from("<Q", blob, off + W_OFF)[0],
                               struct.unpack_from("<Q", blob, off + W_BYTES)[0], struct.unpack_from("<I", blob, off + GROUPS)[0])
    assert g == groups and relu & 2 and w_bytes == c * 9 * span * 2
    W = _unpack_sw128(np.frombuffer(blob, np.float16, c * 9 * span, payload + w_off), c, 9 * span).reshape(c, 9, span)
    cpg = c // groups
    Wsrc = low["ops"][0]["W"].reshape(c, 9, cpg).astype(np.float16)
    for o in range(c):
        base = (o // span) * span            # first input channel of the tile's span
        lo = (o // cpg) * cpg - base         # the group's columns inside it
        np.testing.assert_array_equal(W[o, :, lo:lo + cpg], Wsrc[o])
        assert not np.any(np.delete(W[o], np.s_[lo:lo + cpg], axis=1))


@pytest.mark.parametrize("precision,c,cout,groups", [(builder.PREC_FP16, 96, 96, 4), (builder.PREC_FP16, 64, 128, 4),
                                                     (builder.PREC_FP32, 128, 128, 32)])
def test_builder_writes_row_major_weights_off_the_tensor_cores(precision, c, cout, groups):
    _, _, low = _grouped_case(c, 4, 3, 1, groups, cout=cout)
    blob = builder.build_plan(low, precision, 2)
    version, payload, off = _conv_record(blob)
    cout_phys = struct.unpack_from("<I", blob, off + CIN + 12)[0]
    relu, w_off, w_bytes = (struct.unpack_from("<I", blob, off + RELU)[0], struct.unpack_from("<Q", blob, off + W_OFF)[0],
                            struct.unpack_from("<Q", blob, off + W_BYTES)[0])
    elt, dt = (4, np.float32) if precision == builder.PREC_FP32 else (2, np.float16)
    cpg = c // groups
    assert version == 2 and not relu & 2 and w_bytes == cout_phys * 9 * cpg * elt
    W = np.frombuffer(blob, dt, cout_phys * 9 * cpg, payload + w_off).reshape(cout_phys, 9, cpg)
    np.testing.assert_array_equal(W[:cout], low["ops"][0]["W"].reshape(cout, 9, cpg).astype(dt))
    assert not np.any(W[cout:])


def test_dense_plans_stay_version_1():
    blob = builder.build_resnet_plan(50, builder.PREC_FP16, 8)
    version, payload, offs = _plan_ops(blob)
    assert version == 1 and offs[1] - offs[0] == 176 == builder._OP.size
    assert struct.unpack_from("<I", blob, offs[1] + 64)[0] == builder.OP_CONV  # the stem conv follows the input cast


def test_grouped_engine_metadata(lib):
    _, _, low = _grouped_case(128, 8, 3, 2, 32)
    eng = capi.Engine(builder.build_plan(low, builder.PREC_FP16, 4), inspect_only=True)
    try:
        assert eng.flops(1) == pytest.approx(2.0 * 4 * 4 * 128 * (128 // 32) * 9)  # algorithmic: Cin/g inputs per channel
    finally:
        eng.destroy()


def test_malformed_grouped_ops_are_rejected(lib):
    _, _, low = _grouped_case(128, 6, 3, 1, 32)
    blob = builder.build_plan(low, builder.PREC_FP16, 2)
    _, _, off = _conv_record(blob)
    capi.Engine(blob, inspect_only=True).destroy()

    def mutated(field, fmt, value):
        bad = bytearray(blob)
        struct.pack_into(fmt, bad, off + field, value)
        return bytes(bad)

    w_bytes = struct.unpack_from("<Q", blob, off + W_BYTES)[0]
    relu = struct.unpack_from("<I", blob, off + RELU)[0]
    cases = {
        "groups do not divide the channels": mutated(GROUPS, "<I", 3),
        "zero groups": mutated(GROUPS, "<I", 0),
        "weight size of another layout": mutated(W_BYTES, "<Q", w_bytes // 16),  # the dense cpg-wide row-major size
        "grouped op flagged INT8": mutated(RELU, "<I", relu | 4),
        "packed layout without a tensor-core geometry": mutated(CIN, "<I", 96),  # Cin != Cout (and != its tensor)
    }
    for name, bad in cases.items():
        with pytest.raises(capi.B2Error) as ei:
            capi.Engine(bad, inspect_only=True)
        assert ei.value.code == 1, name


def test_quantize_rejects_grouped_convolutions():
    _, _, low = _grouped_case(64, 4, 3, 1, 8)
    with pytest.raises(ValueError, match="INT8 grouped convolution is not supported") as ei:
        quantize.quantize_lowered(low, np.zeros((1, 64, 4, 4), np.float32))
    assert "conv conv:" in str(ei.value)
    # rejected before calibration: no forward pass is attempted (there are not even weights here)
    with pytest.raises(ValueError, match="res2a_branch2b: INT8 grouped"):
        quantize.quantize_lowered(graph.lower(graph.resnext_caffe(50)), None)
