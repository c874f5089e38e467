"""GoogLeNet without a GPU: the Concat / LRN / Dropout front end and its refusals, the generated BVLC net, the version-4
plan records (channel slices, LRN), the engine's validation of hand-corrupted plans, the two CPU oracles, and round trips
through a .caffemodel and ONNX."""
from __future__ import annotations

import hashlib
import re
import struct

import numpy as np
import pytest

from oracle import numpy_ops
from oracle.caffe_forward import caffe_forward
from tensorrt_laboratory_b200 import builder, caffemodel, capi, graph, onnx_import, onnx_lite, quantize, weights
from tests.cnn_nets import inception_net

PROTOTXT = """
name: "mini"
input: "data"
input_dim: 1 input_dim: 64 input_dim: 14 input_dim: 14
layer { name: "norm" type: "LRN" bottom: "data" top: "norm" }
layer { name: "a" type: "Convolution" bottom: "norm" top: "a" convolution_param { num_output: 16 kernel_size: 1 } }
layer { name: "a_relu" type: "ReLU" bottom: "a" top: "a" }
layer { name: "b" type: "Convolution" bottom: "norm" top: "b" convolution_param { num_output: 32 kernel_size: 3 pad: 1 } }
layer { name: "cat" type: "Concat" bottom: "a" bottom: "b" top: "cat" concat_param { concat_dim: 1 } }
layer { name: "drop" type: "Dropout" bottom: "cat" top: "cat" dropout_param { dropout_ratio: 0.4 } }
layer { name: "pool" type: "Pooling" bottom: "cat" top: "pool" pooling_param { pool: AVE kernel_size: 14 } }
"""


def test_prototxt_layers_and_defaults():
    net = graph.parse_prototxt(PROTOTXT)
    L = {x["name"]: x for x in net["layers"]}
    assert L["norm"]["type"] == "LRN"
    assert (L["norm"]["local_size"], L["norm"]["alpha"], L["norm"]["beta"], L["norm"]["k"]) == (5, 1.0, 0.75, 1.0)
    assert L["cat"]["axis"] == 1 and L["drop"]["type"] == "Dropout"
    assert graph.infer_shapes(net)["cat"] == (48, 14, 14)
    low = graph.lower(net, weights.random_weights(net, 0))
    assert [o["type"] for o in low["ops"]] == ["lrn", "conv", "conv", "avgpool"]
    assert [o.get("out_c0") for o in low["ops"] if o["type"] == "conv"] == [0, 16]
    assert low["ops"][-1]["input"] == "cat" and "a" not in low["tensors"]


@pytest.mark.parametrize("edit, msg", [
    (lambda t: t.replace('top: "norm" }', 'top: "norm" lrn_param { norm_region: WITHIN_CHANNEL } }'), r"LRN norm: .*WITHIN_CHANNEL"),
    (lambda t: t.replace("concat_dim: 1", "axis: 2"), r"Concat cat: .*axis 2"),
    (lambda t: t.replace('type: "Fancy"', ""), None),
])
def test_prototxt_refusals(edit, msg):
    if msg is None:
        with pytest.raises(ValueError, match=r"unsupported layer type 'Fancy' \(x\)"):
            graph.parse_prototxt(PROTOTXT + 'layer { name: "x" type: "Fancy" bottom: "pool" top: "x" }')
        return
    with pytest.raises(ValueError, match=msg):
        graph.parse_prototxt(edit(PROTOTXT))


def _net_with(extra_layers, bottoms=("a", "b")):
    net = graph.parse_prototxt(PROTOTXT)
    layers = [x for x in net["layers"] if x["name"] not in ("cat", "drop", "pool")]
    layers += extra_layers
    layers.append(dict(name="cat", type="Concat", bottoms=list(bottoms), tops=["cat"], axis=1))
    return dict(net, layers=layers)


def test_concat_refusals_name_the_layer():
    pool = dict(name="p", type="Pooling", bottoms=["norm"], tops=["p"], pool="MAX", kernel_size=3, stride=1, pad=1)
    with pytest.raises(ValueError, match=r"Concat cat: input p is not the output of a convolution"):
        graph.lower(_net_with([pool], ("a", "p")))
    other = dict(name="c", type="Convolution", bottoms=["a"], tops=["c"], num_output=8, kernel_size=1, pad=0, stride=1, bias_term=True)
    with pytest.raises(ValueError, match=r"Concat cat: input a is also read by c"):
        graph.lower(_net_with([other]))
    small = dict(name="s", type="Convolution", bottoms=["norm"], tops=["s"], num_output=8, kernel_size=3, pad=0, stride=1, bias_term=True)
    with pytest.raises(ValueError, match=r"Concat cat: input s is 12x12, not 14x14"):
        graph.lower(_net_with([small], ("a", "s")))
    with pytest.raises(ValueError, match=r"Concat cat: input 'a' starts|starts at channel 12"):
        odd = _net_with([dict(name="o", type="Convolution", bottoms=["norm"], tops=["o"], num_output=12, kernel_size=1, pad=0,
                              stride=1, bias_term=True)], ("o", "b"))
        builder.build_plan(graph.lower(odd, weights.random_weights(odd, 0)), builder.PREC_FP16)


def test_precisions_other_than_fp16_are_refused():
    net = inception_net(hw=7)
    low = graph.lower(net, weights.random_weights(net, 0))
    for prec in (builder.PREC_FP32,):
        with pytest.raises(ValueError, match="fp16 only"):
            builder.build_plan(low, prec)
    for fmt in ("int8", "e4m3"):
        with pytest.raises(ValueError, match="fp16 only"):
            quantize.quantize_lowered(low, np.zeros((1, 64, 7, 7), np.float32), fmt=fmt)
    for prec in (builder.PREC_FP32, builder.PREC_INT8, builder.PREC_FP8):
        with pytest.raises(ValueError, match="fp16 only"):
            builder.build_googlenet_plan(prec)


# ---- the generated BVLC net ---------------------------------------------------------------------------------------------
def test_googlenet_shapes_and_flops():
    net = graph.googlenet_caffe()
    names = [x["name"] for x in net["layers"]]
    for n in ("conv1/7x7_s2", "inception_3a/1x1", "inception_3a/output", "pool5/drop_7x7_s1", "loss3/classifier", "prob"):
        assert n in names
    sh = graph.infer_shapes(net)
    want = {"3a": (256, 28), "3b": (480, 28), "4a": (512, 14), "4b": (512, 14), "4c": (512, 14), "4d": (528, 14), "4e": (832, 14),
            "5a": (832, 7), "5b": (1024, 7)}
    for tag, (c, hw) in want.items():
        assert sh[f"inception_{tag}/output"] == (c, hw, hw)
    # 2 x MACs from the shapes: every convolution and the classifier
    flops, cur = 0, {"data": (3, 224, 224)}
    for L in net["layers"]:
        c, h, w = cur[L["bottoms"][0]]
        if L["type"] == "Convolution":
            k, p, s = L["kernel_size"], L["pad"], L["stride"]
            ho, wo = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
            flops += 2 * ho * wo * L["num_output"] * c * k * k
        elif L["type"] == "InnerProduct":
            flops += 2 * c * h * w * L["num_output"]
        cur[L["tops"][0]] = sh[L["tops"][0]] if L["type"] != "Convolution" else (L["num_output"], ho, wo)
    eng = capi.Engine(builder.build_googlenet_plan(max_batch=2), inspect_only=True)
    try:
        assert eng.flops(1) == flops
    finally:
        eng.destroy()


def _records(blob):
    hdr = builder._HEADER.unpack_from(blob, 0)
    version, n_tensors, n_ops = hdr[1], hdr[4], hdr[5]
    tensors = [builder._TENSOR.unpack_from(blob, 128 + i * 96) for i in range(n_tensors)]
    base = 128 + n_tensors * 96
    ops = [builder._OP_V4.unpack_from(blob, base + i * 192) for i in range(n_ops)]
    return version, tensors, ops, base


def test_plan_records_tile_each_concatenated_tensor():
    blob = builder.build_googlenet_plan(max_batch=2)
    version, tensors, ops, _ = _records(blob)
    assert version == builder.VERSION_CONCAT == 4
    slices = {}
    for o in ops:
        if o[27]:
            slices.setdefault(o[4], []).append((o[26], o[27], o[12], o[14], o[0].rstrip(b"\0").decode()))
    assert len(slices) == 9
    for ti, ss in slices.items():
        name, c, c_phys = tensors[ti][0].rstrip(b"\0").decode(), tensors[ti][4], tensors[ti][5]
        ss.sort()
        assert ss[0][0] == 0 and all(a[0] + a[1] == b[0] for a, b in zip(ss, ss[1:])), (name, ss)
        assert ss[-1][0] + ss[-1][1] == c_phys and ss[-1][0] + ss[-1][2] == c, (name, ss)
        assert all(c0 % 8 == 0 and cp == -(-cw // 64) * 64 for c0, cw, _, cp, _ in ss)
    t4d = next(t for t in slices if tensors[t][0].startswith(b"inception_4d/output"))
    assert [(c0, cw) for c0, cw, *_ in sorted(slices[t4d])] == [(0, 112), (112, 288), (400, 64), (464, 112)]
    assert tensors[t4d][4:6] == (528, 576)
    lrn = [o for o in ops if o[1] == builder.OP_LRN]
    assert [o[0].rstrip(b"\0") for o in lrn] == [b"pool1/norm1", b"conv2/norm2"] and all(o[6] == 5 for o in lrn)


def test_existing_plans_keep_their_bytes():
    # SHA-256 of the plans as the builder wrote them before version 4 existed
    assert hashlib.sha256(builder.build_resnet_plan(50)).hexdigest() == "772e777068ec0ec7c17607ac5a60af0263135aa63f88b61b4b96ba737d6a4d74"
    assert hashlib.sha256(builder.build_resnext_plan(50)).hexdigest() == "4002cdf58dccaef6039e5df004b2dee9af3164c3061746f959e42fd1a1d78664"


# ---- hand-corrupted plans ----------------------------------------------------------------------------------------------
def _mutations():
    net = inception_net(hw=7, widths=(16, 32, 48, 112), lrn=dict(local_size=5, alpha=1e-4, beta=0.75, k=1.0))
    blob = builder.build_plan(graph.lower(net, weights.random_weights(net, 0)), builder.PREC_FP16, max_batch=2)
    _, _, ops, base = _records(blob)
    idx = {o[0].rstrip(b"\0").decode(): i for i, o in enumerate(ops)}

    def edit(op, **kw):
        fields = {"res": 3, "k": 6, "c0": 26, "cw": 27}
        rec = list(ops[idx[op]])
        for k, v in kw.items():
            rec[fields[k]] = v
        out = bytearray(blob)
        builder._OP_V4.pack_into(out, base + idx[op] * 192, *rec)
        return bytes(out)

    int8 = bytearray(blob)
    struct.pack_into("<I", int8, 12, builder.PREC_INT8)
    return blob, [
        ("overlap", edit("b/3x3", c0=8), r"conv b/3x3: slice \[8, 40\) of b/output overlaps"),
        ("gap", edit("b/3x3", c0=24), r"conv b/3x3: slice \[24, 56\) of b/output leaves channels \[16, 24\) unwritten"),
        ("misaligned", edit("b/3x3", c0=20), r"conv b/3x3: slice offset 20 is not a multiple of 8"),
        ("past c_phys", edit("b/pool_proj", cw=224), r"conv b/pool_proj: slice \[96, 320\) runs past the 256 channels"),
        ("slice on a pool", edit("b/pool", c0=0, cw=16), r"op b/pool: only a convolution writes an output channel slice"),
        ("residual", edit("b/1x1", res=0), r"conv b/1x1: a slice writer has no residual"),
        ("1-byte plan", bytes(int8), r"(output channel slices exist in fp16 plans only|LRN needs a version-4 fp16 plan)"),
        ("lrn n", edit("norm", k=4), r"lrn norm: local size 4"),
    ]


def test_corrupted_plans_are_refused():
    blob, muts = _mutations()
    capi.Engine(blob, inspect_only=True).destroy()
    for what, bad, msg in muts:
        with pytest.raises(capi.B2Error) as ei:
            capi.Engine(bad, inspect_only=True)
        assert ei.value.code == 1 and re.search(msg, str(ei.value)), (what, str(ei.value))


# ---- oracles and round trips --------------------------------------------------------------------------------------------
def test_torch_oracle_and_numpy_witness_agree():
    import torch
    net = inception_net(cin=16, hw=9, widths=(8, 16, 8, 8), reduce=(8, 8), lrn=dict(local_size=5, alpha=0.05, beta=0.75, k=2.0))
    wts = weights.random_weights(net, 4)
    x = np.random.default_rng(0).standard_normal((2, 16, 9, 9)) * 3
    a = caffe_forward(net, wts, x, dtype=torch.float64)
    b = numpy_ops.forward(net, wts, x)
    assert float(np.abs(a - b).max() / np.abs(b).max()) <= 1e-10
    assert float(np.abs(numpy_ops.lrn(x, 5, 0.05, 0.75, 2.0) - x).max()) > 0.1  # the normalisation matters at this scale


def test_caffemodel_round_trip_gives_the_same_plan():
    net = graph.googlenet_caffe()
    wts = weights.random_weights(net, 2)
    low = graph.lower(net, caffemodel.load_caffemodel(caffemodel.save_caffemodel(net, wts), net))
    assert builder.build_plan(low, builder.PREC_FP16, 2) == builder.build_googlenet_plan(max_batch=2, weights=wts)


def test_onnx_round_trip_gives_the_same_oracle_outputs():
    net = inception_net(cin=16, hw=9, widths=(8, 16, 8, 8), reduce=(8, 8), lrn=dict(local_size=3, alpha=0.05, beta=0.5, k=2.0))
    wts = weights.random_weights(net, 6)
    x = np.random.default_rng(1).standard_normal((2, 16, 9, 9)).astype(np.float32) * 3
    net2, wts2 = onnx_import.import_onnx(onnx_lite.parse_model(onnx_import.export_onnx(net, wts)))
    assert np.allclose(numpy_ops.forward(net2, wts2, x), numpy_ops.forward(net, wts, x), rtol=1e-6, atol=1e-7)
    assert [L["type"] for L in net2["layers"]].count("Concat") == 1 and [L["type"] for L in net2["layers"]].count("LRN") == 1
