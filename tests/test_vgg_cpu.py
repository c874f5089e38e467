"""VGG-16 / VGG-19 without a GPU: the generated nets, hidden fully-connected layers in the lowering and the plan, each
refusal with the layer named, the prototxt / generator / ONNX front ends, the float64 oracle against torchvision, the
streaming FC record's plan refusals, and the bytes of every plan without a hidden FC."""
from __future__ import annotations

import hashlib
import re
import struct

import numpy as np
import pytest
import torch

from oracle.caffe_forward import caffe_forward, lowered_forward_f16emu
from tensorrt_laboratory_b200 import bert, builder, capi, graph, onnx_import, onnx_lite, quantize, vgg, vit, weights
from tests.cnn_nets import fc_net


def _records(blob):
    hdr = builder._HEADER.unpack_from(blob, 0)
    version, n_t, n_o = hdr[1], hdr[4], hdr[5]
    tensors = [builder._TENSOR.unpack_from(blob, 128 + i * 96) for i in range(n_t)]
    base = 128 + n_t * 96
    op_struct = builder._OP_V4 if version == 4 else builder._OP
    ops = [op_struct.unpack_from(blob, base + i * op_struct.size) for i in range(n_o)]
    return version, tensors, ops, base


def _weighted(net):
    return [L["name"] for L in net["layers"] if L["type"] in ("Convolution", "InnerProduct")]


@pytest.mark.parametrize("depth, convs", [(16, 13), (19, 16)])
def test_generator_shapes_and_layer_counts(depth, convs):
    net = graph.vgg_caffe(depth)
    names = _weighted(net)
    assert len(names) == depth and names[-3:] == ["fc6", "fc7", "fc8"] and len(names) - 3 == convs
    shapes = graph.infer_shapes(net)
    assert shapes["pool5"] == (512, 7, 7) and shapes["fc6"] == (4096, 1, 1) and shapes["prob"] == (1000, 1, 1)
    assert [shapes[f"pool{b}"][1] for b in range(1, 6)] == [112, 56, 28, 14, 7]
    assert [L["name"] for L in net["layers"][-8:]] == ["fc6", "relu6", "drop6", "fc7", "relu7", "drop7", "fc8", "prob"]
    with pytest.raises(ValueError, match="VGG depth 11"):
        graph.vgg_caffe(11)


def test_vgg16_flops():
    # 30.94 GFLOP per image, the same count the lowering gave before the FC ReLUs could be lowered
    low = graph.lower(graph.vgg_caffe(16))
    assert graph.conv_flops(low) == 30940528640
    no_fc_relu = dict(graph.vgg_caffe(16))
    no_fc_relu["layers"] = [L for L in no_fc_relu["layers"] if not (L["type"] in ("ReLU", "Dropout") and L["bottoms"][0].startswith("fc"))]
    assert graph.conv_flops(graph.lower(no_fc_relu)) == graph.conv_flops(low)


def test_fc_relu_fuses_and_hidden_outputs_are_fp16():
    low = graph.lower(graph.vgg_caffe(16))
    fcs = {o["name"]: o for o in low["ops"] if o["type"] == graph.OP_FC}
    assert [(fcs[n]["relu"], fcs[n]["hidden"]) for n in ("fc6", "fc7", "fc8")] == [(True, True), (True, True), (False, False)]
    assert fcs["fc7"]["in_chw"] == (4096, 1, 1) and fcs["fc8"]["in_chw"] == (4096, 1, 1)
    assert len(low["ops"]) == 22 and not any(o["type"] == "relu" for o in low["ops"])
    net = fc_net((64, 2, 2), [100, 10], [True, False])
    blob = builder.build_plan(graph.lower(net, weights.random_weights(net, 1)), builder.PREC_FP16, max_batch=4)
    version, tensors, ops, _ = _records(blob)
    t = {r[0].rstrip(b"\0").decode(): r for r in tensors}
    assert version == 4
    assert t["fc1"][1:6] == (builder.T_ACT, 1, 1, 100, 128)  # kind, h, w, c, c_phys = 100 rounded up to 64
    assert t["fc2"][1] == builder.T_VEC and t["fc2"][4] == 10
    fc = [o for o in ops if o[1] == builder.OP_FC]
    assert [o[9] for o in fc] == [builder.FC_STREAM | 1, builder.FC_STREAM]
    assert [(o[11], o[12], o[13], o[14]) for o in fc] == [(256, 100, 256, 128), (100, 10, 128, 128)]  # cin, cout, K, cout_phys
    # one FC with a fused ReLU also streams; one FC without stays on the old path (and its plan's version)
    one = fc_net((64, 2, 2), [100], [True])
    assert _records(builder.build_plan(graph.lower(one, weights.random_weights(one, 1)), builder.PREC_FP16, 4))[2][1][9] == 33
    plain = fc_net((64, 2, 2), [100], [False])
    version, _, ops, _ = _records(builder.build_plan(graph.lower(plain, weights.random_weights(plain, 1)), builder.PREC_FP16, 4))
    assert version == 1 and ops[1][9] == 0


def test_refusals_name_the_layer():
    net = graph.vgg_caffe(16)
    low = graph.lower(net, weights.random_weights(net, 0))
    with pytest.raises(ValueError, match="fc fc6: an InnerProduct with a fused ReLU builds in fp16 only"):
        builder.build_plan(low, builder.PREC_FP32, 2)
    for fmt in ("int8", "e4m3"):
        with pytest.raises(ValueError, match="fc fc6: an InnerProduct with a fused ReLU builds in fp16 only"):
            quantize.quantize_lowered(low, weights.synthetic_input(1, seed=1), fmt=fmt)
    soft = fc_net((64, 1, 1), [10], [False])
    soft["layers"] += [dict(name="prob", type="Softmax", bottoms=["fc1"], tops=["prob"]),
                       dict(name="relu_prob", type="ReLU", bottoms=["prob"], tops=["prob"])]
    with pytest.raises(ValueError, match="ReLU relu_prob: a ReLU on the output of Softmax prob"):
        graph.lower(soft)
    res = fc_net((64, 1, 1), [64, 64], [True, False])
    res["layers"].append(dict(name="sum", type="Eltwise", bottoms=["fc1", "fc2"], tops=["sum"], operation="SUM"))
    with pytest.raises(ValueError, match="Eltwise sum: InnerProduct fc1 cannot take a residual"):
        graph.lower(res)


def _prototxt(depth):
    lines = [f'name: "VGG_ILSVRC_{depth}_layers"', 'input: "data"'] + [f"input_dim: {d}" for d in (10, 3, 224, 224)]
    for L in graph.vgg_caffe(depth)["layers"]:
        body = ""
        if L["type"] == "Convolution":
            body = f"convolution_param {{ num_output: {L['num_output']} pad: 1 kernel_size: 3 }}"
        elif L["type"] == "Pooling":
            body = "pooling_param { pool: MAX kernel_size: 2 stride: 2 }"
        elif L["type"] == "InnerProduct":
            body = f"inner_product_param {{ num_output: {L['num_output']} }}"
        elif L["type"] == "Dropout":
            body = "dropout_param { dropout_ratio: 0.5 }"
        lines.append(f'layers {{ bottom: "{L["bottoms"][0]}" top: "{L["tops"][0]}" name: "{L["name"]}" type: {L["type"]} {body} }}'
                     .replace("layers {", "layer {").replace(f"type: {L['type']}", f'type: "{L["type"]}"'))
    return "\n".join(lines)


def _same_ops(a, b):
    assert [o["type"] for o in a["ops"]] == [o["type"] for o in b["ops"]]
    for x, y in zip(a["ops"], b["ops"]):
        for k in ("cin", "cout", "k", "stride", "pad", "relu", "hidden", "in_chw"):
            assert x.get(k) == y.get(k), (x["name"], k)
        if "W" in x:
            assert np.abs(x["W"] - y["W"]).max() <= 1e-6 and np.abs(x["bias"] - y["bias"]).max() <= 1e-6, x["name"]
    assert a["tensors"] == b["tensors"] or list(a["tensors"].values()) == list(b["tensors"].values())


def test_prototxt_generator_and_onnx_lower_alike():
    net = graph.vgg_caffe(16)
    parsed = graph.parse_prototxt(_prototxt(16))
    parsed["input_dims"][0] = 1
    assert [(L["name"], L["type"]) for L in parsed["layers"]] == [(L["name"], L["type"]) for L in net["layers"]]
    _same_ops(graph.lower(parsed), graph.lower(net))
    # ONNX: Gemm -> Relu, and Flatten / Dropout between Gemms, lower to the same ops (small VGG-style head for speed)
    small = fc_net((32, 4, 4), [48, 40], [True, False])
    small["layers"].insert(2, dict(name="drop1", type="Dropout", bottoms=["fc1"], tops=["fc1"]))
    small["layers"].append(dict(name="prob", type="Softmax", bottoms=["fc2"], tops=["prob"]))
    w = weights.random_weights(small, 3)
    model = onnx_lite.parse_model(onnx_import.export_onnx(small, w))
    assert [n["op"] for n in model["nodes"]] == ["Flatten", "Gemm", "Relu", "Flatten", "Gemm", "Softmax"]
    net2, w2 = onnx_import.import_onnx(model, name=small["name"])
    _same_ops(graph.lower(net2, w2), graph.lower(small, w))


@pytest.mark.parametrize("depth", [16, 19])
def test_float64_oracle_matches_torchvision(depth):
    import torchvision
    torch.manual_seed(depth)
    model = getattr(torchvision.models, f"vgg{depth}")(weights=None).double().eval()
    sd = {k: v.numpy() for k, v in model.state_dict().items()}
    wts = vgg.load_weights(sd, depth)
    x = weights.synthetic_input(2, seed=depth)
    with torch.no_grad():
        want = torch.softmax(model(torch.from_numpy(x).double()), dim=1).numpy()
    got = caffe_forward(graph.vgg_caffe(depth), wts, x, dtype=torch.float64)
    assert float(np.abs(got - want).max()) <= 1e-10
    with pytest.raises(ValueError, match="224 x 224 only"):
        vgg.load_weights(sd, depth, image=256)
    bad = dict(sd)
    del bad["classifier.3.weight"]
    with pytest.raises(KeyError, match="classifier.3.weight"):
        vgg.load_weights(bad, depth)


def test_emulation_tracks_the_float64_oracle():
    """fp16 emulation of a reduced VGG (same head, 32 x 32 input): close to float64 and the same top-1."""
    net = graph.vgg_caffe(16)
    net = dict(net, input_dims=[1, 3, 32, 32])
    net["layers"] = [dict(L, num_output=64) if L["name"] in ("fc6", "fc7") else L for L in net["layers"]]
    wts = weights.random_weights(net, 2)
    x = weights.synthetic_input(2, chw=(3, 32, 32), seed=2)
    ref = caffe_forward(net, wts, x, dtype=torch.float64)
    emu = lowered_forward_f16emu(graph.lower(net, wts), x)
    assert float(np.abs(emu - ref).max()) <= 1e-3 and np.array_equal(emu.argmax(1), ref.argmax(1))


# sha256 of plans at the commit before hidden FC layers existed: plans without one keep their bytes (ResNet-50, ResNeXt-50
# and GoogLeNet are pinned elsewhere)
PLAN_SHA256 = {
    "densenet121": "c850b84e85d997442975a8996875f64cd17c6c510ee824121cc87583e5730a4f",
    "bert_small": "5e096df8a41ebd4b72a7919cde01d56310c9dba2e2f20cf3dea075b4fdbb1410",
    "vit_small": "c037c7d19e67eb685974a5ab8dc07152ed127b63c55b9cd0fdcad23aa536ba63",
    "fc2_fp32": "f402e8e7be8f83d25753e81dfde9099209c15edda43400cb17fe72dac1678a0d",
}


def test_plans_without_hidden_fc_keep_their_bytes():
    def sha(blob):
        return hashlib.sha256(blob).hexdigest()
    assert sha(builder.build_densenet_plan(121, max_batch=8)) == PLAN_SHA256["densenet121"]
    cfg = bert.BertConfig(layers=2, hidden=128, heads=2, ffn=512, seq=64, vocab=1000)
    assert sha(builder.build_bert_plan(cfg, max_batch=4)) == PLAN_SHA256["bert_small"]
    vc = vit.VitConfig(layers=2, hidden=128, heads=2, ffn=256, image=64, classes=10)
    assert sha(builder.build_vit_plan(vc, max_batch=4)) == PLAN_SHA256["vit_small"]
    # two FCs without a ReLU in an fp32 plan: the old fp32 vector path
    net = {"name": "fc2", "input": "data", "input_dims": [1, 64, 2, 2], "layers": [
        dict(name="fc1", type="InnerProduct", bottoms=["data"], tops=["fc1"], num_output=100, bias_term=True),
        dict(name="fc2", type="InnerProduct", bottoms=["fc1"], tops=["fc2"], num_output=10, bias_term=True)]}
    assert sha(builder.build_plan(graph.lower(net, weights.random_weights(net, 0)), builder.PREC_FP32, 4)) == PLAN_SHA256["fc2_fp32"]


# ---- plan refusals of the streaming FC record (plan_format.h, kFcStream) ---------------------------------------------------
def fc_mutations():
    """A two-FC streaming plan and (what, mutated blob, message) triples, one per refusal; used on the GPU too."""
    net = fc_net((64, 1, 1), [100, 10], [True, False])
    blob = builder.build_plan(graph.lower(net, weights.random_weights(net, 0)), builder.PREC_FP16, max_batch=2)
    version, tensors, ops, base = _records(blob)
    assert version == 4
    t_base = 128
    tidx = {r[0].rstrip(b"\0").decode(): i for i, r in enumerate(tensors)}
    oidx = {r[0].rstrip(b"\0").decode(): i for i, r in enumerate(ops)}

    def edit_op(name, **kw):
        fields = {"inp": 2, "relu": 9, "cout_phys": 14}
        rec = list(ops[oidx[name]])
        for k, v in kw.items():
            rec[fields[k]] = v
        out = bytearray(blob)
        builder._OP_V4.pack_into(out, base + oidx[name] * 192, *rec)
        return bytes(out)

    def edit_tensor(name, **kw):
        fields = {"c": 4, "c_phys": 5}
        rec = list(tensors[tidx[name]])
        for k, v in kw.items():
            rec[fields[k]] = v
        out = bytearray(blob)
        builder._TENSOR.pack_into(out, t_base + tidx[name] * 96, *rec)
        return bytes(out)

    fp32 = bytearray(blob)
    struct.pack_into("<I", fp32, 12, builder.PREC_FP32)
    fc1 = ops[oidx["fc1"]]
    return blob, [
        ("flag in an fp32 plan", bytes(fp32), r"fc fc1: a streaming FC layer needs a version-4 fp16 plan"),
        ("K not a multiple of 64", edit_tensor("data", c=72, c_phys=72), r"fc fc1: K = h \* w \* c_phys = 72 .* not a multiple of 64"),
        ("cout_phys", edit_op("fc1", cout_phys=256), r"fc fc1: weights must be 128 x 64 fp16"),
        ("ReLU without the flag", edit_op("fc1", relu=1), r"fc fc1: a fused ReLU exists on streaming \(kFcStream\) FC layers only"),
        ("unknown flag", edit_op("fc1", relu=fc1[9] | 64), r"fc fc1: unknown flags 0x61"),
        ("output c_phys", edit_tensor("fc1", c_phys=192), r"fc fc1: the output is an fp32 \[100\] vector or an fp16 \[1, 1, 100\]"),
        ("output c", edit_tensor("fc1", c=96), r"fc fc1: the output is an fp32"),
        ("input not an fp16 activation", edit_op("fc2", inp=tidx["fc2"]), r"fc fc2: a streaming FC layer reads an fp16 activation"),
    ]


def test_fc_stream_plan_refusals():
    blob, muts = fc_mutations()
    capi.Engine(blob, inspect_only=True).destroy()
    for what, bad, msg in muts:
        with pytest.raises(capi.B2Error) as ei:
            capi.Engine(bad, inspect_only=True)
        assert ei.value.code == 1 and re.search(msg, str(ei.value)), (what, str(ei.value))
