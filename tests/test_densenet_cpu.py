"""DenseNet without a GPU: the generated nets and their FLOPs, round_mode parsing, the lowering of pre-activations, growing
concatenations and commuted transitions (and its refusals), the plan records and the engine's refusal of corrupted ones,
weight loading, and the CPU oracles against each other and against torchvision."""
from __future__ import annotations

import hashlib
import re

import numpy as np
import pytest

from oracle.caffe_forward import caffe_forward, lowered_forward_f16emu
from tensorrt_laboratory_b200 import builder, caffemodel, capi, densenet, graph, weights
from tests.cnn_nets import dense_net
from tests.test_googlenet_cpu import _records


def _raw_flops(net):
    """2 * MAC of the raw layer list (convolutions at their own resolution, classifier included), per image."""
    shapes = graph.infer_shapes(net)
    cur = {net["input"]: tuple(net["input_dims"][1:])}
    total = 0
    for L in net["layers"]:
        c = cur[L["bottoms"][0]][0]
        if L["type"] == "Convolution":
            co, h, w = shapes[L["tops"][0]]
            total += 2 * co * h * w * c * L["kernel_size"] ** 2
        elif L["type"] == "InnerProduct":
            total += 2 * L["num_output"] * int(np.prod(cur[L["bottoms"][0]]))
        cur[L["tops"][0]] = shapes[L["tops"][0]]
    return total


@pytest.mark.parametrize("depth, blocks, final", [(121, (256, 512, 1024, 1024), 1024), (169, (256, 512, 1280, 1664), 1664),
                                                  (201, (256, 512, 1792, 1920), 1920)])
def test_generated_shapes(depth, blocks, final):
    net = graph.densenet_caffe(depth)
    s = graph.infer_shapes(net)
    assert s["conv1"] == (64, 112, 112) and s["pool1"] == (64, 56, 56)
    n = graph._DENSENET_BLOCKS[depth]
    ends = [s[f"concat_{b}_{n[b - 2]}"] for b in (2, 3, 4, 5)]
    assert [e[0] for e in ends] == list(blocks) and [e[1] for e in ends] == [56, 28, 14, 7]
    assert s["pool2"] == (128, 28, 28) and s["pool5"] == (final, 1, 1) and s["fc6"] == (1000, 1, 1)
    low = graph.lower(net)
    # each block is one tensor of the block's final width
    assert {k: v for k, v in low["tensors"].items() if k.startswith("concat_")} == {
        f"concat_{b}_{n[b - 2]}": e for b, e in zip((2, 3, 4, 5), ends)}


def test_flops_as_defined_and_as_lowered():
    net = graph.densenet_caffe(121)
    assert _raw_flops(net) / 1e9 == pytest.approx(5.668, abs=5e-4)
    assert graph.conv_flops(graph.lower(net)) / 1e9 == pytest.approx(5.206, abs=5e-4)
    # the three commuted transitions do a quarter of their work
    assert _raw_flops(net) - graph.conv_flops(graph.lower(net)) == 3 * 3 * 2 * 56 * 56 * 256 * 128 // 4


def test_round_mode_parsing():
    proto = ('name: "p" input: "data" input_dim: 1 input_dim: 8 input_dim: 57 input_dim: 57 '
             'layer { name: "a" type: "Pooling" bottom: "data" top: "a" pooling_param { pool: MAX kernel_size: 3 stride: 2 %s } }')
    assert graph.infer_shapes(graph.parse_prototxt(proto % ""))["a"] == (8, 28, 28)  # CEIL, as before
    assert "ceil_mode" not in graph.parse_prototxt(proto % "")["layers"][0]
    assert graph.infer_shapes(graph.parse_prototxt(proto % "round_mode: CEIL"))["a"] == (8, 28, 28)
    assert graph.infer_shapes(graph.parse_prototxt(proto % "pad: 1 round_mode: FLOOR"))["a"] == (8, 29, 29)
    assert graph.infer_shapes(graph.parse_prototxt(proto % "pad: 1"))["a"] == (8, 29, 29)
    p = proto.replace("57", "112")
    assert graph.infer_shapes(graph.parse_prototxt(p % "pad: 1 round_mode: FLOOR"))["a"] == (8, 56, 56)
    assert graph.infer_shapes(graph.parse_prototxt(p % "pad: 1"))["a"] == (8, 57, 57)
    with pytest.raises(ValueError, match="Pooling a: round_mode UP"):
        graph.parse_prototxt(proto % "round_mode: UP")


def test_lowering():
    low = graph.lower(graph.densenet_caffe(121))
    ops = low["ops"]
    convs = [o for o in ops if o["type"] == graph.OP_CONV]
    assert len(convs) == 120
    assert sum(bool(o.get("pre") or o.get("commuted")) for o in convs) == 61
    prefix = [o for o in convs if o["cin"] < low["tensors"][o["input"]][0]]
    assert len(prefix) == 58 and all(o.get("pre") and o["k"] == 1 for o in prefix)
    assert sum(o["cin"] % 64 != 0 for o in prefix) == 29
    commuted = [o for o in convs if o.get("commuted")]
    assert [o["name"] for o in commuted] == ["conv2_blk", "conv3_blk", "conv4_blk"]
    for o in commuted:
        pool = ops[ops.index(o) - 1]
        assert pool["type"] == graph.OP_AVGPOOL and pool.get("pre") and pool["k"] == 2 and pool["output"] == o["input"]
        assert o["out_c0"] == 0 and not o.get("pre")
    pool1 = next(o for o in ops if o["name"] == "pool1")
    assert pool1["type"] == graph.OP_MAXPOOL and pool1["out_c0"] == 0 and pool1["output"] == "concat_2_6"
    pool5 = next(o for o in ops if o["name"] == "pool5")
    assert pool5["type"] == graph.OP_AVGPOOL and pool5.get("pre") and pool5["input"] == "concat_5_16"
    # the 3x3 of each dense layer writes its 32 channels behind the prefix its 1x1 read
    x2 = next(o for o in ops if o["name"] == "conv3_5/x2")
    assert x2["output"] == "concat_3_12" and x2["out_c0"] == 128 + 4 * 32 and x2["cout"] == 32
    assert next(o for o in ops if o["name"] == "conv3_5/x1")["cin"] == 128 + 4 * 32


def test_prologue_parameters_are_folded_in_float64():
    net = graph.densenet_caffe(121)
    w = weights.random_weights(net, 0)
    op = next(o for o in graph.lower(net, w)["ops"] if o["name"] == "conv3_2/x1")
    scale = w["conv3_2/x1/scale"]["gamma"].astype(np.float64) / np.sqrt(w["conv3_2/x1/bn"]["var"].astype(np.float64) + 1e-5)
    shift = w["conv3_2/x1/scale"]["beta"] - w["conv3_2/x1/bn"]["mean"].astype(np.float64) * scale
    assert op["pre_scale"].dtype == np.float32 and np.array_equal(op["pre_scale"], scale.astype(np.float32))
    assert np.array_equal(op["pre_shift"], shift.astype(np.float32))


def _edit_net(fn):
    net = dense_net(layers=2)
    layers = [dict(L) for L in net["layers"]]
    fn(layers)
    return dict(net, layers=layers)


def _drop(names):
    return lambda layers: layers.__setitem__(slice(None), [L for L in layers if L["name"] not in names])


def _set(name, **kw):
    return lambda layers: next(L for L in layers if L["name"] == name).update(kw)


def _insert_after(name, new):
    def fn(layers):
        i = next(i for i, L in enumerate(layers) if L["name"] == name)
        layers.insert(i + 1, new)
    return fn


@pytest.mark.parametrize("edit, msg", [
    (_drop({"relu2_2/x1"}), r"BatchNorm conv2_2/x1/bn: a pre-activation without ReLU"),
    (_set("conv2_1/x1", kernel_size=3, pad=1), r"BatchNorm conv2_1/x1/bn: a pre-activation before conv2_1/x1, a 3x3"),
    (_insert_after("conv2_1/x1", dict(name="extra", type="Convolution", bottoms=["conv2_1/x1/bn"], tops=["extra"], num_output=8,
                                      kernel_size=1, pad=0, stride=1, bias_term=False)),
     r"BatchNorm conv2_1/x1/bn: its output conv2_1/x1/bn has 2 readers"),
    (_insert_after("relu2_1/x1", dict(name="mp", type="Pooling", bottoms=["conv2_1/x1/bn"], tops=["mp"], pool="MAX", kernel_size=1,
                                      stride=1, pad=0)),
     r"BatchNorm conv2_1/x1/bn: a pre-activation is the input prologue of a 1x1 convolution or an average pool, not of Pooling mp"),
    (_insert_after("concat_2_1", dict(name="peek", type="Convolution", bottoms=["pool1"], tops=["peek"], num_output=8, kernel_size=1,
                                      pad=0, stride=1, bias_term=False)),
     r"Concat concat_2_1: input pool1 is also read by peek"),
    (_set("pool2", kernel_size=3, stride=2), r"Pooling pool2: only global AVE pooling, or a k x k / stride k window"),
    (_drop({"conv2_blk", "pool2", "conv3_1/x1/bn", "conv3_1/x1/scale", "relu3_1/x1", "conv3_1/x1", "conv3_1/x2/bn", "conv3_1/x2/scale",
            "relu3_1/x2", "conv3_1/x2", "concat_3_1", "conv3_2/x1/bn", "conv3_2/x1/scale", "relu3_2/x1", "conv3_2/x1", "conv3_2/x2/bn",
            "conv3_2/x2/scale", "relu3_2/x2", "conv3_2/x2", "concat_3_2", "conv5_blk/bn", "conv5_blk/scale", "relu5_blk", "pool5", "fc6",
            "prob"}),
     r"BatchNorm conv2_blk/bn: its pre-activation has no reader"),
])
def test_lowering_refusals_name_the_layer(edit, msg):
    with pytest.raises(ValueError, match=msg):
        graph.lower(_edit_net(edit))


def test_precisions_other_than_fp16_are_refused():
    for p in (builder.PREC_FP32, builder.PREC_INT8, builder.PREC_FP8):
        with pytest.raises(ValueError, match="fp16 only"):
            builder.build_densenet_plan(max_batch=1, precision=p)


# ---- plans ---------------------------------------------------------------------------------------------------------------
def test_existing_plans_keep_their_bytes():
    assert hashlib.sha256(builder.build_googlenet_plan()).hexdigest() == "f74a9c3cc20cb08d54c4478c9718d39875bc16d22ceca95471a5836f4058f6da"


def test_plan_records():
    blob = builder.build_densenet_plan(121, max_batch=2)
    version, tensors, ops, _ = _records(blob)
    assert version == builder.VERSION_CONCAT
    name = {i: t[0].rstrip(b"\0").decode() for i, t in enumerate(tensors)}
    by = {o[0].rstrip(b"\0").decode(): o for o in ops}
    pre = [n for n, o in by.items() if o[9] & builder.CONV_PREACT]
    assert len([n for n in pre if by[n][1] == builder.OP_CONV]) == 58
    assert sorted(n for n in pre if by[n][1] == builder.OP_AVGPOOL) == ["pool2", "pool3", "pool4", "pool5"]
    p1 = by["pool1"]
    assert p1[1] == builder.OP_MAXPOOL and (p1[26], p1[27]) == (0, 64) and name[p1[4]] == "concat_2_6"
    x1 = by["conv4_3/x1"]  # reads [0, 320) of the block-4 tensor: cin_phys 320, b = bias, scale, shift
    assert (x1[11], x1[13], tensors[x1[2]][4:6]) == (320, 320, (1024, 1024)) and x1[20] == (128 + 2 * 320) * 4
    x1 = by["conv4_2/x1"]
    assert (x1[11], x1[13]) == (288, 320)
    blk = by["conv3_blk"]  # the commuted transition: 1x1 on the pooled tensor, writing [0, 256) of the block-4 tensor
    assert name[blk[2]] == "conv3_blk/pool" and tensors[blk[2]][2:5] == (14, 14, 512) and (blk[26], blk[27]) == (0, 256)
    eng = capi.Engine(blob, inspect_only=True)
    try:
        assert eng.flops(1) == pytest.approx(graph.conv_flops(graph.lower(graph.densenet_caffe(121))))
    finally:
        eng.destroy()


def _mutations():
    net = dense_net(layers=3)
    blob = builder.build_plan(graph.lower(net, weights.random_weights(net, 0)), builder.PREC_FP16, max_batch=2)
    _, _, ops, base = _records(blob)
    idx = {o[0].rstrip(b"\0").decode(): i for i, o in enumerate(ops)}

    def edit(op, blob=blob, **kw):
        fields = {"inp": 2, "res": 3, "k": 6, "stride": 7, "relu": 9, "cin": 11, "cin_phys": 13, "b_bytes": 20, "c0": 26, "cw": 27}
        rec = list(ops[idx[op]])
        for k, v in kw.items():
            rec[fields[k]] = v
        out = bytearray(blob)
        builder._OP_V4.pack_into(out, base + idx[op] * 192, *rec)
        return bytes(out)

    def swap(a, b):  # exchange two op records
        out = bytearray(blob)
        builder._OP_V4.pack_into(out, base + idx[a] * 192, *ops[idx[b]])
        builder._OP_V4.pack_into(out, base + idx[b] * 192, *ops[idx[a]])
        return bytes(out)

    relu = ops[idx["conv2_2/x1"]][9]
    return blob, [
        ("unknown flag", edit("conv2_2/x1", relu=relu | 32), r"conv conv2_2/x1: unknown flags 0x33"),
        ("prologue on a 3x3", edit("conv2_2/x2", relu=ops[idx["conv2_2/x2"]][9] | 16),
         r"conv conv2_2/x2: a BatchNorm \+ ReLU prologue exists for dense 1x1"),
        ("prologue size", edit("conv2_2/x1", b_bytes=ops[idx["conv2_2/x1"]][20] - 4), r"conv conv2_2/x1 weight size mismatch"),
        ("prefix padding", edit("conv2_2/x1", cin_phys=192), r"conv conv2_2/x1: an input prefix reader is a dense 1x1 .* cin_phys = cin"),
        ("prefix of a 3x3", edit("conv2_2/x2", inp=ops[idx["conv2_2/x1"]][2], cin=96),
         r"conv conv2_2/x2: an input prefix reader is a dense 1x1"),
        ("not a boundary", edit("conv2_2/x1", cin=88), r"conv conv2_2/x1: prefix \[0, 88\) of concat_2_3 does not end at a slice boundary"),
        ("read early", swap("conv2_2/x1", "conv2_1/x2"), r"conv conv2_2/x1: reads channels \[0, 96\) of concat_2_3 before conv2_1/x2 writes"),
        ("unsliced input", edit("conv2_2/x2", cin=64, inp=ops[idx["conv3_1/x1"]][4]),
         r"conv conv2_2/x2: (reads channels \[0, 64\) of .* which is not slice-written|an input prefix reader)"),
        ("pool stride", edit("pool2", stride=1), r"avgpool pool2: a prologue pool is a k x k / stride k window"),
        ("pool prologue size", edit("pool2", b_bytes=16), r"avgpool pool2: the prologue parameters must be fp32"),
        ("window without prologue", edit("pool2", relu=0), r"avgpool pool2: a windowed average pool carries a BatchNorm \+ ReLU prologue"),
        ("pool flags", edit("pool5", relu=17), r"avgpool pool5: unknown flags 0x11"),
        ("max pool slice width", edit("pool1", cw=32), r"op pool1: only a convolution writes an output channel slice, and a max pool all 64"),
        ("max pool slice offset", edit("pool1", c0=4), r"op pool1: only a convolution writes an output channel slice, and a max pool"),
    ]


def test_corrupted_plans_are_refused():
    blob, muts = _mutations()
    capi.Engine(blob, inspect_only=True).destroy()
    for what, bad, msg in muts:
        with pytest.raises(capi.B2Error) as ei:
            capi.Engine(bad, inspect_only=True)
        assert ei.value.code == 1 and re.search(msg, str(ei.value)), (what, str(ei.value))


# ---- weights and oracles ------------------------------------------------------------------------------------------------
def test_caffemodel_round_trip_gives_the_same_plan():
    net = graph.densenet_caffe(121)
    wts = weights.random_weights(net, 2)
    low = graph.lower(net, caffemodel.load_caffemodel(caffemodel.save_caffemodel(net, wts), net))
    assert builder.build_plan(low, builder.PREC_FP16, 2) == builder.build_densenet_plan(121, max_batch=2, weights=wts)


def _torchvision_densenet(depth, seed):
    torchvision = pytest.importorskip("torchvision")
    import torch
    torch.manual_seed(seed)
    model = getattr(torchvision.models, f"densenet{depth}")(weights=None).double().eval()
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.BatchNorm2d):  # random statistics, so that every BatchNorm matters
                m.running_mean.copy_(torch.randn(m.num_features, generator=g, dtype=torch.float64) * 0.1)
                m.running_var.copy_(torch.rand(m.num_features, generator=g, dtype=torch.float64) + 0.5)
                m.weight.copy_(torch.rand(m.num_features, generator=g, dtype=torch.float64) * 0.4 + 0.8)
                m.bias.copy_(torch.randn(m.num_features, generator=g, dtype=torch.float64) * 0.1)
    return model


def test_load_weights_matches_torchvision():
    import torch
    model = _torchvision_densenet(121, 0)
    sd = {k: v.float().numpy() for k, v in model.state_dict().items() if not k.endswith("num_batches_tracked")}
    wts = densenet.load_weights(sd, 121)
    net = graph.densenet_caffe(121)
    x = np.random.default_rng(5).standard_normal((2, 3, 224, 224))
    # the float64 oracle on the fp32-stored weights against torchvision's own forward on the same values
    model = model.float().double()
    with torch.no_grad():
        ref = torch.softmax(model(torch.from_numpy(x)), 1).numpy()
    got = caffe_forward(net, wts, x, dtype=torch.float64)
    assert float(np.abs(got - ref).max() / np.abs(ref).max()) <= 1e-10
    bad = dict(sd)
    del bad["features.denseblock3.denselayer7.norm2.running_var"]
    with pytest.raises(KeyError, match=r"features.denseblock3.denselayer7.norm2.running_var"):
        densenet.load_weights(bad, 121)
    bad = dict(sd, **{"features.transition2.conv.weight": np.zeros((256, 512, 3, 3), np.float32)})
    with pytest.raises(ValueError, match=r"features.transition2.conv.weight has shape \(256, 512, 3, 3\), expected \(256, 512, 1, 1\)"):
        densenet.load_weights(bad, 121)


def test_emulation_against_float64():
    import torch
    net = dense_net(layers=3)
    wts = weights.random_weights(net, 1)
    low = graph.lower(net, wts)
    x = weights.synthetic_input(2, chw=(3, 16, 16), seed=9)
    ref = caffe_forward(net, wts, x, dtype=torch.float64, logits=True)
    emu = lowered_forward_f16emu(low, x, logits=True)
    rel = float(np.abs(emu - ref).max() / np.abs(ref).max())
    assert 1e-5 < rel <= 3e-3, rel  # fp16 storage matters, and only that much
    assert np.array_equal(np.argmax(ref, 1), np.argmax(emu, 1))
