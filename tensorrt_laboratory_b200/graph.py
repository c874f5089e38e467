"""Layer-graph IR for the inference hot path.

Two levels:

* **raw Caffe layers** -- a list of plain dicts ``{name, type, bottoms, tops, ...params}`` exactly as a
  deploy prototxt states them (Convolution / BatchNorm / Scale / ReLU / Pooling / Eltwise /
  InnerProduct / Softmax).  Produced either by :func:`parse_prototxt` (front-end for the files the
  reference feeds to ``trtexec --deploy``, reference ``models/setup.py:53-55``) or by
  :func:`resnet_caffe` (a programmatic generator of the same layer list, so the GPU box does not need
  the prototxt).  The CPU oracle executes THIS level, unfused.

* **lowered ops** -- what the engine executes: every Convolution absorbs its BatchNorm+Scale (folded to
  per-channel scale/bias at build time), its ReLU, and -- for the last conv of a bottleneck -- the
  Eltwise SUM + ReLU.  See :func:`lower`.

Caffe semantics that matter (reference ``models/ResNet-50-deploy.prototxt``):
  * Pooling output size uses CEIL:  out = ceil((in + 2p - k)/s) + 1        (``:48-58`` pool1 -> 56)
  * BatchNorm is ``use_global_stats`` followed by a separate Scale layer with ``bias_term``
  * stride 2 sits on the 1x1 ``branch2a`` / ``branch1`` convs (Caffe-v1 ResNet)
  * ``conv1`` has a bias, every other conv says ``bias_term: false``
"""
from __future__ import annotations

import math
import re
from typing import Dict, List, Optional, Tuple

# --------------------------------------------------------------------------------------------------
# prototxt front-end
# --------------------------------------------------------------------------------------------------

_TOKEN = re.compile(r'\s*(?:(#[^\n]*)|([{}:])|"((?:[^"\\]|\\.)*)"|([^\s{}:"#]+))')


def _tokenize(text: str):
    pos = 0
    n = len(text)
    while pos < n:
        m = _TOKEN.match(text, pos)
        if not m:
            if text[pos:].strip() == "":
                return
            raise ValueError(f"prototxt: cannot tokenize at offset {pos}: {text[pos:pos+40]!r}")
        pos = m.end()
        if m.group(1) is not None:
            continue
        if m.group(2) is not None:
            yield ("sym", m.group(2))
        elif m.group(3) is not None:
            yield ("str", m.group(3))
        else:
            yield ("atom", m.group(4))


def _parse_message(tokens, i, top=False):
    """Parse protobuf text format into {field: [values...]} (every field repeated)."""
    out: Dict[str, list] = {}
    while i < len(tokens):
        kind, val = tokens[i]
        if kind == "sym" and val == "}":
            if top:
                raise ValueError("prototxt: unbalanced '}'")
            return out, i + 1
        if kind != "atom":
            raise ValueError(f"prototxt: expected field name, got {val!r}")
        name = val
        i += 1
        kind, val = tokens[i]
        if kind == "sym" and val == ":":
            i += 1
            kind, val = tokens[i]
            if kind == "sym" and val == "{":
                sub, i = _parse_message(tokens, i + 1)
                out.setdefault(name, []).append(sub)
            else:
                out.setdefault(name, []).append(_scalar(kind, val))
                i += 1
        elif kind == "sym" and val == "{":
            sub, i = _parse_message(tokens, i + 1)
            out.setdefault(name, []).append(sub)
        else:
            raise ValueError(f"prototxt: expected ':' or '{{' after {name}")
    if not top:
        raise ValueError("prototxt: missing '}'")
    return out, i


def _scalar(kind, val):
    if kind == "str":
        return val
    if val in ("true", "false"):
        return val == "true"
    try:
        return int(val)
    except ValueError:
        pass
    try:
        return float(val)
    except ValueError:
        return val  # enum such as MAX / AVE


def _one(msg, key, default=None):
    v = msg.get(key)
    return v[0] if v else default


def parse_prototxt(text: str) -> dict:
    """Parse a Caffe deploy prototxt into ``{name, input, input_dims, layers}`` (raw layer dicts)."""
    tokens = list(_tokenize(text))
    msg, _ = _parse_message(tokens, 0, top=True)
    layers = []
    for L in msg.get("layer", []):
        ltype = _one(L, "type")
        rec = {
            "name": _one(L, "name"),
            "type": ltype,
            "bottoms": list(L.get("bottom", [])),
            "tops": list(L.get("top", [])),
        }
        if ltype == "Convolution":
            p = _one(L, "convolution_param", {})
            rec.update(
                num_output=_one(p, "num_output"),
                kernel_size=_one(p, "kernel_size"),
                pad=_one(p, "pad", 0),
                stride=_one(p, "stride", 1),
                bias_term=_one(p, "bias_term", True),
            )
            if "group" in p:  # absent = 1; read everywhere as L.get("group", 1)
                rec["group"] = _one(p, "group")
        elif ltype == "BatchNorm":
            p = _one(L, "batch_norm_param", {})
            rec.update(use_global_stats=_one(p, "use_global_stats", True), eps=_one(p, "eps", 1e-5))
        elif ltype == "Scale":
            p = _one(L, "scale_param", {})
            rec.update(bias_term=_one(p, "bias_term", False))
        elif ltype == "Pooling":
            p = _one(L, "pooling_param", {})
            rec.update(
                pool=_one(p, "pool", "MAX"),
                kernel_size=_one(p, "kernel_size"),
                stride=_one(p, "stride", 1),
                pad=_one(p, "pad", 0),
            )
            round_mode = _one(p, "round_mode", "CEIL")  # absent = Caffe's CEIL
            if round_mode not in ("CEIL", "FLOOR"):
                raise ValueError(f"prototxt: Pooling {rec['name']}: round_mode {round_mode}; CEIL or FLOOR")
            if round_mode == "FLOOR":
                rec["ceil_mode"] = False
        elif ltype == "InnerProduct":
            p = _one(L, "inner_product_param", {})
            rec.update(num_output=_one(p, "num_output"), bias_term=_one(p, "bias_term", True))
        elif ltype == "Eltwise":
            p = _one(L, "eltwise_param", {})
            rec.update(operation=_one(p, "operation", "SUM"))
        elif ltype == "Concat":
            p = _one(L, "concat_param", {})
            axis = _one(p, "axis", _one(p, "concat_dim", 1))
            if axis != 1:
                raise ValueError(f"prototxt: Concat {rec['name']}: concatenation along axis {axis}; only channels (axis 1) are supported")
            rec.update(axis=1)
        elif ltype == "LRN":
            p = _one(L, "lrn_param", {})
            region = _one(p, "norm_region", "ACROSS_CHANNELS")
            if region != "ACROSS_CHANNELS":
                raise ValueError(f"prototxt: LRN {rec['name']}: norm_region {region}; only ACROSS_CHANNELS is supported")
            rec.update(local_size=_one(p, "local_size", 5), alpha=float(_one(p, "alpha", 1.0)), beta=float(_one(p, "beta", 0.75)),
                       k=float(_one(p, "k", 1.0)))
        elif ltype in ("ReLU", "Softmax", "Dropout"):
            pass
        else:
            raise ValueError(f"prototxt: unsupported layer type {ltype!r} ({rec['name']})")
        layers.append(rec)
    dims = [int(d) for d in msg.get("input_dim", [])]
    return {
        "name": _one(msg, "name", "net"),
        "input": _one(msg, "input", "data"),
        "input_dims": dims,  # [1, C, H, W]
        "layers": layers,
    }


# --------------------------------------------------------------------------------------------------
# programmatic generator of the Caffe-v1 ResNet deploy nets (same layer list as the prototxt)
# --------------------------------------------------------------------------------------------------

_RESNET_BLOCKS = {50: (3, 4, 6, 3), 101: (3, 4, 23, 3), 152: (3, 8, 36, 3)}


def _block_names(count: int, stage: int, depth: int) -> List[str]:
    # ResNet-50 names blocks a,b,c,...; the deeper nets name them a, b1, b2, ... in stages 3 and 4.
    if depth == 50 or count <= 3:
        return [chr(ord("a") + i) for i in range(count)]
    return ["a"] + [f"b{i}" for i in range(1, count)]


def resnet_caffe(depth: int = 50) -> dict:
    """Generate the raw layer list of ``models/ResNet-{50,152}-deploy.prototxt`` (reference)."""
    if depth not in _RESNET_BLOCKS:
        raise ValueError(f"unsupported ResNet depth {depth}")
    return _bottleneck_net(f"ResNet-{depth}", depth, [64 << si for si in range(4)], group=1)


def resnext_caffe(depth: int = 50, groups: int = 32, width_per_group: int = 4) -> dict:
    """ResNeXt (Xie et al., "Aggregated Residual Transformations for Deep Neural Networks") in the Caffe conventions of
    :func:`resnet_caffe`: same stem, block names and BatchNorm + Scale pairs.  The bottleneck's 3x3 convolution has
    ``groups`` groups of ``width_per_group * 2**stage`` channels (128, 256, 512, 1024 for 32x4d) and carries the stride, as
    does ``branch1``; the 1x1 ``branch2a`` always has stride 1."""
    if depth not in _RESNET_BLOCKS:
        raise ValueError(f"unsupported ResNeXt depth {depth}")
    widths = [groups * width_per_group << si for si in range(4)]
    return _bottleneck_net(f"ResNeXt-{depth}-{groups}x{width_per_group}d", depth, widths, group=groups)


def _bottleneck_net(name: str, depth: int, widths: List[int], group: int) -> dict:
    """Bottleneck network with stage widths ``widths``; ``group`` > 1 makes the 3x3 grouped and moves the stride onto it."""
    L: List[dict] = []

    def conv(name, bottom, nout, k, pad, stride, bias, g=1):
        L.append(dict(name=name, type="Convolution", bottoms=[bottom], tops=[name], num_output=nout,
                      kernel_size=k, pad=pad, stride=stride, bias_term=bias))
        if g != 1:
            L[-1]["group"] = g

    def bn_scale(suffix, blob):
        L.append(dict(name="bn" + suffix, type="BatchNorm", bottoms=[blob], tops=[blob],
                      use_global_stats=True, eps=1e-5))
        L.append(dict(name="scale" + suffix, type="Scale", bottoms=[blob], tops=[blob], bias_term=True))

    def relu(name, blob):
        L.append(dict(name=name, type="ReLU", bottoms=[blob], tops=[blob]))

    conv("conv1", "data", 64, 7, 3, 2, depth == 50)  # the 152 prototxt says bias_term: false
    bn_scale("_conv1", "conv1")
    relu("conv1_relu", "conv1")
    L.append(dict(name="pool1", type="Pooling", bottoms=["conv1"], tops=["pool1"], pool="MAX",
                  kernel_size=3, stride=2, pad=0))
    prev = "pool1"
    for si, count in enumerate(_RESNET_BLOCKS[depth]):
        stage = si + 2
        mid = widths[si]
        out = 256 << si
        for bi, bname in enumerate(_block_names(count, stage, depth)):
            tag = f"{stage}{bname}"
            stride = 2 if (bi == 0 and stage > 2) else 1
            s_1x1, s_3x3 = (stride, 1) if group == 1 else (1, stride)
            if bi == 0:
                conv(f"res{tag}_branch1", prev, out, 1, 0, stride, False)
                bn_scale(f"{tag}_branch1", f"res{tag}_branch1")
                shortcut = f"res{tag}_branch1"
            else:
                shortcut = prev
            conv(f"res{tag}_branch2a", prev, mid, 1, 0, s_1x1, False)
            bn_scale(f"{tag}_branch2a", f"res{tag}_branch2a")
            relu(f"res{tag}_branch2a_relu", f"res{tag}_branch2a")
            conv(f"res{tag}_branch2b", f"res{tag}_branch2a", mid, 3, 1, s_3x3, False, group)
            bn_scale(f"{tag}_branch2b", f"res{tag}_branch2b")
            relu(f"res{tag}_branch2b_relu", f"res{tag}_branch2b")
            conv(f"res{tag}_branch2c", f"res{tag}_branch2b", out, 1, 0, 1, False)
            bn_scale(f"{tag}_branch2c", f"res{tag}_branch2c")
            L.append(dict(name=f"res{tag}", type="Eltwise", bottoms=[shortcut, f"res{tag}_branch2c"],
                          tops=[f"res{tag}"], operation="SUM"))
            relu(f"res{tag}_relu", f"res{tag}")
            prev = f"res{tag}"
    L.append(dict(name="pool5", type="Pooling", bottoms=[prev], tops=["pool5"], pool="AVE",
                  kernel_size=7, stride=1, pad=0))
    L.append(dict(name="fc1000", type="InnerProduct", bottoms=["pool5"], tops=["fc1000"],
                  num_output=1000, bias_term=True))
    L.append(dict(name="prob", type="Softmax", bottoms=["fc1000"], tops=["prob"]))
    return {"name": name, "input": "data", "input_dims": [1, 3, 224, 224], "layers": L}


# BVLC GoogLeNet inception modules (Szegedy et al., "Going Deeper with Convolutions", Table 1):
# name -> (#1x1, #3x3 reduce, #3x3, #5x5 reduce, #5x5, pool proj)
_INCEPTION = {
    "3a": (64, 96, 128, 16, 32, 32), "3b": (128, 128, 192, 32, 96, 64),
    "4a": (192, 96, 208, 16, 48, 64), "4b": (160, 112, 224, 24, 64, 64), "4c": (128, 128, 256, 24, 64, 64),
    "4d": (112, 144, 288, 32, 64, 64), "4e": (256, 160, 320, 32, 128, 128),
    "5a": (256, 160, 320, 32, 128, 128), "5b": (384, 192, 384, 48, 128, 128),
}


def googlenet_caffe() -> dict:
    """The raw layer list of BVLC GoogLeNet's deploy net (``models/bvlc_googlenet/deploy.prototxt`` of Caffe), without the
    auxiliary classifiers, under the BVLC layer and blob names, so that ``bvlc_googlenet.caffemodel`` loads by name.
    Every convolution has a bias and a ReLU; the LRN layers are local_size 5, alpha 1e-4, beta 0.75."""
    L: List[dict] = []

    def conv(name, bottom, nout, k, pad=0, stride=1, relu="relu"):
        L.append(dict(name=name, type="Convolution", bottoms=[bottom], tops=[name], num_output=nout, kernel_size=k, pad=pad,
                      stride=stride, bias_term=True))
        L.append(dict(name=name.rsplit("/", 1)[0] + "/" + relu, type="ReLU", bottoms=[name], tops=[name]))

    def pool(name, bottom, k, stride, pad=0, kind="MAX"):
        L.append(dict(name=name, type="Pooling", bottoms=[bottom], tops=[name], pool=kind, kernel_size=k, stride=stride, pad=pad))

    def lrn(name, bottom):
        L.append(dict(name=name, type="LRN", bottoms=[bottom], tops=[name], local_size=5, alpha=1e-4, beta=0.75, k=1.0))

    conv("conv1/7x7_s2", "data", 64, 7, 3, 2, "relu_7x7")
    pool("pool1/3x3_s2", "conv1/7x7_s2", 3, 2)
    lrn("pool1/norm1", "pool1/3x3_s2")
    conv("conv2/3x3_reduce", "pool1/norm1", 64, 1, relu="relu_3x3_reduce")
    conv("conv2/3x3", "conv2/3x3_reduce", 192, 3, 1, relu="relu_3x3")
    lrn("conv2/norm2", "conv2/3x3")
    pool("pool2/3x3_s2", "conv2/norm2", 3, 2)
    prev = "pool2/3x3_s2"
    for tag, (n1, r3, n3, r5, n5, pp) in _INCEPTION.items():
        m = f"inception_{tag}"
        conv(f"{m}/1x1", prev, n1, 1, relu="relu_1x1")
        conv(f"{m}/3x3_reduce", prev, r3, 1, relu="relu_3x3_reduce")
        conv(f"{m}/3x3", f"{m}/3x3_reduce", n3, 3, 1, relu="relu_3x3")
        conv(f"{m}/5x5_reduce", prev, r5, 1, relu="relu_5x5_reduce")
        conv(f"{m}/5x5", f"{m}/5x5_reduce", n5, 5, 2, relu="relu_5x5")
        pool(f"{m}/pool", prev, 3, 1, 1)
        conv(f"{m}/pool_proj", f"{m}/pool", pp, 1, relu="relu_pool_proj")
        L.append(dict(name=f"{m}/output", type="Concat", bottoms=[f"{m}/1x1", f"{m}/3x3", f"{m}/5x5", f"{m}/pool_proj"],
                      tops=[f"{m}/output"], axis=1))
        prev = f"{m}/output"
        if tag in ("3b", "4e"):
            pool(f"pool{tag[0]}/3x3_s2", prev, 3, 2)
            prev = f"pool{tag[0]}/3x3_s2"
    pool("pool5/7x7_s1", prev, 7, 1, kind="AVE")
    L.append(dict(name="pool5/drop_7x7_s1", type="Dropout", bottoms=["pool5/7x7_s1"], tops=["pool5/7x7_s1"]))
    L.append(dict(name="loss3/classifier", type="InnerProduct", bottoms=["pool5/7x7_s1"], tops=["loss3/classifier"], num_output=1000,
                  bias_term=True))
    L.append(dict(name="prob", type="Softmax", bottoms=["loss3/classifier"], tops=["prob"]))
    return {"name": "GoogleNet", "input": "data", "input_dims": [1, 3, 224, 224], "layers": L}


# DenseNet (Huang et al., "Densely Connected Convolutional Networks"): dense layers per block, growth 32, a 4 x 32
# bottleneck, compression 1/2 -- torchvision's geometry
_DENSENET_BLOCKS = {121: (6, 12, 24, 16), 169: (6, 12, 32, 32), 201: (6, 12, 48, 32)}


def densenet_caffe(depth: int = 121) -> dict:
    """The raw layer list of DenseNet-{121,169,201} in the usual Caffe form: blocks 2 ... 5, each dense layer
    ``conv{b}_{l}/x1/bn|scale``, ``relu{b}_{l}/x1``, ``conv{b}_{l}/x1`` (1x1, 128), the same with ``x2`` (3x3, 32), then
    ``concat_{b}_{l}`` of the previous concatenation (or ``pool1`` / ``pool{b-1}``) and ``conv{b}_{l}/x2``; transitions
    ``conv{b}_blk/bn|scale``, ``relu{b}_blk``, ``conv{b}_blk`` (1x1, half the channels) and ``pool{b}`` (AVE 2x2/2); the
    stem ``conv1`` (7x7/2, 64), ``conv1/bn|scale``, ``relu1``, ``pool1`` (MAX 3x3/2, pad 1, FLOOR); the head
    ``conv5_blk/bn|scale``, ``relu5_blk``, ``pool5`` (global AVE), ``fc6`` and ``prob``.  Every BatchNorm writes a new blob
    named after it; Scale and ReLU run in place on it.  No convolution has a bias."""
    if depth not in _DENSENET_BLOCKS:
        raise ValueError(f"unsupported DenseNet depth {depth}")
    L: List[dict] = []

    def conv(name, bottom, nout, k, pad=0, stride=1):
        L.append(dict(name=name, type="Convolution", bottoms=[bottom], tops=[name], num_output=nout, kernel_size=k, pad=pad,
                      stride=stride, bias_term=False))

    def bn_scale_relu(prefix, relu, bottom):
        bn = prefix + "/bn"
        L.append(dict(name=bn, type="BatchNorm", bottoms=[bottom], tops=[bn], use_global_stats=True, eps=1e-5))
        L.append(dict(name=prefix + "/scale", type="Scale", bottoms=[bn], tops=[bn], bias_term=True))
        L.append(dict(name=relu, type="ReLU", bottoms=[bn], tops=[bn]))
        return bn

    conv("conv1", "data", 64, 7, 3, 2)
    L.append(dict(name="pool1", type="Pooling", bottoms=[bn_scale_relu("conv1", "relu1", "conv1")], tops=["pool1"], pool="MAX",
                  kernel_size=3, stride=2, pad=1, ceil_mode=False))
    prev, c = "pool1", 64
    for b, n in enumerate(_DENSENET_BLOCKS[depth], 2):
        for l in range(1, n + 1):
            x1, x2 = f"conv{b}_{l}/x1", f"conv{b}_{l}/x2"
            conv(x1, bn_scale_relu(x1, f"relu{b}_{l}/x1", prev), 128, 1)
            conv(x2, bn_scale_relu(x2, f"relu{b}_{l}/x2", x1), 32, 3, 1)
            L.append(dict(name=f"concat_{b}_{l}", type="Concat", bottoms=[prev, x2], tops=[f"concat_{b}_{l}"], axis=1))
            prev, c = f"concat_{b}_{l}", c + 32
        if b < 5:
            c //= 2
            conv(f"conv{b}_blk", bn_scale_relu(f"conv{b}_blk", f"relu{b}_blk", prev), c, 1)
            L.append(dict(name=f"pool{b}", type="Pooling", bottoms=[f"conv{b}_blk"], tops=[f"pool{b}"], pool="AVE", kernel_size=2,
                          stride=2, pad=0))
            prev = f"pool{b}"
    L.append(dict(name="pool5", type="Pooling", bottoms=[bn_scale_relu("conv5_blk", "relu5_blk", prev)], tops=["pool5"], pool="AVE",
                  kernel_size=7, stride=1, pad=0))
    L.append(dict(name="fc6", type="InnerProduct", bottoms=["pool5"], tops=["fc6"], num_output=1000, bias_term=True))
    L.append(dict(name="prob", type="Softmax", bottoms=["fc6"], tops=["prob"]))
    return {"name": f"DenseNet-{depth}", "input": "data", "input_dims": [1, 3, 224, 224], "layers": L}


# VGG (Simonyan and Zisserman, "Very Deep Convolutional Networks for Large-Scale Image Recognition", configurations D
# and E): 3x3 convolutions per block, each block followed by a 2x2 / 2 max pool
_VGG_BLOCKS = {16: (2, 2, 3, 3, 3), 19: (2, 2, 4, 4, 4)}
_VGG_WIDTHS = (64, 128, 256, 512, 512)


def vgg_caffe(depth: int = 16) -> dict:
    """The raw layer list of VGG-{16,19}'s Caffe deploy net (``VGG_ILSVRC_{16,19}_layers_deploy.prototxt``) under its layer
    names, so that ``VGG_ILSVRC_{16,19}_layers.caffemodel`` loads by name: ``conv{b}_{l}`` (3x3, pad 1, stride 1, bias)
    with ``relu{b}_{l}`` in place, ``pool{b}`` (MAX 2x2 / 2) after each block, then ``fc6`` (4096), ``relu6``, ``drop6``,
    ``fc7`` (4096), ``relu7``, ``drop7``, ``fc8`` (1000) and ``prob``.  Input 3 x 224 x 224."""
    if depth not in _VGG_BLOCKS:
        raise ValueError(f"unsupported VGG depth {depth} (16 or 19)")
    L: List[dict] = []
    prev = "data"
    for b, (n, c) in enumerate(zip(_VGG_BLOCKS[depth], _VGG_WIDTHS), 1):
        for l in range(1, n + 1):
            name = f"conv{b}_{l}"
            L.append(dict(name=name, type="Convolution", bottoms=[prev], tops=[name], num_output=c, kernel_size=3, pad=1, stride=1,
                          bias_term=True))
            L.append(dict(name=f"relu{b}_{l}", type="ReLU", bottoms=[name], tops=[name]))
            prev = name
        L.append(dict(name=f"pool{b}", type="Pooling", bottoms=[prev], tops=[f"pool{b}"], pool="MAX", kernel_size=2, stride=2, pad=0))
        prev = f"pool{b}"
    for i, c in ((6, 4096), (7, 4096), (8, 1000)):
        L.append(dict(name=f"fc{i}", type="InnerProduct", bottoms=[prev], tops=[f"fc{i}"], num_output=c, bias_term=True))
        prev = f"fc{i}"
        if i < 8:
            L.append(dict(name=f"relu{i}", type="ReLU", bottoms=[prev], tops=[prev]))
            L.append(dict(name=f"drop{i}", type="Dropout", bottoms=[prev], tops=[prev]))
    L.append(dict(name="prob", type="Softmax", bottoms=[prev], tops=["prob"]))
    return {"name": f"VGG_ILSVRC_{depth}_layers", "input": "data", "input_dims": [1, 3, 224, 224], "layers": L}


# --------------------------------------------------------------------------------------------------
# shape inference on raw layers
# --------------------------------------------------------------------------------------------------

def conv_out(size: int, k: int, pad: int, stride: int) -> int:
    return (size + 2 * pad - k) // stride + 1


def pool_out_ceil(size: int, k: int, pad: int, stride: int, ceil_mode: bool = True) -> int:
    """Caffe pooling: ceil mode, and the last window must start inside the (padded) image.
    ``ceil_mode=False`` is the ONNX/floor convention (used by the MNIST import)."""
    if not ceil_mode:
        return (size + 2 * pad - k) // stride + 1
    out = int(math.ceil((size + 2 * pad - k) / stride)) + 1
    if pad > 0 and (out - 1) * stride >= size + pad:
        out -= 1
    return out


def infer_shapes(net: dict) -> Dict[str, Tuple[int, int, int]]:
    """blob name -> (C, H, W) after the LAST layer that writes it (in-place layers keep the shape)."""
    _, c, h, w = net["input_dims"]
    shapes = {net["input"]: (c, h, w)}
    for L in net["layers"]:
        t = L["type"]
        c, h, w = shapes[L["bottoms"][0]]
        if t == "Convolution":
            k, p, s = L["kernel_size"], L["pad"], L["stride"]
            shapes[L["tops"][0]] = (L["num_output"], conv_out(h, k, p, s), conv_out(w, k, p, s))
        elif t == "Pooling":
            k, p, s = L["kernel_size"], L["pad"], L["stride"]
            cm = L.get("ceil_mode", True)
            shapes[L["tops"][0]] = (c, pool_out_ceil(h, k, p, s, cm), pool_out_ceil(w, k, p, s, cm))
        elif t == "InnerProduct":
            shapes[L["tops"][0]] = (L["num_output"], 1, 1)
        elif t == "Eltwise":
            for b in L["bottoms"][1:]:
                if shapes[b] != (c, h, w):
                    raise ValueError(f"Eltwise {L['name']}: shape mismatch {shapes[b]} vs {(c, h, w)}")
            shapes[L["tops"][0]] = (c, h, w)
        elif t == "Concat":
            for b in L["bottoms"][1:]:
                if shapes[b][1:] != (h, w):
                    raise ValueError(f"Concat {L['name']}: input {b} is {shapes[b][1]}x{shapes[b][2]}, not {h}x{w} like {L['bottoms'][0]}")
            shapes[L["tops"][0]] = (sum(shapes[b][0] for b in L["bottoms"]), h, w)
        else:  # BatchNorm / Scale / ReLU / Softmax / LRN / Dropout
            shapes[L["tops"][0]] = (c, h, w)
    return shapes


# --------------------------------------------------------------------------------------------------
# lowering: raw layers (+ raw weights) -> fused ops (+ folded weights)
# --------------------------------------------------------------------------------------------------

OP_CONV, OP_MAXPOOL, OP_AVGPOOL, OP_FC, OP_SOFTMAX = "conv", "maxpool", "avgpool", "fc", "softmax"
OP_LRN = "lrn"


def _drop_dropout(net: dict) -> dict:
    """``net`` without its Dropout layers (identity at inference): a layer that reads a Dropout's top reads its bottom."""
    if not any(L["type"] == "Dropout" for L in net["layers"]):
        return net
    alias: Dict[str, str] = {}
    layers = []
    for L in net["layers"]:
        bottoms = [alias.get(b, b) for b in L["bottoms"]]
        if L["type"] == "Dropout":
            if L["tops"][0] != bottoms[0]:
                alias[L["tops"][0]] = bottoms[0]
            continue
        layers.append(dict(L, bottoms=bottoms))
    return dict(net, layers=layers)


def lower(net: dict, weights: Optional[dict] = None) -> dict:
    """Fuse Conv+BatchNorm+Scale(+ReLU)(+Eltwise SUM+ReLU) and version in-place blobs.

    Returns ``{name, input, input_shape (C,H,W), tensors {name: (C,H,W)}, ops [...], output}``.
    When ``weights`` (raw, keyed by layer name; see :mod:`weights`) is given each conv/fc op carries
    folded fp32 parameters: ``W`` in OHWI order ``[Cout, kh, kw, Cin]`` already multiplied by the
    per-channel BN*Scale factor, and ``bias`` ``[Cout]``.
    """
    import numpy as np

    net = _drop_dropout(net)
    layers = net["layers"]
    shapes = infer_shapes(net)
    # last writer of each blob decides the SSA tensor that consumers see
    ops: List[dict] = []
    producer: Dict[str, dict] = {}  # blob -> op dict that currently defines it
    tensors: Dict[str, Tuple[int, int, int]] = {net["input"]: shapes[net["input"]]}

    def fold_state(op):
        return op.setdefault("_fold", {"scale": None, "shift": None})

    def readers_of(blob, i):
        """Layers other than layer i that read ``blob``, less the in-place BatchNorm / Scale / ReLU before layer i."""
        return [(j, M) for j, M in enumerate(layers) if j != i and blob in M["bottoms"] and
                not (j < i and M["type"] in ("BatchNorm", "Scale", "ReLU") and M["tops"] == [blob])]

    # Pre-activations: a BatchNorm (+ Scale) + ReLU chain that cannot fold into the convolution before it becomes the input
    # prologue of its one reader.  blob -> {name, input, relu, scale, shift} (scale / shift fp64 while folding)
    preact: Dict[str, dict] = {}
    grown: Dict[str, str] = {}  # nested concatenation: blob -> the Concat top that extends it (channel prefix)

    def take_preact(blob, i, reader):
        pa = preact.pop(blob)
        if not pa["relu"]:
            raise ValueError(f"BatchNorm {pa['name']}: a pre-activation without ReLU is not supported ({reader} reads it)")
        n = len(readers_of(blob, i)) + 1
        if n != 1:
            raise ValueError(f"BatchNorm {pa['name']}: its output {blob} has {n} readers; a pre-activation has exactly one")
        return pa

    def attach_preact(op, pa):
        op["pre"] = True
        if "scale" in pa:
            op["pre_scale"] = pa["scale"].astype(np.float32)
            op["pre_shift"] = pa["shift"].astype(np.float32)

    consumed_by_eltwise = set()
    i = 0
    while i < len(layers):
        L = layers[i]
        t = L["type"]
        name = L["name"]
        for b in L["bottoms"]:
            if b in preact and not (t in ("Scale", "ReLU") and L["tops"] == [b]) and not (
                    t == "Convolution" or (t == "Pooling" and L["pool"] == "AVE")):
                raise ValueError(f"BatchNorm {preact[b]['name']}: a pre-activation is the input prologue of a 1x1 convolution or an "
                                 f"average pool, not of {t} {name}")
        pa_in = None
        if t in ("Convolution", "Pooling") and L["bottoms"][0] in preact:
            pa_in = take_preact(L["bottoms"][0], i, name)
            L = dict(L, bottoms=[pa_in["input"]] + L["bottoms"][1:])
        if t == "Convolution":
            if pa_in is not None and (L["kernel_size"] != 1 or L["stride"] != 1 or L["pad"] != 0 or L.get("group", 1) != 1):
                raise ValueError(f"BatchNorm {pa_in['name']}: a pre-activation before {name}, a {L['kernel_size']}x{L['kernel_size']} "
                                 "convolution, is not supported (only dense 1x1 stride-1 unpadded ones: with padding, "
                                 "relu(shift) != 0 at a zero-padded pixel)")
            cin = tensors[L["bottoms"][0]][0]
            groups = L.get("group", 1)
            if groups < 1 or cin % groups or L["num_output"] % groups:
                raise ValueError(f"Convolution {name}: {groups} groups do not divide {cin} -> {L['num_output']} channels")
            op = dict(type=OP_CONV, name=name, input=L["bottoms"][0], output=L["tops"][0], residual=None,
                      cin=cin, cout=L["num_output"], k=L["kernel_size"], stride=L["stride"], pad=L["pad"],
                      relu=False, groups=groups)
            if weights is not None:
                w = np.asarray(weights[name]["W"], dtype=np.float64)  # [Cout, Cin/groups, k, k]
                b = (np.asarray(weights[name]["b"], dtype=np.float64) if L["bias_term"]
                     else np.zeros(L["num_output"], dtype=np.float64))
                op["_w"], op["_b"] = w, b
            if pa_in is not None:
                attach_preact(op, pa_in)
            ops.append(op)
            producer[L["tops"][0]] = op
            tensors[L["tops"][0]] = shapes[L["tops"][0]]
        elif t == "BatchNorm":
            bottom, top = L["bottoms"][0], L["tops"][0]
            op = producer.get(bottom)
            if (op is None or op["type"] != OP_CONV or op.get("_sealed") or op["output"] != bottom) and top != bottom:
                # a pre-activation (into a new blob): folded into the input prologue of the blob's one reader
                pa = preact[top] = dict(name=name, input=bottom, relu=False)
                if weights is not None:
                    pa["scale"] = 1.0 / np.sqrt(np.asarray(weights[name]["var"], dtype=np.float64) + L.get("eps", 1e-5))
                    pa["shift"] = -np.asarray(weights[name]["mean"], dtype=np.float64) * pa["scale"]
                i += 1
                continue
            if op is None or op["type"] != OP_CONV or op.get("_sealed"):
                raise ValueError(f"BatchNorm {name} does not follow a foldable Convolution")
            if top != bottom:  # folded into the convolution, whose output takes the new blob's name
                others = readers_of(bottom, i)
                if others:
                    raise ValueError(f"BatchNorm {name}: the convolution output {bottom} it normalises is also read by {others[0][1]['name']}")
                op["output"] = top
                del tensors[bottom]
                del producer[bottom]
                tensors[top] = shapes[top]
                producer[top] = op
            if weights is not None:
                mean = np.asarray(weights[name]["mean"], dtype=np.float64)
                var = np.asarray(weights[name]["var"], dtype=np.float64)
                inv = 1.0 / np.sqrt(var + L.get("eps", 1e-5))
                op["_w"] = op["_w"] * inv[:, None, None, None]
                op["_b"] = (op["_b"] - mean) * inv
        elif t == "Scale" and L["bottoms"][0] in preact and L["tops"] == L["bottoms"]:
            pa = preact[L["bottoms"][0]]
            if pa["relu"]:
                raise ValueError(f"Scale {name}: a pre-activation applies its Scale before its ReLU")
            if weights is not None:
                g = np.asarray(weights[name]["gamma"], dtype=np.float64)
                pa["scale"], pa["shift"] = pa["scale"] * g, pa["shift"] * g
                if L.get("bias_term"):
                    pa["shift"] = pa["shift"] + np.asarray(weights[name]["beta"], dtype=np.float64)
        elif t == "Scale":
            op = producer[L["bottoms"][0]]
            if op["type"] != OP_CONV or op.get("_sealed"):
                raise ValueError(f"Scale {name} does not follow a foldable Convolution")
            if weights is not None:
                g = np.asarray(weights[name]["gamma"], dtype=np.float64)
                op["_w"] = op["_w"] * g[:, None, None, None]
                op["_b"] = op["_b"] * g
                if L.get("bias_term"):
                    op["_b"] = op["_b"] + np.asarray(weights[name]["beta"], dtype=np.float64)
        elif t == "ReLU" and L["bottoms"][0] in preact and L["tops"] == L["bottoms"]:
            preact[L["bottoms"][0]]["relu"] = True
        elif t == "ReLU":
            op = producer[L["bottoms"][0]]
            if op["type"] == OP_SOFTMAX:
                raise ValueError(f"ReLU {name}: a ReLU on the output of Softmax {op['name']} is not supported")
            if op["type"] not in (OP_CONV, OP_FC):
                raise ValueError(f"ReLU {name}: only conv-fused ReLU is supported")
            if op["type"] == OP_FC and op.get("_sealed"):
                raise ValueError(f"ReLU {name}: InnerProduct {op['name']} already has a fused ReLU")
            op["relu"] = True
            op["_sealed"] = True
        elif t == "Eltwise":
            if L.get("operation", "SUM") != "SUM" or len(L["bottoms"]) != 2:
                raise ValueError(f"Eltwise {name}: only 2-input SUM is supported")
            a, b = L["bottoms"]
            for x in (a, b):
                if producer.get(x, {}).get("type") == OP_FC:
                    raise ValueError(f"Eltwise {name}: InnerProduct {producer[x]['name']} cannot take a residual")
            # fuse into whichever input was produced LAST by a conv that nobody else has read yet
            cand = [x for x in (a, b) if producer.get(x, {}).get("type") == OP_CONV
                    and not producer[x].get("_sealed") and x not in consumed_by_eltwise]
            if not cand:
                raise ValueError(f"Eltwise {name}: no fusable conv input")
            fuse = max(cand, key=lambda x: ops.index(producer[x]))
            other = b if fuse == a else a
            op = producer[fuse]
            op["residual"] = other
            op["output"] = L["tops"][0]
            op["_sealed"] = True
            del tensors[fuse]
            tensors[L["tops"][0]] = shapes[L["tops"][0]]
            producer[L["tops"][0]] = op
            consumed_by_eltwise.add(fuse)
        elif t == "Pooling":
            c, h, w = tensors[L["bottoms"][0]]
            if L["pool"] == "MAX":
                op = dict(type=OP_MAXPOOL, name=name, input=L["bottoms"][0], output=L["tops"][0],
                          k=L["kernel_size"], stride=L["stride"], pad=L["pad"],
                          ceil_mode=L.get("ceil_mode", True))
            else:
                k = L["kernel_size"]
                glob = k == h == w and L["pad"] == 0
                if not glob and not (L["stride"] == k and L["pad"] == 0 and h % k == 0 and w % k == 0):
                    raise ValueError(f"Pooling {name}: only global AVE pooling, or a k x k / stride k window without padding that "
                                     "tiles the input, is supported")
                conv = producer.get(L["bottoms"][0])
                if (not glob and pa_in is None and conv is not None and conv["type"] == OP_CONV and conv.get("pre") and
                        conv["output"] == L["bottoms"][0] and conv["residual"] is None and not conv["relu"] and
                        not conv.get("_sealed") and not readers_of(L["bottoms"][0], i)):
                    # pre-activation -> 1x1 convolution -> average pool: the two commute exactly, so the pool runs first with
                    # the prologue and the convolution on the pooled tensor (4x less work; the convolution writes the output)
                    mid = conv["name"] + "/pool"
                    pool = dict(type=OP_AVGPOOL, name=name, input=conv["input"], output=mid, k=k, stride=k, pad=0, ceil_mode=True,
                                pre=True)
                    for key in ("pre_scale", "pre_shift"):
                        if key in conv:
                            pool[key] = conv.pop(key)
                    del conv["pre"]
                    ops.insert(ops.index(conv), pool)
                    tensors[mid] = (conv["cin"], h // k, w // k)
                    del tensors[conv["output"]]
                    del producer[conv["output"]]
                    conv.update(input=mid, output=L["tops"][0], commuted=True, _sealed=True)
                    producer[L["tops"][0]] = conv
                    tensors[L["tops"][0]] = shapes[L["tops"][0]]
                    i += 1
                    continue
                op = dict(type=OP_AVGPOOL, name=name, input=L["bottoms"][0], output=L["tops"][0],
                          k=k, stride=k if not glob else L["stride"], pad=0, ceil_mode=True)
                if pa_in is not None:
                    attach_preact(op, pa_in)
            ops.append(op)
            producer[L["tops"][0]] = op
            tensors[L["tops"][0]] = shapes[L["tops"][0]]
        elif t == "InnerProduct":
            c, h, w = tensors[L["bottoms"][0]]
            op = dict(type=OP_FC, name=name, input=L["bottoms"][0], output=L["tops"][0],
                      cin=c * h * w, cout=L["num_output"], in_chw=(c, h, w), relu=False)
            if weights is not None:
                W = np.asarray(weights[name]["W"], dtype=np.float64).reshape(L["num_output"], c, h, w)
                # Caffe flattens C,H,W; the engine keeps activations NHWC -> permute K to (h, w, c)
                op["W"] = np.ascontiguousarray(W.transpose(0, 2, 3, 1).reshape(L["num_output"], -1)).astype(np.float32)
                op["bias"] = (np.asarray(weights[name]["b"], dtype=np.float32) if L["bias_term"]
                              else np.zeros(L["num_output"], np.float32))
            ops.append(op)
            producer[L["tops"][0]] = op
            tensors[L["tops"][0]] = shapes[L["tops"][0]]
        elif t == "Softmax":
            op = dict(type=OP_SOFTMAX, name=name, input=L["bottoms"][0], output=L["tops"][0])
            ops.append(op)
            producer[L["tops"][0]] = op
            tensors[L["tops"][0]] = shapes[L["tops"][0]]
        elif t == "LRN":
            n = L.get("local_size", 5)
            if n < 1 or n % 2 == 0:
                raise ValueError(f"LRN {name}: local_size {n} must be odd")
            if L["tops"][0] == L["bottoms"][0]:
                raise ValueError(f"LRN {name}: in-place LRN is not supported (give the layer its own top)")
            op = dict(type=OP_LRN, name=name, input=L["bottoms"][0], output=L["tops"][0], local_size=n,
                      alpha=float(L.get("alpha", 1.0)), beta=float(L.get("beta", 0.75)), k=float(L.get("k", 1.0)))
            ops.append(op)
            producer[L["tops"][0]] = op
            tensors[L["tops"][0]] = shapes[L["tops"][0]]
        elif t == "Concat":
            # no op: each input convolution writes its own channel range of the output (op["out_c0"])
            top = L["tops"][0]
            if len(set(L["bottoms"])) != len(L["bottoms"]) or top in L["bottoms"]:
                raise ValueError(f"Concat {name}: an input appears twice, or the output overwrites an input")
            c0 = 0
            b0 = L["bottoms"][0]
            p0 = producer.get(b0)
            r0 = readers_of(b0, i)
            # a Concat that grows its first input: an earlier Concat's top, a max pool's output, or a convolution's output
            # that pre-activations (before this Concat) read too.  The whole chain is one tensor, the last Concat's top; each
            # earlier top is a channel prefix of it, and the first input's producer writes its first slice.
            if p0 is not None and (p0["type"] in ("concat", OP_MAXPOOL) or (p0["type"] == OP_CONV and r0)):
                for j, M in r0:
                    if not (j < i and M["type"] == "BatchNorm" and M["tops"][0] != b0 and M["tops"][0] not in tensors):
                        raise ValueError(f"Concat {name}: input {b0} is also read by {M['name']}; the first input of a growing "
                                         "concatenation may be read only by pre-activation BatchNorms before the Concat")
                if p0["type"] != "concat":
                    if p0.get("residual") is not None or p0["output"] != b0 or b0 == net["input"]:
                        raise ValueError(f"Concat {name}: input {b0} is not the output of a convolution without a residual or of a max pool")
                    p0["out_c0"] = 0
                    p0["_sealed"] = True
                    if p0["type"] == OP_MAXPOOL:
                        p0["cout"] = tensors[b0][0]
                grown[b0] = top
                c0 = tensors[b0][0]
            elif p0 is not None and p0["type"] not in (OP_CONV, "concat") and b0 != net["input"]:
                raise ValueError(f"Concat {name}: input {b0} is not the output of a convolution, a max pool or a concatenation")
            for b in (L["bottoms"][1:] if b0 in grown else L["bottoms"]):
                op = producer.get(b)
                if op is None or op["type"] != OP_CONV or op["residual"] is not None or op["output"] != b:
                    raise ValueError(f"Concat {name}: input {b} is not the output of a convolution (only convolutions, "
                                     "without a residual, can be concatenated)")
                # (the convolution's own in-place BatchNorm / Scale / ReLU before the Concat are part of it)
                readers = [M["name"] for j, M in enumerate(layers) if j != i and b in M["bottoms"] and
                           not (j < i and M["type"] in ("BatchNorm", "Scale", "ReLU") and M["tops"] == [b])]
                if readers:
                    raise ValueError(f"Concat {name}: input {b} is also read by {readers[0]}; a concatenated convolution "
                                     "output may have no other reader")
                if b == net["input"]:
                    raise ValueError(f"Concat {name}: the network input cannot be concatenated")
                op["output"] = top
                op["out_c0"] = c0
                op["_sealed"] = True
                c0 += op["cout"]
                del tensors[b]
                del producer[b]
            tensors[top] = shapes[top]
            producer[top] = dict(type="concat", name=name)
        else:
            raise ValueError(f"unsupported layer type {t}")
        i += 1

    if preact:
        pa = next(iter(preact.values()))
        raise ValueError(f"BatchNorm {pa['name']}: its pre-activation has no reader")

    def phys(b):
        while b in grown:
            b = grown[b]
        return b

    for op in ops:  # nested concatenations: every blob of a chain is its last top (the readers' cin keeps the prefix)
        if op.get("input") in grown:
            op["input"] = phys(op["input"])
        if op.get("output") in grown:
            op["output"] = phys(op["output"])
    for b in grown:
        tensors.pop(b, None)
    # an FC whose output another FC reads is a hidden layer: an fp16 activation [C, 1, 1] in fp16 plans (the reader's K
    # order (h, w, c) is then the channel order); the last FC stays an fp32 vector
    fc_inputs = {op["input"] for op in ops if op["type"] == OP_FC}
    for op in ops:
        if op["type"] == OP_FC:
            op["hidden"] = op["output"] in fc_inputs
    for op in ops:
        if op["type"] == OP_CONV and "_w" in op:
            op["W"] = np.ascontiguousarray(op.pop("_w").transpose(0, 2, 3, 1)).astype(np.float32)  # OHWI
            op["bias"] = op.pop("_b").astype(np.float32)
        op.pop("_sealed", None)
        op.pop("_fold", None)
    return {
        "name": net["name"],
        "input": net["input"],
        "input_shape": tuple(shapes[net["input"]]),
        "tensors": tensors,
        "ops": ops,
        "output": ops[-1]["output"],
    }


def conv_flops(lowered: dict) -> int:
    """2*MAC over conv + fc ops, per image (the algorithmic FLOP count used by the roofline).  A grouped convolution
    counts its Cin/groups inputs per output channel, not the zero blocks the tensor-core path multiplies."""
    total = 0
    for op in lowered["ops"]:
        if op["type"] == OP_CONV:
            c, h, w = lowered["tensors"][op["output"]]
            total += 2 * h * w * op["cout"] * (op["cin"] // op.get("groups", 1)) * op["k"] * op["k"]
        elif op["type"] == OP_FC:
            total += 2 * op["cin"] * op["cout"]
    return total
