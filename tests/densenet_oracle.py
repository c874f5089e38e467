"""DenseNet for the CPU oracles (test infrastructure only): BatchNorm and Scale as layers of their own, windowed average
pooling, and the lowered BatchNorm + ReLU input prologues.

* :func:`caffe_forward`          the raw layer list, unfused, in torch float64 (Caffe semantics)
* :func:`lowered_forward_f16emu` the lowered ops with the fp16 engine's rounding points: the prologue's fp16 operand, the
                                 pool-first transitions, prefix reads of the block tensors
* :func:`conv_pre_emu`, :func:`avgpool_pre_ref`  per-op references of the two prologue kernels (plan_format.h, kConvPreAct)
"""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch
import torch.nn.functional as F

from tests.googlenet_oracle import _maxpool_caffe


def caffe_forward(net: dict, weights: Dict[str, dict], x: np.ndarray, logits: bool = False) -> np.ndarray:
    """The raw layer list on x (N, C, H, W) in float64.  Returns the last top (or, with ``logits``, the InnerProduct's
    output) as [N, -1]."""
    blobs = {net["input"]: torch.from_numpy(np.ascontiguousarray(x)).double()}
    fc = None
    with torch.no_grad():
        for L in net["layers"]:
            t, name = L["type"], L["name"]
            a = blobs[L["bottoms"][0]]
            p = weights.get(name, {})
            if t == "Convolution":
                b = torch.from_numpy(p["b"]).double() if L["bias_term"] else None
                y = F.conv2d(a, torch.from_numpy(p["W"]).double(), b, stride=L["stride"], padding=L["pad"], groups=L.get("group", 1))
            elif t == "BatchNorm":
                mean = torch.from_numpy(p["mean"]).double().view(1, -1, 1, 1)
                var = torch.from_numpy(p["var"]).double().view(1, -1, 1, 1)
                y = (a - mean) / torch.sqrt(var + L.get("eps", 1e-5))
            elif t == "Scale":
                y = a * torch.from_numpy(p["gamma"]).double().view(1, -1, 1, 1)
                if L.get("bias_term"):
                    y = y + torch.from_numpy(p["beta"]).double().view(1, -1, 1, 1)
            elif t == "ReLU":
                y = torch.relu(a)
            elif t == "Pooling":
                if L["pool"] == "MAX":
                    y = _maxpool_caffe(a, L["kernel_size"], L["stride"], L["pad"], L.get("ceil_mode", True))
                elif L["kernel_size"] == a.shape[2] == a.shape[3]:
                    y = a.mean(dim=(2, 3), keepdim=True)
                else:
                    y = F.avg_pool2d(a, L["kernel_size"], L["stride"])
            elif t == "Concat":
                y = torch.cat([blobs[b] for b in L["bottoms"]], dim=1)
            elif t == "InnerProduct":
                b = torch.from_numpy(p["b"]).double() if L["bias_term"] else None
                y = F.linear(a.reshape(a.shape[0], -1), torch.from_numpy(p["W"]).double(), b).view(a.shape[0], -1, 1, 1)
                fc = y
            elif t == "Softmax":
                y = torch.softmax(a, dim=1)
            else:
                raise ValueError(f"oracle: unsupported layer {t}")
            blobs[L["tops"][0]] = y
    out = fc if logits else blobs[net["layers"][-1]["tops"][0]]
    return out.reshape(out.shape[0], -1).numpy()


def _r16(t):
    return t.to(torch.float16).to(torch.float64)


def prologue_f32(a: torch.Tensor, scale: np.ndarray, shift: np.ndarray) -> torch.Tensor:
    """max(fmaf(x, scale, shift), 0) in fp32 on fp16 values a (float64 NCHW): x * scale is exact in float64, so one rounding
    of the float64 sum to fp32 is fmaf's."""
    s = torch.from_numpy(scale.astype(np.float32)).double().view(1, -1, 1, 1)
    t = torch.from_numpy(shift.astype(np.float32)).double().view(1, -1, 1, 1)
    return torch.relu((a * s + t).to(torch.float32).double())


def conv_pre_emu(op: dict, a: torch.Tensor) -> torch.Tensor:
    """A prologue 1x1 convolution on fp16 values a (channels [0, cin) of its input): the fp16 operand, fp16 weights, exact
    products and sum, bias, ReLU and one fp16 rounding."""
    a = _r16(prologue_f32(a[:, :op["cin"]], op["pre_scale"], op["pre_shift"]))
    w = _r16(torch.from_numpy(op["W"]).double()).permute(0, 3, 1, 2).contiguous()
    y = F.conv2d(a, w) + torch.from_numpy(op["bias"]).double().view(1, -1, 1, 1)
    return _r16(torch.relu(y) if op["relu"] else y)


def avgpool_pre_ref(a: torch.Tensor, scale: np.ndarray, shift: np.ndarray, k: int) -> torch.Tensor:
    """The prologue average pool's contract, bit for bit: relu(fmaf(x, s, t)) summed in fp32 in row-major window order,
    times fp32(1 / k^2), one fp16 rounding."""
    v = prologue_f32(a, scale, shift).to(torch.float32)
    n, c, h, w = v.shape
    acc = torch.zeros((n, c, h // k, w // k), dtype=torch.float32)
    for r in range(k):
        for s in range(k):
            acc = acc + v[:, :, r::k, s::k]
    return (acc * torch.tensor(1.0 / (k * k), dtype=torch.float32)).to(torch.float16).double()


def lowered_forward_f16emu(lowered: dict, x: np.ndarray, logits: bool = False) -> np.ndarray:
    """The lowered DenseNet ops with the fp16 engine's rounding points.  Returns the output (or the fc logits) as [N, -1]."""
    shapes = lowered["tensors"]
    blobs = {lowered["input"]: _r16(torch.from_numpy(np.ascontiguousarray(x)).double())}
    n = x.shape[0]
    fc = None
    with torch.no_grad():
        for op in lowered["ops"]:
            a = blobs[op["input"]]
            t = op["type"]
            if t == "conv":
                if op.get("pre"):
                    y = conv_pre_emu(op, a)
                else:
                    w = _r16(torch.from_numpy(op["W"]).double()).permute(0, 3, 1, 2).contiguous()
                    y = F.conv2d(a[:, :op["cin"]], w, None, stride=op["stride"], padding=op["pad"])
                    y = y + torch.from_numpy(op["bias"]).double().view(1, -1, 1, 1)
                    y = _r16(torch.relu(y) if op["relu"] else y)
            elif t == "maxpool":
                y = _maxpool_caffe(a, op["k"], op["stride"], op["pad"], op["ceil_mode"])
            elif t == "avgpool":
                y = avgpool_pre_ref(a, op["pre_scale"], op["pre_shift"], op["k"])
            elif t == "fc":
                W = _r16(torch.from_numpy(op["W"]).double())
                flat = a.permute(0, 2, 3, 1).reshape(n, -1)
                y = (flat @ W.t() + torch.from_numpy(op["bias"]).double()).float().double().view(n, -1, 1, 1)
                fc = y
            elif t == "softmax":
                y = torch.softmax(a.float(), dim=1).double()
            else:
                raise ValueError(t)
            if "out_c0" in op:
                c, h, w_ = shapes[op["output"]]
                dst = blobs.setdefault(op["output"], torch.zeros((n, c, h, w_), dtype=torch.float64))
                dst[:, op["out_c0"]:op["out_c0"] + y.shape[1]] = y
            else:
                blobs[op["output"]] = y
    out = fc if logits else blobs[lowered["output"]]
    return out.reshape(n, -1).numpy()



def dense_net(cin: int = 64, hw: int = 16, layers: int = 3, growth: int = 32, bottleneck: int = 128, classes: int = 16) -> dict:
    """A small DenseNet in the layer names and form of ``graph.densenet_caffe``: a 1x1 stem convolution (+ BN, ReLU) of
    ``cin`` channels, the 3x3/2 pad-1 max pool (FLOOR) that starts block 2, ``layers`` dense layers, a transition
    (BN-ReLU-1x1-AVE 2x2/2) into block 3 with ``layers`` more, then BN-ReLU, the global average pool, fc6 and prob."""
    L = []

    def conv(name, bottom, nout, k, pad=0):
        L.append(dict(name=name, type="Convolution", bottoms=[bottom], tops=[name], num_output=nout, kernel_size=k, pad=pad, stride=1,
                      bias_term=False))

    def bsr(prefix, relu, bottom):
        bn = prefix + "/bn"
        L.append(dict(name=bn, type="BatchNorm", bottoms=[bottom], tops=[bn], use_global_stats=True, eps=1e-5))
        L.append(dict(name=prefix + "/scale", type="Scale", bottoms=[bn], tops=[bn], bias_term=True))
        L.append(dict(name=relu, type="ReLU", bottoms=[bn], tops=[bn]))
        return bn

    conv("conv1", "data", cin, 1)
    L.append(dict(name="pool1", type="Pooling", bottoms=[bsr("conv1", "relu1", "conv1")], tops=["pool1"], pool="MAX", kernel_size=3,
                  stride=2, pad=1, ceil_mode=False))
    prev, c = "pool1", cin
    for b in (2, 3):
        for l in range(1, layers + 1):
            x1, x2 = f"conv{b}_{l}/x1", f"conv{b}_{l}/x2"
            conv(x1, bsr(x1, f"relu{b}_{l}/x1", prev), bottleneck, 1)
            conv(x2, bsr(x2, f"relu{b}_{l}/x2", x1), growth, 3, 1)
            L.append(dict(name=f"concat_{b}_{l}", type="Concat", bottoms=[prev, x2], tops=[f"concat_{b}_{l}"], axis=1))
            prev, c = f"concat_{b}_{l}", c + growth
        if b == 2:
            c //= 2
            conv("conv2_blk", bsr("conv2_blk", "relu2_blk", prev), c, 1)
            L.append(dict(name="pool2", type="Pooling", bottoms=["conv2_blk"], tops=["pool2"], pool="AVE", kernel_size=2, stride=2, pad=0))
            prev = "pool2"
    L.append(dict(name="pool5", type="Pooling", bottoms=[bsr("conv5_blk", "relu5_blk", prev)], tops=["pool5"], pool="AVE",
                  kernel_size=hw // 4, stride=1, pad=0))
    L.append(dict(name="fc6", type="InnerProduct", bottoms=["pool5"], tops=["fc6"], num_output=classes, bias_term=True))
    L.append(dict(name="prob", type="Softmax", bottoms=["fc6"], tops=["prob"]))
    return {"name": "dense", "input": "data", "input_dims": [1, 3, hw, hw], "layers": L}
