"""Concat, LRN and Dropout for the CPU oracles (test infrastructure only), the layers GoogLeNet adds to the ResNet
vocabulary that ``oracle/`` restates.

* :func:`caffe_forward`          the raw layer list, unfused, in torch (fp32 or fp64), Caffe semantics
* :func:`lowered_forward_f16emu` the lowered ops with the fp16 engine's rounding points, including LRN's numerics contract
* :func:`numpy_forward`          the second witness: the raw layer list in float64 numpy (``oracle.numpy_ops`` + the new layers)

LRN (Caffe ``ACROSS_CHANNELS``): y_c = x_c (k + alpha / n sum_{|j - c| <= (n - 1) / 2} x_j^2)^(-beta), the window zero-padded at
the channel edges and the divisor always n.  The engine's contract (plan_format.h, OP_LRN): squares summed in fp32 in
channel order, scale = fmaf(fp32(alpha / n), sum, k), powf(scale, -beta) in fp32, the product in fp32, one fp16 rounding.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

from oracle import numpy_ops
from oracle.caffe_forward import _pool_out


def _maxpool_caffe(a, k, s, p, ceil_mode=True):
    ho = _pool_out(a.shape[2], k, p, s, ceil_mode)
    wo = _pool_out(a.shape[3], k, p, s, ceil_mode)
    need_h = (ho - 1) * s + k - a.shape[2] - p
    need_w = (wo - 1) * s + k - a.shape[3] - p
    return F.max_pool2d(F.pad(a, (p, max(need_w, 0), p, max(need_h, 0)), value=float("-inf")), k, s)


def lrn_torch(a: torch.Tensor, n: int, alpha: float, beta: float, k: float) -> torch.Tensor:
    """Caffe ACROSS_CHANNELS LRN in a's dtype (NCHW)."""
    h = (n - 1) // 2
    sq = F.pad(a * a, (0, 0, 0, 0, h, h))
    s = sum(sq[:, d:d + a.shape[1]] for d in range(n))
    return a * torch.pow(k + alpha / n * s, -beta)


def lrn_f16emu(a: torch.Tensor, n: int, alpha: float, beta: float, k: float) -> torch.Tensor:
    """The engine's LRN on fp16 values ``a`` (float64 NCHW holding fp16 numbers) -> float64 holding fp16 numbers."""
    h = (n - 1) // 2
    x = a.to(torch.float32)
    sq = F.pad(x * x, (0, 0, 0, 0, h, h))            # exact squares of fp16 values
    s = torch.zeros_like(x)
    for d in range(n):                                # fp32 sum in channel order c - h ... c + h
        s = s + sq[:, d:d + x.shape[1]]
    alpha_n = np.float32(np.float32(alpha) / np.float32(n))
    scale = (float(alpha_n) * s.double() + float(np.float32(k))).to(torch.float32)   # one rounding (fmaf)
    y = x * torch.pow(scale, -float(np.float32(beta)))
    return y.to(torch.float16).to(torch.float64)


def caffe_forward(net: dict, weights: Dict[str, dict], x: np.ndarray, dtype=torch.float32):
    """The raw layer list (Convolution with bias, ReLU, Pooling, LRN, Concat, Dropout, InnerProduct, Softmax) on x (N,C,H,W).
    Returns the last top as a float64 [N, -1] array."""
    blobs = {net["input"]: torch.from_numpy(np.ascontiguousarray(x)).to(dtype)}
    with torch.no_grad():
        for L in net["layers"]:
            t, name = L["type"], L["name"]
            a = blobs[L["bottoms"][0]]
            if t == "Convolution":
                w = torch.from_numpy(weights[name]["W"]).to(dtype)
                b = torch.from_numpy(weights[name]["b"]).to(dtype) if L["bias_term"] else None
                y = F.conv2d(a, w, b, stride=L["stride"], padding=L["pad"])
            elif t == "ReLU":
                y = torch.relu(a)
            elif t == "Pooling":
                if L["pool"] == "MAX":
                    y = _maxpool_caffe(a, L["kernel_size"], L["stride"], L["pad"], L.get("ceil_mode", True))
                else:
                    y = a.mean(dim=(2, 3), keepdim=True)
            elif t == "LRN":
                y = lrn_torch(a, L["local_size"], L["alpha"], L["beta"], L["k"])
            elif t == "Concat":
                y = torch.cat([blobs[b] for b in L["bottoms"]], dim=1)
            elif t == "Dropout":
                y = a
            elif t == "InnerProduct":
                w = torch.from_numpy(weights[name]["W"]).to(dtype)
                b = torch.from_numpy(weights[name]["b"]).to(dtype) if L["bias_term"] else None
                y = F.linear(a.reshape(a.shape[0], -1), w, b).view(a.shape[0], -1, 1, 1)
            elif t == "Softmax":
                y = torch.softmax(a, dim=1)
            else:
                raise ValueError(f"oracle: unsupported layer {t}")
            blobs[L["tops"][0]] = y
    out = blobs[net["layers"][-1]["tops"][0]]
    return out.reshape(out.shape[0], -1).double().numpy()


def lowered_forward_f16emu(lowered: dict, x: np.ndarray, keep: Optional[list] = None):
    """The lowered ops with the fp16 engine's rounding points (``oracle.caffe_forward.lowered_forward_f16emu``'s plan), plus
    LRN (:func:`lrn_f16emu`) and convolutions that write channel ``out_c0 ...`` of a concatenated tensor.  ``keep``: tensor
    names to return as float64 NCHW arrays, or ``("conv", name)`` for one convolution's own output channels."""
    def r16(t):
        return t.to(torch.float16).to(torch.float64)

    shapes = lowered["tensors"]
    blobs = {lowered["input"]: r16(torch.from_numpy(np.ascontiguousarray(x)).double())}
    snap = {}
    n = x.shape[0]
    with torch.no_grad():
        for op in lowered["ops"]:
            a = blobs[op["input"]]
            t = op["type"]
            if t == "conv":
                w = r16(torch.from_numpy(op["W"]).double()).permute(0, 3, 1, 2).contiguous()
                y = F.conv2d(a, w, None, stride=op["stride"], padding=op["pad"])
                y = y + torch.from_numpy(op["bias"]).double().view(1, -1, 1, 1)
                if op["residual"] is not None:
                    y = y + blobs[op["residual"]]
                if op["relu"]:
                    y = torch.relu(y)
                y = r16(y)
                if keep and ("conv", op["name"]) in keep:
                    snap[("conv", op["name"])] = y.numpy().copy()
                if "out_c0" in op:
                    c, h, w_ = shapes[op["output"]]
                    dst = blobs.setdefault(op["output"], torch.zeros((n, c, h, w_), dtype=torch.float64))
                    dst[:, op["out_c0"]:op["out_c0"] + op["cout"]] = y
                    continue
            elif t == "maxpool":
                y = _maxpool_caffe(a, op["k"], op["stride"], op["pad"], op["ceil_mode"])
            elif t == "avgpool":
                y = r16(a.mean(dim=(2, 3), keepdim=True).float().double())
            elif t == "lrn":
                y = lrn_f16emu(a, op["local_size"], op["alpha"], op["beta"], op["k"])
            elif t == "fc":
                W = r16(torch.from_numpy(op["W"]).double())
                flat = a.permute(0, 2, 3, 1).reshape(a.shape[0], -1)
                y = (flat @ W.t() + torch.from_numpy(op["bias"]).double()).float().double().view(a.shape[0], -1, 1, 1)
            elif t == "softmax":
                y = torch.softmax(a.float(), dim=1).double()
            else:
                raise ValueError(t)
            blobs[op["output"]] = y
    if keep:
        for k in keep:
            if not isinstance(k, tuple):
                snap[k] = blobs[k].numpy().copy()
    out = blobs[lowered["output"]]
    out = out.reshape(out.shape[0], -1).numpy()
    return (out, snap) if keep else out


def lrn_numpy(a: np.ndarray, n: int, alpha: float, beta: float, k: float) -> np.ndarray:
    h = (n - 1) // 2
    c = a.shape[1]
    sq = np.zeros((a.shape[0], c + 2 * h) + a.shape[2:], np.float64)
    sq[:, h:h + c] = a.astype(np.float64) ** 2
    s = np.zeros_like(a, dtype=np.float64)
    for ch in range(c):
        s[:, ch] = sq[:, ch:ch + n].sum(axis=1)
    return a * (k + alpha / n * s) ** (-beta)


def numpy_forward(net: dict, weights: Dict[str, dict], x: np.ndarray) -> np.ndarray:
    """The second witness: the raw layer list in float64 numpy."""
    blobs = {net["input"]: np.asarray(x, np.float64)}
    for L in net["layers"]:
        t, name = L["type"], L["name"]
        a = blobs[L["bottoms"][0]]
        if t == "Convolution":
            y = numpy_ops.conv2d(a, weights[name]["W"], weights[name]["b"] if L["bias_term"] else None, L["stride"], L["pad"])
        elif t == "ReLU":
            y = np.maximum(a, 0.0)
        elif t == "Pooling":
            if L["pool"] == "MAX":
                y = numpy_ops.maxpool(a, L["kernel_size"], L["stride"], L["pad"], L.get("ceil_mode", True))
            else:
                y = numpy_ops.avgpool_global(a)
        elif t == "LRN":
            y = lrn_numpy(a, L["local_size"], L["alpha"], L["beta"], L["k"])
        elif t == "Concat":
            y = np.concatenate([blobs[b] for b in L["bottoms"]], axis=1)
        elif t == "Dropout":
            y = a
        elif t == "InnerProduct":
            y = numpy_ops.inner_product(a, weights[name]["W"], weights[name]["b"] if L["bias_term"] else None)
        elif t == "Softmax":
            y = numpy_ops.softmax(a)
        else:
            raise ValueError(f"numpy witness: unsupported layer {t}")
        blobs[L["tops"][0]] = y
    out = blobs[net["layers"][-1]["tops"][0]]
    return out.reshape(out.shape[0], -1)


def inception_net(cin: int = 64, hw: int = 14, widths=(16, 32, 48, 96), reduce=(24, 16), lrn: Optional[dict] = None,
                  pool_proj: bool = True, name: str = "inception") -> dict:
    """A small inception module in the BVLC names: [LRN ->] 1x1 | 3x3 reduce -> 3x3 | 5x5 reduce -> 5x5 | pool -> pool proj,
    concatenated.  ``widths``: the four branch outputs (the last is the pool projection)."""
    L = []

    def conv(lname, bottom, nout, k, pad=0):
        L.append(dict(name=lname, type="Convolution", bottoms=[bottom], tops=[lname], num_output=nout, kernel_size=k, pad=pad,
                      stride=1, bias_term=True))
        L.append(dict(name=lname + "_relu", type="ReLU", bottoms=[lname], tops=[lname]))

    prev = "data"
    if lrn:
        L.append(dict(name="norm", type="LRN", bottoms=["data"], tops=["norm"], **lrn))
        prev = "norm"
    conv("b/1x1", prev, widths[0], 1)
    conv("b/3x3_reduce", prev, reduce[0], 1)
    conv("b/3x3", "b/3x3_reduce", widths[1], 3, 1)
    conv("b/5x5_reduce", prev, reduce[1], 1)
    conv("b/5x5", "b/5x5_reduce", widths[2], 5, 2)
    L.append(dict(name="b/pool", type="Pooling", bottoms=[prev], tops=["b/pool"], pool="MAX", kernel_size=3, stride=1, pad=1))
    conv("b/pool_proj", "b/pool", widths[3], 1)
    L.append(dict(name="b/output", type="Concat", bottoms=["b/1x1", "b/3x3", "b/5x5", "b/pool_proj"], tops=["b/output"], axis=1))
    return {"name": name, "input": "data", "input_dims": [1, cin, hw, hw], "layers": L}
