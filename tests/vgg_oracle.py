"""VGG for the CPU oracles (test infrastructure only).

* :func:`caffe_forward`          the raw Caffe layer list in torch float64, Dropout as the identity
* :func:`lowered_forward_f16emu` the lowered ops with the fp16 engine's rounding points: every op output rounded to fp16,
                                 hidden FC outputs (bias, then ReLU, in fp32) rounded once to fp16, the logits to fp32
* :func:`fc_ref`                 one streaming FC layer (plan_format.h, kFcStream): the float64 product of the fp16-rounded
                                 operands, bias, ReLU, and the scale sum |w| |x| of its fp32 accumulation error
* :func:`fc_net`                 a network of one or two InnerProduct layers on a [C, H, W] input, for per-op tests
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from tests.googlenet_oracle import _maxpool_caffe


def _r16(t):
    return t.to(torch.float16).to(torch.float64)


def caffe_forward(net: dict, weights: Dict[str, dict], x: np.ndarray) -> np.ndarray:
    """The raw layer list on x (N, C, H, W) in float64; returns the last top as [N, -1]."""
    blobs = {net["input"]: torch.from_numpy(np.ascontiguousarray(x)).double()}
    with torch.no_grad():
        for L in net["layers"]:
            t, name = L["type"], L["name"]
            a = blobs[L["bottoms"][0]]
            p = weights.get(name, {})
            if t == "Convolution":
                b = torch.from_numpy(np.asarray(p["b"])).double() if L["bias_term"] else None
                y = F.conv2d(a, torch.from_numpy(np.asarray(p["W"])).double(), b, stride=L["stride"], padding=L["pad"])
            elif t == "ReLU":
                y = torch.relu(a)
            elif t == "Dropout":
                y = a
            elif t == "Pooling":
                if L["pool"] != "MAX":
                    raise ValueError(f"oracle: {name}: only MAX pooling")
                y = _maxpool_caffe(a, L["kernel_size"], L["stride"], L["pad"], L.get("ceil_mode", True))
            elif t == "InnerProduct":
                b = torch.from_numpy(np.asarray(p["b"])).double() if L["bias_term"] else None
                y = F.linear(a.reshape(a.shape[0], -1), torch.from_numpy(np.asarray(p["W"])).double().reshape(L["num_output"], -1), b)
                y = y.view(a.shape[0], -1, 1, 1)
            elif t == "Softmax":
                y = torch.softmax(a, dim=1)
            else:
                raise ValueError(f"oracle: unsupported layer {t}")
            blobs[L["tops"][0]] = y
    out = blobs[net["layers"][-1]["tops"][0]]
    return out.reshape(out.shape[0], -1).numpy()


def lowered_forward_f16emu(lowered: dict, x: np.ndarray) -> np.ndarray:
    """The lowered VGG ops with the fp16 engine's rounding points; returns the output as [N, -1].  Products and sums are
    exact (float64), so the emulation differs from the engine only by fp32 accumulation order."""
    n = x.shape[0]
    blobs = {lowered["input"]: _r16(torch.from_numpy(np.ascontiguousarray(x)).double())}
    with torch.no_grad():
        for op in lowered["ops"]:
            a = blobs[op["input"]]
            t = op["type"]
            if t == "conv":
                w = _r16(torch.from_numpy(op["W"]).double()).permute(0, 3, 1, 2).contiguous()
                y = F.conv2d(a, w, None, stride=op["stride"], padding=op["pad"]) + torch.from_numpy(op["bias"]).double().view(1, -1, 1, 1)
                y = _r16(torch.relu(y) if op["relu"] else y)
            elif t == "maxpool":
                y = _maxpool_caffe(a, op["k"], op["stride"], op["pad"], op["ceil_mode"])
            elif t == "fc":
                W = _r16(torch.from_numpy(op["W"]).double())
                flat = a.permute(0, 2, 3, 1).reshape(n, -1)
                y = (flat @ W.t() + torch.from_numpy(op["bias"].astype(np.float32)).double()).float().double()
                if op.get("relu"):
                    y = torch.relu(y)
                y = (_r16(y) if op.get("hidden") else y).view(n, -1, 1, 1)
            elif t == "softmax":
                y = torch.softmax(a.float(), dim=1).double()
            else:
                raise ValueError(t)
            blobs[op["output"]] = y
    return blobs[lowered["output"]].reshape(n, -1).numpy()


def fc_ref(op: dict, x16: np.ndarray):
    """One streaming FC layer on fp16 values x16 ([N, K] in the op's (h, w, c) K order): (reference, sum |w| |x|), float64.
    The reference is exact on the fp16-rounded weights; bias and ReLU as the kernel applies them."""
    W = np.asarray(op["W"], np.float32).astype(np.float16).astype(np.float64)
    x = np.asarray(x16, np.float64)
    y = x @ W.T + np.asarray(op["bias"], np.float32).astype(np.float64)
    if op.get("relu"):
        y = np.maximum(y, 0.0)
    return y, np.abs(x) @ np.abs(W).T + np.abs(np.asarray(op["bias"], np.float64))


def fc_net(chw: Sequence[int], couts: Sequence[int], relus: Sequence[bool], name: Optional[str] = None) -> dict:
    """data [C, H, W] -> fc1 (-> relu1) [-> fc2 (-> relu2)]: one or two InnerProduct layers, no softmax, so every FC output
    can be bound."""
    L, prev = [], "data"
    for i, (c, r) in enumerate(zip(couts, relus), 1):
        L.append(dict(name=f"fc{i}", type="InnerProduct", bottoms=[prev], tops=[f"fc{i}"], num_output=c, bias_term=True))
        if r:
            L.append(dict(name=f"relu{i}", type="ReLU", bottoms=[f"fc{i}"], tops=[f"fc{i}"]))
        prev = f"fc{i}"
    tag = "_".join(f"{c}{'r' if r else ''}" for c, r in zip(couts, relus))
    return {"name": name or f"fc_{'x'.join(map(str, chw))}_{tag}", "input": "data", "input_dims": [1, *chw], "layers": L}
