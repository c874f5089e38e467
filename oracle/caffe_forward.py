"""CPU ORACLE -- test infrastructure only.  Never imported by the product package.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs may import this module; it is the checker, never the thing measured as the product or shipped.

What it restates.  The reference (NVIDIA/tensorrt-laboratory) contains no arithmetic of its own for the
forward pass: ``ExecutionContext::Infer`` hands the bindings to closed-source TensorRT
(``trtlab/tensorrt/src/workspace.cc:47,52`` ``enqueueV2``; legacy contract
``examples/10_Internals/README.md:50-52``).  TensorRT 7.1 (``Dockerfile:6``
``nvcr.io/nvidia/tensorrt:20.06-py3``) is absent from /root/reference and cannot be run here, so the
oracle restates the PUBLISHED operator semantics of the model files the reference feeds it:

* Caffe deploy nets ``models/ResNet-{50,152}-deploy.prototxt`` (built by ``models/setup.py:53-55``):
  Convolution, BatchNorm(use_global_stats)+Scale, ReLU, Pooling (MAX/AVE, **ceil** output size),
  Eltwise SUM, InnerProduct, Softmax -- executed UNFUSED, layer by layer, in fp32 (or fp64).
* ONNX opset-8 MNIST ``models/onnx/mnist-v1.3/model.onnx`` (Conv SAME_UPPER, Add, Relu, MaxPool floor,
  Reshape, MatMul) -- expressed with the same layer vocabulary (``ceil_mode=False`` on its pools).
* The layers GoogLeNet, DenseNet and VGG add: grouped Convolution, LRN (ACROSS_CHANNELS), Concat, Dropout
  (the identity at inference), exact windowed AVE pooling, and InnerProduct weights stored 4-D.

Pinning: the MNIST path is pinned against the reference's in-tree golden vectors
(``models/onnx/mnist-v1.3/test_data_set_{0,1,2}``, tolerance ``decimal=3`` as in
``examples/30_PyTensorRT/server.py:31``) by ``tests/test_oracle.py``.  For ResNet-50/152 the reference
holds NO golden vector in-tree (its ResNet fixtures are a network download,
``examples/ONNX/resnet50/fetch.sh:3-9``): **parity unpinned** for those graphs beyond the operator
family that MNIST exercises (conv+bias, relu, maxpool, matmul+bias).

Inputs are fp32 NCHW, the reference's binding contract (``trtlab/tensorrt/src/bindings.cc:128-175``).
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F


def _pool_out(size, k, pad, stride, ceil_mode):
    if not ceil_mode:
        return (size + 2 * pad - k) // stride + 1
    out = int(math.ceil((size + 2 * pad - k) / stride)) + 1
    if pad > 0 and (out - 1) * stride >= size + pad:
        out -= 1
    return out


def _pool_pad_end(size, k, pad, stride, ceil_mode):
    """The right / bottom padding after which a floor-mode torch pool has Caffe's output size and clipped windows."""
    return max((_pool_out(size, k, pad, stride, ceil_mode) - 1) * stride + k - size - pad, 0)


def maxpool_caffe(a: torch.Tensor, k: int, s: int, p: int, ceil_mode: bool = True) -> torch.Tensor:
    """Caffe MAX pooling (NCHW, a's dtype): -inf padding, so windows are clipped to the image."""
    ph, pw = (_pool_pad_end(a.shape[d], k, p, s, ceil_mode) for d in (2, 3))
    return F.max_pool2d(F.pad(a, (p, pw, p, ph), value=float("-inf")), k, s)


def lrn_torch(a: torch.Tensor, n: int, alpha: float, beta: float, k: float) -> torch.Tensor:
    """Caffe ACROSS_CHANNELS LRN in a's dtype (NCHW): y_c = x_c (k + alpha / n sum_{|j - c| <= (n - 1) / 2} x_j^2)^(-beta),
    the window zero-padded at the channel edges and the divisor always n."""
    h = (n - 1) // 2
    sq = F.pad(a * a, (0, 0, 0, 0, h, h))
    s = sum(sq[:, d:d + a.shape[1]] for d in range(n))
    return a * torch.pow(k + alpha / n * s, -beta)


def caffe_forward(net: dict, weights: Dict[str, dict], x: np.ndarray, dtype=torch.float32,
                  keep: Optional[list] = None, threads: Optional[int] = None, logits: bool = False):
    """Run the raw layer list on ``x`` (N,C,H,W fp32).  Returns the last top (with ``logits``, the last InnerProduct's
    output) as a float64 [N, -1] ndarray; with ``keep=[blob names]`` returns (out, {blob: ndarray NCHW}) snapshot right
    after each blob's last in-place writer."""
    if threads:
        torch.set_num_threads(threads)

    def param(name, key):
        return torch.from_numpy(weights[name][key]).to(dtype)

    blobs = {net["input"]: torch.from_numpy(np.ascontiguousarray(x)).to(dtype)}
    snap = {}
    fc = None
    layers = net["layers"]
    last_writer = {}
    for i, L in enumerate(layers):
        last_writer[L["tops"][0]] = i
    with torch.no_grad():
        for i, L in enumerate(layers):
            t = L["type"]
            name = L["name"]
            a = blobs[L["bottoms"][0]]
            if t == "Convolution":
                b = param(name, "b") if L["bias_term"] else None
                y = F.conv2d(a, param(name, "W"), b, stride=L["stride"], padding=L["pad"], groups=L.get("group", 1))
            elif t == "BatchNorm":
                mean = param(name, "mean").view(1, -1, 1, 1)
                var = param(name, "var").view(1, -1, 1, 1)
                y = (a - mean) / torch.sqrt(var + L.get("eps", 1e-5))
            elif t == "Scale":
                y = a * param(name, "gamma").view(1, -1, 1, 1)
                if L.get("bias_term"):
                    y = y + param(name, "beta").view(1, -1, 1, 1)
            elif t == "ReLU":
                y = torch.relu(a)
            elif t == "Dropout":
                y = a
            elif t == "Pooling":
                k, s, p = L["kernel_size"], L["stride"], L["pad"]
                cm = L.get("ceil_mode", True)
                if L["pool"] == "MAX":
                    y = maxpool_caffe(a, k, s, p, cm)
                else:
                    if p or _pool_pad_end(a.shape[2], k, p, s, cm) or _pool_pad_end(a.shape[3], k, p, s, cm):
                        raise ValueError("oracle: only unpadded, exact AVE pooling is restated")
                    y = F.avg_pool2d(a, k, s)
            elif t == "LRN":
                y = lrn_torch(a, L["local_size"], L["alpha"], L["beta"], L["k"])
            elif t == "Concat":
                y = torch.cat([blobs[b] for b in L["bottoms"]], dim=1)
            elif t == "Eltwise":
                y = a
                for bname in L["bottoms"][1:]:
                    y = y + blobs[bname]
            elif t == "InnerProduct":
                w = param(name, "W")
                b = param(name, "b") if L["bias_term"] else None
                y = fc = F.linear(a.reshape(a.shape[0], -1), w.reshape(w.shape[0], -1), b).view(a.shape[0], -1, 1, 1)
            elif t == "Softmax":
                y = torch.softmax(a, dim=1)
            else:
                raise ValueError(f"oracle: unsupported layer {t}")
            blobs[L["tops"][0]] = y
            if keep and L["tops"][0] in keep and last_writer[L["tops"][0]] == i:
                snap[L["tops"][0]] = y.double().numpy().copy()
    out = fc if logits else blobs[layers[-1]["tops"][0]]
    out = out.reshape(out.shape[0], -1).double().numpy()
    return (out, snap) if keep else out


# ------------------------------------------------------------------------------------------------
# fp16-rounding emulation of the ENGINE's numerics plan (separates kernel bugs from rounding)
# ------------------------------------------------------------------------------------------------

def r16(t: torch.Tensor) -> torch.Tensor:
    """float64 values rounded to fp16, held in float64."""
    return t.to(torch.float16).to(torch.float64)


def lrn_f16emu(a: torch.Tensor, n: int, alpha: float, beta: float, k: float) -> torch.Tensor:
    """The engine's LRN (plan_format.h, OP_LRN) on fp16 values ``a`` (float64 NCHW holding fp16 numbers) -> float64
    holding fp16 numbers: squares summed in fp32 in channel order, scale = fmaf(fp32(alpha / n), sum, k),
    powf(scale, -beta) in fp32, the product in fp32, one fp16 rounding."""
    h = (n - 1) // 2
    x = a.to(torch.float32)
    sq = F.pad(x * x, (0, 0, 0, 0, h, h))            # exact squares of fp16 values
    s = torch.zeros_like(x)
    for d in range(n):                                # fp32 sum in channel order c - h ... c + h
        s = s + sq[:, d:d + x.shape[1]]
    alpha_n = np.float32(np.float32(alpha) / np.float32(n))
    scale = (float(alpha_n) * s.double() + float(np.float32(k))).to(torch.float32)   # one rounding (fmaf)
    y = x * torch.pow(scale, -float(np.float32(beta)))
    return r16(y)


def prologue_f32(a: torch.Tensor, scale: np.ndarray, shift: np.ndarray) -> torch.Tensor:
    """max(fmaf(x, scale, shift), 0) in fp32 on fp16 values a (float64 NCHW): x * scale is exact in float64, so one rounding
    of the float64 sum to fp32 is fmaf's."""
    s = torch.from_numpy(scale.astype(np.float32)).double().view(1, -1, 1, 1)
    t = torch.from_numpy(shift.astype(np.float32)).double().view(1, -1, 1, 1)
    return torch.relu((a * s + t).to(torch.float32).double())


def _conv_emu(op: dict, a: torch.Tensor, residual, rnd) -> torch.Tensor:
    """One lowered convolution on the values a of its input tensor: channels [0, cin), the BatchNorm + ReLU prologue's
    rounded operand when ``pre`` is set, rounded OHWI weights, exact products and sums, bias, residual, ReLU, one rounding."""
    if op.get("groups", 1) != 1:
        raise ValueError(f"f16 emulation: conv {op['name']} has {op['groups']} groups; evaluate its dense block-diagonal "
                         "equivalent (tests/grouped_oracle.dense_lowered) instead")
    a = a[:, :op["cin"]]
    if op.get("pre"):
        a = rnd(prologue_f32(a, op["pre_scale"], op["pre_shift"]))
    w = rnd(torch.from_numpy(op["W"]).double()).permute(0, 3, 1, 2).contiguous()  # OHWI->OIHW
    y = F.conv2d(a, w, None, stride=op["stride"], padding=op["pad"])
    y = y + torch.from_numpy(op["bias"]).double().view(1, -1, 1, 1)
    if residual is not None:
        y = y + residual
    if op["relu"]:
        y = torch.relu(y)
    return rnd(y)


def conv_pre_emu(op: dict, a: torch.Tensor) -> torch.Tensor:
    """A prologue 1x1 convolution on fp16 values a (channels [0, cin) of its input): the fp16 operand, fp16 weights, exact
    products and sum, bias, ReLU and one fp16 rounding."""
    return _conv_emu(op, a, None, r16)


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


def fc_ref(op: dict, x16: np.ndarray):
    """One streaming FC layer on fp16 values x16 ([N, K] in the op's (h, w, c) K order): (reference, sum |w| |x|), float64.
    The reference is exact on the fp16-rounded weights; bias and ReLU as the kernel applies them."""
    W = np.asarray(op["W"], np.float32).astype(np.float16).astype(np.float64)
    x = np.asarray(x16, np.float64)
    y = x @ W.T + np.asarray(op["bias"], np.float32).astype(np.float64)
    if op.get("relu"):
        y = np.maximum(y, 0.0)
    return y, np.abs(x) @ np.abs(W).T + np.abs(np.asarray(op["bias"], np.float64))


def lowered_forward_f16emu(lowered: dict, x: np.ndarray, keep: Optional[list] = None, round16: bool = True,
                           logits: bool = False):
    """Execute *lowered* ops (folded fp32 W in OHWI, bias) with the rounding points of the fp16 engine:

    input -> fp16; weights -> fp16; conv reads channels [0, cin) of its input (through the BatchNorm + ReLU prologue,
    :func:`prologue_f32` rounded to fp16, when ``pre`` is set), accumulates in fp32 (here fp64, i.e. exact) then
    ``+bias (+residual) -> relu -> fp16``; max-pool exact in fp16; global avg-pool fp32 sum / HW -> fp16, or
    :func:`avgpool_pre_ref` with a prologue; LRN :func:`lrn_f16emu`; FC fp16 weights, fp32 accumulate + fp32 bias (-> relu)
    -> fp32 logits, or fp16 for a hidden FC; softmax fp32.  An op with ``out_c0`` writes its channels
    ``out_c0 ...`` of a zero-initialised tensor.
    ``round16=False`` evaluates the same fused graph exactly (fp64): used to check BN/Scale folding.
    ``keep``: tensor names, returned as float64 NCHW arrays at the end of the run, or ``("conv", name)`` for one
    convolution's own output channels; returns (out, {key: ndarray}).  ``logits``: return the last FC's output.
    An op feature the emulation does not model raises ``ValueError``.
    """
    rnd = r16 if round16 else (lambda t: t)
    shapes = lowered["tensors"]
    n = x.shape[0]
    blobs = {lowered["input"]: rnd(torch.from_numpy(np.ascontiguousarray(x)).double())}
    snap = {}
    fc = None
    with torch.no_grad():
        for op in lowered["ops"]:
            a = blobs[op["input"]]
            t = op["type"]
            if t == "conv":
                y = _conv_emu(op, a, None if op["residual"] is None else blobs[op["residual"]], rnd)
                if keep and ("conv", op["name"]) in keep:
                    snap[("conv", op["name"])] = y.numpy().copy()
            elif t == "maxpool":
                y = maxpool_caffe(a, op["k"], op["stride"], op["pad"], op["ceil_mode"])
            elif t == "avgpool":
                if "pre_scale" in op:
                    y = avgpool_pre_ref(a, op["pre_scale"], op["pre_shift"], op["k"])
                elif a.shape[2] == a.shape[3] == op["k"]:
                    y = rnd(a.mean(dim=(2, 3), keepdim=True).float().double())
                else:
                    raise ValueError(f"f16 emulation: avgpool {op['name']} is windowed without a prologue")
            elif t == "lrn":
                y = lrn_f16emu(a, op["local_size"], op["alpha"], op["beta"], op["k"])
            elif t == "fc":
                W = rnd(torch.from_numpy(op["W"]).double())  # [out, (h,w,c)]
                flat = a.permute(0, 2, 3, 1).reshape(n, -1)
                y = (flat @ W.t() + torch.from_numpy(op["bias"].astype(np.float32)).double()).float().double()
                if op["relu"]:
                    y = torch.relu(y)
                y = fc = (rnd(y) if op["hidden"] else y).view(n, -1, 1, 1)
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
    for k in keep or ():
        if not isinstance(k, tuple):
            snap[k] = blobs[k].numpy().copy()
    out = fc if logits else blobs[lowered["output"]]
    out = out.reshape(n, -1).numpy()
    return (out, snap) if keep else out
