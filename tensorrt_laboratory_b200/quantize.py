"""INT8 post-training quantization of a lowered graph (the builder-side role of the reference's
``examples/ONNX/resnet50/int8.py:5-22`` + ``calibrator.py:61`` + ``build.py:63-65``: calibrate on a batch set, hand the
scales to the engine builder).

Scheme (what the INT8 kernels of this repository implement, bit for bit):
  * activations: symmetric per-tensor scale ``s = max|x| / 127`` from max-abs calibration over the calibration inputs;
  * weights: symmetric per-OUTPUT-CHANNEL scale ``s_w[c] = max|W[c]| / 127``, ``Wq = clip(rint(W / s_w), -127, 127)``;
  * convolution: ``acc = sum(q_in * Wq)`` exact in int32; epilogue in fp32, two fused multiply-adds (one rounding each)
        t = fma(float(acc), m[c], b[c])               m[c] = fl(s_in * s_w[c] / s_out),  b[c] = fl(bias[c] / s_out)
        t = fma(float(q_res), r, t)                   r = fl(s_res / s_out)                      (fused residual)
        t = max(t, 0)                                                                           (fused ReLU)
        q_out = clip(rint(t), -127, 127)              round-half-even
  * the thin-input stem convolution, the max pool behind it, the classifier (FC) and the softmax stay fp16: a
    ``quantize`` op ``q = clip(rint(fl(float(h) * fl(1/s))), -127, 127)`` sits between the fp16 part and the first INT8
    convolution; the global average pool reads INT8 and writes fp16: ``h = fp16(fl(float(sum q) * fl(s / HW)))``.

A convolution runs in INT8 when both its channel counts are multiples of 64 (all bottleneck convolutions of the ResNets).
With ``grouped=True`` a grouped convolution runs in INT8 / FP8 too, when Cin/g == Cout/g == cpg and cpg divides 128 or is a
multiple of 128 (``builder.grouped_1byte_span``: every grouped layer of ResNeXt-50 32x4d, ResNeXt-101 32x8d / 64x4d, and
depthwise layers); its weights are scaled per output channel over that channel's taps * cpg weights.

FP8 (``fmt="e4m3"``): the same split and the same layouts, with E4M3 codes (the ``e4m3fn`` format: no infinities,
subnormals kept, largest value 448) in place of int8 values.  ``e4m3()`` is round-to-nearest-even, saturating to +-448
(the ``satfinite`` conversion of the tensor-core epilogue):
  * activations: symmetric per-tensor scale ``s = fl32(max(amax, 1e-12) / 448)`` from max-abs calibration;
  * quantize op: ``q = e4m3(fl(float(h) * fl(1/s)))``;
  * weights: symmetric per-OUTPUT-CHANNEL scale ``s_w[c] = max|W[c]| / 448``, ``Wq = e4m3(clamp(fl32(W / s_w), +-448))``,
    stored as raw E4M3 bytes in the ``pack_weights_sw128_i8`` block layout;
  * convolution: ``acc = sum(Wq * q)`` on the tensor core with fp32 accumulators.  Every product is exact in fp32, but the
    order and width of the tensor core's internal accumulation belong to the hardware (Hopper's FP8 MMA keeps fewer bits
    than fp32 there), so the GPU result is not bit-reproducible on the CPU; the tests bound it from the exact sum instead;
  * epilogue: INT8's, except for the last step
        t = fma(acc, m[c], b[c])                      m[c] = fl(s_in * s_w[c] / s_out),  b[c] = fl(bias[c] / s_out)
        t = fma(float(q_res), r, t)                   r = fl(s_res / s_out)                      (fused residual)
        t = fmax(t, 0)                                                                          (fused ReLU)
        q_out = e4m3(t)                               padding output channels are code 0x00
    The max is taken under ReLU only: without it a NaN t stays NaN and becomes a NaN code (0x7F / 0xFF), with it
    fmax gives 0, as CUDA's fmaxf does in every fp16 epilogue.  The quantize op maps NaN to a NaN code and +-inf to
    +-448.  Measured on an H100: the e4m3 tensor-core MMA gives NaN for NaN x 0 and keeps subnormal operands, so a NaN
    input reaches every output whose window holds it (tests/test_gpu_fp8_values.py);
  * average pool: each code converted to fp32 and summed in fp32 in pixel order, ``h = fp16(fl(sum * fl(s / HW)))`` (the
    sum is exact for HW < 73: E4M3 values are multiples of 2^-9 and at most 448);
  * output cast of an FP8 tensor to an fp32 binding: ``y = fl(float(q) * s)``.

The calibration forward pass runs on the host (torch CPU, fp32) -- build-time work like the rest of this module, never
part of the request path.
"""
from __future__ import annotations

import copy
from typing import Dict, Optional

import numpy as np

from . import graph as G

QMAX = 127.0
E4M3_MAX = 448.0
FORMATS = {"int8": "INT8", "e4m3": "FP8"}


def e4m3(x: np.ndarray) -> np.ndarray:
    """float32 values -> E4M3 codes (uint8): round to nearest even, saturating to +-448.  torch's cast is round-to-nearest-
    even but turns values from 464 up into NaN, hence the clamp."""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).clamp(-E4M3_MAX, E4M3_MAX)
    return t.to(torch.float8_e4m3fn).view(torch.uint8).numpy()


def _is_int8_conv(op: dict) -> bool:
    return op["type"] == G.OP_CONV and op["cin"] % 64 == 0 and op["cout"] % 64 == 0


def calibrate(lowered: dict, calib_inputs: np.ndarray) -> Dict[str, float]:
    """max |x| of every tensor of the lowered (fused, folded) graph over ``calib_inputs`` [N, C, H, W], fp32 arithmetic."""
    import torch
    import torch.nn.functional as F

    from .graph import pool_out_ceil

    amax: Dict[str, float] = {}
    with torch.no_grad():
        blobs = {lowered["input"]: torch.from_numpy(np.ascontiguousarray(calib_inputs, dtype=np.float32))}
        amax[lowered["input"]] = float(blobs[lowered["input"]].abs().max())
        for op in lowered["ops"]:
            a = blobs[op["input"]]
            t = op["type"]
            if t == G.OP_CONV:
                w = torch.from_numpy(np.ascontiguousarray(op["W"], dtype=np.float32)).permute(0, 3, 1, 2).contiguous()
                y = F.conv2d(a, w, torch.from_numpy(np.asarray(op["bias"], dtype=np.float32)), stride=op["stride"], padding=op["pad"],
                             groups=op.get("groups", 1))
                if op["residual"] is not None:
                    y = y + blobs[op["residual"]]
                if op["relu"]:
                    y = torch.relu(y)
            elif t == G.OP_MAXPOOL:
                k, s, p = op["k"], op["stride"], op["pad"]
                ho = pool_out_ceil(a.shape[2], k, p, s) if op["ceil_mode"] else (a.shape[2] + 2 * p - k) // s + 1
                wo = pool_out_ceil(a.shape[3], k, p, s) if op["ceil_mode"] else (a.shape[3] + 2 * p - k) // s + 1
                need_h = (ho - 1) * s + k - a.shape[2] - p
                need_w = (wo - 1) * s + k - a.shape[3] - p
                y = F.max_pool2d(F.pad(a, (p, max(need_w, 0), p, max(need_h, 0)), value=float("-inf")), k, s)
            elif t == G.OP_AVGPOOL:
                y = a.mean(dim=(2, 3), keepdim=True)
            elif t == G.OP_FC:
                flat = a.permute(0, 2, 3, 1).reshape(a.shape[0], -1)
                y = (flat @ torch.from_numpy(np.asarray(op["W"], dtype=np.float32)).t() + torch.from_numpy(np.asarray(op["bias"], dtype=np.float32)))
                y = y.view(a.shape[0], -1, 1, 1)
            elif t == G.OP_SOFTMAX:
                y = torch.softmax(a, dim=1)
            else:
                raise ValueError(f"calibrate: unsupported op {t}")
            blobs[op["output"]] = y
            amax[op["output"]] = float(y.abs().max())
    return amax


def quantize_lowered(lowered: dict, calib_inputs: np.ndarray, amax: Optional[Dict[str, float]] = None,
                     fmt: str = "int8", grouped: bool = False) -> dict:
    """-> a lowered graph whose eligible convolutions carry INT8 parameters (``Wq`` int8 OHWI, ``m`` / ``b`` fp32 per
    output channel, ``r`` fp32 or None, ``in_scale`` / ``out_scale``), with ``quantize`` ops inserted where an INT8
    convolution reads an fp16 tensor, ``in_scale`` on an average pool that reads INT8, and ``tensor_scales`` {name: s}
    for every INT8 tensor.  ``lowered`` itself is not modified.  A graph with a grouped convolution is rejected before
    calibration unless ``grouped=True``; then every grouped convolution is quantized like a dense one, and one whose
    geometry the 1-byte kernels do not run (see above) is rejected before calibration instead.

    ``fmt="e4m3"``: the FP8 scheme above instead -- ``Wq`` holds E4M3 codes (uint8), and the graph and its quantized
    convolutions are marked ``fp8`` rather than ``int8``."""
    if fmt not in FORMATS:
        raise ValueError(f"fmt must be one of {sorted(FORMATS)}, not {fmt!r}")
    name = FORMATS[fmt]
    fp8 = fmt == "e4m3"
    qmax = E4M3_MAX if fp8 else QMAX
    from .builder import grouped_1byte_span
    for op in lowered["ops"]:
        if op["type"] == G.OP_FC and op.get("relu"):
            raise ValueError(f"fc {op['name']}: an InnerProduct with a fused ReLU builds in fp16 only; {name} hidden "
                             "fully-connected layers are not supported")
        if "out_c0" in op or op["type"] == G.OP_LRN:
            raise ValueError(f"{op['name']}: a graph with a Concat or LRN layer builds in fp16 only; {name} channel "
                             "concatenation and LRN are not supported")
    for op in lowered["ops"]:
        if op["type"] == G.OP_CONV and op.get("groups", 1) != 1:
            if not grouped:
                raise ValueError(f"conv {op['name']}: {name} grouped convolution is not supported ({op['groups']} groups); "
                                 "build this model in fp16 or fp32")
            if not grouped_1byte_span(op["cin"], op["cout"], op["groups"]):
                raise ValueError(f"conv {op['name']}: {name} grouped convolution needs Cin/g == Cout/g dividing 128 or a multiple "
                                 f"of 128 ({op['cin']} -> {op['cout']} channels, {op['groups']} groups); build this model in "
                                 "fp16 or fp32")
    amax = amax or calibrate(lowered, calib_inputs)
    q = copy.copy(lowered)
    q["tensors"] = dict(lowered["tensors"])
    q["fp8" if fp8 else "int8"] = True
    scales: Dict[str, float] = {}   # 1-byte tensors only
    ops = []
    alias: Dict[str, str] = {}      # fp16 tensor -> its quantized copy

    def scale_of(name: str) -> float:
        # scales are fp32 numbers (that is what the plan stores); everything derived from them starts from the rounded value
        return float(np.float32(max(amax[name], 1e-12) / qmax))

    for op in lowered["ops"]:
        op = dict(op)
        if _is_int8_conv(op) or (op["type"] == G.OP_CONV and op.get("groups", 1) != 1):  # grouped: admitted above
            src = op["input"]
            if src not in scales:  # produced by the fp16 part: quantize it once
                if src not in alias:
                    qn = src + "_q"
                    alias[src] = qn
                    q["tensors"][qn] = q["tensors"][src]
                    scales[qn] = scale_of(src)
                    ops.append(dict(type="quantize", name="quantize:" + src, input=src, output=qn, scale=scales[qn],
                                    inv_scale=np.float32(1.0 / scales[qn])))
                op["input"] = alias[src]
            if op["residual"] is not None:
                if op["residual"] not in scales:
                    raise ValueError(f"conv {op['name']}: the residual input of an {name} convolution must be an {name} tensor")
            s_in = scales[op["input"]]
            s_out = scale_of(op["output"])
            W = np.asarray(op["W"], dtype=np.float64)                      # [O, kh, kw, I]
            s_w = np.maximum(np.abs(W).reshape(W.shape[0], -1).max(axis=1), 1e-12) / qmax
            if fp8:
                op["Wq"] = e4m3(np.clip((W / s_w[:, None, None, None]).astype(np.float32), -E4M3_MAX, E4M3_MAX))
            else:
                op["Wq"] = np.clip(np.rint(W / s_w[:, None, None, None]), -QMAX, QMAX).astype(np.int8)
            op["m"] = (s_in * s_w / s_out).astype(np.float32)
            op["b"] = (np.asarray(op["bias"], dtype=np.float64) / s_out).astype(np.float32)
            op["r"] = np.float32(scales[op["residual"]] / s_out) if op["residual"] is not None else None
            op["in_scale"], op["out_scale"], op["w_scale"] = s_in, s_out, s_w
            op["fp8" if fp8 else "int8"] = True
            scales[op["output"]] = s_out
        else:
            for key in ("input", "residual"):
                if op.get(key) in scales and op["type"] != G.OP_AVGPOOL:
                    raise ValueError(f"{op['name']}: an fp16 operator reads the {name} tensor {op[key]}")
            if op["type"] == G.OP_AVGPOOL and op["input"] in scales:
                c, h, w = q["tensors"][op["input"]]
                op["in_scale"] = scales[op["input"]]
                op["k_scale"] = np.float32(scales[op["input"]] / float(h * w))
        ops.append(op)
    q["ops"] = ops
    q["tensor_scales"] = scales
    q["calib_amax"] = amax
    return q
