"""FP8 (E4M3) CPU ORACLE -- test infrastructure only.  Never imported by the product package.

The FP8 twin of ``int8_forward.py``: executes a graph quantized by ``quantize.quantize_lowered(..., fmt="e4m3")`` with the
explicit rounding steps of the scheme (quantize.py).  One step is not reproducible on the CPU: the tensor core sums the
exact E4M3 products with an accumulator whose internal width and order belong to the hardware.  So for every
convolution the oracle computes the EXACT accumulator ``A`` and the magnitude sum ``P = sum |Wq * q|``; a GPU result is
held to the codes the epilogue gives between ``A - eps * P`` and ``A + eps * P`` (tests/test_gpu_fp8.py), and the oracle
itself continues from the exact ``A``.

Rounding contract (every ``fl`` / ``fma`` is one IEEE fp32 operation, round-to-nearest-even; ``e4m3`` rounds to nearest
even and saturates to +-448):
    quantize   q = e4m3(fl(h * inv_s))                                           h: the fp16 value as fp32
    conv       t = fma(fl32(acc), m[c], b[c]);  t = fma(float(q_res), r, t);  t = fmax(t, 0);  q = e4m3(t)
               (fmax under ReLU only: it takes 0 for a NaN t, which without ReLU stays NaN and becomes a NaN code)
    avg pool   h = fp16(fl(sum * k)),  the values summed in fp32 in pixel order
    output     y = fl(float(q) * s)                                              (FP8 tensor exposed as fp32 binding)
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

from oracle.caffe_forward import _pool_out
from oracle.int8_forward import fma32

f32 = np.float32
E4M3_MAX = 448.0
# value of every code (0x7F / 0xFF are NaN); exact in fp32
E4M3_VALUES = torch.arange(256, dtype=torch.int32).to(torch.uint8).view(torch.float8_e4m3fn).float().numpy()


def e4m3(x: np.ndarray) -> np.ndarray:
    """fp32 values -> E4M3 codes (uint8): round to nearest even, saturating to +-448 (NaN stays NaN).  torch's cast rounds
    to nearest even but maps values from 464 up to NaN, so the clamp comes first."""
    t = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).clamp(-E4M3_MAX, E4M3_MAX)
    return t.to(torch.float8_e4m3fn).view(torch.uint8).numpy()


def value(codes: np.ndarray) -> np.ndarray:
    """E4M3 codes -> their fp32 values."""
    return E4M3_VALUES[np.asarray(codes, dtype=np.uint8)]


def conv_fp8(q: np.ndarray, op: dict, with_p: bool = True):
    """Codes [N, C, H, W] -> (A, P): the exact accumulator and sum |Wq * q|, float64 [N, Cout, Ho, Wo].  Exact: products are
    multiples of 2^-18 below 2^18, and K <= 2^13 of them stay below 2^31, so every partial sum fits float64's 53 bits."""
    w = torch.from_numpy(value(op["Wq"]).astype(np.float64)).permute(0, 3, 1, 2).contiguous()  # OHWI -> OIHW
    a = torch.from_numpy(value(q).astype(np.float64))
    A = F.conv2d(a, w, None, stride=op["stride"], padding=op["pad"]).numpy()
    P = F.conv2d(a.abs(), w.abs(), None, stride=op["stride"], padding=op["pad"]).numpy() if with_p else None
    return A, P


def requant(acc: np.ndarray, op: dict, res_q: Optional[np.ndarray]) -> np.ndarray:
    """Accumulator values [N, C, H, W] (rounded to fp32 first, as the fp32 accumulator holds them) -> E4M3 codes."""
    m = np.broadcast_to(op["m"].astype(f32).reshape(1, -1, 1, 1), acc.shape)
    b = np.broadcast_to(op["b"].astype(f32).reshape(1, -1, 1, 1), acc.shape)
    t = fma32(np.asarray(acc).astype(f32), m, b)
    if res_q is not None:
        t = fma32(value(res_q), np.broadcast_to(f32(op["r"]), acc.shape), t)
    if op["relu"]:
        t = np.fmax(t, f32(0))  # CUDA's fmaxf: NaN -> 0
    return e4m3(t)


def avgpool_fp8(q: np.ndarray, k_scale) -> np.ndarray:
    """Codes [N, C, H, W] -> fp16 values [N, C, 1, 1] as float64: fp32 sum in pixel order, times k, to fp16."""
    v = value(q).reshape(q.shape[0], q.shape[1], -1)
    s = np.zeros(v.shape[:2], f32)
    for i in range(v.shape[2]):
        s = (s + v[:, :, i]).astype(f32)
    return (s * f32(k_scale)).astype(f32).astype(np.float16).astype(np.float64)[:, :, None, None]


def fp8_forward(lowered_q: dict, x: np.ndarray, keep: Optional[list] = None, start_from: Optional[Dict[str, np.ndarray]] = None):
    """Run the FP8 graph on ``x`` [N, C, H, W], each convolution from its exact accumulator.  fp16 parts follow the fp16
    engine's numerics plan (as ``int8_forward``).  ``start_from`` {tensor: values}: take these tensors as given (fp16
    values, or E4M3 codes for FP8 tensors) and skip the ops that produce them.  Returns (out [N, -1] float64, {tensor:
    ndarray}) -- FP8 tensors as uint8 code arrays."""
    def r16(t):
        return t.to(torch.float16).to(torch.float64)

    scales = lowered_q["tensor_scales"]
    blobs: Dict[str, object] = {lowered_q["input"]: r16(torch.from_numpy(np.ascontiguousarray(x)).double())}
    given = dict(start_from or {})
    for k, v in given.items():
        blobs[k] = np.asarray(v).astype(np.uint8) if k in scales else torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64))
    snap = {}
    with torch.no_grad():
        for op in lowered_q["ops"]:
            if op["output"] in given:
                continue
            t = op["type"]
            a = blobs[op["input"]]
            if t == "quantize":
                h = a.numpy().astype(f32)                      # exact: fp16 values
                y = e4m3(h * f32(op["inv_scale"]))
            elif t == "conv" and op.get("fp8"):
                res = blobs[op["residual"]] if op["residual"] is not None else None
                y = requant(conv_fp8(a, op, with_p=False)[0], op, res)
            elif t == "conv":
                w = r16(torch.from_numpy(op["W"]).double()).permute(0, 3, 1, 2).contiguous()
                y = F.conv2d(a, w, None, stride=op["stride"], padding=op["pad"])
                y = y + torch.from_numpy(op["bias"]).double().view(1, -1, 1, 1)
                if op["residual"] is not None:
                    y = y + blobs[op["residual"]]
                if op["relu"]:
                    y = torch.relu(y)
                y = r16(y)
            elif t == "maxpool":
                k, s, p = op["k"], op["stride"], op["pad"]
                ho = _pool_out(a.shape[2], k, p, s, op["ceil_mode"])
                wo = _pool_out(a.shape[3], k, p, s, op["ceil_mode"])
                need_h = (ho - 1) * s + k - a.shape[2] - p
                need_w = (wo - 1) * s + k - a.shape[3] - p
                y = F.max_pool2d(F.pad(a, (p, max(need_w, 0), p, max(need_h, 0)), value=float("-inf")), k, s)
            elif t == "avgpool":
                if "k_scale" in op:  # FP8 in, fp16 out
                    y = torch.from_numpy(avgpool_fp8(a, op["k_scale"]))
                else:
                    y = r16(a.mean(dim=(2, 3), keepdim=True).float().double())
            elif t == "fc":
                W = r16(torch.from_numpy(op["W"]).double())
                flat = a.permute(0, 2, 3, 1).reshape(a.shape[0], -1)
                y = (flat @ W.t() + torch.from_numpy(op["bias"]).double()).float().double().view(a.shape[0], -1, 1, 1)
            elif t == "softmax":
                y = torch.softmax(a.float(), dim=1).double()
            else:
                raise ValueError(f"fp8 oracle: unsupported op {t}")
            blobs[op["output"]] = y
            if keep and op["output"] in keep:
                snap[op["output"]] = y.copy() if isinstance(y, np.ndarray) else y.numpy().copy()
    out = blobs[lowered_q["output"]]
    if isinstance(out, np.ndarray):  # FP8 graph output: dequantised the way the output cast does
        out = (value(out) * f32(scales[lowered_q["output"]])).astype(f32).astype(np.float64)
    else:
        out = out.numpy()
    out = out.reshape(out.shape[0], -1)
    return (out, snap) if keep is not None else out
