"""Grouped INT8 / FP8 convolutions for the CPU oracles (test infrastructure only).

``oracle/int8_forward.py`` and ``oracle/fp8_forward.py`` restate dense convolutions.  As for fp16 (``grouped_oracle.py``),
a grouped convolution reaches them as its dense block-diagonal expansion: the zero weights (int8 0, E4M3 code 0x00 = +0)
add exact zeros to the integer accumulator, to the exact FP8 accumulator A and to P = sum |Wq * q|, so the results are
the grouped convolution's, bit for bit.

  * :func:`dense_quantized`    quantized graph -> the same graph with every grouped op's ``Wq`` (and ``W``) expanded
  * :func:`conv_int8_grouped`  the exact integer accumulator of a grouped op, from ``F.conv2d(..., groups=g)``
  * :func:`conv_fp8_grouped`   (A, P) of a grouped FP8 op, from ``F.conv2d(..., groups=g)``

The last two are the direct grouped evaluation the expansion is checked against (tests/test_grouped_1byte_cpu.py).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle import fp8_forward as O8
from tests.grouped_oracle import dense_weight


def dense_quantized(lq: dict) -> dict:
    """-> a quantized graph whose grouped conv ops carry dense OHWI ``Wq`` / ``W`` [Cout, kh, kw, Cin] and groups = 1."""
    out = dict(lq)
    ops = []
    for op in lq["ops"]:
        if op["type"] == "conv" and op.get("groups", 1) != 1:
            g = op["groups"]
            op = dict(op, groups=1, W=dense_weight(np.asarray(op["W"]), g, axis=3))
            if "Wq" in op:
                op["Wq"] = dense_weight(op["Wq"], g, axis=3)
        ops.append(op)
    out["ops"] = ops
    return out


def conv_int8_grouped(qx: np.ndarray, op: dict) -> np.ndarray:
    """int8 values [N, Cin, H, W] -> exact accumulator int64 [N, Cout, Ho, Wo] of the grouped convolution ``op``."""
    w = torch.from_numpy(op["Wq"].astype(np.float64)).permute(0, 3, 1, 2).contiguous()
    y = F.conv2d(torch.from_numpy(qx.astype(np.float64)), w, None, stride=op["stride"], padding=op["pad"], groups=op["groups"])
    return np.rint(y.numpy()).astype(np.int64)


def conv_fp8_grouped(q: np.ndarray, op: dict):
    """E4M3 codes [N, Cin, H, W] -> (A, P) float64 of the grouped convolution ``op``."""
    w = torch.from_numpy(O8.value(op["Wq"]).astype(np.float64)).permute(0, 3, 1, 2).contiguous()
    a = torch.from_numpy(O8.value(q).astype(np.float64))
    kw = dict(stride=op["stride"], padding=op["pad"], groups=op["groups"])
    return F.conv2d(a, w, None, **kw).numpy(), F.conv2d(a.abs(), w.abs(), None, **kw).numpy()
