"""Grouped convolutions for the CPU oracles (test infrastructure only).

The oracles under ``oracle/`` restate dense convolutions.  A convolution with ``groups`` groups is the dense convolution
whose [Cout, Cin, kh, kw] weight is block-diagonal: output channel o of group g = o // (Cout/groups) carries its
[Cin/groups, kh, kw] weights at input channels g*Cin/groups ... (g+1)*Cin/groups - 1 and zeros everywhere else.  The
zeros add exact zeros to every sum, so the unmodified oracles evaluate a grouped network through these rewrites:

  * :func:`dense_net`      raw layer list + raw weights -> the same net without ``group``, weights expanded
  * :func:`dense_lowered`  lowered graph (OHWI weights [Cout, kh, kw, Cin/groups]) -> the same graph with dense weights

:func:`numpy_conv2d` is the independent second witness: ``numpy_ops.conv2d`` applied group by group to channel slices.
"""
from __future__ import annotations

import copy

import numpy as np

from oracle import numpy_ops


def dense_weight(W: np.ndarray, groups: int, axis: int = 1) -> np.ndarray:
    """Grouped weight -> dense block-diagonal weight.  ``axis``: the input-channel axis (1 for OIHW, 3 for OHWI)."""
    if groups == 1:
        return W
    cout, cg = W.shape[0], W.shape[axis]
    shape = list(W.shape)
    shape[axis] = cg * groups
    out = np.zeros(shape, W.dtype)
    per = cout // groups
    for g in range(groups):
        idx = [slice(g * per, (g + 1) * per)] + [slice(None)] * (W.ndim - 1)
        dst = list(idx)
        dst[axis] = slice(g * cg, (g + 1) * cg)
        out[tuple(dst)] = W[tuple(idx)]
    return out


def dense_net(net: dict, weights: dict):
    """-> (net, weights) with every grouped Convolution rewritten as its dense block-diagonal equivalent."""
    net2 = copy.deepcopy(net)
    w2 = dict(weights)
    for L in net2["layers"]:
        if L["type"] == "Convolution" and L.get("group", 1) != 1:
            w2[L["name"]] = dict(weights[L["name"]], W=dense_weight(np.asarray(weights[L["name"]]["W"]), L["group"]))
            del L["group"]
    return net2, w2


def dense_lowered(lowered: dict) -> dict:
    """-> a lowered graph whose grouped conv ops carry dense OHWI weights [Cout, kh, kw, Cin] and groups = 1."""
    low = dict(lowered)
    ops = []
    for op in lowered["ops"]:
        if op["type"] == "conv" and op.get("groups", 1) != 1:
            op = dict(op, W=dense_weight(op["W"], op["groups"], axis=3), groups=1)
        ops.append(op)
    low["ops"] = ops
    return low


def numpy_conv2d(x, w, b, stride, pad, groups=1):
    """x [N, C, H, W], w [O, C/groups, kh, kw] (float64), evaluated group by group with ``numpy_ops.conv2d``."""
    c, o = x.shape[1], w.shape[0]
    ci, co = c // groups, o // groups
    y = np.concatenate([numpy_ops.conv2d(x[:, g * ci:(g + 1) * ci], w[g * co:(g + 1) * co], None, stride, pad)
                        for g in range(groups)], axis=1)
    if b is not None:
        y += np.asarray(b, np.float64).reshape(1, -1, 1, 1)
    return y
