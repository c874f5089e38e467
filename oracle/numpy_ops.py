"""SECOND CPU ORACLE (test infrastructure only; never imported by the product package).

A plain-numpy restatement, written independently of ``caffe_forward.py`` (which leans on torch), of the operator
semantics the reference's MNIST golden vectors do NOT pin: BatchNorm(use_global_stats)+Scale (and their folding into the
preceding convolution), Caffe's ceil-mode MAX pooling with clipped windows, global AVE pooling, Eltwise SUM, Softmax --
plus a direct (loop over taps) convolution so whole small networks can be evaluated.  ``tests/test_oracle_second_witness.py``
checks the two oracles against each other; parity for these ops therefore rests on two witnesses, not one.

Semantics restated (Caffe, as consumed by the reference through ``models/ResNet-50-deploy.prototxt`` ->
``models/setup.py:53-55`` trtexec --deploy):
  * BatchNorm (use_global_stats: true):  y = (x - mean) / sqrt(var + eps)              (prototxt lines 22-33 et al.)
  * Scale (bias_term: true):             y = gamma * x + beta                          (prototxt lines 35-46)
  * Pooling MAX k/s/p: out = ceil((in + 2p - k) / s) + 1, minus one if the last window would start in the padding;
    windows are clipped to the image (-inf padding)                                   (prototxt lines 48-58: 3x3/2)
  * Pooling AVE, global 7x7: arithmetic mean over the window                          (prototxt lines 2292-2302)
  * Eltwise SUM, ReLU, InnerProduct, Softmax over channels.
  * GoogLeNet's LRN (ACROSS_CHANNELS):    y_c = x_c (k + alpha / n sum_{|j - c| <= (n - 1) / 2} x_j^2)^(-beta);
    Concat over channels; Dropout as the identity.
"""
from __future__ import annotations

import math

import numpy as np


def conv2d(x, w, b, stride, pad):
    """x [N,C,H,W], w [O,C,kh,kw] (float64 accumulate), zero padding, no dilation / groups."""
    n, c, h, wd = x.shape
    o, _, kh, kw = w.shape
    ho = (h + 2 * pad - kh) // stride + 1
    wo = (wd + 2 * pad - kw) // stride + 1
    xp = np.zeros((n, c, h + 2 * pad, wd + 2 * pad), np.float64)
    xp[:, :, pad:pad + h, pad:pad + wd] = x
    y = np.zeros((n, o, ho, wo), np.float64)
    for r in range(kh):
        for s in range(kw):
            patch = xp[:, :, r:r + (ho - 1) * stride + 1:stride, s:s + (wo - 1) * stride + 1:stride]  # [N,C,ho,wo]
            y += np.einsum("nchw,oc->nohw", patch, w[:, :, r, s].astype(np.float64))
    if b is not None:
        y += np.asarray(b, np.float64).reshape(1, -1, 1, 1)
    return y


def batchnorm(x, mean, var, eps=1e-5):
    return (x - mean.reshape(1, -1, 1, 1)) / np.sqrt(var.reshape(1, -1, 1, 1).astype(np.float64) + eps)


def scale(x, gamma, beta=None):
    y = x * gamma.reshape(1, -1, 1, 1)
    return y + beta.reshape(1, -1, 1, 1) if beta is not None else y


def fold_bn_scale(w, b, mean, var, gamma, beta, eps=1e-5):
    """conv -> BN -> Scale as ONE conv: W' = W * gamma / sqrt(var + eps), b' = (b - mean) * gamma / sqrt(var + eps) + beta."""
    k = gamma.astype(np.float64) / np.sqrt(var.astype(np.float64) + eps)
    b0 = np.zeros_like(mean, dtype=np.float64) if b is None else b.astype(np.float64)
    return w.astype(np.float64) * k.reshape(-1, 1, 1, 1), (b0 - mean) * k + (0.0 if beta is None else beta)


def pool_out_size(size, k, pad, stride, ceil_mode=True):
    if not ceil_mode:
        return (size + 2 * pad - k) // stride + 1
    out = int(math.ceil((size + 2 * pad - k) / float(stride))) + 1
    if pad > 0 and (out - 1) * stride >= size + pad:
        out -= 1
    return out


def maxpool(x, k, stride, pad, ceil_mode=True):
    n, c, h, w = x.shape
    ho, wo = pool_out_size(h, k, pad, stride, ceil_mode), pool_out_size(w, k, pad, stride, ceil_mode)
    y = np.full((n, c, ho, wo), -np.inf, np.float64)
    for p in range(ho):
        h0, h1 = max(p * stride - pad, 0), min(p * stride - pad + k, h)
        for q in range(wo):
            w0, w1 = max(q * stride - pad, 0), min(q * stride - pad + k, w)
            y[:, :, p, q] = x[:, :, h0:h1, w0:w1].max(axis=(2, 3))
    return y


def avgpool_global(x):
    return x.astype(np.float64).sum(axis=(2, 3), keepdims=True) / float(x.shape[2] * x.shape[3])


def lrn(x, n, alpha, beta, k):
    """Caffe ACROSS_CHANNELS LRN: the n-channel window zero-padded at the channel edges, the divisor always n."""
    h = (n - 1) // 2
    c = x.shape[1]
    sq = np.zeros((x.shape[0], c + 2 * h) + x.shape[2:], np.float64)
    sq[:, h:h + c] = x.astype(np.float64) ** 2
    s = np.zeros_like(x, dtype=np.float64)
    for ch in range(c):
        s[:, ch] = sq[:, ch:ch + n].sum(axis=1)
    return x * (k + alpha / n * s) ** (-beta)


def eltwise_sum(*xs):
    y = xs[0].astype(np.float64)
    for t in xs[1:]:
        y = y + t
    return y


def inner_product(x, w, b):
    y = x.reshape(x.shape[0], -1).astype(np.float64) @ w.astype(np.float64).T
    return (y + b if b is not None else y).reshape(x.shape[0], -1, 1, 1)


def softmax(x):
    z = x.reshape(x.shape[0], -1).astype(np.float64)
    z = z - z.max(axis=1, keepdims=True)
    e = np.exp(z)
    return (e / e.sum(axis=1, keepdims=True)).reshape(x.shape)


def forward(net: dict, weights: dict, x: np.ndarray):
    """The raw Caffe layer list, unfused, in float64 (same net / weights dictionaries as caffe_forward)."""
    blobs = {net["input"]: np.asarray(x, np.float64)}
    for L in net["layers"]:
        t, name = L["type"], L["name"]
        a = blobs[L["bottoms"][0]]
        if t == "Convolution":
            y = conv2d(a, weights[name]["W"], weights[name]["b"] if L["bias_term"] else None, L["stride"], L["pad"])
        elif t == "BatchNorm":
            y = batchnorm(a, weights[name]["mean"], weights[name]["var"], L.get("eps", 1e-5))
        elif t == "Scale":
            y = scale(a, weights[name]["gamma"], weights[name]["beta"] if L.get("bias_term") else None)
        elif t == "ReLU":
            y = np.maximum(a, 0.0)
        elif t == "Pooling":
            if L["pool"] == "MAX":
                y = maxpool(a, L["kernel_size"], L["stride"], L["pad"], L.get("ceil_mode", True))
            else:
                if L["kernel_size"] != a.shape[2] or a.shape[2] != a.shape[3] or L["pad"]:
                    raise ValueError("numpy oracle: only global AVE pooling is restated")
                y = avgpool_global(a)
        elif t == "LRN":
            y = lrn(a, L["local_size"], L["alpha"], L["beta"], L["k"])
        elif t == "Concat":
            y = np.concatenate([blobs[b] for b in L["bottoms"]], axis=1)
        elif t == "Dropout":
            y = a
        elif t == "Eltwise":
            y = eltwise_sum(a, *[blobs[b] for b in L["bottoms"][1:]])
        elif t == "InnerProduct":
            y = inner_product(a, weights[name]["W"], weights[name]["b"] if L["bias_term"] else None)
        elif t == "Softmax":
            y = softmax(a)
        else:
            raise ValueError(f"numpy oracle: unsupported layer {t}")
        blobs[L["tops"][0]] = y
    out = blobs[net["layers"][-1]["tops"][0]]
    return out.reshape(out.shape[0], -1)
