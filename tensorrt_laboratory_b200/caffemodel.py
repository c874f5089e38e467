"""Caffe ``.caffemodel`` reader / writer (the real-weights half of the prototxt front end, SURVEY.md 8f N4).

The reference builds its Caffe engines with ``trtexec --deploy=<prototxt>`` (``models/setup.py:53-55``) and, for real
weights, ``--model=<caffemodel>``; the weights file is a binary ``caffe.NetParameter`` protobuf.  Only the fields that carry
learned parameters are needed, so the wire format is decoded by hand (no protobuf / caffe dependency):

    NetParameter    .name = 1 (string), .layer = 100 (repeated LayerParameter)          [V1: .layers = 2 is not supported]
    LayerParameter  .name = 1, .type = 2, .blobs = 7 (repeated BlobProto)
    BlobProto       .shape = 7 (BlobShape{ .dim = 1, packed int64 }), .data = 5 (packed float),
                    legacy .num/.channels/.height/.width = 1..4

Blob conventions restated from Caffe's layers:
    Convolution / InnerProduct   blobs[0] = weights [Cout, Cin/group, kh, kw] / [Cout, K], blobs[1] = bias (if bias_term)
    BatchNorm                    blobs[0] = mean * f, blobs[1] = variance * f, blobs[2] = [f]  (moving-average factor;
                                 the statistics are blobs / f, and 0 when f == 0)
    Scale                        blobs[0] = gamma, blobs[1] = beta (if bias_term)

``load_caffemodel`` returns the ``{layer name: {W, b} | {mean, var} | {gamma, beta}}`` dictionary that ``graph.lower`` and the
oracle consume (the layout of :func:`weights.random_weights`); ``save_caffemodel`` writes the same conventions (used by the
round-trip test and to hand synthetic weights to other tools).
"""
from __future__ import annotations

import struct
from typing import Dict, List

import numpy as np

from .graph import infer_shapes
from .onnx_lite import _fields, _packed_varints


def _blob(buf: bytes) -> np.ndarray:
    dims: List[int] = []
    legacy = {}
    data = None
    for field, wt, v in _fields(buf):
        if field == 7 and wt == 2:  # BlobShape
            for f2, w2, v2 in _fields(v):
                if f2 == 1:
                    dims += _packed_varints(v2) if w2 == 2 else [v2]
        elif field == 5:
            if wt == 2:
                data = np.frombuffer(v, dtype="<f4").copy() if data is None else np.concatenate([data, np.frombuffer(v, dtype="<f4")])
            elif wt == 5:
                val = np.frombuffer(struct.pack("<I", v), dtype="<f4")
                data = val.copy() if data is None else np.concatenate([data, val])
        elif field in (1, 2, 3, 4) and wt == 0:
            legacy[field] = v
        elif field == 8:
            raise ValueError("caffemodel: double-precision blobs (BlobProto.double_data) are not supported")
    if data is None:
        data = np.zeros(0, np.float32)
    if not dims and legacy:
        dims = [legacy.get(i, 1) for i in (1, 2, 3, 4)]
    if dims and int(np.prod(dims)) == data.size:
        data = data.reshape(dims)
    return data.astype(np.float32)


def read_layers(buf: bytes) -> List[dict]:
    """-> [{name, type, blobs: [ndarray]}] in file order.  A truncated or corrupt file is a ValueError, whatever the
    low-level symptom (a varint running off the end, a length past the buffer, bytes that are not UTF-8 ...)."""
    try:
        return _read_layers(buf)
    except ValueError:
        raise
    except (IndexError, struct.error, OverflowError, MemoryError) as ex:
        raise ValueError(f"caffemodel: truncated or corrupt NetParameter ({type(ex).__name__}: {ex})") from ex


def _read_layers(buf: bytes) -> List[dict]:
    layers = []
    for field, wt, v in _fields(buf):
        if field == 2 and wt == 2:
            raise ValueError("caffemodel: V1 layer format (NetParameter.layers) is not supported; upgrade with upgrade_net_proto_binary")
        if field != 100 or wt != 2:
            continue
        rec = {"name": "", "type": "", "blobs": []}
        for f2, w2, v2 in _fields(v):
            if f2 == 1 and w2 == 2:
                rec["name"] = bytes(v2).decode()
            elif f2 == 2 and w2 == 2:
                rec["type"] = bytes(v2).decode()
            elif f2 == 7 and w2 == 2:
                rec["blobs"].append(_blob(v2))
        layers.append(rec)
    return layers


def load_caffemodel(path_or_bytes, net: dict) -> Dict[str, dict]:
    """Weights of ``net`` (a parsed deploy prototxt / generated layer list) from a .caffemodel; checks every shape."""
    buf = path_or_bytes if isinstance(path_or_bytes, (bytes, bytearray)) else open(path_or_bytes, "rb").read()
    by_name = {L["name"]: L for L in read_layers(bytes(buf))}
    out: Dict[str, dict] = {}
    for L in net["layers"]:
        t, name = L["type"], L["name"]
        if t not in ("Convolution", "InnerProduct", "BatchNorm", "Scale"):
            continue
        if name not in by_name:
            raise ValueError(f"caffemodel has no layer {name!r}")
        blobs = by_name[name]["blobs"]
        if t in ("Convolution", "InnerProduct"):
            need = 2 if L.get("bias_term", True) else 1
            if len(blobs) < need:
                raise ValueError(f"{name}: expected {need} blobs, found {len(blobs)}")
            W = blobs[0]
            if W.shape[0] != L["num_output"]:
                raise ValueError(f"{name}: weight blob {W.shape} does not match num_output {L['num_output']}")
            if t == "InnerProduct":
                W = W.reshape(L["num_output"], -1)
            elif W.ndim != 4 or W.shape[2] != L["kernel_size"] or W.shape[3] != L["kernel_size"]:
                raise ValueError(f"{name}: weight blob {W.shape} does not match kernel_size {L['kernel_size']}")
            elif L.get("group", 1) != 1:  # a grouped blob is [Cout, Cin/group, k, k]
                cin = infer_shapes(net)[L["bottoms"][0]][0]
                if W.shape[1] * L["group"] != cin:
                    raise ValueError(f"{name}: weight blob {W.shape} does not match {cin} input channels in {L['group']} groups")
            rec = {"W": np.ascontiguousarray(W, np.float32)}
            if need == 2:
                rec["b"] = blobs[1].reshape(-1).astype(np.float32)
            out[name] = rec
        elif t == "BatchNorm":
            if len(blobs) < 3:
                raise ValueError(f"{name}: BatchNorm needs mean, variance and the moving-average factor")
            f = float(blobs[2].reshape(-1)[0])
            k = 0.0 if f == 0.0 else 1.0 / f
            out[name] = {"mean": (blobs[0].reshape(-1) * k).astype(np.float32), "var": (blobs[1].reshape(-1) * k).astype(np.float32)}
        else:  # Scale
            rec = {"gamma": blobs[0].reshape(-1).astype(np.float32)}
            if L.get("bias_term"):
                if len(blobs) < 2:
                    raise ValueError(f"{name}: Scale with bias_term needs two blobs")
                rec["beta"] = blobs[1].reshape(-1).astype(np.float32)
            out[name] = rec
    return out


# ---- writer ------------------------------------------------------------------------------------------------------
def _vi(x: int) -> bytes:
    out = bytearray()
    while True:
        b = x & 0x7F
        x >>= 7
        out.append(b | (0x80 if x else 0))
        if not x:
            return bytes(out)


def _ld(field: int, payload: bytes) -> bytes:
    return _vi((field << 3) | 2) + _vi(len(payload)) + payload


def _blob_bytes(a: np.ndarray) -> bytes:
    a = np.ascontiguousarray(a, dtype="<f4")
    shape = _ld(1, b"".join(_vi(int(d)) for d in a.shape))
    return _ld(7, shape) + _ld(5, a.tobytes())


def save_caffemodel(net: dict, weights: Dict[str, dict], bn_factor: float = 1.0) -> bytes:
    """Serialize ``weights`` for ``net`` with Caffe's blob conventions (BatchNorm statistics scaled by ``bn_factor``)."""
    out = bytearray(_ld(1, net.get("name", "net").encode()))
    for L in net["layers"]:
        t, name = L["type"], L["name"]
        blobs: List[np.ndarray] = []
        w = weights.get(name)
        if t == "Convolution":
            blobs = [w["W"]] + ([w["b"]] if L.get("bias_term", True) else [])
        elif t == "InnerProduct":
            blobs = [w["W"].reshape(L["num_output"], -1)] + ([w["b"]] if L.get("bias_term", True) else [])
        elif t == "BatchNorm":
            blobs = [w["mean"] * bn_factor, w["var"] * bn_factor, np.array([bn_factor], np.float32)]
        elif t == "Scale":
            blobs = [w["gamma"]] + ([w["beta"]] if L.get("bias_term") else [])
        body = _ld(1, name.encode()) + _ld(2, t.encode()) + b"".join(_ld(7, _blob_bytes(b)) for b in blobs)
        out += _ld(100, body)
    return bytes(out)
