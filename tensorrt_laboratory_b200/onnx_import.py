"""ONNX graph import for CNN classifiers (SURVEY.md 8f N4: the on-disk model format in front of the hot path;
reference ``examples/ONNX/resnet50/build.py`` hands an ONNX ResNet-50 to ``trtexec --onnx``).

``import_onnx(model)`` turns a parsed ONNX graph (:func:`onnx_lite.parse_model`) into the same raw Caffe-style layer list
+ raw weights the prototxt front-end produces, so everything downstream (lowering / folding, plan builder, oracle) is
shared.  Supported operators -- the ones ONNX-zoo ResNets and the reference's MNIST model use:

  Conv (any group, dilation 1, symmetric pads or SAME_UPPER that resolves symmetric) / BatchNormalization / Relu /
  Add (two activations -> Eltwise SUM; activation + constant -> bias) / MaxPool (pads, ceil_mode) / AveragePool /
  GlobalAveragePool / Flatten / Reshape (activation flatten or constant reshape) / Gemm (alpha = beta = 1, transB 0|1) /
  MatMul / Softmax.

``export_onnx(net, weights)`` is the inverse for the layer lists of this repository (BatchNorm + Scale pairs merge into
one BatchNormalization): it exists so the importer can be round-trip tested without a third-party ONNX writer, and as a
way to hand a model built here to other ONNX consumers.  No ``onnx`` / ``protobuf`` dependency in either direction.
"""
from __future__ import annotations

import struct
from typing import Dict, List, Optional, Tuple

import numpy as np

from . import onnx_lite


# --------------------------------------------------------------------------------------------------
# import
# --------------------------------------------------------------------------------------------------
def import_onnx(model: dict, input_dims: Optional[List[int]] = None, name: str = "onnx-model") -> Tuple[dict, Dict[str, dict]]:
    """-> (net, weights) in the raw layer-list format of :mod:`graph` / :mod:`weights`.

    ``input_dims`` ([1, C, H, W]) is required unless the model's input value_info carries a static shape that
    :func:`onnx_lite.parse_model` recorded under ``model["input_shapes"]``."""
    inits: Dict[str, np.ndarray] = dict(model["initializers"])
    consts: Dict[str, np.ndarray] = {}
    layers: List[dict] = []
    weights: Dict[str, dict] = {}
    alias: Dict[str, str] = {}
    inp = model["inputs"][0]
    if input_dims is None:
        input_dims = (model.get("input_shapes") or {}).get(inp)
    if not input_dims or len(input_dims) != 4:
        raise ValueError("onnx import: a static [1, C, H, W] input shape is required")
    input_dims = [1] + [int(d) for d in input_dims[1:]]
    shapes: Dict[str, Tuple[int, int, int]] = {inp: tuple(input_dims[1:])}
    used = set()

    def res(n: str) -> str:
        while n in alias:
            n = alias[n]
        return n

    def const_of(n: str):
        return consts.get(n, inits.get(n))

    def uname(node, fallback):
        base = node["name"] or fallback
        n, k = base, 1
        while n in used:
            n, k = f"{base}_{k}", k + 1
        used.add(n)
        return n

    def last_writer(blob: str) -> dict:
        for L in reversed(layers):
            if L["tops"][0] == blob:
                return L
        raise ValueError(f"onnx import: no producer for {blob}")

    def conv_out(h, k, p0, p1, s):
        return (h + p0 + p1 - k) // s + 1

    for node in model["nodes"]:
        op, attrs = node["op"], node["attrs"]
        ins = [res(x) for x in node["inputs"]]
        out = node["outputs"][0]
        if op == "Constant":
            consts[out] = np.asarray(attrs["value"])
        elif op == "Conv":
            W = np.asarray(const_of(ins[1]), np.float32)
            if any(int(d) != 1 for d in attrs.get("dilations", [1, 1])):
                raise ValueError("onnx import: dilated Conv is not supported")
            group = int(attrs.get("group", 1))
            kh, kw = int(W.shape[2]), int(W.shape[3])
            st = [int(s) for s in attrs.get("strides", [1, 1])]
            c, h, w = shapes[ins[0]]
            if group < 1 or c % group or W.shape[0] % group or W.shape[1] != c // group:
                raise ValueError(f"onnx import: Conv {node['name'] or out}: weight {tuple(W.shape)} does not fit {c} input "
                                 f"channels in {group} groups")
            if attrs.get("auto_pad") in ("SAME_UPPER", "SAME_LOWER"):
                ph, pw = onnx_lite.same_upper_pads(h, kh, st[0]), onnx_lite.same_upper_pads(w, kw, st[1])
                pads = [ph[0], pw[0], ph[1], pw[1]]
            else:
                pads = [int(p) for p in attrs.get("pads", [0, 0, 0, 0])]
            if kh != kw or st[0] != st[1] or len(set(pads)) != 1:
                raise ValueError(f"onnx import: Conv {node['name'] or out} needs a square kernel, one stride and symmetric pads")
            lname = uname(node, out)
            bias = len(ins) > 2
            layers.append(dict(name=lname, type="Convolution", bottoms=[ins[0]], tops=[out], num_output=int(W.shape[0]),
                               kernel_size=kh, pad=pads[0], stride=st[0], bias_term=True))
            if group != 1:
                layers[-1]["group"] = group
            weights[lname] = {"W": W, "b": np.asarray(const_of(ins[2]), np.float32).reshape(-1) if bias else np.zeros(W.shape[0], np.float32)}
            shapes[out] = (int(W.shape[0]), conv_out(h, kh, pads[0], pads[2], st[0]), conv_out(w, kw, pads[1], pads[3], st[1]))
        elif op == "BatchNormalization":
            gamma, beta, mean, var = (np.asarray(const_of(x), np.float32) for x in ins[1:5])
            lname = uname(node, out)
            blob = ins[0]
            layers.append(dict(name=lname, type="BatchNorm", bottoms=[blob], tops=[blob], use_global_stats=True,
                               eps=float(attrs.get("epsilon", 1e-5))))
            weights[lname] = {"mean": mean, "var": var}
            layers.append(dict(name=lname + "_scale", type="Scale", bottoms=[blob], tops=[blob], bias_term=True))
            used.add(lname + "_scale")
            weights[lname + "_scale"] = {"gamma": gamma, "beta": beta}
            alias[out] = blob
        elif op == "Relu":
            layers.append(dict(name=uname(node, out), type="ReLU", bottoms=[ins[0]], tops=[ins[0]]))
            alias[out] = ins[0]
        elif op == "Add":
            a, b = ins
            ca, cb = const_of(a), const_of(b)
            if ca is None and cb is None:
                if shapes[a] != shapes[b]:
                    raise ValueError("onnx import: Add of differently shaped activations")
                layers.append(dict(name=uname(node, out), type="Eltwise", bottoms=[a, b], tops=[out], operation="SUM"))
                shapes[out] = shapes[a]
            else:  # bias of the producing Conv / MatMul
                act, cst = (b, ca) if ca is not None else (a, cb)
                target = last_writer(act)
                if target["type"] not in ("Convolution", "InnerProduct"):
                    raise ValueError("onnx import: constant Add must follow a Conv or MatMul")
                weights[target["name"]]["b"] = weights[target["name"]]["b"] + np.asarray(cst, np.float32).reshape(-1)
                alias[out] = act
        elif op in ("MaxPool", "AveragePool"):
            ks = [int(k) for k in attrs["kernel_shape"]]
            st = [int(s) for s in attrs.get("strides", [1, 1])]
            pads = [int(p) for p in attrs.get("pads", [0, 0, 0, 0])]
            if ks[0] != ks[1] or st[0] != st[1] or len(set(pads)) != 1:
                raise ValueError(f"onnx import: {op} needs a square window, one stride and symmetric pads")
            c, h, w = shapes[ins[0]]
            ceil_mode = bool(int(attrs.get("ceil_mode", 0)))
            layers.append(dict(name=uname(node, out), type="Pooling", bottoms=[ins[0]], tops=[out],
                               pool="MAX" if op == "MaxPool" else "AVE", kernel_size=ks[0], stride=st[0], pad=pads[0],
                               ceil_mode=ceil_mode))
            from .graph import pool_out_ceil
            shapes[out] = (c, pool_out_ceil(h, ks[0], pads[0], st[0], ceil_mode), pool_out_ceil(w, ks[0], pads[0], st[0], ceil_mode))
        elif op == "GlobalAveragePool":
            c, h, w = shapes[ins[0]]
            if h != w:
                raise ValueError("onnx import: GlobalAveragePool over a non-square plane")
            layers.append(dict(name=uname(node, out), type="Pooling", bottoms=[ins[0]], tops=[out], pool="AVE",
                               kernel_size=h, stride=1, pad=0))
            shapes[out] = (c, 1, 1)
        elif op in ("Flatten", "Reshape", "Squeeze", "Identity", "Dropout"):
            cst = const_of(ins[0])
            if cst is not None and op == "Reshape":
                shape = [int(x) for x in (const_of(ins[1]) if len(ins) > 1 else attrs["shape"])]
                consts[out] = np.asarray(cst).reshape(shape)
            else:
                alias[out] = ins[0]  # InnerProduct flattens (C, H, W) itself
        elif op in ("Gemm", "MatMul"):
            Wm = np.asarray(const_of(ins[1]), np.float32)
            if op == "Gemm":
                if float(attrs.get("alpha", 1.0)) != 1.0 or float(attrs.get("beta", 1.0)) != 1.0 or int(attrs.get("transA", 0)):
                    raise ValueError("onnx import: Gemm with alpha/beta != 1 or transA is not supported")
                if not int(attrs.get("transB", 0)):
                    Wm = Wm.T
            else:
                Wm = Wm.T  # MatMul: [K, N]
            lname = uname(node, out)
            bias = op == "Gemm" and len(ins) > 2
            layers.append(dict(name=lname, type="InnerProduct", bottoms=[ins[0]], tops=[out], num_output=int(Wm.shape[0]),
                               bias_term=True))
            weights[lname] = {"W": np.ascontiguousarray(Wm), "b": np.asarray(const_of(ins[2]), np.float32).reshape(-1) if bias
                              else np.zeros(Wm.shape[0], np.float32)}
            shapes[out] = (int(Wm.shape[0]), 1, 1)
        elif op == "Softmax":
            layers.append(dict(name=uname(node, out), type="Softmax", bottoms=[ins[0]], tops=[out]))
            shapes[out] = shapes[ins[0]]
        elif op == "Concat":
            if int(attrs.get("axis", 1)) != 1:
                raise ValueError(f"onnx import: Concat {node['name'] or out} along axis {attrs.get('axis')}; only channels (axis 1)")
            layers.append(dict(name=uname(node, out), type="Concat", bottoms=ins, tops=[out], axis=1))
            shapes[out] = (sum(shapes[x][0] for x in ins),) + shapes[ins[0]][1:]
        elif op == "LRN":
            size = int(attrs["size"])
            if size % 2 == 0:
                raise ValueError(f"onnx import: LRN {node['name'] or out}: even size {size} (the window is centred only for odd sizes)")
            layers.append(dict(name=uname(node, out), type="LRN", bottoms=[ins[0]], tops=[out], local_size=size,
                               alpha=float(attrs.get("alpha", 1e-4)), beta=float(attrs.get("beta", 0.75)), k=float(attrs.get("bias", 1.0))))
            shapes[out] = shapes[ins[0]]
        else:
            raise ValueError(f"onnx import: unsupported operator {op}")
    net = {"name": name, "input": inp, "input_dims": input_dims, "layers": layers}
    return net, weights


# --------------------------------------------------------------------------------------------------
# export (protobuf wire encoder, onnx.proto3 field numbers)
# --------------------------------------------------------------------------------------------------
def _vi(x: int) -> bytes:
    x &= (1 << 64) - 1
    out = bytearray()
    while True:
        b = x & 0x7F
        x >>= 7
        out.append(b | (0x80 if x else 0))
        if not x:
            return bytes(out)


def _f_varint(fno: int, v: int) -> bytes:
    return _vi(fno << 3) + _vi(v)


def _f_bytes(fno: int, v: bytes) -> bytes:
    return _vi((fno << 3) | 2) + _vi(len(v)) + v


def _tensor(name: str, arr: np.ndarray) -> bytes:
    arr = np.ascontiguousarray(arr)
    dt = {np.dtype(np.float32): 1, np.dtype(np.int64): 7}[arr.dtype]
    return b"".join(_f_varint(1, int(d)) for d in arr.shape) + _f_varint(2, dt) + _f_bytes(8, name.encode()) + _f_bytes(9, arr.tobytes())


def _attr(name: str, value) -> bytes:
    body = _f_bytes(1, name.encode())
    if isinstance(value, float):
        body += _vi((2 << 3) | 5) + struct.pack("<f", value) + _f_varint(20, 1)
    elif isinstance(value, int):
        body += _f_varint(3, value) + _f_varint(20, 2)
    elif isinstance(value, str):
        body += _f_bytes(4, value.encode()) + _f_varint(20, 3)
    else:  # list of ints
        body += b"".join(_f_varint(8, int(v)) for v in value) + _f_varint(20, 7)
    return body


def _node(op: str, inputs: List[str], outputs: List[str], name: str, **attrs) -> bytes:
    body = b"".join(_f_bytes(1, i.encode()) for i in inputs) + b"".join(_f_bytes(2, o.encode()) for o in outputs)
    body += _f_bytes(3, name.encode()) + _f_bytes(4, op.encode())
    body += b"".join(_f_bytes(5, _attr(k, v)) for k, v in attrs.items())
    return body


def _value_info(name: str, dims: List[int]) -> bytes:
    shape = b"".join(_f_bytes(1, _f_varint(1, int(d))) for d in dims)            # TensorShapeProto.dim{dim_value}
    tensor_type = _f_varint(1, 1) + _f_bytes(2, shape)                            # elem_type FLOAT, shape
    return _f_bytes(1, name.encode()) + _f_bytes(2, _f_bytes(1, tensor_type))     # TypeProto.tensor_type


def export_onnx(net: dict, weights: Dict[str, dict], opset: int = 11) -> bytes:
    """Serialize a raw layer list + raw weights as an ONNX ModelProto (BatchNorm+Scale pairs -> BatchNormalization)."""
    layers = net["layers"]
    nodes: List[bytes] = []
    inits: List[bytes] = []
    cur: Dict[str, str] = {}  # blob -> ONNX tensor currently holding it (in-place layers create new tensor names)
    counter = [0]

    def t(blob):
        return cur.get(blob, blob)

    def fresh(blob):
        counter[0] += 1
        cur[blob] = f"{blob}__{counter[0]}"
        return cur[blob]

    i = 0
    while i < len(layers):
        L = layers[i]
        ty, name = L["type"], L["name"]
        if ty == "Convolution":
            ins = [t(L["bottoms"][0]), name + "_W"]
            inits.append(_tensor(name + "_W", np.asarray(weights[name]["W"], np.float32)))
            if L["bias_term"]:
                ins.append(name + "_b")
                inits.append(_tensor(name + "_b", np.asarray(weights[name]["b"], np.float32)))
            k, p, s = L["kernel_size"], L["pad"], L["stride"]
            extra = {"group": L["group"]} if L.get("group", 1) != 1 else {}
            nodes.append(_node("Conv", ins, [fresh(L["tops"][0])], name, kernel_shape=[k, k], pads=[p, p, p, p], strides=[s, s],
                               **extra))
        elif ty == "BatchNorm":
            nxt = layers[i + 1] if i + 1 < len(layers) else None
            c = len(weights[name]["mean"])
            gamma, beta = np.ones(c, np.float32), np.zeros(c, np.float32)
            if nxt is not None and nxt["type"] == "Scale" and nxt["bottoms"][0] == L["bottoms"][0]:
                gamma = np.asarray(weights[nxt["name"]]["gamma"], np.float32)
                if nxt.get("bias_term"):
                    beta = np.asarray(weights[nxt["name"]]["beta"], np.float32)
                i += 1
            for suffix, arr in (("_gamma", gamma), ("_beta", beta), ("_mean", weights[name]["mean"]), ("_var", weights[name]["var"])):
                inits.append(_tensor(name + suffix, np.asarray(arr, np.float32)))
            src = t(L["bottoms"][0])
            nodes.append(_node("BatchNormalization", [src, name + "_gamma", name + "_beta", name + "_mean", name + "_var"],
                               [fresh(L["tops"][0])], name, epsilon=float(L.get("eps", 1e-5))))
        elif ty == "Scale":
            raise ValueError("export_onnx: a Scale layer that does not follow its BatchNorm")
        elif ty == "ReLU":
            src = t(L["bottoms"][0])
            nodes.append(_node("Relu", [src], [fresh(L["tops"][0])], name))
        elif ty == "Eltwise":
            a, b = (t(x) for x in L["bottoms"])
            nodes.append(_node("Add", [a, b], [fresh(L["tops"][0])], name))
        elif ty == "Pooling":
            k, p, s = L["kernel_size"], L["pad"], L["stride"]
            src = t(L["bottoms"][0])
            if L["pool"] == "AVE":
                nodes.append(_node("GlobalAveragePool", [src], [fresh(L["tops"][0])], name))
            else:
                nodes.append(_node("MaxPool", [src], [fresh(L["tops"][0])], name, kernel_shape=[k, k], pads=[p, p, p, p],
                                   strides=[s, s], ceil_mode=1 if L.get("ceil_mode", True) else 0))
        elif ty == "InnerProduct":
            src = t(L["bottoms"][0])
            flat = src + "__flat"
            nodes.append(_node("Flatten", [src], [flat], name + "_flatten", axis=1))
            inits.append(_tensor(name + "_W", np.asarray(weights[name]["W"], np.float32)))
            ins = [flat, name + "_W"]
            if L["bias_term"]:
                inits.append(_tensor(name + "_b", np.asarray(weights[name]["b"], np.float32)))
                ins.append(name + "_b")
            nodes.append(_node("Gemm", ins, [fresh(L["tops"][0])], name, alpha=1.0, beta=1.0, transB=1))
        elif ty == "Softmax":
            src = t(L["bottoms"][0])
            nodes.append(_node("Softmax", [src], [fresh(L["tops"][0])], name, axis=1))
        elif ty == "Concat":
            srcs = [t(b) for b in L["bottoms"]]
            nodes.append(_node("Concat", srcs, [fresh(L["tops"][0])], name, axis=1))
        elif ty == "LRN":
            src = t(L["bottoms"][0])
            nodes.append(_node("LRN", [src], [fresh(L["tops"][0])], name, size=int(L["local_size"]), alpha=float(L["alpha"]),
                               beta=float(L["beta"]), bias=float(L["k"])))
        elif ty == "Dropout":  # identity at inference
            cur[L["tops"][0]] = t(L["bottoms"][0])
        else:
            raise ValueError(f"export_onnx: unsupported layer type {ty}")
        i += 1
    out_blob = layers[-1]["tops"][0]
    graph = b"".join(_f_bytes(1, n) for n in nodes) + _f_bytes(2, net["name"].encode())
    graph += b"".join(_f_bytes(5, x) for x in inits)
    graph += _f_bytes(11, _value_info(net["input"], net["input_dims"]))
    graph += _f_bytes(12, _value_info(t(out_blob), []))
    opset_id = _f_bytes(1, b"") + _f_varint(2, opset)
    return _f_varint(1, 6) + _f_bytes(2, b"tensorrt_laboratory_b200") + _f_bytes(7, graph) + _f_bytes(8, opset_id)
