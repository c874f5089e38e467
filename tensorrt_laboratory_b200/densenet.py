"""DenseNet weights: a torchvision ``densenet{121,169,201}`` ``state_dict`` -> raw weights under the Caffe layer names of
:func:`graph.densenet_caffe`, so real ImageNet weights run without this project downloading anything.

Save the state dict as ``.npz`` (``np.savez(f, **{k: v.numpy() for k, v in model.state_dict().items()})``) and pass the
file or the loaded mapping to :func:`load_weights`; ``builder.build_densenet_plan(depth, weights=...)`` takes the result.
Seeded weights come from ``weights.random_weights(graph.densenet_caffe(depth))`` and ``.caffemodel`` files from
``caffemodel``.  torchvision's BatchNorm (eps 1e-5) becomes a Caffe BatchNorm (mean, var) and a Scale (gamma, beta).
"""
from __future__ import annotations

from typing import Dict, Union

import numpy as np

from . import graph


def _bn_pairs(depth: int):
    """(torchvision BatchNorm prefix, Caffe layer prefix) and (torchvision conv, Caffe conv) name pairs."""
    bns, convs = [("features.norm0", "conv1")], [("features.conv0", "conv1")]
    for b, n in enumerate(graph._DENSENET_BLOCKS[depth], 1):
        for l in range(1, n + 1):
            tv, cf = f"features.denseblock{b}.denselayer{l}", f"conv{b + 1}_{l}"
            bns += [(tv + ".norm1", cf + "/x1"), (tv + ".norm2", cf + "/x2")]
            convs += [(tv + ".conv1", cf + "/x1"), (tv + ".conv2", cf + "/x2")]
        if b < 4:
            bns.append((f"features.transition{b}.norm", f"conv{b + 1}_blk"))
            convs.append((f"features.transition{b}.conv", f"conv{b + 1}_blk"))
    bns.append(("features.norm5", "conv5_blk"))
    return bns, convs


def load_weights(npz: Union[str, Dict[str, np.ndarray]], depth: int = 121) -> dict:
    """Raw weights of :func:`graph.densenet_caffe(depth) <graph.densenet_caffe>` from a torchvision state dict (``.npz``
    path or mapping).  A missing key or a wrong shape raises ``KeyError`` / ``ValueError`` naming the key."""
    if depth not in graph._DENSENET_BLOCKS:
        raise ValueError(f"unsupported DenseNet depth {depth}")
    src = np.load(npz) if isinstance(npz, str) else npz
    net = graph.densenet_caffe(depth)
    layers = {L["name"]: L for L in net["layers"]}
    shapes = graph.infer_shapes(net)
    in_c = {L["name"]: shapes[L["bottoms"][0]][0] for L in net["layers"] if L["bottoms"][0] in shapes}
    in_c["conv1"] = 3

    def get(key, shape):
        if key not in src:
            raise KeyError(f"densenet{depth} weights: missing {key}")
        v = np.asarray(src[key], dtype=np.float32)
        if v.shape != tuple(shape):
            raise ValueError(f"densenet{depth} weights: {key} has shape {v.shape}, expected {tuple(shape)}")
        return v

    bns, convs = _bn_pairs(depth)
    out: dict = {}
    for tv, cf in convs:
        L = layers[cf]
        out[cf] = {"W": get(tv + ".weight", (L["num_output"], in_c[cf], L["kernel_size"], L["kernel_size"]))}
    for tv, cf in bns:
        c = in_c[cf + "/bn"]
        out[cf + "/bn"] = {"mean": get(tv + ".running_mean", (c,)), "var": get(tv + ".running_var", (c,))}
        out[cf + "/scale"] = {"gamma": get(tv + ".weight", (c,)), "beta": get(tv + ".bias", (c,))}
    c = in_c["fc6"]
    out["fc6"] = {"W": get("classifier.weight", (1000, c)), "b": get("classifier.bias", (1000,))}
    return out
