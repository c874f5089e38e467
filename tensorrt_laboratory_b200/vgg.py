"""VGG weights: a torchvision ``vgg16`` / ``vgg19`` ``state_dict`` -> raw weights under the Caffe layer names of
:func:`graph.vgg_caffe`, so real ImageNet weights run without this project downloading anything.

Save the state dict as ``.npz`` (``np.savez(f, **{k: v.numpy() for k, v in model.state_dict().items()})``) and pass the
file or the loaded mapping to :func:`load_weights`; ``builder.build_vgg_plan(depth, weights=...)`` takes the result.
Seeded weights come from ``weights.random_weights(graph.vgg_caffe(depth))`` and ``VGG_ILSVRC_{16,19}_layers.caffemodel``
files from ``caffemodel``.

torchvision's ``features.{i}`` convolutions map in order onto ``conv{b}_{l}`` and ``classifier.{0,3,6}`` onto ``fc6``,
``fc7`` and ``fc8``.  Between the features and the classifier torchvision has an ``AdaptiveAvgPool2d((7, 7))``: at a
224 x 224 input pool5 is already 7 x 7, so that pool is the identity and the Caffe net (which has none) computes the same
function.  At any other input size it is not, so the loader refuses other sizes.
"""
from __future__ import annotations

from typing import Dict, Union

import numpy as np

from . import graph


def load_weights(npz: Union[str, Dict[str, np.ndarray]], depth: int = 16, image: int = 224) -> dict:
    """Raw weights of :func:`graph.vgg_caffe(depth) <graph.vgg_caffe>` from a torchvision state dict (``.npz`` path or
    mapping).  ``image`` is the input size the weights will run at; only 224 keeps torchvision's adaptive 7 x 7 pool the
    identity.  A missing key or a wrong shape raises ``KeyError`` / ``ValueError`` naming the key."""
    if depth not in graph._VGG_BLOCKS:
        raise ValueError(f"unsupported VGG depth {depth} (16 or 19)")
    if image != 224:
        raise ValueError(f"VGG weights from torchvision run at 224 x 224 only: at {image} x {image} torchvision's "
                         "AdaptiveAvgPool2d((7, 7)) is not the identity, and the Caffe net has no such pool")
    src = np.load(npz) if isinstance(npz, str) else npz

    def get(key, shape):
        if key not in src:
            raise KeyError(f"vgg{depth} weights: missing {key}")
        v = np.asarray(src[key], dtype=np.float32)
        if v.shape != tuple(shape):
            raise ValueError(f"vgg{depth} weights: {key} has shape {v.shape}, expected {tuple(shape)}")
        return v

    out: dict = {}
    i, cin = 0, 3
    for b, (n, c) in enumerate(zip(graph._VGG_BLOCKS[depth], graph._VGG_WIDTHS), 1):
        for l in range(1, n + 1):
            out[f"conv{b}_{l}"] = {"W": get(f"features.{i}.weight", (c, cin, 3, 3)), "b": get(f"features.{i}.bias", (c,))}
            i, cin = i + 2, c  # Conv2d, ReLU
        i += 1  # MaxPool2d
    for name, idx, (cout, k) in (("fc6", 0, (4096, 512 * 7 * 7)), ("fc7", 3, (4096, 4096)), ("fc8", 6, (1000, 4096))):
        out[name] = {"W": get(f"classifier.{idx}.weight", (cout, k)), "b": get(f"classifier.{idx}.bias", (cout,))}
    return out
