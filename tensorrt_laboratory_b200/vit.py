"""Vision Transformer (ViT) image classifiers: configuration, seeded weights and a weight loader.

Parameter names and shapes are those of Hugging Face ``ViTForImageClassification`` (``vit.embeddings.cls_token``,
``vit.encoder.layer.{i}.attention.attention.query.weight`` [out, in], ``classifier.weight`` ...), so weights exported from
such a model with numpy (``np.savez(f, **{k: v.numpy() for k, v in model.state_dict().items()})``) load as they are.  The
plan built from them is described in ``builder.build_vit_plan``.
"""
from __future__ import annotations

import dataclasses
from typing import Dict, Mapping, Union

import numpy as np


@dataclasses.dataclass(frozen=True)
class VitConfig:
    layers: int = 12
    hidden: int = 768
    heads: int = 12
    ffn: int = 3072
    patch: int = 16
    image: int = 224        # input images of image x image_width pixels, 3 channels
    classes: int = 1000
    eps: float = 1e-12      # LayerNorm epsilon: Hugging Face ViT uses 1e-12, torchvision 1e-6
    image_width: int = 0    # 0: square images

    @property
    def width(self) -> int:
        return self.image_width or self.image

    @property
    def patches(self) -> int:
        return (self.image // self.patch) * (self.width // self.patch)

    @property
    def tokens(self) -> int:
        """L: the patches and the class token"""
        return self.patches + 1


VIT_B16 = VitConfig()
VIT_B32 = VitConfig(patch=32)
VIT_L16 = VitConfig(layers=24, hidden=1024, heads=16, ffn=4096)


def param_shapes(cfg: VitConfig) -> Dict[str, tuple]:
    """Every parameter of the model, Hugging Face names without the ``vit.`` prefix -> shape."""
    H, F, p, L = cfg.hidden, cfg.ffn, cfg.patch, cfg.tokens
    s = {
        "embeddings.cls_token": (1, 1, H),
        "embeddings.position_embeddings": (1, L, H),
        "embeddings.patch_embeddings.projection.weight": (H, 3, p, p),
        "embeddings.patch_embeddings.projection.bias": (H,),
    }
    for i in range(cfg.layers):
        q = f"encoder.layer.{i}."
        s[q + "layernorm_before.weight"] = (H,)
        s[q + "layernorm_before.bias"] = (H,)
        for m in ("query", "key", "value"):
            s[q + f"attention.attention.{m}.weight"] = (H, H)
            s[q + f"attention.attention.{m}.bias"] = (H,)
        s[q + "attention.output.dense.weight"] = (H, H)
        s[q + "attention.output.dense.bias"] = (H,)
        s[q + "layernorm_after.weight"] = (H,)
        s[q + "layernorm_after.bias"] = (H,)
        s[q + "intermediate.dense.weight"] = (F, H)
        s[q + "intermediate.dense.bias"] = (F,)
        s[q + "output.dense.weight"] = (H, F)
        s[q + "output.dense.bias"] = (H,)
    s["layernorm.weight"] = (H,)
    s["layernorm.bias"] = (H,)
    s["classifier.weight"] = (cfg.classes, H)
    s["classifier.bias"] = (cfg.classes,)
    return s


def random_weights(cfg: VitConfig = VIT_B16, seed: int = 0) -> Dict[str, np.ndarray]:
    """Seeded fp32 weights drawn the way ViT initialises them: N(0, 0.02) for every matrix, the patch projection, the class
    token and the position embeddings; LayerNorm gamma = 1 + N(0, 0.02).  Biases and LayerNorm beta are N(0, 0.02) rather
    than zeros, so that every bias path is exercised.

    The classifier is the exception: W ~ N(0, 1 / H) and b ~ N(0, 0.02).  The final LayerNorm gives the class token unit
    scale, so the logits have unit scale too and the gaps between the largest ones (about 0.3 for 1000 classes) stay far
    above the fp16 error of the engine, which makes a top-1 comparison on N(0, 1) images meaningful.  At N(0, 0.02) the
    logits would be 0.55 wide and the bias would matter as much as the image."""
    rng = np.random.default_rng(seed)
    out = {}
    for k, shp in param_shapes(cfg).items():
        v = rng.standard_normal(shp, dtype=np.float32) * np.float32(0.02)
        if k.endswith(("layernorm_before.weight", "layernorm_after.weight")) or k == "layernorm.weight":
            v += np.float32(1.0)
        if k == "classifier.weight":
            v *= np.float32(1.0 / (0.02 * np.sqrt(cfg.hidden)))
        out[k] = v
    return out


def load_weights(src: Union[str, Mapping[str, np.ndarray]], cfg: VitConfig = VIT_B16) -> Dict[str, np.ndarray]:
    """Weights from a dict or an ``.npz`` file with Hugging Face ``ViTForImageClassification`` names, with or without the
    ``vit.`` prefix (``vit.pooler.*`` is ignored).  Every parameter must be present with its exact shape; the error names
    the offending key."""
    if isinstance(src, str):
        with np.load(src) as z:
            src = {k: z[k] for k in z.files}
    items = {}
    for k, v in src.items():
        name = k[len("vit."):] if k.startswith("vit.") else k
        if name.startswith("pooler."):
            continue
        items[name] = v
    out = {}
    for k, shp in param_shapes(cfg).items():
        if k not in items:
            raise KeyError(f"ViT weights: missing parameter {k!r} (shape {shp})")
        v = np.asarray(items[k])
        if tuple(v.shape) != shp:
            raise ValueError(f"ViT weights: parameter {k!r} has shape {tuple(v.shape)}, the configuration needs {shp}")
        out[k] = np.ascontiguousarray(v, dtype=np.float32)
    return out
