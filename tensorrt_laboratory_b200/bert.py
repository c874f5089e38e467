"""BERT-base encoder model: configuration, seeded weights and a weight loader.

Parameter names and shapes are those of Hugging Face ``BertModel`` (``embeddings.word_embeddings.weight``,
``encoder.layer.{i}.attention.self.query.weight`` [out, in], ...), so weights exported from such a model with numpy
(``np.savez(f, **{k: v.numpy() for k, v in model.state_dict().items()})``) load as they are.  The plan built from them is
described in ``builder.build_bert_plan``.
"""
from __future__ import annotations

import dataclasses
from typing import Dict, Mapping, Union

import numpy as np


@dataclasses.dataclass(frozen=True)
class BertConfig:
    layers: int = 12
    hidden: int = 768
    heads: int = 12
    ffn: int = 3072
    vocab: int = 30522
    positions: int = 512
    types: int = 2
    seq: int = 128          # the sequence length S a plan is built for (64, 128, 256, 384 or 512; at most positions)
    eps: float = 1e-12      # LayerNorm epsilon


BERT_BASE = BertConfig()


def param_shapes(cfg: BertConfig) -> Dict[str, tuple]:
    """Every parameter of the encoder + pooler, Hugging Face names (no ``bert.`` prefix) -> shape."""
    H, F = cfg.hidden, cfg.ffn
    s = {
        "embeddings.word_embeddings.weight": (cfg.vocab, H),
        "embeddings.position_embeddings.weight": (cfg.positions, H),
        "embeddings.token_type_embeddings.weight": (cfg.types, H),
        "embeddings.LayerNorm.weight": (H,),
        "embeddings.LayerNorm.bias": (H,),
    }
    for i in range(cfg.layers):
        p = f"encoder.layer.{i}."
        for m in ("query", "key", "value"):
            s[p + f"attention.self.{m}.weight"] = (H, H)
            s[p + f"attention.self.{m}.bias"] = (H,)
        s[p + "attention.output.dense.weight"] = (H, H)
        s[p + "attention.output.dense.bias"] = (H,)
        s[p + "attention.output.LayerNorm.weight"] = (H,)
        s[p + "attention.output.LayerNorm.bias"] = (H,)
        s[p + "intermediate.dense.weight"] = (F, H)
        s[p + "intermediate.dense.bias"] = (F,)
        s[p + "output.dense.weight"] = (H, F)
        s[p + "output.dense.bias"] = (H,)
        s[p + "output.LayerNorm.weight"] = (H,)
        s[p + "output.LayerNorm.bias"] = (H,)
    s["pooler.dense.weight"] = (H, H)
    s["pooler.dense.bias"] = (H,)
    return s


def random_weights(cfg: BertConfig = BERT_BASE, seed: int = 0) -> Dict[str, np.ndarray]:
    """Seeded fp32 weights drawn the way BERT initialises them: N(0, 0.02) for every matrix and embedding table, LayerNorm
    gamma = 1 + N(0, 0.02).  Biases and LayerNorm beta are N(0, 0.02) rather than BERT's zeros, so that every bias path is
    exercised."""
    rng = np.random.default_rng(seed)
    out = {}
    for k, shp in param_shapes(cfg).items():
        v = rng.standard_normal(shp, dtype=np.float32) * np.float32(0.02)
        if k.endswith("LayerNorm.weight"):
            v += np.float32(1.0)
        out[k] = v
    return out


def load_weights(src: Union[str, Mapping[str, np.ndarray]], cfg: BertConfig = BERT_BASE) -> Dict[str, np.ndarray]:
    """Weights from a dict or an ``.npz`` file with Hugging Face ``BertModel`` names, with or without the ``bert.`` prefix
    (keys of task heads, e.g. ``cls.*``, are ignored).  Every parameter must be present with its exact shape; the error
    names the offending key."""
    if isinstance(src, str):
        with np.load(src) as z:
            src = {k: z[k] for k in z.files}
    items = {}
    for k, v in src.items():
        name = k[len("bert."):] if k.startswith("bert.") else k
        items[name] = v
    out = {}
    for k, shp in param_shapes(cfg).items():
        if k not in items:
            raise KeyError(f"BERT weights: missing parameter {k!r} (shape {shp})")
        v = np.asarray(items[k])
        if tuple(v.shape) != shp:
            raise ValueError(f"BERT weights: parameter {k!r} has shape {tuple(v.shape)}, the configuration needs {shp}")
        out[k] = np.ascontiguousarray(v, dtype=np.float32)
    return out
