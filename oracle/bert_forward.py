"""CPU oracles of the BERT encoder plan (``builder.build_bert_plan``), torch on the CPU; used by the tests only.

* :func:`forward_fp32` -- the model in fp32 (the reference answer).
* :func:`forward_fp16` -- an emulation of the engine's numerics contract (DESIGN.md, "BERT numerics"): fp16 tables and
  weights, fp16 activations between operators, fp32 inside them, with the rounding points of the kernels.
* :func:`witness_layers` -- the second witness: ``torch.nn.TransformerEncoderLayer`` loaded with the same weights.

Weights are dicts in Hugging Face ``BertModel`` names (``bert.load_weights``).  Inputs are int arrays [N, S].
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn.functional as TF

MASK_ADD = -10000.0


def _t(a) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))


def _h(x: torch.Tensor) -> torch.Tensor:
    """round to fp16, keep computing in fp32"""
    return x.to(torch.float16).to(torch.float32)


def _ln(x: torch.Tensor, g, b, eps: float) -> torch.Tensor:
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    return (x - mean) * (1.0 / torch.sqrt(var + eps)) * _t(g) + _t(b)


def _mask_add(mask: np.ndarray) -> torch.Tensor:
    return torch.where(torch.from_numpy(np.asarray(mask) != 0), 0.0, MASK_ADD).to(torch.float32)


def _embed_rows(W, cfg, ids, segs, rnd):
    """(word + position) + type rows, clamped ids; `rnd` rounds the tables (fp16 storage) or not."""
    ids = np.clip(np.asarray(ids, dtype=np.int64), 0, cfg.vocab - 1)
    segs = np.clip(np.asarray(segs, dtype=np.int64), 0, cfg.types - 1)
    S = ids.shape[1]
    wt = rnd(_t(W["embeddings.word_embeddings.weight"]))
    pt = rnd(_t(W["embeddings.position_embeddings.weight"]))
    tt = rnd(_t(W["embeddings.token_type_embeddings.weight"]))
    return (wt[torch.from_numpy(ids)] + pt[:S][None]) + tt[torch.from_numpy(segs)]


def _forward(W: Dict[str, np.ndarray], cfg, ids, segs, mask, fp16: bool, record: Optional[List[dict]] = None):
    r = _h if fp16 else (lambda x: x)
    H, nh = cfg.hidden, cfg.heads
    madd = _mask_add(mask)                                    # [N, S]
    x = r(_ln(_embed_rows(W, cfg, ids, segs, r), W["embeddings.LayerNorm.weight"], W["embeddings.LayerNorm.bias"], cfg.eps))
    if record is not None:
        record.append({"embeddings": x})
    N, S, _ = x.shape

    def gemm(a, w, b, res=None, gelu=False):
        y = a @ r(_t(w)).T + _t(b)
        if res is not None:
            y = y + res
        if gelu:
            y = TF.gelu(y)
        return r(y)

    for i in range(cfg.layers):
        p = f"encoder.layer.{i}."
        Wqkv = np.concatenate([W[p + f"attention.self.{m}.weight"] for m in ("query", "key", "value")])
        bqkv = np.concatenate([W[p + f"attention.self.{m}.bias"] for m in ("query", "key", "value")])
        qkv = gemm(x, Wqkv, bqkv)
        q, k, v = (qkv[..., j * H:(j + 1) * H].reshape(N, S, nh, 64).transpose(1, 2) for j in range(3))
        s = (q @ k.transpose(-1, -2)) * 0.125 + madd[:, None, None, :]
        e = torch.exp(s - s.amax(-1, keepdim=True))
        P = r(e / e.sum(-1, keepdim=True))                    # normalised before P V, rounded to fp16
        ctx = r((P @ v).transpose(1, 2).reshape(N, S, H))
        att = gemm(ctx, W[p + "attention.output.dense.weight"], W[p + "attention.output.dense.bias"], res=x)
        h1 = r(_ln(att, W[p + "attention.output.LayerNorm.weight"], W[p + "attention.output.LayerNorm.bias"], cfg.eps))
        f = gemm(h1, W[p + "intermediate.dense.weight"], W[p + "intermediate.dense.bias"], gelu=True)
        fs = gemm(f, W[p + "output.dense.weight"], W[p + "output.dense.bias"], res=h1)
        x = r(_ln(fs, W[p + "output.LayerNorm.weight"], W[p + "output.LayerNorm.bias"], cfg.eps))
        if record is not None:
            record.append({"qkv": qkv, "context": ctx, "attn_sum": att, "attn_ln": h1, "ffn": f, "ffn_sum": fs, "out": x})
    pooled = torch.tanh(x[:, 0] @ r(_t(W["pooler.dense.weight"])).T + _t(W["pooler.dense.bias"]))
    return x.numpy(), pooled.numpy()


@torch.no_grad()
def forward_fp32(W, cfg, ids, segs, mask, record: Optional[List[dict]] = None):
    """-> (last_hidden_state [N, S, H], pooled_output [N, H]) in fp32."""
    return _forward(W, cfg, ids, segs, mask, False, record)


@torch.no_grad()
def forward_fp16(W, cfg, ids, segs, mask, record: Optional[List[dict]] = None):
    """The engine's numerics contract:
    - embedding tables in fp16, rows summed in fp32 as (word + position) + type, LayerNorm in fp32, rounded to fp16;
    - GEMMs: fp16 operands, fp32 accumulation, + bias (+ residual) (+ GELU, erf form) in fp32, rounded to fp16;
    - attention: scores Q K^T in fp32 times 0.125, + (-10000 where input_mask == 0); softmax in fp32 with the maximum
      subtracted; P = fp16(exp(s - max) / sum) (normalised before P V); P V accumulated in fp32, rounded to fp16;
    - LayerNorm: fp16 in, mean and variance in fp32, gamma / beta applied in fp32, fp16 out;
    - pooler: tanh(W h[CLS] + b) from fp16 weights and activations, fp32 out."""
    return _forward(W, cfg, ids, segs, mask, True, record)


def emulate_ops(W, cfg, layer: int, madd_mask, taps: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
    """Per-operator emulation of one layer from the ENGINE's own fp16 inputs (``taps``: [N, S, C] arrays read back from
    the plan's tap bindings), so each operator is judged on its own: -> expected value of each tap."""
    p = f"encoder.layer.{layer}."
    H, nh = cfg.hidden, cfg.heads
    T = {k: _t(v) for k, v in taps.items()}
    madd = _mask_add(madd_mask)
    N, S, _ = T["qkv"].shape

    def gemm(a, w, b, res=None, gelu=False):
        y = a @ _h(_t(w)).T + _t(b)
        if res is not None:
            y = y + res
        return _h(TF.gelu(y) if gelu else y)

    out = {}
    Wqkv = np.concatenate([W[p + f"attention.self.{m}.weight"] for m in ("query", "key", "value")])
    bqkv = np.concatenate([W[p + f"attention.self.{m}.bias"] for m in ("query", "key", "value")])
    out["qkv"] = gemm(T["x"], Wqkv, bqkv)
    q, k, v = (T["qkv"][..., j * H:(j + 1) * H].reshape(N, S, nh, 64).transpose(1, 2) for j in range(3))
    s = (q @ k.transpose(-1, -2)) * 0.125 + madd[:, None, None, :]
    e = torch.exp(s - s.amax(-1, keepdim=True))
    out["context"] = _h((_h(e / e.sum(-1, keepdim=True)) @ v).transpose(1, 2).reshape(N, S, H))
    out["attn_sum"] = gemm(T["context"], W[p + "attention.output.dense.weight"], W[p + "attention.output.dense.bias"], res=T["x"])
    out["attn_ln"] = _h(_ln(T["attn_sum"], W[p + "attention.output.LayerNorm.weight"], W[p + "attention.output.LayerNorm.bias"], cfg.eps))
    out["ffn"] = gemm(T["attn_ln"], W[p + "intermediate.dense.weight"], W[p + "intermediate.dense.bias"], gelu=True)
    out["ffn_sum"] = gemm(T["ffn"], W[p + "output.dense.weight"], W[p + "output.dense.bias"], res=T["attn_ln"])
    out["out"] = _h(_ln(T["ffn_sum"], W[p + "output.LayerNorm.weight"], W[p + "output.LayerNorm.bias"], cfg.eps))
    return {k: v.numpy() for k, v in out.items()}


def emulate_embeddings(W, cfg, ids, segs) -> np.ndarray:
    return _h(_ln(_embed_rows(W, cfg, ids, segs, _h), W["embeddings.LayerNorm.weight"], W["embeddings.LayerNorm.bias"], cfg.eps)).numpy()


@torch.no_grad()
def witness_layers(W, cfg, x0: np.ndarray, mask) -> List[np.ndarray]:
    """Runs ``torch.nn.TransformerEncoderLayer(H, heads, FFN, dropout=0, activation="gelu", layer_norm_eps=eps,
    batch_first=True)`` with the BERT weights, layer after layer from the fp32 embedding output ``x0``, with the
    key-padding mask; -> the output of every layer.  (-10000 and -inf give the same exp = 0 on every row with a valid key.)"""
    H = cfg.hidden
    kpm = torch.from_numpy(np.asarray(mask) == 0)
    x = _t(x0)
    outs = []
    for i in range(cfg.layers):
        p = f"encoder.layer.{i}."
        layer = torch.nn.TransformerEncoderLayer(H, cfg.heads, cfg.ffn, dropout=0.0, activation="gelu", layer_norm_eps=cfg.eps,
                                                 batch_first=True)
        layer.train()  # the reference (non-fused) path: every position is computed, padded ones included
        sd = {
            "self_attn.in_proj_weight": np.concatenate([W[p + f"attention.self.{m}.weight"] for m in ("query", "key", "value")]),
            "self_attn.in_proj_bias": np.concatenate([W[p + f"attention.self.{m}.bias"] for m in ("query", "key", "value")]),
            "self_attn.out_proj.weight": W[p + "attention.output.dense.weight"],
            "self_attn.out_proj.bias": W[p + "attention.output.dense.bias"],
            "linear1.weight": W[p + "intermediate.dense.weight"], "linear1.bias": W[p + "intermediate.dense.bias"],
            "linear2.weight": W[p + "output.dense.weight"], "linear2.bias": W[p + "output.dense.bias"],
            "norm1.weight": W[p + "attention.output.LayerNorm.weight"], "norm1.bias": W[p + "attention.output.LayerNorm.bias"],
            "norm2.weight": W[p + "output.LayerNorm.weight"], "norm2.bias": W[p + "output.LayerNorm.bias"],
        }
        layer.load_state_dict({k: _t(v) for k, v in sd.items()})
        x = layer(x, src_key_padding_mask=kpm)
        outs.append(x.numpy().copy())
    return outs
