"""CPU oracles of the Vision Transformer plan (``builder.build_vit_plan``), torch on the CPU; used by the tests only.

* :func:`forward_fp32` -- the model with Hugging Face ViT semantics in float64 (the reference answer).
* :func:`forward_fp16` -- an emulation of the engine's numerics contract (DESIGN.md, "ViT numerics"), built from the BERT
  oracle's LayerNorm, GEMM and GELU helpers.
* :func:`emulate_ops` / :func:`emulate_front` / :func:`emulate_head` -- the same operators applied to the engine's own
  tapped inputs, so each operator is judged on its own.
* ``ref_*`` -- float64 references with elementwise error bounds (``bert_forward``'s), for the operators ViT shares with BERT.

Weights are dicts in Hugging Face ``ViTForImageClassification`` names (``vit.load_weights``).  Images are fp32 [N, 3, H, W].
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn.functional as TF

from oracle.bert_forward import _gelu, _h, _ln, _t, ref_attention as _bert_ref_attention, ref_layernorm, ref_gelu_gemm  # noqa: F401

KEY_BLOCK = 128  # keys per warpgroup of the key-split attention kernel (S_k >= 256)


def _d(a) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64))


def patch_rows(x: np.ndarray, p: int) -> np.ndarray:
    """[N, 3, H, W] -> [N, P, 3 p^2]: patch t = (py, px) in row-major order, element (c, dy, dx) at column c p^2 + dy p + dx
    (the engine's OP_PATCHIFY layout, in the input's dtype)."""
    N, C, Hh, Ww = x.shape
    r = x.reshape(N, C, Hh // p, p, Ww // p, p).transpose(0, 2, 4, 1, 3, 5)
    return np.ascontiguousarray(r.reshape(N, (Hh // p) * (Ww // p), C * p * p))


# ---- float64 model --------------------------------------------------------------------------------------------------
@torch.no_grad()
def forward_fp32(W: Dict[str, np.ndarray], cfg, x: np.ndarray):
    """-> (logits [N, classes], prob [N, classes]), Hugging Face ViT semantics in float64: conv2d patch embedding with
    stride p, pre-LN layers, softmax attention over all L tokens, erf GELU, final LayerNorm on the class token."""
    H, nh, p = cfg.hidden, cfg.heads, cfg.patch
    y = TF.conv2d(_d(x), _d(W["embeddings.patch_embeddings.projection.weight"]), _d(W["embeddings.patch_embeddings.projection.bias"]),
                  stride=p)
    N = y.shape[0]
    y = y.flatten(2).transpose(1, 2)                                              # [N, P, H]
    h = torch.cat([_d(W["embeddings.cls_token"]).expand(N, 1, H), y], 1) + _d(W["embeddings.position_embeddings"])
    L = h.shape[1]

    def ln(t, prefix):
        return TF.layer_norm(t, (H,), _d(W[prefix + ".weight"]), _d(W[prefix + ".bias"]), cfg.eps)

    def lin(t, prefix):
        return t @ _d(W[prefix + ".weight"]).T + _d(W[prefix + ".bias"])

    for i in range(cfg.layers):
        q = f"encoder.layer.{i}."
        a = ln(h, q + "layernorm_before")
        qh, kh, vh = (lin(a, q + f"attention.attention.{m}").reshape(N, L, nh, 64).transpose(1, 2) for m in ("query", "key", "value"))
        s = (qh @ kh.transpose(-1, -2)) * 0.125
        ctx = (torch.softmax(s, -1) @ vh).transpose(1, 2).reshape(N, L, H)
        h = h + lin(ctx, q + "attention.output.dense")
        f = TF.gelu(lin(ln(h, q + "layernorm_after"), q + "intermediate.dense"))
        h = h + lin(f, q + "output.dense")
    logits = lin(ln(h[:, 0], "layernorm"), "classifier")
    return logits.numpy(), torch.softmax(logits, -1).numpy()


# ---- the engine's numerics contract -------------------------------------------------------------------------------------
def _gemm(a, w, b, res=None, gelu=False):
    """fp16 operands, fp32 accumulation, + bias (+ residual) (+ GELU) in fp32, rounded to fp16"""
    y = a @ _h(_t(w)).T + _t(b)
    if res is not None:
        y = y + res
    return _h(_gelu(y) if gelu else y)


def _attend_blocks(q, k, v) -> torch.Tensor:
    """q, k, v [N, heads, L, 64] fp16 values -> P V (before the fp16 rounding of O), reduced over the keys in blocks of 128
    in block order as the key-split kernel does: scores in fp32 times 0.125, the row maximum over all keys, each block's
    exp sum and partial P V in fp32, the blocks added in order; P = fp16(exp / sum) before P V."""
    s = (q @ k.transpose(-1, -2)) * 0.125
    e = torch.exp(s - s.amax(-1, keepdim=True))
    L = s.shape[-1]
    blocks = range(0, L, KEY_BLOCK)
    total = None
    for b0 in blocks:
        part = e[..., b0:b0 + KEY_BLOCK].sum(-1, keepdim=True)
        total = part if total is None else total + part
    P = _h(e / total)
    out = None
    for b0 in blocks:
        part = P[..., b0:b0 + KEY_BLOCK] @ v[..., b0:b0 + KEY_BLOCK, :]
        out = part if out is None else out + part
    return out


def _attention(qkv: torch.Tensor, heads: int) -> torch.Tensor:
    """fused QKV [N, L, 3H] (channel part * H + 64 * head + d) -> context [N, L, H], rounded to fp16"""
    N, L, C3 = qkv.shape
    H = C3 // 3
    qh, kh, vh = (qkv[..., j * H:(j + 1) * H].reshape(N, L, heads, 64).transpose(1, 2) for j in range(3))
    return _h(_attend_blocks(qh, kh, vh).transpose(1, 2).reshape(N, L, H))


def _layer(W, cfg, i: int, x: torch.Tensor, T: Optional[Dict[str, torch.Tensor]] = None) -> Dict[str, torch.Tensor]:
    """One pre-LN layer; with T (tapped engine tensors) every operator reads the engine's own input instead of the
    emulation's previous result."""
    q = f"encoder.layer.{i}."
    nh = cfg.heads
    src = (lambda k, v: T[k]) if T is not None else (lambda k, v: v)  # noqa: E731
    out = {}
    out["ln1"] = _h(_ln(x, W[q + "layernorm_before.weight"], W[q + "layernorm_before.bias"], cfg.eps))
    Wqkv = np.concatenate([W[q + f"attention.attention.{m}.weight"] for m in ("query", "key", "value")])
    bqkv = np.concatenate([W[q + f"attention.attention.{m}.bias"] for m in ("query", "key", "value")])
    out["qkv"] = _gemm(src("ln1", out["ln1"]), Wqkv, bqkv)
    out["context"] = _attention(src("qkv", out["qkv"]), nh)
    out["attn_sum"] = _gemm(src("context", out["context"]), W[q + "attention.output.dense.weight"], W[q + "attention.output.dense.bias"], res=x)
    x1 = src("attn_sum", out["attn_sum"])
    out["ln2"] = _h(_ln(x1, W[q + "layernorm_after.weight"], W[q + "layernorm_after.bias"], cfg.eps))
    out["ffn"] = _gemm(src("ln2", out["ln2"]), W[q + "intermediate.dense.weight"], W[q + "intermediate.dense.bias"], gelu=True)
    out["out"] = _gemm(src("ffn", out["ffn"]), W[q + "output.dense.weight"], W[q + "output.dense.bias"], res=x1)
    return out


def _front(W, cfg, x: np.ndarray) -> Dict[str, torch.Tensor]:
    H, p = cfg.hidden, cfg.patch
    patches = _h(_t(patch_rows(np.asarray(x, np.float32), p)))
    pe = _gemm(patches, W["embeddings.patch_embeddings.projection.weight"].reshape(H, 3 * p * p), W["embeddings.patch_embeddings.projection.bias"])
    return {"patches": patches, "patch_embed": pe}


def _tokens(W, cfg, pe: torch.Tensor) -> torch.Tensor:
    """row 0 = fp16(cls + pos_0), row t = fp16(pe[t - 1] + pos_t), fp16 tables, fp32 sums"""
    H = cfg.hidden
    cls = _h(_t(W["embeddings.cls_token"].reshape(1, 1, H)))
    pos = _h(_t(W["embeddings.position_embeddings"].reshape(1, -1, H)))
    return _h(torch.cat([cls.expand(pe.shape[0], 1, H), pe], 1) + pos)


def _head(W, cfg, h0: torch.Tensor):
    """h0 [N, H]: the class-token rows -> (final LayerNorm rows, logits fp32, prob)"""
    f = _h(_ln(h0, W["layernorm.weight"], W["layernorm.bias"], cfg.eps))
    logits = f @ _h(_t(W["classifier.weight"])).T + _t(W["classifier.bias"])
    return f, logits, torch.softmax(logits, -1)


@torch.no_grad()
def forward_fp16(W, cfg, x: np.ndarray, record: Optional[List[dict]] = None):
    """The engine's numerics contract -> (logits [N, classes], prob [N, classes]):
    - patches: the fp32 image rounded to fp16 (round to nearest), laid out as :func:`patch_rows`;
    - GEMMs (patch projection, QKV, attention output, FFN): fp16 operands, fp32 accumulation, + bias (+ residual)
      (+ GELU, erf form) in fp32, rounded to fp16;
    - tokens: fp16 class token and position tables, row 0 = fp16(cls + pos_0), row t = fp16(y[t - 1] + pos_t);
    - LayerNorm: fp16 in, mean and variance in fp32, gamma / beta in fp32, fp16 out;
    - attention (no mask, all L tokens): scores in fp32 times 0.125, softmax in fp32 with the maximum subtracted, keys
      reduced in blocks of 128 in block order, P = fp16(exp(s - max) / sum) before P V, P V in fp32, rounded to fp16;
    - head: the final LayerNorm of the class token (fp16 result), logits = b + W h in fp32 from fp16 weights, fp32
      softmax.
    ``record``: gets {"patches", "patch_embed", "tokens"}, one dict per layer (``_layer``'s names) and {"final_ln",
    "logits"}."""
    fr = _front(W, cfg, x)
    h = _tokens(W, cfg, fr["patch_embed"])
    if record is not None:
        record.append({**fr, "tokens": h})
    for i in range(cfg.layers):
        o = _layer(W, cfg, i, h)
        if record is not None:
            record.append(o)
        h = o["out"]
    f, logits, prob = _head(W, cfg, h[:, 0])
    if record is not None:
        record.append({"final_ln": f, "logits": logits})
    return logits.numpy(), prob.numpy()


@torch.no_grad()
def emulate_front(W, cfg, x: np.ndarray, patch_embed: Optional[np.ndarray] = None) -> Dict[str, np.ndarray]:
    """patches and patch_embed from the image, tokens from ``patch_embed`` (the engine's, when given)"""
    fr = _front(W, cfg, x)
    pe = _t(patch_embed) if patch_embed is not None else fr["patch_embed"]
    return {"patches": fr["patches"].numpy(), "patch_embed": fr["patch_embed"].numpy(), "tokens": _tokens(W, cfg, pe).numpy()}


@torch.no_grad()
def emulate_ops(W, cfg, layer: int, taps: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
    """Every operator of one layer from the engine's own fp16 inputs (``taps``: [N, L, C] arrays named x -- the layer
    input -- ln1, qkv, context, attn_sum, ln2, ffn) -> the expected value of each tap (ln1 ... out)."""
    T = {k: _t(v) for k, v in taps.items()}
    return {k: v.numpy() for k, v in _layer(W, cfg, layer, T["x"], T).items()}


@torch.no_grad()
def emulate_attention(qkv: np.ndarray, heads: int) -> np.ndarray:
    """the attention operator of the contract from the engine's QKV tensor [N, L, 3H]"""
    return _attention(_t(qkv), heads).numpy()


@torch.no_grad()
def emulate_head(W, cfg, last: np.ndarray, final_ln: Optional[np.ndarray] = None):
    """-> (final LayerNorm of every token [N, L, H], logits [N, classes]) from the last layer's output; the logits from
    the engine's ``final_ln`` class-token rows when given."""
    f_all = _h(_ln(_t(last), W["layernorm.weight"], W["layernorm.bias"], cfg.eps))
    h0 = _t(final_ln)[:, 0] if final_ln is not None else f_all[:, 0]
    logits = h0 @ _h(_t(W["classifier.weight"])).T + _t(W["classifier.bias"])
    return f_all.numpy(), logits.numpy()


# ---- float64 references with elementwise bounds -------------------------------------------------------------------------
def ref_attention(qkv, heads: int):
    """``bert_forward.ref_attention`` over all L tokens (no mask): qkv [N, L, 3H] fp16 values -> (O [N, L, H], bound)"""
    qkv = np.asarray(qkv)
    return _bert_ref_attention(qkv, np.ones(qkv.shape[:2], np.int32), heads)


def ref_head(W, final_ln_rows):
    """logits = fp16(W) h + b in float64 from the class-token rows h [N, H] (fp16 values) -> (logits, bound): the products
    are exact in fp32, the lanes' in-order sums and the butterfly are within H U32 sum|w h|, the bias add rounds once."""
    from oracle.bert_forward import U32, _f64, _w16
    h = _f64(final_ln_rows)
    w = _w16(W["classifier.weight"])
    t = h @ w.T + _f64(np.asarray(W["classifier.bias"], np.float32))
    return t, h.shape[-1] * U32 * (np.abs(h) @ np.abs(w).T) + U32 * np.abs(t) + 1e-30
