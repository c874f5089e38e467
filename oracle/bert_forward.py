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


# The operators of the emulation, one function each, so a test can replace one of them (tests/test_bert_values_cpu.py
# checks that deliberately wrong versions break the float64 bounds below).
def _gelu(y: torch.Tensor) -> torch.Tensor:
    return TF.gelu(y)


def _attend(q, k, v, madd, r) -> torch.Tensor:
    """q, k, v [N, heads, S, 64], madd [N, S] -> P V [N, heads, S, 64] (before the fp16 rounding of O)"""
    s = (q @ k.transpose(-1, -2)) * 0.125 + madd[:, None, None, :]
    e = torch.exp(s - s.amax(-1, keepdim=True))
    P = r(e / e.sum(-1, keepdim=True))                        # normalised before P V, rounded to fp16
    return P @ v


def _pool(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """x [N, S, H] -> tanh(W x[:, 0] + b), token 0 = [CLS]"""
    return torch.tanh(x[:, 0] @ w.T + b)


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
            y = _gelu(y)
        return r(y)

    for i in range(cfg.layers):
        p = f"encoder.layer.{i}."
        Wqkv = np.concatenate([W[p + f"attention.self.{m}.weight"] for m in ("query", "key", "value")])
        bqkv = np.concatenate([W[p + f"attention.self.{m}.bias"] for m in ("query", "key", "value")])
        qkv = gemm(x, Wqkv, bqkv)
        q, k, v = (qkv[..., j * H:(j + 1) * H].reshape(N, S, nh, 64).transpose(1, 2) for j in range(3))
        ctx = r(_attend(q, k, v, madd, r).transpose(1, 2).reshape(N, S, H))
        att = gemm(ctx, W[p + "attention.output.dense.weight"], W[p + "attention.output.dense.bias"], res=x)
        h1 = r(_ln(att, W[p + "attention.output.LayerNorm.weight"], W[p + "attention.output.LayerNorm.bias"], cfg.eps))
        f = gemm(h1, W[p + "intermediate.dense.weight"], W[p + "intermediate.dense.bias"], gelu=True)
        fs = gemm(f, W[p + "output.dense.weight"], W[p + "output.dense.bias"], res=h1)
        x = r(_ln(fs, W[p + "output.LayerNorm.weight"], W[p + "output.LayerNorm.bias"], cfg.eps))
        if record is not None:
            record.append({"qkv": qkv, "context": ctx, "attn_sum": att, "attn_ln": h1, "ffn": f, "ffn_sum": fs, "out": x})
    pooled = _pool(x, r(_t(W["pooler.dense.weight"])), _t(W["pooler.dense.bias"]))
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
        return _h(_gelu(y) if gelu else y)

    out = {}
    Wqkv = np.concatenate([W[p + f"attention.self.{m}.weight"] for m in ("query", "key", "value")])
    bqkv = np.concatenate([W[p + f"attention.self.{m}.bias"] for m in ("query", "key", "value")])
    out["qkv"] = gemm(T["x"], Wqkv, bqkv)
    q, k, v = (T["qkv"][..., j * H:(j + 1) * H].reshape(N, S, nh, 64).transpose(1, 2) for j in range(3))
    out["context"] = _h(_attend(q, k, v, madd, _h).transpose(1, 2).reshape(N, S, H))
    out["attn_sum"] = gemm(T["context"], W[p + "attention.output.dense.weight"], W[p + "attention.output.dense.bias"], res=T["x"])
    out["attn_ln"] = _h(_ln(T["attn_sum"], W[p + "attention.output.LayerNorm.weight"], W[p + "attention.output.LayerNorm.bias"], cfg.eps))
    out["ffn"] = gemm(T["attn_ln"], W[p + "intermediate.dense.weight"], W[p + "intermediate.dense.bias"], gelu=True)
    out["ffn_sum"] = gemm(T["ffn"], W[p + "output.dense.weight"], W[p + "output.dense.bias"], res=T["attn_ln"])
    out["out"] = _h(_ln(T["ffn_sum"], W[p + "output.LayerNorm.weight"], W[p + "output.LayerNorm.bias"], cfg.eps))
    return {k: v.numpy() for k, v in out.items()}


def emulate_embeddings(W, cfg, ids, segs) -> np.ndarray:
    return _h(_ln(_embed_rows(W, cfg, ids, segs, _h), W["embeddings.LayerNorm.weight"], W["embeddings.LayerNorm.bias"], cfg.eps)).numpy()


# ---- float64 references with elementwise error bounds ---------------------------------------------------------------
# Each reference computes an operator exactly (float64) from the engine's own fp16 inputs and returns (value, bound):
# any implementation of the contract above -- fp32 arithmetic inside the operator, rounded to fp16 where the contract
# rounds -- lies within `bound` of `value`, element by element.  Unlike the scale-relative 2-ulp bar, the bound of a small
# element is small, so an error in GELU's negative tail or in a small LayerNorm output is not hidden by the tensor's
# largest element.  The bounds are first-order worst cases built from these constants:
U16 = 2.0 ** -11   # fp16 unit roundoff: |fp16(y) - y| <= U16 |y| for a normal result ...
SUB16 = 2.0 ** -25  # ... and <= SUB16 where the result is subnormal (spacing 2^-24)
U32 = 2.0 ** -24   # fp32 unit roundoff (one IEEE operation)
UMMA = 2.0 ** -23  # per term of a tensor-core fp32 accumulation (products exact, sums possibly truncated: 1 ulp)


def _f64(a) -> np.ndarray:
    return np.asarray(a, dtype=np.float64)


def _w16(a) -> np.ndarray:
    return np.asarray(a, np.float32).astype(np.float16).astype(np.float64)


def _rounded16(y: np.ndarray, e) -> np.ndarray:
    """bound of |fp16(y') - y| given |y' - y| <= e"""
    return e * (1.0 + 2.0 * U16) + U16 * np.abs(y) + SUB16


def _erf(x: np.ndarray) -> np.ndarray:
    from scipy.special import erf
    return erf(x)


def ref_gelu_gemm(a, w, b):
    """FFN1: y = gelu(t), t = a . fp16(w) + b, gelu(t) = t/2 (1 + erf(t / sqrt 2)); a [.., K] fp16 values, w [F, K],
    b [F] fp32 -> (y, bound).

    Rounding points: the K products are exact in fp32 and accumulated there (error <= K UMMA sum|a w|), the bias add
    rounds once (U32 |t|): dt = K UMMA sum|a w| + U32 |t|, which moves gelu by <= |gelu'(t)| dt + 0.4 dt^2 (|gelu''| <= 0.8).
    gelu_erf: CUDA's erff is within 2 ulp (<= 2 U32 absolute, |erf| < 1), its argument's rounding moves it by <= 0.5 U32,
    and 1 + erf rounds by <= 2 U32; the two products round by U32 |y| each.  The fp16 output rounds by U16 |y| or, below
    2^-14, by SUB16.  In GELU's negative tail 1 + erff cancels, so the erf term is absolute, a multiple of U32 |t| / 2,
    not relative to the tiny y.  It is taken as 16 U32 |t| / 2: torch's vectorised fp32 GELU on the CPU (the emulation)
    is off by up to 12.2 U32 |t| / 2 over [-8, 8]; CUDA's erff by at most 4.5."""
    a, w = _f64(a), _w16(w)
    b = _f64(np.asarray(b, np.float32))
    K = a.shape[-1]
    t = a @ w.T + b
    y = 0.5 * t * (1.0 + _erf(t / np.sqrt(2.0)))
    dt = K * UMMA * (np.abs(a) @ np.abs(w).T) + U32 * np.abs(t)
    phi = np.exp(-0.5 * t * t) / np.sqrt(2.0 * np.pi)
    dgelu = np.abs(0.5 * (1.0 + _erf(t / np.sqrt(2.0))) + t * phi)
    e = dgelu * dt + 0.4 * dt * dt + 8.0 * U32 * np.abs(t) + 2.0 * U32 * np.abs(y)
    return y, _rounded16(y, e)


def ref_attention(qkv, mask, heads: int):
    """Attention from the QKV tensor [N, S, 3H] (fp16 values, channel part * H + 64 * head + d) and input_mask [N, S]
    -> (O [N, S, H], bound).

    s = q k / 8 + (-10000 where mask == 0), P = softmax(s), and -- as the contract rounds P to fp16 before P V --
    O = fp16(P) V, all in float64.  Engine: the score's 64 products accumulate in fp32 (64 UMMA sum|q k| / 8) and the mask
    add rounds (U32 |s|); s - max rounds (U32 |s - max|), expf is within 2 ulp: exp(s_j - max) is off by a factor within
    exp(+-r_j), r_j = ds_j + U32 |s_j - max| + 2 U32 (an error of the maximum itself cancels between numerator and sum).
    The sum of the S terms (each lane its S/4 in order, a butterfly, the key blocks in order) is within (S + 4) U32 of the
    sum of the computed terms, so the fp32 P_j is within eps_j = (1 + r_j)(1 + U32) / ((1 - R)(1 - (S + 4) U32)) - 1 of
    P_j, R = sum_i P_i r_i.  Rounded to fp16 it equals fp16(P_j) unless P_j (1 +- eps_j) straddles an fp16 rounding
    boundary, and then differs by at most the spacing f_j = fp16(P_j (1 + eps_j)) - fp16(P_j (1 - eps_j)).  P V accumulates
    S terms in fp32 ((S + 8) UMMA sum P|V|, with the key-block partials) and rounds to fp16 once:
    bound = U16 |O| + SUB16 + sum_j f_j |V_jd| + (S + 8) UMMA sum_j (fp16(P_j) + f_j) |V_jd|.
    So P's fp16 rounding is part of the value, not of the bound: normalising after P V (no rounded P) is an error here."""
    qkv = _f64(qkv)
    N, S, C3 = qkv.shape
    H = C3 // 3
    q, k, v = (qkv[..., j * H:(j + 1) * H].reshape(N, S, heads, 64).transpose(0, 2, 1, 3) for j in range(3))
    madd = np.where(np.asarray(mask) != 0, 0.0, MASK_ADD)[:, None, None, :]
    s = (q @ k.transpose(0, 1, 3, 2)) * 0.125 + madd
    m = s.max(-1, keepdims=True)
    ex = np.exp(s - m)
    P = ex / ex.sum(-1, keepdims=True)
    P16 = P.astype(np.float16).astype(np.float64)
    ds = 64 * UMMA * 0.125 * (np.abs(q) @ np.abs(k).transpose(0, 1, 3, 2)) + U32 * np.abs(s)
    r = np.expm1(ds + U32 * np.abs(s - m) + 2.0 * U32)
    R = (P * r).sum(-1, keepdims=True)
    eps = (1.0 + r) * (1.0 + U32) / ((1.0 - R) * (1.0 - (S + 4) * U32)) - 1.0
    f = (P * (1.0 + eps)).astype(np.float16).astype(np.float64) - (P * (1.0 - eps)).astype(np.float16).astype(np.float64)
    av = np.abs(v)
    O = P16 @ v
    e = f @ av + (S + 8) * UMMA * ((P16 + f) @ av)
    to = lambda x: x.transpose(0, 2, 1, 3).reshape(N, S, H)  # noqa: E731
    return to(O), to(_rounded16(O, e))


def ref_layernorm(x, gamma, beta, eps: float, dx=0.0):
    """LayerNorm over the last axis of x [.., C] (float64 values; dx: a bound of the engine's error in x itself, for the
    embedding sum) -> (y, bound), y = (x - mean) / sqrt(var + eps) * gamma + beta.

    Engine: mean = fp32 sum of C terms / C: dmu = C U32 mean|x| + U32 |mean| + mean(dx).  Each x_j - mean is then off by
    the common dmu plus its own rho_j = dx_j + U32 (|x_j - mean| + dmu + dx_j).  Since sum(x - mean) = 0, the squares sum to
    C var + C dmu^2 + 2 sum d_j rho_j - 2 dmu sum rho_j + sum rho^2: dvar = dmu^2 + (2 sqrt(sum d^2 sum rho^2) +
    2 dmu sum|rho| + sum rho^2) / C, plus the fp32 accumulation of the squares ((C + 2) U32 (var + dvar)).  rstd is the
    value of 1 / sqrt(var + eps) anywhere in var +- dvar, plus 3 U32 for the add, sqrt and division.  y is then off by
    |gamma| (|d| drstd + (dmu + rho) (rstd + drstd)), the three operations round by U32 (2 |gamma d rstd| + |y|), and the
    fp16 output by U16 |y| (or SUB16).  A row whose elements are all equal has d = 0, and an implementation of the
    contract gives beta there exactly (the sum of C equal fp16 values is exact in fp32); the bound does not assume it."""
    x = _f64(x)
    C = x.shape[-1]
    g = _f64(np.asarray(gamma, np.float32))
    b = _f64(np.asarray(beta, np.float32))
    dx = np.broadcast_to(_f64(dx), x.shape)
    mu = x.mean(-1, keepdims=True)
    d = x - mu
    var = (d * d).mean(-1, keepdims=True)
    rstd = 1.0 / np.sqrt(var + eps)
    y = d * rstd * g + b
    dmu = C * U32 * np.abs(x).mean(-1, keepdims=True) + U32 * np.abs(mu) + dx.mean(-1, keepdims=True)
    rho = dx + U32 * (np.abs(d) + dmu + dx)
    dvar = dmu * dmu + (2.0 * np.sqrt((d * d).sum(-1, keepdims=True) * (rho * rho).sum(-1, keepdims=True))
                        + 2.0 * dmu * rho.sum(-1, keepdims=True) + (rho * rho).sum(-1, keepdims=True)) / C
    dvar = dvar + (C + 2) * U32 * (var + dvar)
    lo = 1.0 / np.sqrt(np.maximum(var - dvar, 0.0) + eps)
    drstd = np.maximum(lo - rstd, rstd - 1.0 / np.sqrt(var + dvar + eps)) + 3.0 * U32 * lo
    e = np.abs(g) * (np.abs(d) * drstd + (dmu + rho) * (rstd + drstd)) + U32 * (2.0 * np.abs(g * d * rstd) + np.abs(y))
    return y, _rounded16(y, e)


def ref_embeddings(W, cfg, ids, segs):
    """The embedding operator: LayerNorm of (word + position) + type rows of the fp16 tables -> (y [N, S, H], bound).
    The two fp32 additions are off by <= U32 (|w + p| + |w + p + t|), which enters ref_layernorm as dx."""
    ids = np.clip(np.asarray(ids, dtype=np.int64), 0, cfg.vocab - 1)
    segs = np.clip(np.asarray(segs, dtype=np.int64), 0, cfg.types - 1)
    S = ids.shape[1]
    wp = _w16(W["embeddings.word_embeddings.weight"])[ids] + _w16(W["embeddings.position_embeddings.weight"])[:S][None]
    x = wp + _w16(W["embeddings.token_type_embeddings.weight"])[segs]
    dx = U32 * (np.abs(wp) + np.abs(x))
    return ref_layernorm(x, W["embeddings.LayerNorm.weight"], W["embeddings.LayerNorm.bias"], cfg.eps, dx)


def ref_pooler(W, last_hidden):
    """pooled = tanh(t), t = fp16(W) h[:, 0] + b from last_hidden_state [N, S, H] (fp16 values) -> (y [N, H], bound).
    Engine: the products are exact in fp32; each lane sums its 8 ceil(C / 256) terms in order and the warp adds lanes by
    a 5-step butterfly, within C U32 sum|w h| for C >= 64, and the bias add rounds (U32 |t|): dt moves tanh by
    <= (1 - y^2) dt + 0.4 dt^2 (|tanh''| <= 0.77); tanhf is within 2 ulp (4 U32 |y|).  The output is fp32."""
    h = _f64(last_hidden)[:, 0]
    w = _w16(W["pooler.dense.weight"])
    b = _f64(np.asarray(W["pooler.dense.bias"], np.float32))
    C = h.shape[-1]
    t = h @ w.T + b
    y = np.tanh(t)
    dt = C * U32 * (np.abs(h) @ np.abs(w).T) + U32 * np.abs(t)
    return y, (1.0 - y * y) * dt + 0.4 * dt * dt + 4.0 * U32 * np.abs(y) + 1e-30


def ref_ops(W, cfg, layer: int, mask, taps: Dict[str, np.ndarray]) -> Dict[str, tuple]:
    """The float64 references of one layer from the engine's taps (``emulate_ops``' names: x, qkv, attn_sum, ffn_sum
    ...) -> {"context", "attn_ln", "ffn", "out"}: (value, bound)."""
    p = f"encoder.layer.{layer}."
    return {
        "context": ref_attention(taps["qkv"], mask, cfg.heads),
        "attn_ln": ref_layernorm(taps["attn_sum"], W[p + "attention.output.LayerNorm.weight"],
                                 W[p + "attention.output.LayerNorm.bias"], cfg.eps),
        "ffn": ref_gelu_gemm(taps["attn_ln"], W[p + "intermediate.dense.weight"], W[p + "intermediate.dense.bias"]),
        "out": ref_layernorm(taps["ffn_sum"], W[p + "output.LayerNorm.weight"], W[p + "output.LayerNorm.bias"], cfg.eps),
    }


def bound_ratio(got, ref) -> float:
    """max |got - value| / bound over the elements (inf where got is not finite)"""
    value, bound = ref
    got = _f64(got)
    if not np.isfinite(got).all():
        return float("inf")
    return float((np.abs(got - value) / bound).max())


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
