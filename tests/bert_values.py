"""Value sets for the BERT kernels: weights and inputs that push softmax, GELU, LayerNorm and the pooler into the regimes
of trained checkpoints -- peaked attention, scores beyond expf's range, wide FFN activations, LayerNorm rows with a large
common offset, outlier channels or no variance at all, saturated tanh -- which seeded N(0, 0.02) weights never reach.
Each set starts from ``bert.random_weights`` and scales or overwrites some of it.  Shared by
tests/test_bert_values_cpu.py (each set reaches its regime; the fp16 emulation meets the float64 bounds, wrong
emulations do not) and tests/test_gpu_bert_values.py (the kernels meet them)."""
from __future__ import annotations

import numpy as np

from oracle import bert_forward as O
from tensorrt_laboratory_b200 import bert

BASE = bert.BertConfig(layers=1, hidden=256, heads=4, ffn=1024, vocab=1000, positions=512, seq=128)

SETS = ("seeded", "peaked", "one_hot", "shifted", "masked_dominant", "tied_maxima", "last_block", "gelu_wide",
        "ln_offset", "ln_constant", "pooler_wide")

CONST_TOKEN = 5          # ln_constant: the token whose word row is constant
CONST_WORD, CONST_EMB_BETA, CONST_ATTN_BIAS = 0.75, 0.5, 0.25  # fp16-exact, and so is every sum of them
SHIFT_KEY_BIAS = 1200.0  # shifted: added to channel 0 of every head's key


def config(S: int, **kw) -> bert.BertConfig:
    return bert.BertConfig(**{**BASE.__dict__, "seq": S, **kw})


def inputs(cfg, N: int, seed: int = 1):
    """random tokens and segments, every key valid"""
    rng = np.random.default_rng(seed)
    S = cfg.seq
    return dict(input_ids=rng.integers(0, cfg.vocab, (N, S)).astype(np.int32),
                segment_ids=rng.integers(0, cfg.types, (N, S)).astype(np.int32),
                input_mask=np.ones((N, S), np.int32))


def scale(W, cfg, keys, f):
    """W[layer parameter] *= f for every layer and each of `keys` (names after ``encoder.layer.{i}.``)"""
    for i in range(cfg.layers):
        for k in keys:
            W[f"encoder.layer.{i}.{k}"] = (W[f"encoder.layer.{i}.{k}"] * np.float32(f)).astype(np.float32)


_QK = ("attention.self.query.weight", "attention.self.query.bias", "attention.self.key.weight", "attention.self.key.bias")


def _layer0_scores(W, cfg, inp):
    """the emulation's attention scores of layer 0 (mask not applied) [N, heads, S, S]; the QKV GEMM does not depend on
    the mask"""
    rec = []
    O.forward_fp16(W, cfg, inp["input_ids"], inp["segment_ids"], np.ones_like(inp["input_mask"]), record=rec)
    H = cfg.hidden
    N, S, _ = rec[1]["qkv"].shape
    q, k = (rec[1]["qkv"][..., j * H:(j + 1) * H].reshape(N, S, cfg.heads, 64).transpose(1, 2) for j in range(2))
    return ((q @ k.transpose(-1, -2)) * 0.125).numpy()


def dominant_key(W, cfg, inp, n: int = 0) -> int:
    """the key of sequence n that is the row maximum of the most (head, query) rows"""
    s = _layer0_scores(W, cfg, inp)[n]
    return int(np.bincount(s.argmax(-1).ravel(), minlength=cfg.seq).argmax())


def make(name: str, cfg, N: int = 2, seed: int = 3):
    """-> (weights, inputs) of value set `name` for configuration `cfg`"""
    W = bert.random_weights(cfg, seed)
    inp = inputs(cfg, N)
    S = cfg.seq
    if name == "seeded":
        inp["input_mask"][-1, S - S // 8:] = 0  # a padded tail
    elif name in ("peaked", "shifted", "masked_dominant", "tied_maxima", "last_block"):
        scale(W, cfg, _QK, 8)   # query and key x 8: scores x 64, the median row's largest P about 0.6
        if name == "shifted":
            # + B on channel 0 of every head's key shifts row i of the scores by q_i0 B / 8: rows with q_i0 > 1 sit
            # wholly above expf's overflow (88.7), rows with q_i0 < -1 wholly below its underflow (-103)
            for i in range(cfg.layers):
                b = W[f"encoder.layer.{i}.attention.self.key.bias"]
                b[::64] += np.float32(SHIFT_KEY_BIAS)
        elif name == "masked_dominant":
            inp["input_mask"][0, dominant_key(W, cfg, inp)] = 0   # the maximum must come from another key
        elif name == "tied_maxima":
            # key j2 (half a sequence away: another 128-key block from S = 256) made identical to the dominant key j1:
            # same token, segment and position row, so every row whose maximum was j1 has two equal maxima
            j1 = dominant_key(W, cfg, inp)
            j2 = (j1 + S // 2) % S
            inp["input_ids"][0, j2] = inp["input_ids"][0, j1]
            inp["segment_ids"][0, j2] = inp["segment_ids"][0, j1]
            W["embeddings.position_embeddings.weight"][j2] = W["embeddings.position_embeddings.weight"][j1]
        elif name == "last_block":
            inp["input_mask"][-1, :S - (128 if S > 128 else S // 2)] = 0  # valid keys in the last block only
    elif name == "one_hot":
        scale(W, cfg, _QK, 30)  # scores up to about +-470: one key takes nearly all of P
    elif name == "gelu_wide":
        scale(W, cfg, ("intermediate.dense.weight",), 12)  # FFN1 pre-activations over about +-18
    elif name == "ln_offset":
        for i in range(cfg.layers):
            p = f"encoder.layer.{i}."
            W[p + "attention.output.dense.bias"] += np.float32(500.0)  # attn_ln: |mean| about 500 x its std
            b = W[p + "output.dense.bias"]
            b += np.float32(300.0)                                      # out: an offset and outlier channels
            b[[7, cfg.hidden // 2 + 3, cfg.hidden - 9]] += np.float32([3000.0, -3000.0, 2500.0])
    elif name == "ln_constant":
        # rows of token CONST_TOKEN: the embedding sum is the constant CONST_WORD (zero position and type rows), so
        # the embedding LayerNorm has var = 0 and must give its beta = CONST_EMB_BETA exactly; with the attention
        # output weights 0 and bias CONST_ATTN_BIAS the attention sum of those rows is constant too, and attn_ln gives
        # its beta (rounded to fp16 here, so "exactly" means the same bits)
        W["embeddings.word_embeddings.weight"][CONST_TOKEN] = CONST_WORD
        W["embeddings.position_embeddings.weight"][:] = 0.0
        W["embeddings.token_type_embeddings.weight"][:] = 0.0
        W["embeddings.LayerNorm.bias"][:] = CONST_EMB_BETA
        for i in range(cfg.layers):
            p = f"encoder.layer.{i}."
            W[p + "attention.output.dense.weight"][:] = 0.0
            W[p + "attention.output.dense.bias"][:] = CONST_ATTN_BIAS
            W[p + "attention.output.LayerNorm.bias"] = W[p + "attention.output.LayerNorm.bias"].astype(np.float16).astype(np.float32)
        inp["input_ids"][:, ::3] = CONST_TOKEN
        inp["input_ids"][-1, :] = CONST_TOKEN   # a sequence of equal rows: uniform attention
    elif name == "pooler_wide":
        # output channel j of the pooler scaled by 10^(-1 ... 2): tanh from its linear part to saturation
        W["pooler.dense.weight"] *= np.logspace(-1, 2, cfg.hidden, dtype=np.float32)[:, None]
    else:
        raise KeyError(name)
    return W, inp


def const_rows(inp) -> np.ndarray:
    """ln_constant: [N, S] True where the token is CONST_TOKEN"""
    return inp["input_ids"] == CONST_TOKEN


MASK_VALUES = (2, -1, -2 ** 31)  # non-zero input_mask values: each attends like 1


def with_mask_value(inp, value: int):
    out = {k: v.copy() for k, v in inp.items()}
    out["input_mask"][out["input_mask"] != 0] = value
    return out


def references(W, cfg, inp, taps, last_hidden):
    """float64 references of layer 0 from the engine's (or the emulation's) taps -> {tap: (value, bound)}:
    embeddings, context, ffn, attn_ln, out, and pooled_output from last_hidden_state"""
    ref = O.ref_ops(W, cfg, 0, inp["input_mask"], taps)
    ref["embeddings"] = O.ref_embeddings(W, cfg, inp["input_ids"], inp["segment_ids"])
    ref["pooled_output"] = O.ref_pooler(W, last_hidden)
    return ref
