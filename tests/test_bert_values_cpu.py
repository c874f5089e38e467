"""CPU: the BERT value sets (tests/bert_values.py) and the float64 per-operator references with elementwise bounds
(oracle/bert_forward.py, ref_*), without a device.

* Every value set reaches the regime it is there for, so a later change to ``bert.random_weights`` cannot quietly flatten
  one of them.
* The fp16 emulation of the engine's numerics contract meets every elementwise bound on every set.
* Each of these wrong emulations breaks at least one bound on at least one set: tanh-form GELU, softmax without the
  maximum subtracted, one-pass variance E[x^2] - mean^2 in LayerNorm, the mask applied one key late, V of adjacent keys
  swapped, P normalised after P V instead of before (no fp16 P), and the pooler reading token 1.  The scale-relative
  2-ulp bar (TOL) of the older tests lets the first three through on seeded weights, and P normalised after P V as
  well; the mask and V mutations and the pooler reading token 1 fail it.
"""
import functools

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

from oracle import bert_forward as O
from tests import bert_values as BV
from tests.helpers import rel_err

TOL = 2.0 ** -9  # the scale-relative 2-ulp bar of the GPU tests (tests/test_gpu_conv.py)
FP16_MAX = 65504.0
CHECKED = ("embeddings", "context", "ffn", "attn_ln", "out", "pooled_output")


def _emulate(name, S, N=2):
    cfg = BV.config(S)
    W, inp = BV.make(name, cfg, N)
    rec = []
    h, p = O.forward_fp16(W, cfg, inp["input_ids"], inp["segment_ids"], inp["input_mask"], record=rec)
    taps = {"x": rec[0]["embeddings"].numpy(), **{k: v.numpy() for k, v in rec[1].items()}}
    return cfg, W, inp, taps, h, p


_cached = functools.lru_cache(maxsize=None)(_emulate)


def _ratios(cfg, W, inp, taps, h, p):
    ref = BV.references(W, cfg, inp, taps, h)
    got = {"embeddings": taps["x"], "pooled_output": p, **taps}
    return {k: O.bound_ratio(got[k], ref[k]) for k in CHECKED}


def _scores(cfg, taps):
    qkv = taps["qkv"].astype(np.float64)
    N, S, _ = qkv.shape
    H = cfg.hidden
    q, k = (qkv[..., j * H:(j + 1) * H].reshape(N, S, cfg.heads, 64).transpose(0, 2, 1, 3) for j in range(2))
    return (q @ k.transpose(0, 1, 3, 2)) * 0.125  # [N, heads, S, S], no mask


def _softmax(s, mask):
    s = s + np.where(mask != 0, 0.0, O.MASK_ADD)[:, None, None, :]
    e = np.exp(s - s.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


# ---- every set reaches its regime ------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", BV.SETS)
def test_every_tap_is_finite_and_fits_fp16(name):
    _, _, _, taps, _, p = _cached(name, 128)
    for k, v in taps.items():
        assert np.isfinite(v).all() and np.abs(v).max() < FP16_MAX, k
    assert np.isfinite(p).all()


def test_seeded_weights_stay_in_the_flat_regime():
    # the reason for the other sets: seeded BERT attention is nearly uniform, GELU near-linear, LayerNorm rows centred
    cfg, W, inp, taps, _, _ = _cached("seeded", 128)
    s = _scores(cfg, taps)
    assert np.abs(s).max() < 2.0 and _softmax(s, inp["input_mask"]).max() < 0.05
    assert np.abs(taps["attn_sum"].mean(-1)).max() < 0.5


def test_peaked_attention():
    cfg, _, inp, taps, _, _ = _cached("peaked", 128)
    med = float(np.median(_softmax(_scores(cfg, taps), inp["input_mask"]).max(-1)))
    assert 0.45 < med < 0.85, med


def test_one_hot_attention_exceeds_expf_range():
    cfg, _, inp, taps, _, _ = _cached("one_hot", 128)
    s = _scores(cfg, taps)
    rmax = s.max(-1)
    assert s.max() > 300 and np.median(rmax) > 88.7 and rmax.min() > 20, (s.max(), np.median(rmax), rmax.min())
    assert np.median(_softmax(s, inp["input_mask"]).max(-1)) > 0.99


def test_shifted_rows_lie_wholly_beyond_expf_range():
    cfg, _, _, taps, _, _ = _cached("shifted", 128)
    s = _scores(cfg, taps)
    assert (s.min(-1) > 88.7).sum() >= 16, "rows whose every exp(s) overflows without the maximum subtracted"
    assert (s.max(-1) < -103.0).sum() >= 16, "rows whose every exp(s) underflows without the maximum subtracted"


def test_masked_dominant_key():
    cfg, W, inp, taps, _, _ = _cached("masked_dominant", 128)
    j = int(np.flatnonzero(inp["input_mask"][0] == 0)[0])
    s = _scores(cfg, taps)[0]
    assert (s.argmax(-1) == j).sum() >= 8, "the masked key was the maximum of many rows"
    assert (_softmax(s[None], inp["input_mask"][:1])[..., j] == 0).all()


@pytest.mark.parametrize("S", [128, 384])
def test_tied_maxima_in_two_key_blocks(S):
    cfg, W, inp, taps, _, _ = _cached("tied_maxima", S)
    s = _scores(cfg, taps)[0]
    rmax = s.max(-1)
    ties = (s == rmax[..., None]).sum(-1) >= 2
    assert ties.sum() >= 4, "rows whose maximum is reached by two keys"
    keys = np.argwhere(s[ties] == rmax[ties][..., None])[:, 1]
    if S > 128:
        assert len(set(keys // 128)) >= 2, "the tied keys lie in different 128-key blocks"


@pytest.mark.parametrize("S", [128, 384])
def test_last_block_only(S):
    _, _, inp, _, _, _ = _cached("last_block", S)
    valid = np.flatnonzero(inp["input_mask"][-1])
    assert valid.min() >= S - (128 if S > 128 else S // 2) and len(valid) == (128 if S > 128 else S // 2)


def test_gelu_wide_reaches_the_negative_tail():
    _, W, _, taps, _, _ = _cached("gelu_wide", 128)
    w16 = W["encoder.layer.0.intermediate.dense.weight"].astype(np.float16).astype(np.float64)
    t = taps["attn_ln"].astype(np.float64) @ w16.T + W["encoder.layer.0.intermediate.dense.bias"]
    assert t.min() < -15 and t.max() > 15, (t.min(), t.max())
    assert ((t > -6) & (t < -3)).mean() > 0.1


def test_ln_offset_mean_dwarfs_std():
    _, _, _, taps, _, _ = _cached("ln_offset", 128)
    a = taps["attn_sum"].astype(np.float64)
    assert np.median(np.abs(a.mean(-1)) / a.std(-1)) > 100
    f = taps["ffn_sum"].astype(np.float64)
    assert np.abs(f).max() > 2000 and np.abs(f.mean(-1)).min() > 200


def test_ln_constant_rows_give_beta_exactly():
    cfg, W, inp, taps, _, _ = _cached("ln_constant", 128)
    rows = BV.const_rows(inp)
    assert rows.sum() > cfg.seq
    beta = np.float32(W["embeddings.LayerNorm.bias"]).astype(np.float16).astype(np.float32)
    assert np.array_equal(taps["x"][rows], np.broadcast_to(beta, taps["x"][rows].shape))
    a = taps["attn_sum"][rows]
    assert (a == a[:, :1]).all(), "var = 0 rows into attn_ln"
    beta = W["encoder.layer.0.attention.output.LayerNorm.bias"]
    assert np.array_equal(taps["attn_ln"][rows], np.broadcast_to(beta, a.shape))


def test_pooler_wide_spans_linear_to_saturated():
    _, W, _, _, h, _ = _cached("pooler_wide", 128)
    t = h[:, 0].astype(np.float64) @ W["pooler.dense.weight"].astype(np.float16).astype(np.float64).T
    assert (np.abs(t) > 10).any(axis=0).sum() >= 16 and (np.abs(t) < 0.1).all(axis=0).sum() >= 4


# ---- the emulation meets every bound -----------------------------------------------------------------------------------

@pytest.mark.parametrize("name", BV.SETS)
def test_emulation_meets_every_bound(name):
    r = _ratios(*_cached(name, 128))
    print(name, {k: f"{v:.3f}" for k, v in r.items()})  # the worst |error| / bound of each operator
    assert max(r.values()) <= 1.0, r


@pytest.mark.parametrize("name", ["shifted", "tied_maxima", "last_block", "ln_offset"])
def test_emulation_meets_every_bound_at_384(name):
    r = _ratios(*_cached(name, 384))
    assert max(r.values()) <= 1.0, r


# ---- wrong emulations break them ---------------------------------------------------------------------------------------

def _attend_no_max(q, k, v, madd, r):
    e = torch.exp((q @ k.transpose(-1, -2)) * 0.125 + madd[:, None, None, :])
    return r(e / e.sum(-1, keepdim=True)) @ v


def _attend_mask_late(q, k, v, madd, r):
    late = torch.cat([torch.zeros_like(madd[:, :1]), madd[:, :-1]], 1)
    return ATTEND(q, k, v, late, r)


def _attend_v_swapped(q, k, v, madd, r):
    S = v.shape[-2]
    return ATTEND(q, k, v[..., torch.arange(S).view(-1, 2).flip(-1).reshape(-1), :], madd, r)


def _attend_normalised_after(q, k, v, madd, r):
    s = (q @ k.transpose(-1, -2)) * 0.125 + madd[:, None, None, :]
    e = torch.exp(s - s.amax(-1, keepdim=True))
    return (e @ v) / e.sum(-1, keepdim=True)


def _ln_one_pass(x, g, b, eps):
    mean = x.mean(-1, keepdim=True)
    var = (x * x).mean(-1, keepdim=True) - mean * mean
    return (x - mean) * (1.0 / torch.sqrt(var + eps)) * O._t(g) + O._t(b)


ATTEND = O._attend
MUTATIONS = {
    "tanh_gelu": ("_gelu", lambda y: TF.gelu(y, approximate="tanh")),
    "no_max_subtraction": ("_attend", _attend_no_max),
    "one_pass_variance": ("_ln", _ln_one_pass),
    "mask_one_key_late": ("_attend", _attend_mask_late),
    "v_adjacent_keys_swapped": ("_attend", _attend_v_swapped),
    "p_normalised_after_pv": ("_attend", _attend_normalised_after),
    "pooler_reads_token_1": ("_pool", lambda x, w, b: torch.tanh(x[:, 1] @ w.T + b)),
}
# which of them the scale-relative 2-ulp bar lets through on seeded weights (S = 128), each operator judged on the
# mutated emulation's own inputs as the GPU tests judge the kernels
PASS_TOL_ON_SEEDED = {"tanh_gelu", "no_max_subtraction", "one_pass_variance", "p_normalised_after_pv"}


def _tol_errors(cfg, W, inp, taps, h, p):
    want = O.emulate_ops(W, cfg, 0, inp["input_mask"], taps)
    err = {k: rel_err(taps[k], v) for k, v in want.items()}
    err["embeddings"] = rel_err(taps["x"], O.emulate_embeddings(W, cfg, inp["input_ids"], inp["segment_ids"]))
    with torch.no_grad():
        ref = O._pool(torch.from_numpy(np.ascontiguousarray(h)), O._h(O._t(W["pooler.dense.weight"])), O._t(W["pooler.dense.bias"]))
    err["pooled_output"] = rel_err(p, ref.numpy())
    return err


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_mutation_breaks_a_bound(monkeypatch, mutation):
    attr, fn = MUTATIONS[mutation]
    with monkeypatch.context() as m:
        m.setattr(O, attr, fn)
        seeded = _emulate("seeded", 128)
    # the 2-ulp bar: the mutated emulation's taps against the correct emulation of each operator on those taps
    tol = max(_tol_errors(*seeded).values()) if all(np.isfinite(v).all() for v in seeded[3].values()) else float("inf")
    assert (tol <= TOL) == (mutation in PASS_TOL_ON_SEEDED), (mutation, tol)
    broken = {}
    for name in BV.SETS:
        with monkeypatch.context() as m:
            m.setattr(O, attr, fn)
            run = seeded if name == "seeded" else _emulate(name, 128)
        r = _ratios(*run)
        worst = max(r, key=r.get)
        if r[worst] > 1.0:
            broken[name] = (worst, r[worst])
            break
    print(mutation, f"2-ulp bar error on seeded {tol:.2e}", broken)
    assert broken, f"{mutation} meets every bound on every set"
