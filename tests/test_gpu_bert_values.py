"""GPU: the BERT kernels on the value sets of tests/bert_values.py -- peaked and one-hot attention, scores beyond expf's
range, masks that move or tie a row's maximum, GELU's negative tail, LayerNorm rows with a large offset, outlier channels
or no variance, saturated tanh in the pooler -- and at geometries seeded BERT-base never produces (hidden 64, 320 and
1024, QKV widths 192 and 960, FFN widths 320 and 1088, partial 128-row GEMM tiles).  Every operator is held to the
2-ulp bar against the fp16 emulation and to the elementwise float64 bounds (oracle/bert_forward.py, ref_*), each on
the engine's own inputs read back through tap bindings; launch names show which attention kernel ran."""
import numpy as np
import pytest

from oracle import bert_forward as O
from tensorrt_laboratory_b200 import builder, capi
from tests import bert_values as BV
from tests.helpers import rel_err
from tests.test_gpu_bert import TAPS
from tests.test_gpu_conv import TOL

pytestmark = pytest.mark.gpu

CHECKED = ("embeddings", "context", "ffn", "attn_ln", "out", "pooled_output")


class _Plan:
    def __init__(self, cfg, W, max_batch):
        self.eng = capi.Engine(builder.build_bert_plan(cfg, W, max_batch=max_batch, taps=TAPS))
        self.s = capi.Session(self.eng)

    def launch_names(self, N):
        return [self.s._lib.b2_context_launch_name(self.s.ctx, N, i).decode() for i in range(self.s.nb_launches(N))]

    def close(self):
        self.s.close()
        self.eng.destroy()


def _run(cfg, W, inp):
    N = inp["input_ids"].shape[0]
    p = _Plan(cfg, W, N)
    try:
        return p.s.infer_bindings(inp), p.launch_names(N)
    finally:
        p.close()


def _check(cfg, W, inp, out):
    """the 2-ulp bar and the elementwise bounds of every operator of layer 0 -> {tap: worst |error| / bound}"""
    taps = {k.split(".", 1)[-1] if k != "embeddings" else "x": v for k, v in out.items() if k in TAPS}
    want = O.emulate_ops(W, cfg, 0, inp["input_mask"], taps)
    for k, v in want.items():
        err = rel_err(taps[k], v)
        assert err <= TOL, f"{k}: rel err {err:.3e} > {TOL:.3e}"
    assert rel_err(out["embeddings"], O.emulate_embeddings(W, cfg, inp["input_ids"], inp["segment_ids"])) <= TOL
    assert np.array_equal(out["last_hidden_state"], out["l0.out"])
    ref = BV.references(W, cfg, inp, taps, out["last_hidden_state"])
    got = {"embeddings": taps["x"], "pooled_output": out["pooled_output"], **taps}
    ratios = {k: O.bound_ratio(got[k], ref[k]) for k in CHECKED}
    print(cfg.hidden, cfg.ffn, cfg.seq, {k: f"{v:.3f}" for k, v in ratios.items()})  # the worst |error| / bound
    bad = {k: v for k, v in ratios.items() if not v <= 1.0}
    assert not bad, f"elementwise bound exceeded (|error| / bound): {bad}"
    return ratios


def _attention_kernel(names, S):
    attn = [n.split(":")[0] for n in names if n.startswith("attention_f16_wgmma")]
    assert attn == ["attention_f16_wgmma_ks" if S > 128 else "attention_f16_wgmma"], names


@pytest.mark.parametrize("S", [64, 128, 384, 512])
@pytest.mark.parametrize("name", BV.SETS)
def test_value_set(gpu, name, S):
    cfg = BV.config(S)
    W, inp = BV.make(name, cfg)
    out, names = _run(cfg, W, inp)
    _attention_kernel(names, S)
    _check(cfg, W, inp, out)
    if name == "ln_constant":
        rows = BV.const_rows(inp)
        beta = W["embeddings.LayerNorm.bias"].astype(np.float16).astype(np.float32)
        assert np.array_equal(out["embeddings"][rows], np.broadcast_to(beta, out["embeddings"][rows].shape))
        beta = W["encoder.layer.0.attention.output.LayerNorm.bias"]
        assert np.array_equal(out["l0.attn_ln"][rows], np.broadcast_to(beta, out["l0.attn_ln"][rows].shape))


@pytest.mark.parametrize("S", [64, 384])
def test_non_binary_mask_values_attend_like_1(gpu, S):
    cfg = BV.config(S)
    W, inp = BV.make("last_block", cfg)
    p = _Plan(cfg, W, 2)
    try:
        want = p.s.infer_bindings(inp)
        for value in BV.MASK_VALUES:
            got = p.s.infer_bindings(BV.with_mask_value(inp, value))
            for k in want:
                assert np.array_equal(got[k], want[k]), (value, k)
    finally:
        p.close()


# hidden 64: one head, lanes 8-31 of the row kernels own no vector; 320: lanes own 2 or 1 vectors, QKV 960 (not a
# multiple of 128); 1024: BERT-large's 16 heads, every lane 4 vectors; FFN 1088 and 320: odd numbers of 64-wide blocks
# (FFN2 then has an odd number of K blocks, the last double-width step holds one); S = 64 at N = 1 and 3: M = 64 and
# 192, partial 128-row tiles through the GELU and residual epilogues
GEOMETRY = [
    dict(hidden=64, heads=1, ffn=256, seq=128, N=2),
    dict(hidden=64, heads=1, ffn=256, seq=512, N=2),
    dict(hidden=320, heads=5, ffn=1280, seq=384, N=2),
    dict(hidden=1024, heads=16, ffn=4096, seq=128, N=2),
    dict(hidden=1024, heads=16, ffn=4096, seq=512, N=1),
    dict(hidden=256, heads=4, ffn=1088, seq=128, N=2),
    dict(hidden=256, heads=4, ffn=320, seq=128, N=2),
    dict(hidden=256, heads=4, ffn=1024, seq=64, N=1),
    dict(hidden=256, heads=4, ffn=1024, seq=64, N=3),
]


@pytest.mark.parametrize("g", GEOMETRY, ids=lambda g: f"h{g['hidden']}_f{g['ffn']}_s{g['seq']}_n{g['N']}")
def test_geometry(gpu, g):
    g = dict(g)
    N = g.pop("N")
    cfg = BV.config(g.pop("seq"), **g)
    W, inp = BV.make("peaked", cfg, N)
    BV.scale(W, cfg, ("intermediate.dense.weight",), 12)  # and GELU's tails
    out, names = _run(cfg, W, inp)
    _attention_kernel(names, cfg.seq)
    _check(cfg, W, inp, out)


@pytest.mark.parametrize("hidden", [64, 320, 1024])
def test_pooler_operator(gpu, hidden):
    cfg = BV.config(128, hidden=hidden, heads=hidden // 64, ffn=2 * hidden)
    W, inp = BV.make("pooler_wide", cfg, 3)
    out, _ = _run(cfg, W, inp)
    ref = O.ref_pooler(W, out["last_hidden_state"])
    r = O.bound_ratio(out["pooled_output"], ref)
    assert r <= 1.0, r
    assert (1.0 - np.abs(ref[0]) < 1e-7).any() and (np.abs(ref[0]) < 0.1).any()  # saturated channels and linear ones


def test_peaked_batch_position_invariance_and_partial_batch(gpu):
    cfg = BV.config(64)
    W, inp = BV.make("peaked", cfg, 3)
    p = _Plan(cfg, W, 3)
    try:
        full = p.s.infer_bindings(inp)
        rev = p.s.infer_bindings({k: v[::-1].copy() for k, v in inp.items()})
        part = p.s.infer_bindings({k: v[1:2].copy() for k, v in inp.items()})
    finally:
        p.close()
    for k in full:
        assert np.array_equal(rev[k][::-1], full[k]), k
        assert np.array_equal(part[k], full[k][1:2]), k
