"""GPU: packed (padding-free) BERT plans, ``build_bert_plan(..., remove_padding=True)`` -- valid rows bit-identical to the
padded plan for right-padded masks at every sequence length, the zero-row and pooler contract, left padding and holes
against the oracle, every operator through taps, tactics, graph replay, contexts, InferenceManager, and the launch list."""
import numpy as np
import pytest

from oracle import bert_forward as O
from tensorrt_laboratory_b200 import bert, builder, capi
from tests.bert_packed_ref import packed_forward, right_padded
from tests.helpers import rel_err
from tests.test_gpu_bert import E2E_FP32_MARGIN
from tests.test_gpu_conv import TOL

pytestmark = pytest.mark.gpu

SMALL = bert.BertConfig(layers=2, hidden=256, heads=4, ffn=1024, vocab=1000, positions=128, seq=64)
TAPS = ["embeddings", "l0.qkv", "l0.context", "l0.attn_sum", "l0.attn_ln", "l0.ffn", "l0.ffn_sum", "l0.out"]


def _tokens(cfg, mask, seed=1):
    rng = np.random.default_rng(seed)
    N, S = mask.shape
    return dict(input_ids=rng.integers(0, cfg.vocab, (N, S)).astype(np.int32),
                segment_ids=rng.integers(0, cfg.types, (N, S)).astype(np.int32), input_mask=mask.astype(np.int32))


def _lengths(S, N=16, seed=0):
    """right-padded lengths that cross the 64-row key blocks, the 128-key blocks and the 128-row GEMM tiles"""
    special = [L for L in (1, 63, 64, 65, 127, 128, 129, S) if L <= S]
    rng = np.random.default_rng(seed)
    return special + [int(v) for v in rng.integers(1, S + 1, N - len(special))]


def _run(blob, inputs, options=None):
    eng = capi.Engine(blob)
    s = capi.Session(eng, options)
    try:
        return s.infer_bindings(inputs)
    finally:
        s.close()
        eng.destroy()


def _assert_valid_rows_identical(packed, padded, mask, keys):
    valid = mask != 0
    for k in keys:
        assert np.array_equal(packed[k][valid], padded[k][valid]), k
        assert not packed[k][~valid].any(), f"{k}: masked rows are not 0"


@pytest.mark.parametrize("S", [64, 128, 256, 384, 512])
def test_right_padded_valid_rows_bit_identical(gpu, S):
    cfg = bert.BertConfig(layers=2, seq=S)  # BERT-base widths; two layers keep the oracle-free comparison quick
    W = bert.random_weights(cfg, 1)
    mask = right_padded(S, _lengths(S))
    inp = _tokens(cfg, mask)
    taps = ["l0.context", "l1.qkv", "l1.ffn"]
    padded = _run(builder.build_bert_plan(cfg, W, max_batch=16, taps=taps), inp)
    packed = _run(builder.build_bert_plan(cfg, W, max_batch=16, taps=taps, remove_padding=True), inp)
    _assert_valid_rows_identical(packed, padded, mask, ["last_hidden_state"] + taps)
    assert np.array_equal(packed["pooled_output"], padded["pooled_output"])


def test_full_masks_give_the_padded_bits(gpu):
    cfg = bert.BertConfig(layers=2, seq=128)
    W = bert.random_weights(cfg, 2)
    inp = _tokens(cfg, np.ones((16, 128), np.int32))
    padded = _run(builder.build_bert_plan(cfg, W, max_batch=16, taps=TAPS), inp)
    packed = _run(builder.build_bert_plan(cfg, W, max_batch=16, taps=TAPS, remove_padding=True), inp)
    assert padded.keys() == packed.keys()
    for k in padded:
        assert np.array_equal(packed[k], padded[k]), k


def test_fully_masked_item_between_neighbours(gpu):
    cfg = bert.BertConfig(layers=2, seq=128)
    W = bert.random_weights(cfg, 3)
    mask = right_padded(128, [128, 70, 1, 0, 129 - 2, 64, 0, 33])
    inp = _tokens(cfg, mask)
    padded = _run(builder.build_bert_plan(cfg, W, max_batch=8), inp)
    packed = _run(builder.build_bert_plan(cfg, W, max_batch=8, remove_padding=True), inp)
    for n in (3, 6):
        assert not packed["last_hidden_state"][n].any()
        want = np.tanh(np.asarray(W["pooler.dense.bias"], np.float32))
        assert np.allclose(packed["pooled_output"][n], want, rtol=1e-6, atol=1e-7)
    keep = [n for n in range(8) if n not in (3, 6)]
    _assert_valid_rows_identical({k: v[keep] for k, v in packed.items()}, {k: v[keep] for k, v in padded.items()}, mask[keep],
                                 ["last_hidden_state"])
    assert np.array_equal(packed["pooled_output"][keep], padded["pooled_output"][keep])


def _ragged_masks(S, N, seed=4):
    """left padding, holes, position 0 masked, a single token, an empty item"""
    rng = np.random.default_rng(seed)
    mask = np.zeros((N, S), np.int32)
    for n in range(N):
        kind = n % 4
        if kind == 0:
            mask[n, S - int(rng.integers(1, S + 1)):] = 1                 # left padding
        elif kind == 1:
            mask[n] = rng.random(S) < 0.5                                  # holes
        elif kind == 2:
            mask[n, int(rng.integers(0, S)):int(rng.integers(S // 2, S + 1))] = 1
        else:
            mask[n] = rng.random(S) < 0.9
    mask[1, 0] = 0
    mask[2] = 0
    mask[5] = 0
    mask[5, int(S * 0.7)] = 1
    return mask


@pytest.mark.parametrize("S", [64, 128, 256])
def test_left_padding_and_holes_against_the_oracle(gpu, S):
    cfg = bert.BertConfig(**{**SMALL.__dict__, "seq": S, "positions": max(S, 128)})
    W = bert.random_weights(cfg, 5)
    mask = _ragged_masks(S, 8)
    inp = _tokens(cfg, mask)
    out = _run(builder.build_bert_plan(cfg, W, max_batch=8, remove_padding=True), inp)
    kw = dict(ids=inp["input_ids"], segs=inp["segment_ids"], mask=mask)
    h16, p16 = packed_forward(W, cfg, fp16=True, **kw)
    h32, p32 = packed_forward(W, cfg, fp16=False, **kw)
    assert not out["last_hidden_state"][mask == 0].any()
    for k, emu, ref in (("last_hidden_state", h16, h32), ("pooled_output", p16, p32)):
        gap = rel_err(emu, ref)
        assert rel_err(out[k], ref) <= gap + E2E_FP32_MARGIN, (k, rel_err(out[k], ref), gap)
        assert rel_err(out[k], emu) <= 2 * gap + 1e-6, (k, rel_err(out[k], emu), gap)


@pytest.mark.parametrize("S", [128, 384])
def test_every_operator_at_2_ulp_on_mixed_lengths(gpu, S):
    cfg = bert.BertConfig(**{**SMALL.__dict__, "layers": 1, "seq": S, "positions": S})
    W = bert.random_weights(cfg, 6)
    mask = _ragged_masks(S, 6)
    inp = _tokens(cfg, mask)
    out = _run(builder.build_bert_plan(cfg, W, max_batch=6, taps=TAPS, remove_padding=True), inp)
    valid = mask != 0
    # the oracle's padded attention gives the zero rows of the unpacked taps the weight exp(-10000) = 0: it attends over
    # each item's valid tokens, as the packed kernels do
    taps = {k.split(".", 1)[-1] if k != "embeddings" else "x": v for k, v in out.items() if k in TAPS}
    want = O.emulate_ops(W, cfg, 0, mask, taps)
    for k, v in want.items():
        err = rel_err(taps[k][valid], v[valid])
        assert err <= TOL, f"{k}: rel err {err:.3e} > {TOL:.3e}"
        assert not taps[k][~valid].any(), k


# GEMM tactics of the live-row kernels: N tile, ring depth (shallower and deeper than the K loop), double-width stages,
# and refused tactics (persistent, cluster, split-K) that must fall back to the tile kernel
TACTICS = [{}, {"bn": 32}, {"bn": 64}, {"bn": 128}, {"bn": 256}, {"stages": 1}, {"stages": 2}, {"stages": 8}, {"sps": 2},
           {"ws": 1}, {"cn": 2}, {"splits": 2}, {"autotune": 0}, {"graph": 0}]


@pytest.mark.parametrize("cfg", [SMALL, bert.BertConfig(layers=1, seq=128)], ids=["small", "base-1-layer"])
def test_tactics_and_graph_modes_bit_identical(gpu, cfg):
    W = bert.random_weights(cfg, 7)
    mask = right_padded(cfg.seq, _lengths(cfg.seq, 8, seed=2))
    inp = _tokens(cfg, mask)
    blob = builder.build_bert_plan(cfg, W, max_batch=8, taps=["l0.ffn"], remove_padding=True)
    padded = _run(builder.build_bert_plan(cfg, W, max_batch=8, taps=["l0.ffn"]), inp)
    base = None
    for opt in TACTICS:
        out = _run(blob, inp, opt)
        if base is None:
            base = out
            _assert_valid_rows_identical(out, padded, mask, ["last_hidden_state", "l0.ffn"])
        for k in base:
            assert np.array_equal(out[k], base[k]), (opt, k)


@pytest.fixture(scope="module")
def packed_base(gpu):
    cfg = bert.BertConfig(layers=2, seq=128)
    W = bert.random_weights(cfg, 8)
    blob = builder.build_bert_plan(cfg, W, max_batch=16, remove_padding=True)
    eng = capi.Engine(blob)
    s = capi.Session(eng)
    yield cfg, blob, s
    s.close()
    eng.destroy()


def test_partial_batch_replay_and_second_context(packed_base):
    cfg, blob, s = packed_base
    mask = _ragged_masks(128, 16, seed=9)
    inp = _tokens(cfg, mask, seed=3)
    full = s.infer_bindings(inp)
    again = s.infer_bindings(inp)  # graph replay with the same bindings
    part = s.infer_bindings({k: v[3:8].copy() for k, v in inp.items()})  # 5 items through the 16-item plan
    eng2 = capi.Engine(blob)
    s2 = capi.Session(eng2)
    try:
        other = s2.infer_bindings(inp)
    finally:
        s2.close()
        eng2.destroy()
    for k in full:
        assert np.array_equal(again[k], full[k]), k
        assert np.array_equal(part[k], full[k][3:8]), k
        assert np.array_equal(other[k], full[k]), k


def test_tuned_inference_manager_equals_direct(packed_base):
    cfg, blob, s = packed_base
    eng = capi.Engine(blob)
    eng.tune(4)
    tuned = builder.attach_tactics(blob, eng.tactics())
    eng.destroy()
    inps = [_tokens(cfg, _ragged_masks(128, 16, seed=k), seed=k) for k in (11, 12)]
    m = capi.InferenceManager(max_exec_concurrency=1)
    try:
        m.register_model("bert", tuned)
        m.update_resources()
        for inp in (inps[0], inps[1], inps[0]):  # one context: every request re-points the graph's binding nodes
            got = m.infer_bindings("bert", inp)
            want = s.infer_bindings(inp)
            for k in want:
                assert np.array_equal(got[k], want[k]), k
    finally:
        m.close()


@pytest.mark.parametrize("S", [128, 384])
def test_launch_list(gpu, S):
    cfg = bert.BertConfig(layers=2, seq=S)
    names = {}
    for packed in (False, True):
        eng = capi.Engine(builder.build_bert_plan(cfg, max_batch=4, remove_padding=packed))
        s = capi.Session(eng)
        names[packed] = [s._lib.b2_context_launch_name(s.ctx, 4, i).decode() for i in range(s.nb_launches(4))]
        s.close()
        eng.destroy()
    assert len(names[True]) <= len(names[False]) + 1
    attn = "attention_f16_wgmma_ks_varlen:" if S > 128 else "attention_f16_wgmma_varlen:"
    assert sum(n.startswith(attn) for n in names[True]) == cfg.layers, names[True]
    gemms = [n for n in names[True] if n.startswith("conv_tcgen05:")]
    assert len(gemms) == 4 * cfg.layers and all(" live" in n and " tiled" in n and " ws=" not in n for n in gemms), gemms
    assert any(" gelu" in n for n in gemms)
    assert not any(" live" in n or "varlen" in n for n in names[False])
    assert sum(n.startswith("output_unpack_rows:") for n in names[True]) == 1
