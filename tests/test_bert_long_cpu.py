"""CPU: BERT plans at S = 256, 384 and 512 without a device -- the builder's range, the engine's validation of the plans
(bindings, FLOP count, refusals of other S), the oracle against its second witness and the emulation gap at S = 384."""
import importlib.util
import os
import re

import numpy as np
import pytest

from oracle import bert_forward as O
from tensorrt_laboratory_b200 import bert, builder, capi
from tests.test_bert_cpu import _inputs, _patch, _rel, _tensor_at

LONG = (256, 384, 512)
SMALL512 = bert.BertConfig(layers=2, hidden=256, heads=4, ffn=1024, vocab=1000, positions=512, seq=64)


def _cfg(base, S, **kw):
    return bert.BertConfig(**{**base.__dict__, "seq": S, **kw})


def _bench_bert():
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "bench_bert.py")
    spec = importlib.util.spec_from_file_location("bench_bert", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("S", LONG)
@pytest.mark.parametrize("base", [bert.BERT_BASE, SMALL512], ids=["base", "small"])
def test_long_plans_load_with_their_bindings(lib, base, S):
    cfg = _cfg(base, S, layers=1)
    eng = capi.Engine(builder.build_bert_plan(cfg, max_batch=2), inspect_only=True)
    try:
        b = {x["name"]: x for x in eng.bindings}
        assert all(b[n]["np_dtype"] == np.int32 and b[n]["shape"] == (S,) and b[n]["is_input"]
                   for n in ("input_ids", "segment_ids", "input_mask"))
        assert b["last_hidden_state"]["shape"] == (S, cfg.hidden) and b["pooled_output"]["shape"] == (cfg.hidden,)
    finally:
        eng.destroy()


# GFLOP per sequence of BERT-base: GEMMs 2 S H (3H + H + 2F) per layer + the pooler, attention 4 S^2 H per layer
BASE_GFLOP = {256: 45.90, 384: 70.67, 512: 96.64}


@pytest.mark.parametrize("S", LONG)
def test_bert_base_flops_follow_the_bench_formula(lib, S):
    cfg = _cfg(bert.BERT_BASE, S)
    eng = capi.Engine(builder.build_bert_plan(cfg, max_batch=1), inspect_only=True)
    try:
        want = _bench_bert().algorithmic_flops_per_sequence(cfg)
        assert abs(eng.flops(1) - want["total"]) <= 1e-9 * want["total"]
        assert abs(eng.flops(1) - BASE_GFLOP[S] * 1e9) < 0.01e9
        if S == 384:
            assert abs(want["gemm"] - 65.23e9) < 0.01e9 and abs(want["attention"] - 5.44e9) < 0.01e9
    finally:
        eng.destroy()


def test_builder_refuses_sequence_lengths_outside_the_set():
    for S in (320, 640):
        with pytest.raises(ValueError, match="multiple of 64"):
            builder.build_bert_plan(_cfg(SMALL512, S))
    with pytest.raises(ValueError, match="positions"):
        builder.build_bert_plan(_cfg(SMALL512, 384, positions=256))


@pytest.mark.parametrize("S", [320, 640])
def test_engine_refuses_attention_at_other_sequence_lengths(lib, S):
    blob = builder.build_bert_plan(_cfg(SMALL512, 384), max_batch=2)
    capi.Engine(blob, inspect_only=True).destroy()
    bad = _patch(_patch(_patch(blob, _tensor_at(blob, "l0.qkv") + 72, "<I", S), _tensor_at(blob, "l0.context") + 72, "<I", S),
                 _tensor_at(blob, "attention_mask_add") + 76, "<I", S)
    with pytest.raises(capi.B2Error) as ei:
        capi.Engine(bad, inspect_only=True)
    assert ei.value.code == 1 and re.search(f"S = {S}|S does not match|mask tensor", str(ei.value)), str(ei.value)


def test_oracle_matches_transformer_encoder_layer_at_384():
    cfg = _cfg(SMALL512, 384)
    W = bert.random_weights(cfg, 0)
    ids, segs, mask = _inputs(cfg, 3)
    rec = []
    O.forward_fp32(W, cfg, ids, segs, mask, record=rec)
    outs = O.witness_layers(W, cfg, rec[0]["embeddings"].numpy(), mask)
    for i, (w, r) in enumerate(zip(outs, rec[1:])):
        assert _rel(w, r["out"].numpy()) <= 1e-5, f"layer {i}"


def test_emulation_gap_on_seeded_bert_base_at_384():
    # the whole-network bars of tests/test_gpu_bert_long.py at S = 384: measured 2.1e-3 (hidden state, relative to its
    # max) and 3.0e-3 (pooled output), the size of the gap at S = 128
    cfg = _cfg(bert.BERT_BASE, 384)
    W = bert.random_weights(cfg, 0)
    ids, segs, mask = _inputs(cfg, 2)
    h32, p32 = O.forward_fp32(W, cfg, ids, segs, mask)
    h16, p16 = O.forward_fp16(W, cfg, ids, segs, mask)
    assert 2e-4 < _rel(h16, h32) < 4e-3
    assert _rel(p16, p32) < 5e-3
