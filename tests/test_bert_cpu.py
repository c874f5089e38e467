"""CPU: the BERT encoder path without a device -- the oracle against its second witness, the weight loader, the builder's
refusals, version-3 plan validation in the engine (b2_engine_inspect), and CNN plans that stay byte-identical."""
import hashlib
import struct

import numpy as np
import pytest

from oracle import bert_forward as O
from tensorrt_laboratory_b200 import bert, builder, capi

SMALL = bert.BertConfig(layers=2, hidden=256, heads=4, ffn=1024, vocab=1000, positions=128, seq=64)


def _inputs(cfg, N, seed=1):
    rng = np.random.default_rng(seed)
    mask = np.ones((N, cfg.seq), np.int32)
    for n in range(1, N):
        mask[n, cfg.seq - 7 * n:] = 0
    return (rng.integers(0, cfg.vocab, (N, cfg.seq)), rng.integers(0, cfg.types, (N, cfg.seq)), mask)


def _rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


@pytest.mark.parametrize("cfg", [SMALL, bert.BertConfig(layers=2)], ids=["small", "base-2-layers"])
def test_oracle_matches_transformer_encoder_layer(cfg):
    W = bert.random_weights(cfg, 0)
    ids, segs, mask = _inputs(cfg, 3)
    rec = []
    O.forward_fp32(W, cfg, ids, segs, mask, record=rec)
    outs = O.witness_layers(W, cfg, rec[0]["embeddings"].numpy(), mask)
    for i, (w, r) in enumerate(zip(outs, rec[1:])):
        assert _rel(w, r["out"].numpy()) <= 1e-5, f"layer {i}"


def test_emulation_gap_on_seeded_bert_base():
    # the gap between the fp16 emulation and the fp32 model on seeded BERT-base sets the whole-network bars of
    # tests/test_gpu_bert.py: measured 2.2e-3 (hidden state, relative to its max) and 2.8e-3 (pooled output)
    W = bert.random_weights(bert.BERT_BASE, 0)
    ids, segs, mask = _inputs(bert.BERT_BASE, 2)
    h32, p32 = O.forward_fp32(W, bert.BERT_BASE, ids, segs, mask)
    h16, p16 = O.forward_fp16(W, bert.BERT_BASE, ids, segs, mask)
    assert 2e-4 < _rel(h16, h32) < 4e-3
    assert _rel(p16, p32) < 5e-3


def test_loader_round_trip_and_errors(tmp_path):
    W = bert.random_weights(SMALL, 2)
    f = tmp_path / "w.npz"
    np.savez(f, **{"bert." + k: v for k, v in W.items()}, **{"cls.predictions.bias": np.zeros(3, np.float32)})
    got = bert.load_weights(str(f), SMALL)
    assert got.keys() == W.keys() and all(np.array_equal(got[k], W[k]) for k in W)
    assert builder.build_bert_plan(SMALL, str(f), max_batch=2) == builder.build_bert_plan(SMALL, W, max_batch=2)
    bad = dict(W)
    bad["encoder.layer.1.intermediate.dense.weight"] = np.zeros((1024, 255), np.float32)
    with pytest.raises(ValueError, match=r"encoder\.layer\.1\.intermediate\.dense\.weight"):
        bert.load_weights(bad, SMALL)
    del bad["encoder.layer.1.intermediate.dense.weight"]
    with pytest.raises(KeyError, match=r"encoder\.layer\.1\.intermediate\.dense\.weight"):
        bert.load_weights(bad, SMALL)


def test_builder_refuses_other_precisions_and_sequence_lengths():
    with pytest.raises(ValueError, match="fp16 only"):
        builder.build_bert_plan(SMALL, precision=builder.PREC_FP32)
    with pytest.raises(ValueError, match="INT8"):
        builder.build_bert_plan(SMALL, precision=builder.PREC_INT8)
    for S in (96, 192, 0):
        with pytest.raises(ValueError, match="multiple of 64"):
            builder.build_bert_plan(bert.BertConfig(**{**SMALL.__dict__, "seq": S}))


# sha256 of the plan blobs at the commit before transformer plans existed: CNN plans must stay byte-identical
CNN_PLAN_SHA256 = {
    "resnet50": "772e777068ec0ec7c17607ac5a60af0263135aa63f88b61b4b96ba737d6a4d74",
    "resnext50": "4002cdf58dccaef6039e5df004b2dee9af3164c3061746f959e42fd1a1d78664",
}


def test_cnn_plans_are_byte_identical():
    assert hashlib.sha256(builder.build_resnet_plan(50)).hexdigest() == CNN_PLAN_SHA256["resnet50"]
    assert hashlib.sha256(builder.build_resnext_plan(50)).hexdigest() == CNN_PLAN_SHA256["resnext50"]


def test_bert_plan_metadata(lib):
    blob = builder.build_bert_plan(bert.BERT_BASE, max_batch=16)
    assert struct.unpack_from("<I", blob, 8)[0] == builder.VERSION_TRANSFORMER
    eng = capi.Engine(blob, inspect_only=True)
    try:
        b = {x["name"]: x for x in eng.bindings}
        assert [x["name"] for x in eng.bindings] == ["input_ids", "segment_ids", "input_mask", "last_hidden_state", "pooled_output"]
        assert all(b[n]["np_dtype"] == np.int32 and b[n]["shape"] == (128,) and b[n]["is_input"]
                   for n in ("input_ids", "segment_ids", "input_mask"))
        assert b["last_hidden_state"]["shape"] == (128, 768) and b["pooled_output"]["shape"] == (768,)
        # 21.7 GFLOP of GEMMs + 0.6 GFLOP of attention per sequence
        assert abs(eng.flops(1) - 22.35e9) < 0.01e9
    finally:
        eng.destroy()


# ---- engine validation of version-3 records (plan_format.h OpRecV3) ----
_OPV3 = 224


def _layout(blob):
    nt, nops, nb = struct.unpack_from("<III", blob, 20)
    ops_at = 128 + nt * 96
    return nt, nops, nb, ops_at, ops_at + nops * _OPV3


def _op_index(blob, name):
    _, nops, _, ops_at, _ = _layout(blob)
    for i in range(nops):
        if blob[ops_at + i * _OPV3:ops_at + i * _OPV3 + 64].rstrip(b"\0").decode() == name:
            return ops_at + i * _OPV3
    raise KeyError(name)


def _tensor_at(blob, name):
    nt = struct.unpack_from("<I", blob, 20)[0]
    for i in range(nt):
        if blob[128 + i * 96:128 + i * 96 + 64].rstrip(b"\0").decode() == name:
            return 128 + i * 96
    raise KeyError(name)


def _patch(blob, off, fmt, value):
    b = bytearray(blob)
    struct.pack_into(fmt, b, off, value)
    return bytes(b)


# (description, mutation, message fragment)
def _mutations(blob):
    att, emb, ln, ffn1 = (_op_index(blob, n) for n in ("l0.attention", "embeddings", "l0.attn_ln", "l0.ffn1"))
    _, _, _, _, bind_at = _layout(blob)
    cast = _op_index(blob, "cast:last_hidden_state")
    return [
        ("heads*64 != hidden", _patch(blob, att + 180, "<I", 3), "heads \\* 64"),
        ("S of the mask tensor", _patch(blob, _tensor_at(blob, "attention_mask_add") + 76, "<I", 32), "S does not match|mask tensor"),
        ("S above 128", _patch(_patch(_patch(blob, _tensor_at(blob, "l0.qkv") + 72, "<I", 192), _tensor_at(blob, "l0.context") + 72, "<I", 192),
                               _tensor_at(blob, "attention_mask_add") + 76, "<I", 192), "S = 192|S does not match|mask tensor"),
        ("gamma/beta size", _patch(blob, ln + 152, "<Q", 256 * 4), "gamma / beta"),
        ("embedding table size", _patch(blob, emb + 136, "<Q", 16), "table / gamma / beta"),
        ("GELU with ReLU", _patch(blob, ffn1 + 96, "<I", 2 | 8 | 1), "GELU excludes ReLU"),
        ("int32 binding into a cast", _patch(blob, cast + 80, "<i", 0), "disagree|int32 binding"),
        ("int32 binding as a tensor's storage", _patch(blob, _tensor_at(blob, "l0.qkv") + 84, "<i", 0), "int32 binding input_ids"),
        ("embedding reads a float binding", _patch(blob, bind_at + 68, "<I", 0), "int32 input"),
        ("binding of S + 1 tokens", _patch(blob, bind_at + 128 + 80, "<i", 65), "shape \\[S"),
    ]


def test_malformed_transformer_ops_are_rejected(lib):
    blob = builder.build_bert_plan(SMALL, max_batch=2)
    capi.Engine(blob, inspect_only=True).destroy()
    for what, bad, msg in _mutations(blob):
        with pytest.raises(capi.B2Error) as ei:
            capi.Engine(bad, inspect_only=True)
        assert ei.value.code == 1 and __import__("re").search(msg, str(ei.value)), (what, str(ei.value))


def test_transformer_ops_need_a_version_3_plan(lib):
    blob = builder.build_bert_plan(SMALL, max_batch=2)
    with pytest.raises(capi.B2Error, match="version"):
        capi.Engine(_patch(blob, 8, "<I", 2), inspect_only=True)
