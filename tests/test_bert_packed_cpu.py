"""CPU: packed (padding-free) BERT plans without a device -- same bindings as the padded plan, padded plans that keep
their bytes, engine validation of packed op records (b2_engine_inspect), and the packed contract's reference against the
padded oracle."""
import hashlib
import re
import struct

import numpy as np
import pytest

from oracle import bert_forward as O
from tensorrt_laboratory_b200 import bert, builder, capi
from tests.bert_packed_ref import packed_forward, right_padded

SMALL = bert.BertConfig(layers=2, hidden=256, heads=4, ffn=1024, vocab=1000, positions=128, seq=64)
_OPV3 = 224
_FLAGS = 176 + 4 * 9  # OpRecV3.flags: after OpRec and groups, heads, vocab, positions, types, binding2, binding3, out2, eps


def _inspect(blob):
    eng = capi.Engine(blob, inspect_only=True)
    try:
        return [dict(x) for x in eng.bindings]
    finally:
        eng.destroy()


def test_packed_plan_has_the_padded_bindings(lib):
    for cfg in (SMALL, bert.BertConfig(seq=384)):
        kw = dict(max_batch=16, taps=["embeddings", "l0.context"])
        assert _inspect(builder.build_bert_plan(cfg, remove_padding=True, **kw)) == _inspect(builder.build_bert_plan(cfg, **kw))


# sha256 of padded BERT plans at the commit before packed plans existed: padded plans must keep their bytes
PADDED_PLAN_SHA256 = {
    "small_taps": "95092d1b0c695b5ce15f73e233b877a0846b26c23ae5806129c58de95a32e1b4",
    "base_s384": "ef7c4e228fd2b7da41043b108540cc6030315634d5b66cd646b51f9f70402778",
}


def test_padded_bert_plans_are_byte_identical():
    small = builder.build_bert_plan(SMALL, max_batch=4, taps=["embeddings", "l0.context"])
    assert hashlib.sha256(small).hexdigest() == PADDED_PLAN_SHA256["small_taps"]
    base = builder.build_bert_plan(bert.BertConfig(seq=384), max_batch=16)
    assert hashlib.sha256(base).hexdigest() == PADDED_PLAN_SHA256["base_s384"]
    assert builder.build_bert_plan(SMALL, max_batch=4, remove_padding=False) == builder.build_bert_plan(SMALL, max_batch=4)


def _ops(blob):
    nt, nops = struct.unpack_from("<II", blob, 20)
    at = 128 + nt * 96
    return {blob[at + i * _OPV3:at + i * _OPV3 + 64].rstrip(b"\0").decode(): at + i * _OPV3 for i in range(nops)}


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


def test_packed_flag_offset_matches_the_builder():
    ops = _ops(builder.build_bert_plan(SMALL, max_batch=2, remove_padding=True))
    blob = builder.build_bert_plan(SMALL, max_batch=2, remove_padding=True)
    assert struct.unpack_from("<I", blob, ops["l0.ffn1"] + _FLAGS)[0] == builder.FLAG_PACKED
    assert struct.unpack_from("<I", blob, ops["cast:last_hidden_state"] + _FLAGS)[0] == builder.FLAG_PACKED | builder.FLAG_ROWS_OUT


def _mutations(packed, padded):
    ops = _ops(packed)
    f = lambda name: ops[name] + _FLAGS  # noqa: E731
    pops = _ops(padded)
    qkv = ops["l0.qkv"]
    return [
        ("a GEMM not marked packed", _patch(packed, f("l0.ffn2"), "<I", 0), "not marked packed"),
        ("a LayerNorm not marked packed", _patch(packed, f("l1.out_ln"), "<I", 0), "not marked packed"),
        ("the pooler not marked packed", _patch(packed, f("pooler"), "<I", 0), "not marked packed"),
        ("attention not marked packed", _patch(packed, f("l0.attention"), "<I", 0), "not marked packed|S does not match"),
        ("cast not marked packed", _patch(packed, f("cast:last_hidden_state"), "<I", 1), "not marked packed"),
        ("packed cast without the rows layout", _patch(packed, f("cast:last_hidden_state"), "<I", 2), "packed plan holds"),
        ("packed op in a padded plan", _patch(padded, pops["l0.ffn1"] + _FLAGS, "<I", 2), "without a packed embedding"),
        ("packing index of S words", _patch(packed, _tensor_at(packed, "packing_index") + 76, "<I", SMALL.seq),
         "packing index|S does not match"),
        ("packed GEMM with a 3x3 window", _patch(packed, qkv + 84, "<I", 3), "dense 1x1|bad geometry"),
        ("packed GEMM with ReLU", _patch(packed, qkv + 96, "<I", 2 | 1), "dense 1x1"),
        ("attention reading another tensor", _patch(packed, ops["l0.attention"] + 72, "<i", _tensor_index(packed, "l0.qkv")),
         "packing index|S does not match|mask"),
    ]


def _tensor_index(blob, name):
    return (_tensor_at(blob, name) - 128) // 96


def test_malformed_packed_ops_are_rejected(lib):
    packed = builder.build_bert_plan(SMALL, max_batch=2, remove_padding=True)
    padded = builder.build_bert_plan(SMALL, max_batch=2)
    capi.Engine(packed, inspect_only=True).destroy()
    for what, bad, msg in _mutations(packed, padded):
        with pytest.raises(capi.B2Error) as ei:
            capi.Engine(bad, inspect_only=True)
        assert ei.value.code == 1 and re.search(msg, str(ei.value)), (what, str(ei.value))


def test_two_packed_embeddings_are_rejected(lib):
    # the embedding record copied over the first GEMM: two packed embeddings in one plan
    packed = builder.build_bert_plan(SMALL, max_batch=2, remove_padding=True)
    ops = _ops(packed)
    b = bytearray(packed)
    b[ops["l0.qkv"]:ops["l0.qkv"] + _OPV3] = packed[ops["embeddings"]:ops["embeddings"] + _OPV3]
    with pytest.raises(capi.B2Error) as ei:
        capi.Engine(bytes(b), inspect_only=True)
    assert ei.value.code == 1


@pytest.mark.parametrize("fp16", [False, True], ids=["fp32", "fp16"])
def test_packed_reference_is_the_padded_forward_on_valid_rows(fp16):
    cfg = SMALL
    W = bert.random_weights(cfg, 7)
    rng = np.random.default_rng(3)
    N, S = 5, cfg.seq
    ids = rng.integers(0, cfg.vocab, (N, S)).astype(np.int32)
    segs = rng.integers(0, cfg.types, (N, S)).astype(np.int32)
    mask = right_padded(S, [S, 1, 40, 0, 63])
    mask[4] = (rng.random(S) < 0.6).astype(np.int32)  # holes
    mask[4, 0] = 0  # position 0 masked: the pooler reads a zero row
    fwd = O.forward_fp16 if fp16 else O.forward_fp32
    h_pad, p_pad = fwd(W, cfg, ids, segs, mask)
    h, p = packed_forward(W, cfg, ids, segs, mask, fp16)
    valid = mask != 0
    assert not h[~valid].any(), "masked rows are exactly 0"
    # the padded forward gives a masked key the weight exp(-10000) = 0: its valid rows are the packed contract, up to
    # the summation order of two different torch computations (and, in fp16, the roundings that order moves)
    tol = 2e-3 if fp16 else 1e-5
    assert np.abs(h[valid] - h_pad[valid]).max() <= tol * np.abs(h_pad[valid]).max()
    bias = np.tanh(np.asarray(W["pooler.dense.bias"], np.float32))
    for n in range(N):
        want = p_pad[n] if mask[n, 0] else bias
        assert np.abs(p[n] - want).max() <= tol, n
    assert np.array_equal(p[3], np.tanh(np.asarray(W["pooler.dense.bias"], np.float32)))  # the empty item
