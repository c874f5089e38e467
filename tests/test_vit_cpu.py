"""CPU: Vision Transformer plans without a device -- the weight loader, the patch layout against a convolution, the fp16
emulation against the float64 model, the plan the builder writes and the engine's validation of ViT op records
(b2_engine_inspect)."""
import re
import struct

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

from oracle import vit_forward as V
from tensorrt_laboratory_b200 import builder, capi, vit
from tests.helpers import rel_err

SMALL = vit.VitConfig(layers=2, hidden=128, heads=2, ffn=256, patch=16, image=64, classes=10)
_OPV3 = 224
_FLAGS = 176 + 4 * 9


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


def _binding_at(blob, name):
    nt, nops, nb = struct.unpack_from("<III", blob, 20)
    at = 128 + nt * 96 + nops * _OPV3
    for i in range(nb):
        if blob[at + i * 128:at + i * 128 + 64].rstrip(b"\0").decode() == name:
            return at + i * 128
    raise KeyError(name)


def _patch(blob, off, fmt, value):
    b = bytearray(blob)
    struct.pack_into(fmt, b, off, value)
    return bytes(b)


def _hf_state_dict(cfg, seed):
    """the layout of a ViTForImageClassification state dict: "vit." on the encoder, the classifier without it, a pooler"""
    W = vit.random_weights(cfg, seed)
    sd = {("" if k.startswith("classifier.") else "vit.") + k: v for k, v in W.items()}
    sd["vit.pooler.dense.weight"] = np.zeros((cfg.hidden, cfg.hidden), np.float32)
    return W, sd


def test_load_weights_round_trip(tmp_path):
    W, sd = _hf_state_dict(SMALL, 3)
    for src in (sd, W):
        path = str(tmp_path / "w.npz")
        np.savez(path, **src)
        got = vit.load_weights(path, SMALL)
        assert got.keys() == W.keys()
        for k in W:
            assert np.array_equal(got[k], W[k]), k


def test_load_weights_names_the_bad_key():
    W, sd = _hf_state_dict(SMALL, 3)
    del sd["vit.encoder.layer.1.layernorm_after.bias"]
    with pytest.raises(KeyError, match=r"encoder\.layer\.1\.layernorm_after\.bias"):
        vit.load_weights(sd, SMALL)
    W["embeddings.position_embeddings"] = W["embeddings.position_embeddings"][:, :-1]
    with pytest.raises(ValueError, match=r"embeddings\.position_embeddings"):
        vit.load_weights(W, SMALL)


@pytest.mark.parametrize("p", [16, 32])
def test_patch_rows_times_the_reshaped_weight_is_the_convolution(p):
    rng = np.random.default_rng(p)
    x = rng.standard_normal((2, 3, 224, 224))
    w = rng.standard_normal((64, 3, p, p))
    want = TF.conv2d(torch.from_numpy(x), torch.from_numpy(w), stride=p).flatten(2).transpose(1, 2).numpy()
    got = V.patch_rows(x, p) @ w.reshape(64, 3 * p * p).T
    assert got.shape == want.shape == (2, (224 // p) ** 2, 64)
    assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()


# the emulation's distance from the float64 model on seeded ViT-B/16 (8 N(0, 1) images: 1.35e-3 of the largest logit);
# the GPU whole-network bars are built on this gap
B16_GAP_BOUND = 4e-3


def test_fp16_emulation_is_within_fp16_error_of_fp32():
    cfg = vit.VIT_B16
    W = vit.random_weights(cfg, 0)
    x = np.random.default_rng(1).standard_normal((2, 3, 224, 224)).astype(np.float32)
    l32, p32 = V.forward_fp32(W, cfg, x)
    l16, p16 = V.forward_fp16(W, cfg, x)
    gap = rel_err(l16, l32)
    assert 0 < gap <= B16_GAP_BOUND, gap
    assert np.abs(p16 - p32).max() <= 1e-3
    assert np.array_equal(l16.argmax(1), l32.argmax(1))
    # the logits depend on the image: the comparisons of top-1 classes are not all the same comparison
    assert np.abs(l32[0] - l32[1]).max() > 0.1 * np.abs(l32).max()


def test_blockwise_attention_is_attention():
    rng = np.random.default_rng(5)
    q, k, v = (torch.from_numpy(rng.standard_normal((1, 2, 197, 64)).astype(np.float32)) for _ in range(3))
    want = torch.softmax((q.double() @ k.double().transpose(-1, -2)) * 0.125, -1) @ v.double()
    got = V._attend_blocks(q, k, v)
    assert rel_err(got.numpy(), want.numpy()) < 2e-3


def test_plan_ops_and_bindings(lib):
    blob = builder.build_vit_plan(SMALL, max_batch=4, taps=["patches", "l0.qkv", "final_ln"])
    assert struct.unpack_from("<I", blob, 8)[0] == builder.VERSION_TRANSFORMER
    ops = _ops(blob)
    names = list(ops)
    layer = ["ln1", "qkv", "attention", "attn_out", "ln2", "ffn1", "ffn2"]
    assert names == (["patchify", "patch_embed", "tokens"] + [f"l{i}.{n}" for i in range(2) for n in layer] +
                     ["final_ln", "cls_head", "softmax", "cast:patches", "cast:l0.qkv", "cast:final_ln"])
    types = [struct.unpack_from("<I", blob, ops[n] + 64)[0] for n in names]
    assert types[:3] == [builder.OP_PATCHIFY, builder.OP_CONV, builder.OP_TOKENS]
    assert types[3:10] == [builder.OP_LAYERNORM, builder.OP_CONV, builder.OP_ATTENTION, builder.OP_CONV, builder.OP_LAYERNORM,
                           builder.OP_CONV, builder.OP_CONV]
    assert types[-6:-3] == [builder.OP_LAYERNORM, builder.OP_CLS_HEAD, builder.OP_SOFTMAX]
    flags = {n: struct.unpack_from("<I", blob, ops[n] + _FLAGS)[0] for n in names}
    assert flags["patchify"] == flags["patch_embed"] == flags["softmax"] == 0
    assert all(flags[n] == builder.FLAG_PACKED for n in names[2:-4])
    assert flags["cast:patches"] == builder.FLAG_ROWS_OUT
    assert flags["cast:l0.qkv"] == builder.FLAG_ROWS_OUT | builder.FLAG_PACKED
    eng = capi.Engine(blob, inspect_only=True)
    try:
        got = [(b["name"], b["is_input"], b["shape"]) for b in eng.bindings]
        flops = eng.flops(1)
    finally:
        eng.destroy()
    assert got == [("data", True, (3, 64, 64)), ("prob", False, (10,)), ("logits", False, (10,)), ("patches", False, (16, 768)),
                   ("l0.qkv", False, (17, 384)), ("final_ln", False, (17, 128))]
    assert flops > 0


def vit_gflop(cfg) -> float:
    """algorithmic GFLOP per image from the shapes: GEMMs, attention and the head"""
    H, F, P, L = cfg.hidden, cfg.ffn, cfg.patches, cfg.tokens
    layer = 2 * L * H * (3 * H + H + 2 * F) + 4 * L * L * H
    return (2 * P * H * 3 * cfg.patch ** 2 + cfg.layers * layer + 2 * H * cfg.classes) / 1e9


def test_engine_flop_count_matches_the_shapes(lib):
    for cfg, want in ((vit.VIT_B16, 35.1), (vit.VIT_B32, 8.8), (vit.VIT_L16, 123.2)):
        assert abs(vit_gflop(cfg) - want) < 0.1, (cfg, vit_gflop(cfg))  # the rounded figures DESIGN.md quotes
        eng = capi.Engine(builder.build_vit_plan(cfg, max_batch=1), inspect_only=True)
        try:
            assert abs(eng.flops(1) / 1e9 - vit_gflop(cfg)) < 0.001 * want
        finally:
            eng.destroy()


@pytest.mark.parametrize("kw, msg", [
    (dict(patch=14, image=224), "3 p\\^2 must be a multiple of 64"),
    (dict(hidden=800), "heads \\* 64"),
    (dict(heads=20, hidden=1280, ffn=1280), "at most 1024"),
    (dict(image=384), "at most 512"),
    (dict(image=232), "divisible by the patch size"),
    (dict(ffn=3000), "multiple of 64"),
])
def test_builder_refuses_bad_geometry(kw, msg):
    with pytest.raises(ValueError, match=msg):
        builder.build_vit_plan(vit.VitConfig(**{**SMALL.__dict__, **kw}), max_batch=1)


@pytest.mark.parametrize("prec", [builder.PREC_FP32, builder.PREC_INT8, builder.PREC_FP8, 7])
def test_builder_refuses_every_precision_but_fp16(prec):
    with pytest.raises(ValueError, match="(?i)fp16"):
        builder.build_vit_plan(SMALL, max_batch=1, precision=prec)


def vit_mutations(blob):
    """hand-corrupted copies of a ViT plan, one per validation rule -> [(what, blob, message pattern)]"""
    ops = _ops(blob)
    data = _binding_at(blob, "data")
    swapped = bytearray(blob)
    a, b = ops["tokens"], ops["l0.ln1"]
    swapped[a:a + _OPV3], swapped[b:b + _OPV3] = blob[b:b + _OPV3], blob[a:a + _OPV3]
    return [
        ("patch size 8 against 3 p^2 = 768 columns", _patch(blob, ops["patchify"] + 84, "<I", 8), "patchify"),
        ("patch size 12", _patch(blob, ops["patchify"] + 84, "<I", 12), "patchify"),
        ("image not divisible by the patch", _patch(blob, data + 84, "<i", 70), "patchify"),
        ("patch count against the tensor rows", _patch(blob, data + 88, "<i", 80), "patchify"),
        ("position table one row short", _patch(blob, ops["tokens"] + 136, "<Q", 17 * 128 * 2), "tokens"),
        ("index tensor of L + 1 words", _patch(blob, _tensor_at(blob, "packing_index") + 76, "<I", 18), "tokens.*packing index|packing index"),
        ("head weight of classes - 1 rows", _patch(blob, ops["cls_head"] + 136, "<Q", 9 * 128 * 2), "cls_head"),
        ("head of another class count", _patch(blob, ops["cls_head"] + 108, "<I", 9), "cls_head"),
        ("an encoder op before OP_TOKENS", bytes(swapped), "runs before the packed embedding"),
        ("tokens not marked packed", _patch(blob, ops["tokens"] + _FLAGS, "<I", 0), "tokens"),
    ]


def test_engine_refuses_corrupted_vit_plans(lib):
    blob = builder.build_vit_plan(SMALL, max_batch=2)
    capi.Engine(blob, inspect_only=True).destroy()
    for what, bad, msg in vit_mutations(blob):
        with pytest.raises(capi.B2Error) as ei:
            capi.Engine(bad, inspect_only=True)
        assert ei.value.code == 1 and re.search(msg, str(ei.value)), (what, str(ei.value))


def test_unpacked_attention_keeps_its_sequence_rule(lib):
    # a ViT attention record whose packed flag is cleared: S = 17 is refused as on any unpacked plan
    blob = builder.build_vit_plan(SMALL, max_batch=2)
    bad = _patch(blob, _ops(blob)["l0.attention"] + _FLAGS, "<I", 0)
    with pytest.raises(capi.B2Error, match="attention"):
        capi.Engine(bad, inspect_only=True)
