"""GPU: Vision Transformer plans (``builder.build_vit_plan``) -- the patch and token kernels bit for bit, every operator at
2 fp16 ulp of the emulation on its own tapped inputs, attention at lengths that cross the 64-row and 128-key blocks, whole
networks against the float64 model, determinism (batch position, partial batch, replay, contexts, tactics, InferenceManager),
the launch list and the validation of corrupted plans on a device."""
import re

import numpy as np
import pytest

from oracle import bert_forward as BO
from oracle import vit_forward as V
from tensorrt_laboratory_b200 import builder, capi, vit
from tests.helpers import rel_err
from tests.test_gpu_bert import E2E_FP32_MARGIN
from tests.test_gpu_conv import TOL
from tests.test_vit_cpu import SMALL, vit_mutations

pytestmark = pytest.mark.gpu


def _images(n, cfg, seed):
    return np.random.default_rng(seed).standard_normal((n, 3, cfg.image, cfg.width)).astype(np.float32)


def _run(blob, x, options=None):
    eng = capi.Engine(blob)
    s = capi.Session(eng, options)
    try:
        return s.infer_bindings({"data": x})
    finally:
        s.close()
        eng.destroy()


def _tiny(patch, image=224, width=0, layers=1):
    return vit.VitConfig(layers=layers, hidden=128, heads=2, ffn=256, patch=patch, image=image, image_width=width, classes=10)


@pytest.mark.parametrize("p", [16, 32])
def test_patchify_is_exact(gpu, p):
    cfg = _tiny(p)
    blob = builder.build_vit_plan(cfg, max_batch=8, taps=["patches"])
    for n in (1, 3, 8):
        x = _images(n, cfg, seed=n) * 100.0  # values across the fp16 range, rounding at every binade
        got = _run(blob, x)["patches"]
        want = V.patch_rows(x, p).astype(np.float16).astype(np.float32)
        assert got.shape == want.shape
        assert np.array_equal(got, want), (p, n)


def test_tokens_are_exact_at_full_and_partial_batch(gpu):
    cfg = _tiny(16)
    W = vit.random_weights(cfg, 1)
    blob = builder.build_vit_plan(cfg, W, max_batch=8, taps=["patch_embed", "tokens"])
    x = _images(8, cfg, seed=2)
    full = _run(blob, x)
    for n in (8, 3):
        out = _run(blob, x[:n]) if n < 8 else full
        want = V.emulate_front(W, cfg, x[:n], patch_embed=out["patch_embed"])["tokens"]
        assert np.array_equal(out["tokens"], want), n  # rows of every item read back through the packing index
        for k in out:
            assert np.array_equal(out[k], full[k][:n]), (n, k)


def _taps(cfg):
    last = cfg.layers - 1
    return (["patches", "patch_embed", "tokens"] + [f"l0.{k}" for k in ("ln1", "qkv", "context", "attn_sum", "ln2", "ffn", "out")] +
            [f"l{last}.out", "final_ln"])


@pytest.mark.parametrize("cfg", [vit.VIT_B16, vit.VIT_B32], ids=["b16", "b32"])
def test_every_operator_at_2_ulp(gpu, cfg):
    W = vit.random_weights(cfg, 3)
    x = _images(4, cfg, seed=4)
    out = _run(builder.build_vit_plan(cfg, W, max_batch=4, taps=_taps(cfg)), x)
    front = V.emulate_front(W, cfg, x, patch_embed=out["patch_embed"])
    assert np.array_equal(out["patches"], front["patches"])
    assert rel_err(out["patch_embed"], front["patch_embed"]) <= TOL
    assert np.array_equal(out["tokens"], front["tokens"])
    T = {"x": out["tokens"], **{k: out["l0." + k] for k in ("ln1", "qkv", "context", "attn_sum", "ln2", "ffn")}}
    want = V.emulate_ops(W, cfg, 0, T)
    for k, v in want.items():
        err = rel_err(out["l0." + k], v)
        assert err <= TOL, f"l0.{k}: rel err {err:.3e} > {TOL:.3e}"
    # attention (L = 197 on the key-split kernel at S_k = 256; L = 50 on the 64-key kernel) against the float64 bound
    assert BO.bound_ratio(out["l0.context"], V.ref_attention(out["l0.qkv"], cfg.heads)) <= 1.0
    final_ln, logits = V.emulate_head(W, cfg, out[f"l{cfg.layers - 1}.out"], final_ln=out["final_ln"])
    assert rel_err(out["final_ln"], final_ln) <= TOL
    assert rel_err(out["logits"], logits) <= TOL
    assert BO.bound_ratio(out["logits"], V.ref_head(W, out["final_ln"][:, 0])) <= 1.0


# L = 50, 65, 129, 197, 257: P = 49 (7 x 7), 64 (8 x 8), 128 (8 x 16), 196 (14 x 14), 256 (16 x 16) patches of 16 pixels
LENGTHS = {50: (112, 112), 65: (128, 128), 129: (128, 256), 197: (224, 224), 257: (256, 256)}


@pytest.mark.parametrize("L", sorted(LENGTHS))
def test_attention_across_block_edges(gpu, L):
    h, w = LENGTHS[L]
    cfg = _tiny(16, h, w)
    assert cfg.tokens == L
    W = vit.random_weights(cfg, L)
    blob = builder.build_vit_plan(cfg, W, max_batch=4, taps=["l0.qkv", "l0.context"])
    x = _images(3, cfg, seed=L)
    out = _run(blob, x)
    assert BO.bound_ratio(out["l0.context"], V.ref_attention(out["l0.qkv"], cfg.heads)) <= 1.0, L
    assert rel_err(out["l0.context"], V.emulate_attention(out["l0.qkv"], cfg.heads)) <= TOL, L
    # rows of neighbouring items never leak: a different item 1 leaves items 0 and 2 as they were
    y = x.copy()
    y[1] = _images(1, cfg, seed=L + 1000)[0]
    other = _run(blob, y)
    for n in (0, 2):
        assert np.array_equal(other["l0.context"][n], out["l0.context"][n]), (L, n)
    assert not np.array_equal(other["l0.context"][1], out["l0.context"][1])


_E2E = {}


def _oracles(cfg, W, x):
    key = (cfg, x.shape[0], float(x[0, 0, 0, 0]))
    if key not in _E2E:
        _E2E[key] = (V.forward_fp32(W, cfg, x), V.forward_fp16(W, cfg, x))
    return _E2E[key]


@pytest.mark.parametrize("cfg, n, max_batch", [(vit.VIT_B16, 8, 8), (vit.VIT_B16, 3, 8), (vit.VIT_B32, 8, 8), (vit.VIT_L16, 2, 2)],
                         ids=["b16-8", "b16-partial-3", "b32-8", "l16-2"])
def test_whole_network_against_the_fp32_model(gpu, cfg, n, max_batch):
    W = vit.random_weights(cfg, 0)
    x = _images(n, cfg, seed=11)
    out = _run(builder.build_vit_plan(cfg, W, max_batch=max_batch), x)
    (l32, p32), (l16, p16) = _oracles(cfg, W, x)
    gap = max(rel_err(l16[i], l32[i]) for i in range(n))
    for i in range(n):
        assert rel_err(out["logits"][i], l32[i]) <= gap + E2E_FP32_MARGIN, i
        # the engine and the emulation round the same values to fp16 after differently ordered fp32 sums, so across 12 to
        # 24 layers they drift apart by about the emulation's own distance from fp32 (measured on an H100: 1.1e-3 to
        # 1.6e-3 of the largest logit, against gaps of 1.3e-3 to 1.6e-3), as the packed BERT test allows
        assert rel_err(out["logits"][i], l16[i]) <= 2 * gap + 1e-6, i
    assert np.abs(out["prob"] - p32).max() <= np.abs(p16 - p32).max() + E2E_FP32_MARGIN
    assert np.abs(out["prob"] - p16).max() <= 1e-3
    # top-1: the fp32 model's class wherever its lead over the second class exceeds twice the measured distance
    dist = np.abs(out["logits"] - l32).max(1)
    top2 = np.sort(l32, 1)[:, -2:]
    clear = top2[:, 1] - top2[:, 0] > 2 * dist
    assert clear.sum() * 2 >= n, (clear, top2, dist)
    assert np.array_equal(out["logits"].argmax(1)[clear], l32.argmax(1)[clear])


@pytest.fixture(scope="module")
def b16(gpu):
    cfg = vit.VIT_B16
    W = vit.random_weights(cfg, 5)
    blob = builder.build_vit_plan(cfg, W, max_batch=8)
    eng = capi.Engine(blob)
    s = capi.Session(eng)
    yield cfg, blob, s
    s.close()
    eng.destroy()


def test_batch_position_partial_batch_replay_and_second_context(b16):
    cfg, blob, s = b16
    x = _images(8, cfg, seed=21)
    full = s.infer_bindings({"data": x})
    again = s.infer_bindings({"data": x})
    perm = np.random.default_rng(0).permutation(8)
    permuted = s.infer_bindings({"data": x[perm]})
    part = s.infer_bindings({"data": x[:3]})
    eng2 = capi.Engine(blob)
    s2 = capi.Session(eng2)
    try:
        other = s2.infer_bindings({"data": x})
    finally:
        s2.close()
        eng2.destroy()
    for k in full:
        assert np.array_equal(again[k], full[k]), k
        assert np.array_equal(permuted[k], full[k][perm]), k
        assert np.array_equal(part[k], full[k][:3]), k
        assert np.array_equal(other[k], full[k]), k


def test_tuned_engine_and_inference_manager_give_the_direct_bits(b16):
    cfg, blob, s = b16
    eng = capi.Engine(blob)
    assert eng.tune(4) > 0
    tuned = builder.attach_tactics(blob, eng.tactics())
    eng.destroy()
    x = _images(8, cfg, seed=31)
    want = s.infer_bindings({"data": x})
    got = _run(tuned, x)
    for k in want:
        assert np.array_equal(got[k], want[k]), k
    m = capi.InferenceManager(max_exec_concurrency=1)
    try:
        m.register_model("vit", blob)  # untuned plan: tuned at registration
        m.update_resources()
        for batch in (x, x[:5], x):
            got = m.infer_bindings("vit", {"data": batch})
            direct = s.infer_bindings({"data": batch})
            for k in direct:
                assert np.array_equal(got[k], direct[k]), k
    finally:
        m.close()


@pytest.mark.parametrize("cfg, sk", [(vit.VIT_B16, 256), (vit.VIT_B32, 64)], ids=["b16", "b32"])
def test_launch_list(gpu, cfg, sk):
    eng = capi.Engine(builder.build_vit_plan(cfg, max_batch=4))
    s = capi.Session(eng)
    try:
        names = [s._lib.b2_context_launch_name(s.ctx, 4, i).decode() for i in range(s.nb_launches(4))]
    finally:
        s.close()
        eng.destroy()
    for k in ("patchify:", "tokens:", "cls_head:", "softmax:"):
        assert sum(n.startswith(k) for n in names) == 1, (k, names)
    assert not any(n.startswith("conv_simt") for n in names)
    attn = [n for n in names if n.startswith("attention")]
    kernel = "attention_f16_wgmma_ks_varlen:" if sk > 128 else "attention_f16_wgmma_varlen:"
    assert len(attn) == cfg.layers and all(n.startswith(kernel) and n.endswith(f" sk={sk}") for n in attn), attn
    gemms = [n for n in names if n.startswith("conv_tcgen05:")]
    assert len(gemms) == 1 + 4 * cfg.layers
    assert " live" not in gemms[0] and all(" live" in n for n in gemms[1:]), gemms


def test_device_refuses_corrupted_vit_plans(gpu):
    blob = builder.build_vit_plan(SMALL, max_batch=2)
    capi.Engine(blob).destroy()
    for what, bad, msg in vit_mutations(blob):
        with pytest.raises(capi.B2Error) as ei:
            capi.Engine(bad)
        assert ei.value.code == 1 and re.search(msg, str(ei.value)), (what, str(ei.value))
