"""GPU: the BERT encoder path -- every operator against the fp16-emulating oracle at the 2-ulp bar (each judged on the
engine's own inputs, read back through tap bindings), GELU GEMM tactics, a small model and BERT-base end to end, padding
and batch-position invariance, and InferenceManager with tuned tactics."""
import numpy as np
import pytest

from oracle import bert_forward as O
from tensorrt_laboratory_b200 import bert, builder, capi
from tests.helpers import rel_err
from tests.test_gpu_conv import TOL

pytestmark = pytest.mark.gpu

SMALL = bert.BertConfig(layers=2, hidden=256, heads=4, ffn=1024, vocab=1000, positions=128, seq=64)
TAPS = ["embeddings", "l0.qkv", "l0.context", "l0.attn_sum", "l0.attn_ln", "l0.ffn", "l0.ffn_sum", "l0.out"]
# Whole-network bars.  Every operator matches the emulation to 2 ulp on its own inputs, but over 12 layers the last-bit
# differences of two fp16 computations (kernels and emulation, each rounding after every operator) grow to the size of
# the fp16 error itself: measured on the CPU (tests/test_bert_cpu.py), the emulation is 1.4e-3 (small model) and 2.2e-3
# (BERT-base; hidden state, relative to its max) from the fp32 model.  So the engine must be within the emulation's own
# gap (+ a margin) of fp32 -- the accuracy bar -- and within twice that gap of the emulation.
E2E_FP32_MARGIN = 1e-3


def _inputs(cfg, N, ragged=True, seed=1):
    rng = np.random.default_rng(seed)
    S = cfg.seq
    ids = rng.integers(0, cfg.vocab, (N, S)).astype(np.int32)
    segs = rng.integers(0, cfg.types, (N, S)).astype(np.int32)
    mask = np.ones((N, S), np.int32)
    if ragged:
        for n in range(N):
            mask[n, S - (n * 7) % S:] = 0 if n else 1  # sequence n has n*7 padded tokens (sequence 0 none)
    return dict(input_ids=ids, segment_ids=segs, input_mask=mask)


def _run(blob, inputs, options=None):
    eng = capi.Engine(blob)
    s = capi.Session(eng, options)
    try:
        return s.infer_bindings(inputs)
    finally:
        s.close()
        eng.destroy()


@pytest.mark.parametrize("S", [64, 128])
@pytest.mark.parametrize("ragged", [False, True])
def test_every_operator_at_2_ulp(gpu, S, ragged):
    cfg = bert.BertConfig(**{**SMALL.__dict__, "layers": 1, "seq": S})
    W = bert.random_weights(cfg, 3)
    inp = _inputs(cfg, 4, ragged)
    out = _run(builder.build_bert_plan(cfg, W, max_batch=4, taps=TAPS), inp)
    emb = O.emulate_embeddings(W, cfg, inp["input_ids"], inp["segment_ids"])
    assert rel_err(out["embeddings"], emb) <= TOL
    taps = {k.split(".", 1)[-1] if k != "embeddings" else "x": v for k, v in out.items() if k in TAPS}
    want = O.emulate_ops(W, cfg, 0, inp["input_mask"], taps)
    for k, v in want.items():
        err = rel_err(taps[k], v)
        assert err <= TOL, f"{k}: rel err {err:.3e} > {TOL:.3e}"
    assert np.array_equal(out["last_hidden_state"], out["l0.out"])


def test_clamped_ids_and_fully_padded_sequence(gpu):
    cfg = bert.BertConfig(**{**SMALL.__dict__, "layers": 1})
    W = bert.random_weights(cfg, 4)
    inp = _inputs(cfg, 2, ragged=False)
    inp["input_ids"][0, :5] = [-3, cfg.vocab, cfg.vocab + 100, 2**31 - 1, -(2**31)]
    inp["segment_ids"][0, :3] = [-1, 2, 99]
    inp["input_mask"][1] = 0  # no valid key at all: uniform attention, finite result
    out = _run(builder.build_bert_plan(cfg, W, max_batch=2, taps=["embeddings"]), inp)
    emb = O.emulate_embeddings(W, cfg, inp["input_ids"], inp["segment_ids"])
    assert rel_err(out["embeddings"], emb) <= TOL
    assert np.isfinite(out["last_hidden_state"]).all() and np.isfinite(out["pooled_output"]).all()


# every tactic a GELU layer can be given: N tile, ring depth, double-width stages, clusters, and (refused for GELU
# layers, so they must fall back to the tile kernel there) the persistent kernel; split-K changes the summation order
TACTICS = [{}, {"bn": 32}, {"bn": 64}, {"bn": 128}, {"bn": 256}, {"stages": 1}, {"stages": 4}, {"sps": 2}, {"cn": 2},
           {"ws": 1}, {"autotune": 0}]


def test_gelu_gemm_tactics_bit_identical(gpu):
    # hidden 512: every GEMM has K >= 8 blocks of 64, so split-K (at least 4 blocks per split) applies too
    cfg = bert.BertConfig(**{**SMALL.__dict__, "layers": 1, "hidden": 512, "heads": 8})
    W = bert.random_weights(cfg, 5)
    inp = _inputs(cfg, 4)
    blob = builder.build_bert_plan(cfg, W, max_batch=4, taps=TAPS)
    base = None
    for opt in TACTICS:
        out = _run(blob, inp, opt)
        want = O.emulate_ops(W, cfg, 0, inp["input_mask"], {k.split(".", 1)[-1] if k != "embeddings" else "x": v
                                                                   for k, v in out.items() if k in TAPS})
        assert rel_err(out["l0.ffn"], want["ffn"]) <= TOL, opt
        if base is None:
            base = out
        for k in base:
            assert np.array_equal(out[k], base[k]), (opt, k)
    for opt in ({"splits": 2}, {"simt": 1}):  # other summation orders: the 2-ulp bar against the emulation
        out = _run(blob, inp, opt)
        taps = {k.split(".", 1)[-1] if k != "embeddings" else "x": v for k, v in out.items() if k in TAPS}
        want = O.emulate_ops(W, cfg, 0, inp["input_mask"], taps)
        assert rel_err(taps["ffn"], want["ffn"]) <= TOL, opt


def test_gelu_layer_never_takes_the_persistent_kernel(gpu):
    cfg = bert.BertConfig(**{**SMALL.__dict__, "layers": 1})
    eng = capi.Engine(builder.build_bert_plan(cfg, max_batch=4))
    s = capi.Session(eng, {"ws": 1})
    names = [s._lib.b2_context_launch_name(s.ctx, 4, i).decode() for i in range(s.nb_launches(4))]
    s.close()
    ffn1 = [n for n in names if ":l0.ffn1" in n]
    assert len(ffn1) == 1 and ffn1[0].startswith("conv_tcgen05:") and " ws=" not in ffn1[0] and " gelu" in ffn1[0], names
    eng.destroy()


def test_small_model_end_to_end(gpu):
    W = bert.random_weights(SMALL, 6)
    inp = _inputs(SMALL, 8)
    out = _run(builder.build_bert_plan(SMALL, W, max_batch=8), inp)
    h16, p16 = O.forward_fp16(W, SMALL, **_kw(inp))
    h32, p32 = O.forward_fp32(W, SMALL, **_kw(inp))
    _check_e2e(out, h16, p16, h32, p32)


def _check_e2e(out, h16, p16, h32, p32):
    for k, emu, ref in (("last_hidden_state", h16, h32), ("pooled_output", p16, p32)):
        gap = rel_err(emu, ref)
        assert rel_err(out[k], ref) <= gap + E2E_FP32_MARGIN, (k, rel_err(out[k], ref), gap)
        assert rel_err(out[k], emu) <= 2 * gap, (k, rel_err(out[k], emu), gap)


def _kw(inp):
    return dict(ids=inp["input_ids"], segs=inp["segment_ids"], mask=inp["input_mask"])


@pytest.fixture(scope="module")
def base(gpu):
    W = bert.random_weights(bert.BERT_BASE, 0)
    blob = builder.build_bert_plan(bert.BERT_BASE, W, max_batch=16)
    eng = capi.Engine(blob)
    s = capi.Session(eng)
    yield W, blob, s
    s.close()
    eng.destroy()


def test_bert_base_matches_oracles(base):
    W, _, s = base
    inp = _inputs(bert.BERT_BASE, 16)
    out = s.infer_bindings(inp)
    h16, p16 = O.forward_fp16(W, bert.BERT_BASE, **_kw(inp))
    h32, p32 = O.forward_fp32(W, bert.BERT_BASE, **_kw(inp))
    _check_e2e(out, h16, p16, h32, p32)


def test_bert_base_batch_position_invariance_and_partial_batch(base):
    _, _, s = base
    inp = _inputs(bert.BERT_BASE, 16)
    full = s.infer_bindings(inp)
    rev = s.infer_bindings({k: v[::-1].copy() for k, v in inp.items()})
    part = s.infer_bindings({k: v[3:8].copy() for k, v in inp.items()})
    for k in full:
        assert np.array_equal(rev[k][::-1], full[k]), k
        assert np.array_equal(part[k], full[k][3:8]), k


def test_padding_invariance(base):
    _, _, s = base
    inp = _inputs(bert.BERT_BASE, 16)
    other = {k: v.copy() for k, v in inp.items()}
    pad = inp["input_mask"] == 0
    assert pad.any()
    other["input_ids"][pad] = np.random.default_rng(9).integers(0, bert.BERT_BASE.vocab, int(pad.sum()))
    a, b = s.infer_bindings(inp), s.infer_bindings(other)
    valid = ~pad
    assert np.array_equal(a["last_hidden_state"][valid], b["last_hidden_state"][valid])
    assert np.array_equal(a["pooled_output"], b["pooled_output"])


def test_inference_manager_tuned_equals_direct(base):
    _, blob, s = base
    inp1 = _inputs(bert.BERT_BASE, 16, seed=11)
    inp2 = _inputs(bert.BERT_BASE, 16, seed=12)
    eng = capi.Engine(blob)
    eng.tune(4)
    tuned = builder.attach_tactics(blob, eng.tactics())
    eng.destroy()
    m = capi.InferenceManager(max_exec_concurrency=1)
    try:
        m.register_model("bert", tuned)
        m.update_resources()
        for inp in (inp1, inp2, inp1):  # one context: every request re-points the graph's binding nodes
            got = m.infer_bindings("bert", inp)
            want = s.infer_bindings(inp)
            for k in want:
                assert np.array_equal(got[k], want[k]), k
    finally:
        m.close()
