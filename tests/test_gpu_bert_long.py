"""GPU: BERT encoders at S = 256, 384 and 512 on the key-split attention kernel -- every operator against the
fp16-emulating oracle at the 2-ulp bar (on the engine's own taps), masks that put a row's maximum in any key block, a
fully padded sequence, which attention kernel runs, BERT-base at S = 384 end to end, exact batch-position and padding
invariance, and InferenceManager with tuned tactics."""
import numpy as np
import pytest

from oracle import bert_forward as O
from tensorrt_laboratory_b200 import bert, builder, capi
from tests.helpers import rel_err
from tests.test_gpu_bert import TAPS, _check_e2e, _inputs, _kw, _run
from tests.test_gpu_conv import TOL

pytestmark = pytest.mark.gpu

SMALL512 = bert.BertConfig(layers=1, hidden=256, heads=4, ffn=1024, vocab=1000, positions=512, seq=384)
BASE384 = bert.BertConfig(seq=384)


def _cfg(S, **kw):
    return bert.BertConfig(**{**SMALL512.__dict__, "seq": S, **kw})


def _check_ops(cfg, W, inp, out):
    emb = O.emulate_embeddings(W, cfg, inp["input_ids"], inp["segment_ids"])
    assert rel_err(out["embeddings"], emb) <= TOL
    taps = {k.split(".", 1)[-1] if k != "embeddings" else "x": v for k, v in out.items() if k in TAPS}
    want = O.emulate_ops(W, cfg, 0, inp["input_mask"], taps)
    for k, v in want.items():
        err = rel_err(taps[k], v)
        assert err <= TOL, f"{k}: rel err {err:.3e} > {TOL:.3e}"
    assert np.array_equal(out["last_hidden_state"], out["l0.out"])


@pytest.mark.parametrize("N", [3, 4])
@pytest.mark.parametrize("S", [256, 384, 512])
@pytest.mark.parametrize("ragged", [False, True])
def test_every_operator_at_2_ulp(gpu, S, ragged, N):
    cfg = _cfg(S)
    W = bert.random_weights(cfg, 3)
    inp = _inputs(cfg, N, ragged)
    _check_ops(cfg, W, inp, _run(builder.build_bert_plan(cfg, W, max_batch=N, taps=TAPS), inp))


def test_row_maximum_in_any_key_block(gpu):
    cfg = _cfg(384)
    S = cfg.seq
    W = bert.random_weights(cfg, 7)
    inp = _inputs(cfg, 4, ragged=False)
    m = inp["input_mask"]
    m[1, :256] = 0       # valid keys in the last 128-key block only
    m[2, 10:] = 0        # valid keys in the first 10 tokens only
    m[3, :S - 1] = 0     # a single valid key, the last one
    _check_ops(cfg, W, inp, _run(builder.build_bert_plan(cfg, W, max_batch=4, taps=TAPS), inp))


def test_fully_padded_sequence(gpu):
    cfg = _cfg(512)
    W = bert.random_weights(cfg, 8)
    inp = _inputs(cfg, 2)
    inp["input_mask"][1] = 0  # no valid key at all: uniform attention over every key block
    out = _run(builder.build_bert_plan(cfg, W, max_batch=2, taps=TAPS), inp)
    assert np.isfinite(out["last_hidden_state"]).all() and np.isfinite(out["pooled_output"]).all()
    _check_ops(cfg, W, inp, out)


@pytest.mark.parametrize("S", [128, 256, 384, 512])
def test_attention_kernel_by_sequence_length(gpu, S):
    cfg = _cfg(S, layers=2)
    eng = capi.Engine(builder.build_bert_plan(cfg, max_batch=2))
    s = capi.Session(eng)
    try:
        names = [s._lib.b2_context_launch_name(s.ctx, 2, i).decode() for i in range(s.nb_launches(2))]
    finally:
        s.close()
        eng.destroy()
    attn = [n for n in names if n.startswith("attention_f16_wgmma")]
    kernel = "attention_f16_wgmma_ks" if S > 128 else "attention_f16_wgmma"
    assert [n.split(":")[0] for n in attn] == [kernel] * 2, names


@pytest.fixture(scope="module")
def base384(gpu):
    W = bert.random_weights(BASE384, 0)
    blob = builder.build_bert_plan(BASE384, W, max_batch=8)
    eng = capi.Engine(blob)
    s = capi.Session(eng)
    yield W, blob, s
    s.close()
    eng.destroy()


def test_bert_base_384_matches_oracles(base384):
    W, _, s = base384
    inp = _inputs(BASE384, 8)
    out = s.infer_bindings(inp)
    h16, p16 = O.forward_fp16(W, BASE384, **_kw(inp))
    h32, p32 = O.forward_fp32(W, BASE384, **_kw(inp))
    _check_e2e(out, h16, p16, h32, p32)


def test_bert_base_384_batch_position_invariance_and_partial_batch(base384):
    _, _, s = base384
    inp = _inputs(BASE384, 8)
    full = s.infer_bindings(inp)
    rev = s.infer_bindings({k: v[::-1].copy() for k, v in inp.items()})
    part = s.infer_bindings({k: v[3:6].copy() for k, v in inp.items()})
    for k in full:
        assert np.array_equal(rev[k][::-1], full[k]), k
        assert np.array_equal(part[k], full[k][3:6]), k


def test_bert_base_384_padding_invariance(base384):
    _, _, s = base384
    inp = _inputs(BASE384, 8)
    other = {k: v.copy() for k, v in inp.items()}
    pad = inp["input_mask"] == 0
    assert pad.any()
    other["input_ids"][pad] = np.random.default_rng(9).integers(0, BASE384.vocab, int(pad.sum()))
    a, b = s.infer_bindings(inp), s.infer_bindings(other)
    valid = ~pad
    assert np.array_equal(a["last_hidden_state"][valid], b["last_hidden_state"][valid])
    assert np.array_equal(a["pooled_output"], b["pooled_output"])


def test_bert_base_384_inference_manager_tuned_equals_direct(base384):
    _, blob, s = base384
    inp1 = _inputs(BASE384, 8, seed=11)
    inp2 = _inputs(BASE384, 8, seed=12)
    eng = capi.Engine(blob)
    eng.tune(4)
    tuned = builder.attach_tactics(blob, eng.tactics())
    eng.destroy()
    m = capi.InferenceManager(max_exec_concurrency=1)
    try:
        m.register_model("bert", tuned)
        m.update_resources()
        for inp in (inp1, inp2, inp1):
            got = m.infer_bindings("bert", inp)
            want = s.infer_bindings(inp)
            for k in want:
                assert np.array_equal(got[k], want[k]), k
    finally:
        m.close()
