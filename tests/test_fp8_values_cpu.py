"""The crafted FP8 cases of tests/fp8_values.py on the CPU: every plan builds and the engine accepts it, each category
holds the values it is meant to (ties are ties, near-ties one fp32 ulp off, saturating values at least 464), and a small
numpy model of each plausible wrong kernel disagrees with the FP8 oracle on at least one crafted position of the set
that targets it -- so tests/test_gpu_fp8_values.py would fail on a kernel built that way."""
import numpy as np
import pytest

from oracle import fp8_forward as O8
from oracle.int8_forward import fma32
from tensorrt_laboratory_b200 import builder, capi
from tests import fp8_values as V
from tests import test_gpu_fp8_values as G

f32 = np.float32
E4M3_MAX = f32(448)


def _e4m3_no_sat(t):
    """A conversion without satfinite: |t| >= 464 (rounds past 448) becomes NaN."""
    q = O8.e4m3(t)
    q[np.abs(t) >= 464] = 0x7F
    return q


def _e4m3_half_away(t):
    """Round half away from zero, saturating: the even neighbour of a tie replaced by the one away from zero."""
    q = O8.e4m3(t)
    v = O8.value(q).astype(np.float64)
    with np.errstate(invalid="ignore"):                                # sign(0) * inf
        up = O8.e4m3(np.nextafter(t, np.sign(t) * np.inf).astype(f32))  # the neighbour away from zero at a tie
    tie = (np.abs(t.astype(np.float64) - v) > 0) & np.isin(np.abs(t), V.TIES)
    q[tie] = up[tie]
    return q


def _e4m3_trunc(t):
    """Round toward zero (saturating)."""
    q = O8.e4m3(t)
    over = np.abs(O8.value(q).astype(np.float64)) > np.abs(t.astype(np.float64))
    q[over] = np.where(q[over] & 0x7F, q[over] - 1, q[over])          # one code toward zero
    return q


def _epilogue_set():
    lq, x = V.crafted(G.EPI_GEOMS[1], relu=False)
    (A, res, op), = V.epilogue_inputs(lq, x).values()
    return lq, x, A, op


def _wrong(A, op, res=None, kind=None, relu=None):
    """requant with one contract step replaced by the wrong model `kind`."""
    relu = op["relu"] if relu is None else relu
    Af = A.astype(f32)
    m = np.broadcast_to(op["m"].reshape(1, -1, 1, 1), A.shape)
    b = np.broadcast_to(op["b"].reshape(1, -1, 1, 1), A.shape)
    t = ((Af * m).astype(f32) + b).astype(f32) if kind == "two_roundings" else fma32(Af, m, b)
    if relu and kind == "relu_first":
        t = np.fmax(t, f32(0))
    if res is not None:
        r = np.broadcast_to(f32(op["r"]), A.shape)
        t = ((O8.value(res) * r).astype(f32) + t).astype(f32) if kind == "res_mul_add" else fma32(O8.value(res), r, t)
    if relu and kind != "relu_first":
        t = np.fmax(t, f32(0))
    if kind == "via_fp16":
        with np.errstate(over="ignore"):  # |t| > 65504 becomes inf, then 448
            return O8.e4m3(t.astype(np.float16).astype(f32))
    if kind == "half_away":
        return _e4m3_half_away(t)
    if kind == "trunc":
        return _e4m3_trunc(t)
    if kind == "no_sat":
        return _e4m3_no_sat(t)
    return O8.e4m3(t)


def _disagree(a, b):
    va, vb = O8.value(a), O8.value(b)
    return int((~((va == vb) | (np.isnan(va) & np.isnan(vb)))).sum())


# ------------------------------------------------------------------------------------------------------------------
# the crafted plans
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,geom,residual,relu", G.all_crafted_cases(), ids=lambda v: str(v) if isinstance(v, str) else None)
def test_every_crafted_plan_builds_and_is_accepted(name, geom, residual, relu):
    lq, x = V.crafted(geom, relu=relu, residual=residual)
    blob = builder.build_plan(lq, builder.PREC_FP8, x.shape[0], outputs=list(lq["tensor_scales"]))
    eng = capi.Engine(blob, inspect_only=True)
    try:
        assert eng.precision_name == "fp8"
    finally:
        eng.destroy()
    snap = V.expected(lq, x)
    assert np.array_equal(snap["data_q"], O8.e4m3(x))                # s = 1: the input codes are the inputs
    for op in lq["ops"]:
        if op.get("fp8"):
            assert (op["Wq"] == V.ONE).sum(axis=(1, 2, 3)).tolist() == [1] * op["cout"]
            assert ((op["Wq"] == 0) | (op["Wq"] == V.ONE)).all()


def test_one_hot_rows_reach_every_k_block_and_tap():
    """The probes' input channels fall in the first, middle, last and partial last 128-channel blocks, at every tap."""
    for geom in [G.EPI_DEEP, (320, 14, 14, 192, 3, 1, 1), (192, 14, 14, 320, 3, 1, 1)]:
        cin, k = geom[0], geom[4]
        lq, _ = V.crafted(geom)
        picks = next(op for op in lq["ops"] if op.get("fp8"))["picks"]
        blocks = {ci // 128 for _, ci in picks}
        assert blocks == set(range((cin + 127) // 128)), (geom, blocks)
        assert {tap for tap, _ in picks} == set(range(k * k))
        # the tie, near-tie and saturation probes (class 0) reach every block
        assert {ci // 128 for (_, ci), p in zip(picks, V.PROBES * 8) if p[0] == 0} == blocks, geom


def test_categories_hold_the_values_they_are_meant_to():
    lq, x, A, op = _epilogue_set()
    t = V.t_values(A, op, None)
    kinds = np.array([V.PROBES[c % len(V.PROBES)][3] for c in range(op["cout"])])
    per_c = lambda kind: np.broadcast_to(np.isin(kinds, kind).reshape(1, -1, 1, 1), t.shape)  # noqa: E731
    interior = A != 0
    at = np.abs(t)
    # ties: exactly midway between neighbouring E4M3 values, in the normal and in the subnormal binade
    ties = at[per_c("tie") & interior]
    assert np.isin(ties, V.TIES).all() and (ties < 2.0 ** -6).any() and (ties > 1).any()
    # near-ties: one fp32 ulp from a tie, on both sides
    near = at[per_c("near") & interior]
    up, down = np.nextafter(near, f32(0)), np.nextafter(near, f32(np.inf))
    assert (np.isin(up, V.TIES) | np.isin(down, V.TIES)).all()
    assert np.isin(up, V.TIES).any() and np.isin(down, V.TIES).any()
    # saturation: 448 <= |t| < 464 and |t| >= 464, both signs
    sat = t[per_c("sat") & interior]
    assert ((np.abs(sat) >= 448) & (np.abs(sat) < 464)).any() and (sat >= 464).any() and (sat <= -464).any()
    # bias-only at the padded border taps: A = 0 with t = b a tie
    border = per_c("bias") & ~interior
    assert border.any() and np.isin(at[border], V.TIES).any()
    # subnormal input codes are read
    assert (np.abs(O8.value(V.expected(lq, x)["data_q"])) < 2.0 ** -6).sum() > 1000
    # the case is exact: one-hot accumulators equal the input value they select
    assert np.isin(np.abs(A[interior]), V.MAGS).all()


@pytest.mark.parametrize("kind", ["two_roundings", "via_fp16", "half_away", "trunc", "no_sat"])
def test_wrong_epilogues_are_caught(kind):
    _, _, A, op = _epilogue_set()
    right = O8.requant(A, op, None)
    n = _disagree(_wrong(A, op, None, kind), right)
    print(f"[fp8 values] {kind}: {n} of {right.size} codes differ")
    assert n > 0


@pytest.mark.parametrize("kind,relu", [("res_mul_add", False), ("res_mul_add", True), ("relu_first", True)])
def test_wrong_residual_epilogues_are_caught(kind, relu):
    lq, x = V.crafted(G.EPI_GEOMS[1], relu=relu, residual=True)
    res_in = V.epilogue_inputs(lq, x)
    A, res, op = next(v for v in res_in.values() if v[1] is not None)
    right = O8.requant(A, op, res)
    n = _disagree(_wrong(A, op, res, kind), right)
    print(f"[fp8 values] {kind} relu={relu}: {n} of {right.size} codes differ")
    assert n > 0


def test_requant_keeps_nan_without_relu_and_zeroes_it_with_relu():
    op = dict(m=np.ones(2, f32), b=np.zeros(2, f32), r=f32(1), relu=False)
    A = np.array([np.nan, 1.0]).reshape(1, 2, 1, 1)
    q = O8.requant(A, op, None).ravel()
    assert (q[0] & 0x7F) == 0x7F and q[1] == V.ONE
    op["relu"] = True
    np.testing.assert_array_equal(O8.requant(A, op, None).ravel(), [0x00, V.ONE])


# ------------------------------------------------------------------------------------------------------------------
# quantize and average pool
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", G.QUANT_SCALES)
def test_quantize_set_discriminates(s):
    """q = e4m3(fl(h * fl(1/s))): h / s, the product in fp16, and a conversion without saturation each differ somewhere."""
    x = V.quantize_input(V.quantize_values(), s, G.QUANT_SHAPE, 0).ravel()
    inv = f32(1.0 / float(f32(s)))
    right = O8.e4m3((x * inv).astype(f32))
    wrong = {"no_sat": _e4m3_no_sat((x * inv).astype(f32))}
    if s != 1:  # at s = 1 the product is exact in any format
        wrong["fp16_product"] = O8.e4m3((x.astype(np.float16) * np.float16(inv)).astype(f32))
        wrong["divide"] = O8.e4m3((x / f32(s)).astype(f32))
    for k, q in wrong.items():
        assert _disagree(q, right) > 0, k
    # the set holds ties of the conversion at s = 1, subnormals, +-0 and values past 448 * s
    if s == 1:
        assert np.isin(np.abs(x), V.TIES).sum() >= 2 * len(V.TIES)
    assert (x == 0).any() and (np.abs(x) * inv >= 464).any() and ((np.abs(x) > 0) & (np.abs(x) * inv < 2.0 ** -6)).sum() > 100


@pytest.mark.parametrize("hw", G.POOL_HW)
def test_pool_sets_are_order_sensitive_where_the_sum_rounds(hw):
    """The pool kernel sums in pixel order: from HW >= 74 a reversed or pairwise sum gives other bits on the crafted set;
    below it the sum is exact and every order agrees."""
    q = V.pool_input_values(G.POOL_BATCH, G.POOL_C, hw, hw)
    k = f32(1.0 / (hw * hw))
    right = O8.avgpool_fp8(q, k).reshape(q.shape[:2])
    fwd, rev, pair = (V.pool_finish(s, k) for s in V._pool_orders(O8.value(q).reshape(q.shape[0], q.shape[1], -1)))
    np.testing.assert_array_equal(fwd, right)
    n_rev, n_pair = int((rev != right).sum()), int((pair != right).sum())
    print(f"[fp8 values] pool hw={hw}: reversed differs on {n_rev}, pairwise on {n_pair} of {right.size}")
    if hw * hw >= 74:
        assert n_rev > 0 and n_pair > 0
    else:
        assert n_rev == 0 and n_pair == 0


def test_gpu_file_case_counts():
    """The GPU file runs few engines: state them here so that growth is a decision."""
    assert G.engine_runs() <= 60, G.engine_runs()
