"""FP8 (E4M3) on the GPU at values and geometries ResNet never produces: the convolution epilogue bit for bit on exact
accumulators, the quantize kernel's ties, subnormals and saturation, the INT8 geometry cases of test_gpu_geometry.py
(section e) in FP8, inputs past the calibrated range, ResNet-50 at 200x264, and NaN / Inf inputs.

Crafted cases (tests/fp8_values.py) give every output channel a one-hot weight row, so each accumulator is exact and the
device's codes must equal the oracle's ``requant(A)`` exactly -- no accumulation interval.  Random-data twins of the
geometry cases are held to the interval of tests/test_gpu_fp8.py.  Every test asserts the launch names of the kernels
under test (conv_f8_tcgen05, quantize_f8, avgpool_f8, output_cast_f8), so a fallback cannot pass for them.
tests/test_fp8_values_cpu.py shows that each crafted set rejects a model of a plausible wrong kernel."""
import math

import numpy as np
import pytest

from oracle import fp8_forward as O8
from oracle.caffe_forward import caffe_forward
from tensorrt_laboratory_b200 import builder, graph, quantize, weights
from tests import fp8_values as V
from tests import helpers
from tests.test_gpu_fp8 import W_BITS, _codes, _within
from tests.test_gpu_geometry import I8_CHANNELS, I8_DEEP, I8_GEOMS, I8_POOL_HW, I8_TILES, resnet50_200x264

pytestmark = pytest.mark.gpu

FP8 = builder.PREC_FP8
f32 = np.float32
EPI_DEEP = I8_DEEP                                             # 3x3 through im2col, 18 K blocks: every ring wraps
EPI_GEOMS = [(320, 14, 14, 256, 1, 1, 0), EPI_DEEP]            # 1x1 tiled with a partial last K block; 3x3 im2col
QUANT_SCALES = [1.0, 0.875]                                    # fl(1 / 0.875) * 0.875 > 1: not a power of two
QUANT_SHAPE = (2, 64, 16, 16)
POOL_HW = I8_POOL_HW + [9]                                     # HW = 81: the fp32 sum rounds
POOL_BATCH, POOL_C = 3, 192
OVERDRIVE = 8.0                                                # inputs at 8x the calibration amax
SAT_SHARE = {False: 0.05, True: 0.05}                          # least share of +-448 codes past the calibrated range


def all_crafted_cases():
    """(name, geom, residual, relu) of every crafted convolution plan this file runs."""
    cases = [("epilogue", g, False, False) for g in EPI_GEOMS]
    cases += [("relu_residual", g, res, relu) for g in EPI_GEOMS for res, relu in [(False, True), (True, False), (True, True)]]
    cases += [("geometry", g, res, not res) for g in I8_GEOMS for res in (False, True)]
    cases += [("channels", (cin, 14, 14, cout, 3, 1, 1), False, False) for cin, cout in I8_CHANNELS]
    return cases


def engine_runs():
    """Engines this file builds and runs."""
    return (len(EPI_GEOMS) * len(I8_TILES) + len(EPI_GEOMS) * (1 + 2 * 2) + len(QUANT_SCALES) + 2 * len(I8_GEOMS) * 2
            + 2 * len(I8_CHANNELS) * 2 + 2 * len(POOL_HW) + 2 + 1 + 2 + 1)


def _launch(names, kind, op=None):
    return next((n for n in names if n.split(" ")[0].split(":")[0] == kind and (op is None or n.split(" ")[0] == f"{kind}:{op}")), None)


def _assert_kernels(names, *kinds):
    for k in kinds:
        assert _launch(names, k) is not None, (k, names)


def _same_values(got, want, what):
    """E4M3 values equal, NaN where NaN, +0 and -0 alike."""
    g, w = O8.value(got), O8.value(want)
    bad = ~((g == w) | (np.isnan(g) & np.isnan(w)))
    if bad.any():
        idx = np.argwhere(bad)[:5]
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} codes differ, e.g. at {idx.tolist()}: "
                             f"{g[bad][:5]} vs {w[bad][:5]}")


def _run_crafted(lq, x, options=None):
    """-> ({FP8 tensor: codes [N, C, H, W]}, launch names).  Every scale is 1, so each output is an E4M3 value."""
    names = list(lq["tensor_scales"])
    out = helpers.run_engine(lq, x, FP8, options=options, outputs=names)
    launches = list(helpers.LAST_LAUNCH_NAMES)
    codes = {}
    for k in names:
        y = np.asarray(out[k], f32)
        q = O8.e4m3(y)
        np.testing.assert_array_equal(O8.value(q), y)        # the output cast at s = 1 gives the values themselves
        codes[k] = q.reshape(x.shape[0], -1, *y.shape[2:])
    _assert_kernels(launches, "conv_f8_tcgen05", "quantize_f8", "output_cast_f8")
    return codes, launches


def _check_crafted(geom, relu=False, residual=False, options=None, seed=0):
    lq, x = V.crafted(geom, relu=relu, residual=residual, seed=seed)
    got, names = _run_crafted(lq, x, options)
    want = V.expected(lq, x)
    for k in lq["tensor_scales"]:
        _same_values(got[k], want[k], k)
    return lq, x, got, names


# ------------------------------------------------------------------------------------------------------------------
# 1. the epilogue, bit for bit on exact accumulators
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bn,st", I8_TILES)
@pytest.mark.parametrize("geom", EPI_GEOMS, ids=["1x1-tiled", "3x3-im2col-18kb"])
def test_fp8_epilogue_bit_exact_every_tactic(gpu, geom, bn, st):
    """Ties (normal and subnormal binades) and one fp32 ulp either side, fma-sensitive values, 448 <= |t| < 464 and
    |t| >= 464 with ReLU off, t = b at the padded border, subnormal operands: every code equals requant(A)."""
    _, _, _, names = _check_crafted(geom, options={"i8_bn": bn, "i8_stages": st})
    name = _launch(names, "conv_f8_tcgen05", "conv")
    assert f" bn={bn} st={st} " in name and (" tiled" in name) == (geom[4] == 1), name
    if geom == EPI_DEEP:
        assert " kblk=18" in name, name


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("relu,residual", [(False, True), (True, True)], ids=["res", "res-relu"])
@pytest.mark.parametrize("geom", EPI_GEOMS, ids=["1x1-tiled", "3x3-im2col-18kb"])
def test_fp8_fused_residual_bit_exact(gpu, geom, relu, residual, bn):
    """The residual codes of a one-hot shortcut, r != 1: t = fma(value(q_res), r, fma(A, m, b)), then [ReLU]."""
    _, _, _, names = _check_crafted(geom, relu=relu, residual=residual, options={"i8_bn": bn})
    assert sum(f" bn={bn} " in n for n in names if n.startswith("conv_f8_tcgen05")) == 2, names


@pytest.mark.parametrize("geom", EPI_GEOMS, ids=["1x1-tiled", "3x3-im2col-18kb"])
def test_fp8_relu_epilogue_bit_exact(gpu, geom):
    _check_crafted(geom, relu=True)


# ------------------------------------------------------------------------------------------------------------------
# 2. the quantize kernel, bit for bit
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", QUANT_SCALES)
def test_fp8_quantize_bit_exact(gpu, s):
    """Every E4M3 tie and one fp16 ulp either side, the subnormal range, +-0, values past 448 * s up to 65504."""
    lq = V.base_plan(64, QUANT_SHAPE[2], QUANT_SHAPE[3], 64, 1, 1, 0)
    V.set_scale(lq, "data_q", s)
    x = V.quantize_input(V.quantize_values(), s, QUANT_SHAPE, 1)
    out = helpers.run_engine(lq, x, FP8, outputs=["data_q"])
    _assert_kernels(helpers.LAST_LAUNCH_NAMES, "quantize_f8", "output_cast_f8")
    want = V.expected(lq, x, keep=["data_q"])["data_q"]
    np.testing.assert_array_equal(O8.e4m3((x * lq["ops"][0]["inv_scale"]).astype(f32)), want)
    np.testing.assert_array_equal(out["data_q"], (O8.value(want) * f32(s)).astype(f32))   # and the output cast


# ------------------------------------------------------------------------------------------------------------------
# 3. geometries and channel counts ResNet never produces (FP8 twins of test_gpu_geometry.py section e)
# ------------------------------------------------------------------------------------------------------------------
def _random_check(cin, h, w, cout, k, s, p, relu, residual, options=None, seed=0):
    """Random data, calibrated on itself: quantize bit-exact, every conv code within the accumulation interval."""
    net = builder.single_conv_net(cin, h, w, cout, k, s, p, relu=relu, residual=residual)
    low = graph.lower(net, weights.random_weights(net, seed))
    x = np.random.default_rng(seed + 1).standard_normal((3, cin, h, w)).astype(np.float16).astype(f32)
    lq = quantize.quantize_lowered(low, x, fmt="e4m3")
    names = list(lq["tensor_scales"])
    out = helpers.run_engine(lq, x, FP8, options=options, outputs=names)
    launches = list(helpers.LAST_LAUNCH_NAMES)
    _assert_kernels(launches, "conv_f8_tcgen05", "quantize_f8", "output_cast_f8")
    got = {n: _codes(out[n], lq["tensor_scales"][n]).reshape(3, -1, *out[n].shape[2:]) for n in names}
    np.testing.assert_array_equal(got["data_q"], V.expected(lq, x, keep=["data_q"])["data_q"])
    for op in lq["ops"]:
        if op.get("fp8"):
            _within(op, got[op["input"]], got[op["output"]], res=got[op["residual"]] if op["residual"] else None)
    return launches


@pytest.mark.parametrize("residual", [False, True], ids=["plain", "res"])
@pytest.mark.parametrize("geom", I8_GEOMS, ids=lambda g: f"{g[0]}x{g[1]}x{g[2]}-{g[3]}-k{g[4]}s{g[5]}p{g[6]}")
def test_fp8_geometry(gpu, geom, residual):
    """Stride 2 whose last window ends on the far edge, a non-square strided 1x1 through im2col, a non-square 3x3."""
    names = _random_check(*geom, relu=not residual, residual=residual, seed=15)
    _, _, _, names2 = _check_crafted(geom, relu=not residual, residual=residual, seed=16)
    for n in (names, names2):
        assert (" im2col" in _launch(n, "conv_f8_tcgen05", "conv")) == (geom[4] != 1 or geom[5] != 1), n


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("cin,cout", I8_CHANNELS)
def test_fp8_partial_channel_blocks(gpu, cin, cout, bn):
    """Cin 192 / 320: the last 128-channel K block is half full (last_cb_mmas).  Cout 320 pads to 384: N tile 256 does not
    divide it and falls back to 128, whose last tile holds 64 real channels (cout_real)."""
    used = bn if (cout + 127) // 128 * 128 % bn == 0 else 128
    names = _random_check(cin, 14, 14, cout, 3, 1, 1, relu=False, residual=False, options={"i8_bn": bn}, seed=13)
    _, _, _, names2 = _check_crafted((cin, 14, 14, cout, 3, 1, 1), options={"i8_bn": bn}, seed=14)
    for n in (names, names2):
        assert f" bn={used} " in _launch(n, "conv_f8_tcgen05", "conv"), n


@pytest.mark.parametrize("hw", POOL_HW)
def test_fp8_global_average_pool(gpu, hw):
    """fp32 sums in pixel order, bit for bit against avgpool_fp8 -- on random data, and on crafted codes where, at
    HW = 81, the sum rounds and another order would give other bits."""
    net = builder.single_conv_net(64, hw, hw, 320, 1, 1, 0, relu=False)
    net["layers"].append(dict(name="pool", type="Pooling", bottoms=["conv"], tops=["pool"], pool="AVE", kernel_size=hw, stride=1, pad=0))
    low = graph.lower(net, weights.random_weights(net, 19))
    x = np.random.default_rng(20).standard_normal((3, 64, hw, hw)).astype(np.float16).astype(f32)
    lq = quantize.quantize_lowered(low, x, fmt="e4m3")
    out = helpers.run_engine(lq, x, FP8, outputs=["conv", "pool"])
    _assert_kernels(helpers.LAST_LAUNCH_NAMES, "conv_f8_tcgen05", "avgpool_f8", "output_cast_f8")
    conv = _codes(out["conv"], lq["tensor_scales"]["conv"]).reshape(3, 320, hw, hw)
    pool_op = next(o for o in lq["ops"] if o["type"] == "avgpool")
    np.testing.assert_array_equal(out["pool"].reshape(3, -1), O8.avgpool_fp8(conv, pool_op["k_scale"]).reshape(3, -1).astype(f32))
    # crafted: the one-hot conv passes chosen codes through
    lq = V.pool_plan(POOL_C, hw, POOL_C)
    q = V.pool_input_values(POOL_BATCH, POOL_C, hw, hw)
    x = O8.value(q).astype(f32)
    out = helpers.run_engine(lq, x, FP8, outputs=["conv", "pool"])
    _assert_kernels(helpers.LAST_LAUNCH_NAMES, "conv_f8_tcgen05", "avgpool_f8", "output_cast_f8")
    np.testing.assert_array_equal(out["conv"], x)
    np.testing.assert_array_equal(out["pool"].reshape(POOL_BATCH, -1),
                                  O8.avgpool_fp8(q, f32(1.0 / (hw * hw))).reshape(POOL_BATCH, -1).astype(f32))


# ------------------------------------------------------------------------------------------------------------------
# 4. past the calibrated range
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("residual", [False, True], ids=["plain", "res"])
def test_fp8_inputs_past_the_calibrated_range(gpu, residual):
    """Calibrated on x, served 8x: the quantize kernel saturates bit for bit, every conv code lies in the interval, a
    share of them is +-448, and none is NaN."""
    net = builder.single_conv_net(128, 14, 14, 256, 3, 1, 1, relu=False, residual=residual)
    low = graph.lower(net, weights.random_weights(net, 31))
    x = np.random.default_rng(32).standard_normal((3, 128, 14, 14)).astype(np.float16).astype(f32)
    lq = quantize.quantize_lowered(low, x, fmt="e4m3")
    xs = (x * f32(OVERDRIVE)).astype(f32)                         # exact: a power of two
    names = list(lq["tensor_scales"])
    out = helpers.run_engine(lq, xs, FP8, outputs=names)
    _assert_kernels(helpers.LAST_LAUNCH_NAMES, "conv_f8_tcgen05", "quantize_f8", "output_cast_f8")
    got = {n: _codes(out[n], lq["tensor_scales"][n]).reshape(3, -1, 14, 14) for n in names}
    want_q = V.expected(lq, xs, keep=["data_q"])["data_q"]
    np.testing.assert_array_equal(got["data_q"], want_q)
    assert (np.abs(O8.value(want_q)) == 448).mean() > 0.3
    for op in lq["ops"]:
        if op.get("fp8"):
            c = got[op["output"]]
            _within(op, got[op["input"]], c, res=got[op["residual"]] if op["residual"] else None)
            v = O8.value(c)
            share = float((np.abs(v) == 448).mean())
            print(f"[fp8 values] {op['name']} at {OVERDRIVE}x amax: {share:.3f} of codes are +-448")
            assert not np.isnan(v).any() and share >= SAT_SHARE[residual]


def test_fp8_resnet50_200x264(gpu):
    """test_resnet50_200x264_int8's scheme with test_gpu_fp8._full_net_check's rules: the fp16 stem within fp16 tolerance,
    every bottleneck convolution on conv_f8_tcgen05, and downstream of the GPU's pool1 the last tensor no further from
    the FP8 oracle than that oracle is from the fp32 model (+ 1e-3).  The net ends at res5c (no classifier), so the
    distances are relative 2-norms: under the max norm of test_gpu_fp8 a single code one step away on the largest value
    of the 2 x 2048 x 7 x 9 map would decide."""
    net = resnet50_200x264()
    wts = weights.random_weights(net, 0)
    low = graph.lower(net, wts)
    lq = quantize.quantize_lowered(low, weights.synthetic_input(4, chw=(3, 200, 264), seed=4321), fmt="e4m3")
    x = weights.synthetic_input(2, chw=(3, 200, 264), seed=21)
    last = lq["output"]
    out = helpers.run_engine(lq, x, FP8, outputs=["pool1", last])
    names = helpers.LAST_LAUNCH_NAMES
    assert sum(n.startswith("conv_f8_tcgen05:") for n in names) == sum(1 for o in lq["ops"] if o.get("fp8"))
    assert not any(n.startswith("conv_i8") for n in names)
    _assert_kernels(names, "quantize_f8", "output_cast_f8")
    _, snaps = O8.fp8_forward(lq, x, keep=["pool1"])
    assert helpers.rel_err(out["pool1"], snaps["pool1"]) <= 4e-3
    oracle = O8.fp8_forward(lq, x, start_from={"pool1": out["pool1"].astype(np.float64)})
    ref = caffe_forward(net, wts, x).reshape(2, -1)
    def rel2(a, b):
        return float(np.linalg.norm(np.asarray(a, np.float64) - b) / np.linalg.norm(b))

    gap, dist = rel2(oracle, ref), rel2(out[last].reshape(2, -1), oracle)
    print(f"[fp8 values] ResNet-50 200x264: {last} distance {dist:.2e}, oracle vs fp32 {gap:.2e}")
    assert dist <= gap + 1e-3, (dist, gap)


# ------------------------------------------------------------------------------------------------------------------
# 5. NaN and Inf inputs
# ------------------------------------------------------------------------------------------------------------------
NAN_AT, PINF_AT, NINF_AT = (0, 5, 3, 4), (1, 7, 9, 9), (2, 0, 0, 13)


@pytest.mark.parametrize("relu", [False, True], ids=["linear", "relu"])
def test_fp8_non_finite_inputs(gpu, relu):
    """Dense weights without a zero code: quantize gives NaN -> NaN and +-Inf -> +-448; the convolution gives NaN at every
    output whose window holds the NaN pixel without ReLU, 0 there with ReLU (fmaxf), and the interval elsewhere."""
    net = builder.single_conv_net(128, 14, 14, 128, 3, 1, 1, relu=relu)
    low = graph.lower(net, weights.random_weights(net, 41))
    x = np.random.default_rng(42).standard_normal((3, 128, 14, 14)).astype(np.float16).astype(f32)
    lq = quantize.quantize_lowered(low, x, fmt="e4m3")
    conv = lq["ops"][1]
    conv["Wq"] = np.where(conv["Wq"] & 0x7F, conv["Wq"], np.uint8(0x01))   # no zero weight: no NaN x 0 in this test
    x[NAN_AT], x[PINF_AT], x[NINF_AT] = np.nan, np.inf, -np.inf
    out = helpers.run_engine(lq, x, FP8, outputs=["data_q", "conv"])
    _assert_kernels(helpers.LAST_LAUNCH_NAMES, "conv_f8_tcgen05", "quantize_f8", "output_cast_f8")
    s = lq["tensor_scales"]
    yq = out["data_q"]
    assert np.isnan(yq[NAN_AT]) and yq[PINF_AT] == f32(448 * f32(s["data_q"])) and yq[NINF_AT] == -f32(448 * f32(s["data_q"]))
    finite = np.isfinite(x)
    q = np.full(x.shape, 0x7F, np.uint8)
    q[finite] = _codes(yq[finite], s["data_q"])
    q[PINF_AT], q[NINF_AT] = 0x7E, 0xFE
    np.testing.assert_array_equal(q, V.expected(lq, x, keep=["data_q"])["data_q"])
    y = out["conv"]
    A, P = O8.conv_fp8(q, conv)
    hit = np.isnan(A)
    assert hit.sum() == 3 * 3 * 128                                 # the 3x3 window positions, every output channel
    v = np.full(y.shape, np.nan, f32)
    v[~np.isnan(y)] = O8.value(_codes(y[~np.isnan(y)], s["conv"]))
    if relu:
        assert (v[hit] == 0).all(), v[hit][:8]
    else:
        assert np.isnan(v[hit]).all(), f"{int((~np.isnan(v[hit])).sum())} outputs lost the NaN, e.g. {v[hit][~np.isnan(v[hit])][:5]}"
    assert not np.isnan(v[~hit]).any()
    K = 9 * 128
    eps = math.ceil(K / 32) * 2.0 ** -W_BITS
    lo = O8.value(O8.requant(np.where(hit, 0, A - eps * P), conv, None))[~hit]
    hi = O8.value(O8.requant(np.where(hit, 0, A + eps * P), conv, None))[~hit]
    assert ((lo <= v[~hit]) & (v[~hit] <= hi)).all()


def test_fp8_nan_times_zero_weight(gpu):
    """One-hot weights: one output channel multiplies the NaN input code by 1.0, every other output whose window holds it
    multiplies it by the zero code.  IEEE gives NaN for NaN x 0, and so does the oracle."""
    geom = (128, 8, 8, 128, 3, 1, 1)
    lq, x = V.crafted(geom)
    conv = next(op for op in lq["ops"] if op.get("fp8"))
    tap, ci = conv["picks"][0]
    x[0, ci, 4, 4] = np.nan
    got, _ = _run_crafted(lq, x)
    want = V.expected(lq, x)
    A, _ = O8.conv_fp8(want["data_q"], conv, with_p=False)
    hit = np.isnan(A)
    g = O8.value(got["conv"])
    direct = hit & (np.arange(128) == 0).reshape(1, -1, 1, 1) & (A != A)
    assert np.isnan(g[direct]).any()
    print(f"[fp8 values] NaN x 0: {int(np.isnan(g[hit]).sum())} of {int(hit.sum())} outputs whose window holds the NaN are NaN")
    _same_values(got["conv"], want["conv"], "conv")
