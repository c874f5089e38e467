"""GPU: the CNN kernels at geometries the shipped models never produce.

ResNet, ResNeXt and MNIST only ever give the kernels square images, channel counts that are multiples of 64, stride-2
layers whose window division leaves a remainder and a classifier tail of 7x7x2048 -> 1000.  The ONNX and prototxt front
ends accept much more, so every case here is one of those other geometries: non-square images, stride-2 layers whose
last window ends exactly on the far edge, padded channel counts, every max-pool window rule, the pooling / FC / softmax
tail at other shapes, the input cast of every thin channel count, INT8 at odd channel counts and geometries, and
ResNet-50 at 200x264.

Each operator is judged against a float64 (or exact integer) reference of the same operation, on the engine's own input
where it has one (read back through tap outputs), and the launch names show which kernel ran, so a fallback cannot pass
for the path under test.  Every case is built through the public builder and run through the C ABI."""
import functools
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle.caffe_forward import caffe_forward, lowered_forward_f16emu
from oracle.int8_forward import int8_forward
from tensorrt_laboratory_b200 import builder, capi, graph, quantize, weights
from tests import helpers

pytestmark = pytest.mark.gpu

TOL = 2.0 ** -9    # 2 ulp of fp16 at the top binade, relative to max|ref| (tests/test_gpu_conv.py)
U32 = 2.0 ** -24   # unit roundoff of fp32
FP16, FP32, INT8 = builder.PREC_FP16, builder.PREC_FP32, builder.PREC_INT8


# ------------------------------------------------------------------------------------------------------------------
# geometries (tests/test_geometry_cpu.py builds every one of them without a GPU)
# ------------------------------------------------------------------------------------------------------------------
# (cin, h, w, cout, k, stride, pad, fused residual, batch); the batch leaves a ragged last 128-row M tile
CONV_CASES = [
    (64, 15, 15, 128, 3, 2, 1, False, 3),    # 15 + 2 - 3 = 14 = 7 * 2: the last window ends on the far edge; odd size
    (64, 7, 7, 64, 3, 2, 1, False, 3),       # Ho = 4: a single small tile
    (256, 13, 17, 512, 1, 2, 0, False, 3),   # non-square, edge case (13 - 1 = 6 * 2), strided 1x1 through im2col
    (256, 13, 17, 512, 1, 2, 0, True, 3),    # ... with a fused residual
    (64, 20, 60, 64, 3, 1, 1, False, 3),     # non-square halo tile: R = 128 // 62 = 2 rows
    (128, 9, 40, 128, 3, 1, 0, False, 3),    # valid padding
    (64, 24, 10, 128, 5, 1, 2, False, 3),    # tall image, k = 5
    (3, 199, 257, 64, 7, 2, 3, False, 1),    # odd-width stem: no space-to-depth, generic 8-channel path
    (3, 200, 264, 64, 7, 2, 3, False, 1),    # non-square space-to-depth stem, row-folded
    (16, 30, 40, 64, 3, 1, 1, False, 3),     # Cin 16 padded to 64
    (96, 14, 14, 200, 3, 1, 1, False, 3),    # Cin 96 -> 128, Cout 200 -> 256
    (64, 14, 18, 10, 1, 1, 0, False, 3),     # Cout 10 -> 64
    (64, 14, 14, 3, 3, 1, 1, False, 3),      # Cout 3 -> 8 physical channels: SIMT convolution
    (6, 32, 48, 64, 3, 1, 0, False, 3),      # thin input outside the stem: K blocks of 8 channels
    (64, 16, 24, 128, 2, 2, 0, False, 3),    # even kernel size
]
EDGE_CASES = [CONV_CASES[0], CONV_CASES[3]]  # the 15x15 and 13x17 stride-2 layers, under forced tactics
COUT320 = (64, 28, 28, 320, 1, 1, 0, False, 3)

# (h, w, k, stride, pad, ceil mode) of the max pool behind a 3x3 convolution
POOL_CASES = [
    (13, 17, 3, 2, 0, True),   # ceil: partial last window in W only (17 - 3 = 14 = 7 * 2 fits; 13 - 3 = 10 too)
    (14, 18, 3, 2, 0, True),   # ceil: partial last window in both directions
    (14, 18, 3, 2, 1, True),   # padded, ceil
    (14, 18, 3, 3, 1, True),   # padded, ceil: a last row of windows that would start in the padding is dropped
    (15, 21, 2, 2, 0, False),  # floor mode: the last row and column are never read
    (9, 11, 3, 1, 1, True),    # stride 1, padded
]

# (batch, H = W, C, Cout) of  conv 1x1 -> global AVE -> InnerProduct -> Softmax
TAIL_CASES = [
    (1, 1, 256, 1),
    (3, 2, 768, 10),
    (9, 7, 2048, 1000),    # N > 8: the FC stages the pooled rows in two passes
    (17, 10, 512, 1001),   # HW > 64: every pool slice loops twice
    (2, 14, 1280, 2100),   # Cout > 2048: the softmax re-reads its row
    (4, 7, 100, 37),       # C_phys 128: the fused tail is refused, generic FC
    (4, 7, 2560, 10),      # K > 2048: the fused tail is refused, generic FC
]

# (H, W, C, Cout) of  conv 3x3 -> InnerProduct  on the spatial tensor (K = H * W * C_phys)
FC_CASES = [
    (4, 5, 64, 50),   # K = 1280: fc_h8
    (4, 5, 24, 50),   # 24 channels padded to 64: K = 1280 with zero weights on the padding, fc_h8
    (7, 7, 64, 50),   # K = 3136: generic FC
]

CAST_CHANNELS = [1, 3, 4, 5, 8, 9, 16]
CAST_WIDTHS = [26, 25]   # even: space-to-depth stem where C <= 4; odd: never

I8_TILES = [(128, 1), (128, 2), (128, 3), (128, 4), (256, 1), (256, 2), (256, 3)]   # every conv_i8_tcgen05 instantiation
I8_DEEP = (256, 14, 14, 256, 3, 1, 1)   # 18 K blocks of 128: every ring depth wraps its barrier phases
I8_CHANNELS = [(192, 320), (320, 192)]  # Cin / Cout with a partial last 128-channel block
I8_GEOMS = [(128, 15, 15, 128, 3, 2, 1), (256, 13, 17, 256, 1, 2, 0), (128, 14, 20, 128, 3, 1, 1)]
I8_POOL_HW = [4, 10]


def _case_id(case):
    cin, h, w, cout, k, s, p, res, batch = case
    return f"{cin}x{h}x{w}-{cout}-k{k}s{s}p{p}" + ("-res" if res else "")


def _inputs(shape, seed):
    return np.random.default_rng(seed).standard_normal(shape, dtype=np.float32)


def _fp16_exact(x):
    return x.astype(np.float16).astype(np.float32)


def _launch(names, kind, op):
    """The launch of op `op` by kernel family `kind`, or None."""
    return next((n for n in names if n.split(" ")[0] == f"{kind}:{op}"), None)


def _run_blob(blob, x, options=None):
    """helpers.run_engine for a prebuilt plan -> (outputs, launch names)."""
    eng = capi.Engine(blob)
    sess = capi.Session(eng, options)
    try:
        out = sess.infer(x)
        names = [capi.load().b2_context_launch_name(sess.ctx, x.shape[0], i).decode() for i in range(sess.nb_launches(x.shape[0]))]
    finally:
        sess.close()
        eng.destroy()
    return out, names


# ------------------------------------------------------------------------------------------------------------------
# nets and own-input references (tests/test_geometry_cpu.py checks the references against torch in float64)
# ------------------------------------------------------------------------------------------------------------------
def conv_net(case, relu=True):
    cin, h, w, cout, k, s, p, res, _ = case
    return builder.single_conv_net(cin, h, w, cout, k, s, p, relu=relu, residual=res)


def pool_size(n, k, s, p, ceil):
    """Caffe pooling output size; in ceil mode a last window that would start in the far padding is dropped."""
    if not ceil:
        return (n + 2 * p - k) // s + 1
    o = -(-(n + 2 * p - k) // s) + 1
    if p > 0 and (o - 1) * s >= n + p:
        o -= 1
    return o


def conv_pool_net(c, h, w, k, s, p, ceil):
    """conv 3x3 / 1 / 1 WITHOUT ReLU (negative inputs to the pool), then a max pool."""
    net = builder.single_conv_net(c, h, w, c, 3, 1, 1, relu=False)
    net["layers"].append(dict(name="pool", type="Pooling", bottoms=["conv"], tops=["pool"], pool="MAX", kernel_size=k, stride=s,
                              pad=p, ceil_mode=ceil))
    return net


def maxpool_ref(x, k, s, p, ceil):
    """Max over each window clipped to the image; a window wholly in the padding is an error of the output size."""
    n, c, h, w = x.shape
    ho, wo = pool_size(h, k, s, p, ceil), pool_size(w, k, s, p, ceil)
    out = np.empty((n, c, ho, wo), x.dtype)
    for i in range(ho):
        r0 = i * s - p
        rows = slice(max(r0, 0), min(r0 + k, h))
        for j in range(wo):
            c0 = j * s - p
            win = x[:, :, rows, max(c0, 0):min(c0 + k, w)]
            assert win.shape[2] > 0 and win.shape[3] > 0, f"window ({i}, {j}) lies in the padding"
            out[:, :, i, j] = win.max(axis=(2, 3))
    return out


def tail_net(hw, c, cout, cin=64):
    """conv 1x1 (ReLU) -> global AVE -> InnerProduct -> Softmax."""
    net = builder.single_conv_net(cin, hw, hw, c, 1, 1, 0, relu=True)
    net["layers"] += [
        dict(name="pool", type="Pooling", bottoms=["conv"], tops=["pool"], pool="AVE", kernel_size=hw, stride=1, pad=0),
        dict(name="fc", type="InnerProduct", bottoms=["pool"], tops=["fc"], num_output=cout, bias_term=True),
        dict(name="prob", type="Softmax", bottoms=["fc"], tops=["prob"]),
    ]
    return net


def fc_net(h, w, c, cout, cin=16):
    """conv 3x3 / 1 / 1 (no ReLU) -> InnerProduct over the whole H x W x C tensor."""
    net = builder.single_conv_net(cin, h, w, c, 3, 1, 1, relu=False)
    net["layers"].append(dict(name="fc", type="InnerProduct", bottoms=["conv"], tops=["fc"], num_output=cout, bias_term=True))
    return net


def mean_ref(x):
    """[N, C, H, W] -> [N, C] float64 mean."""
    return np.asarray(x, np.float64).reshape(x.shape[0], x.shape[1], -1).mean(axis=2)


def fc_ref(x, W, b):
    """Caffe InnerProduct: x flattened in (C, H, W) order times W [Cout, C*H*W], in float64 -> (y, sum |w x| + |b|)."""
    flat = np.asarray(x, np.float64).reshape(x.shape[0], -1)
    W = np.asarray(W, np.float64)
    b = np.asarray(b, np.float64)
    return flat @ W.T + b, np.abs(flat) @ np.abs(W).T + np.abs(b)


def fc_bound(K, mag):
    """fp32 accumulation of K products plus the bias, in any order (fused or not): K + 1 roundings of a partial sum."""
    return (K + 1) * U32 * mag


def softmax_ref(x):
    x = np.asarray(x, np.float64)
    e = np.exp(x - x.max(axis=1, keepdims=True))
    return e / e.sum(axis=1, keepdims=True)


def softmax_rel_bound(x):
    """Relative error of an fp32 softmax  y_i = expf(x_i - m) * (1 / sum_j expf(x_j - m))  per row, in units of 2^-24:
    x_i - m rounds (relative error |x_i - m| of the exponential), expf is within 2 ulp (4), the C-term sum adds C - 1,
    the reciprocal and the product one each -- numerator and denominator together (C + 8 + 2 max|x - m|) * 2^-24, plus
    2 for slack."""
    x = np.asarray(x, np.float64)
    spread = (x.max(axis=1, keepdims=True) - x.min(axis=1, keepdims=True))
    return (x.shape[1] + 10 + 2 * spread) * U32


def fp16_ulp(v):
    return np.spacing(np.abs(np.asarray(v, np.float64)).astype(np.float16)).astype(np.float64)


def resnet50_200x264():
    """ResNet-50 on 3x200x264 without pool5 / fc1000 / prob (a global AVE needs a square map; res5c is 7x9).  Its stem is a
    non-square space-to-depth convolution, pool1 a ceil max pool with a partial window, res4a / res5a are stride-2 layers
    whose last window ends on the edge (25x33 -> 13x17 -> 7x9), and its 3x3 halo tiles have R = 1, 3, 6 and 7 rows."""
    net = graph.resnet_caffe(50)
    assert [L["name"] for L in net["layers"][-3:]] == ["pool5", "fc1000", "prob"]
    net["layers"] = net["layers"][:-3]
    net["input_dims"] = [1, 3, 200, 264]
    return net


# ------------------------------------------------------------------------------------------------------------------
# a. convolutions
# ------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _conv_graph(case, relu):
    net = conv_net(case, relu)
    low = graph.lower(net, weights.random_weights(net, 0))
    cin, h, w = case[0], case[1], case[2]
    x = _inputs((case[-1], cin, h, w), 1)
    return low, x, lowered_forward_f16emu(low, x)


def _conv(case, relu, options=None):
    low, x, ref = _conv_graph(case, relu)
    out = helpers.run_engine(low, x, FP16, options)
    got = list(out.values())[0].reshape(x.shape[0], -1)
    assert got.shape == ref.shape and np.isfinite(got).all()
    err = helpers.rel_err(got, ref)
    return got, list(helpers.LAST_LAUNCH_NAMES), err


def _expected_kb(case, no_fold=False):
    cin, h, w, cout, k, s, p, res, _ = case
    if builder.phys_channels(cin, FP16) % 64 == 0:
        return 64
    s2d = cin <= 4 and s == 2 and w % 2 == 0 and k >= 3   # builder.build_plan's space-to-depth rule
    fold = s2d and ((k - 1 - p) // 2 - (0 - p) // 2 + 1) * 8 * 2 == 64   # k x kw2 filter rows of 64 bytes
    return 32 if fold and not no_fold else 8


@pytest.mark.parametrize("relu", [True, False], ids=["relu", "linear"])
@pytest.mark.parametrize("case", CONV_CASES, ids=_case_id)
def test_conv_geometry(gpu, case, relu):
    got, names, err = _conv(case, relu)
    assert err <= TOL, f"rel err {err:.3e} > {TOL:.3e}"
    if not relu:
        assert (got < 0).any()
    simt = builder.phys_channels(case[3], FP16) % 32 != 0
    name = _launch(names, "conv_simt" if simt else "conv_tcgen05", "conv")
    assert name is not None, names
    if not simt:
        assert f" kb={_expected_kb(case)} " in name, name


def test_conv_halo_on_a_non_square_image(gpu):
    """R = 2 rows of a 60-wide image per tile: the halo kernel must give the im2col kernel's bits."""
    case = CONV_CASES[4]
    for relu in (True, False):
        a, names_a, err_a = _conv(case, relu, {"bn": 64, "halo": 1})
        assert " halo" in _launch(names_a, "conv_tcgen05", "conv"), names_a
        b, names_b, err_b = _conv(case, relu, {"bn": 64, "halo": -1})
        assert " halo" not in _launch(names_b, "conv_tcgen05", "conv")
        assert max(err_a, err_b) <= TOL
        np.testing.assert_array_equal(a, b)


def test_non_square_stem_row_folded_equals_generic_taps(gpu):
    case = CONV_CASES[8]
    a, names_a, err_a = _conv(case, True, {"no_fold": 0})
    assert " kb=32 " in _launch(names_a, "conv_tcgen05", "conv")
    b, names_b, err_b = _conv(case, True, {"no_fold": 1})
    assert " kb=8 " in _launch(names_b, "conv_tcgen05", "conv")
    assert max(err_a, err_b) <= TOL
    np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("bn", [32, 64, 128, 256])
def test_forced_n_tile_on_cout_320(gpu, bn):
    """320 output channels admit N tiles 32 and 64 only; a forced 128 or 256 falls back.  Every tile computes the
    autotune=0 bits."""
    base, _, err = _conv(COUT320, True, {"autotune": 0})
    assert err <= TOL
    got, names, _ = _conv(COUT320, True, {"bn": bn})
    used = int(re.search(r" bn=(\d+) ", _launch(names, "conv_tcgen05", "conv")).group(1))
    assert used == bn if 320 % bn == 0 else (used != bn and 320 % used == 0), (bn, used)
    np.testing.assert_array_equal(got, base)


@pytest.mark.parametrize("case", EDGE_CASES, ids=_case_id)
def test_edge_window_layers_under_forced_tactics(gpu, case):
    """Ring depth, double-width stages and clusters change no bit; split-K reorders the sum and is held to TOL."""
    base, _, err = _conv(case, True, {"autotune": 0})
    assert err <= TOL
    tactics = set()
    for opts in [{"stages": 1}, {"stages": 2}, {"stages": 4}, {"stages": 8}, {"sps": 2}, {"bn": 64, "stages": 2, "sps": 2},
                 {"cn": 2}, {"cn": 4}, {"bn": 64, "cn": 2}, {"bn": 32, "stages": 4}]:
        got, names, _ = _conv(case, True, opts)
        tactics.add(re.sub(r" grid=\S+", "", _launch(names, "conv_tcgen05", "conv")))
        np.testing.assert_array_equal(got, base, err_msg=str(opts))
    assert len(tactics) >= 4, tactics
    # split-K: the 15x15 3x3 has 9 K blocks, two splits of at least 4; the 13x17 1x1 has 4, so the forced split count is
    # dropped and the cost model's unsplit tactic runs (it used to fail the plan with "no kernel configuration")
    got, names, err = _conv(case, True, {"bn": 64, "stages": 2, "splits": 2})
    split = int(re.search(r" grid=\d+x\d+x(\d+) ", _launch(names, "conv_tcgen05", "conv")).group(1))
    if case[4] == 3:
        assert split == 2 and err <= TOL, (split, err)
    else:
        assert split == 1
        np.testing.assert_array_equal(got, base)


# ------------------------------------------------------------------------------------------------------------------
# b. max pool, judged on its own (tapped) input
# ------------------------------------------------------------------------------------------------------------------
def _pool_run(case, c, precision):
    h, w, k, s, p, ceil = case
    net = conv_pool_net(c, h, w, k, s, p, ceil)
    low = graph.lower(net, weights.random_weights(net, 2))
    x = _inputs((3, c, h, w), 3)
    out = helpers.run_engine(low, x, precision, outputs=["conv", "pool"])
    return net, low, x, out, list(helpers.LAST_LAUNCH_NAMES)


@pytest.mark.parametrize("c", [64, 3])
@pytest.mark.parametrize("case", POOL_CASES, ids=lambda t: f"{t[0]}x{t[1]}-k{t[2]}s{t[3]}p{t[4]}-{'ceil' if t[5] else 'floor'}")
def test_maxpool_windows(gpu, case, c):
    h, w, k, s, p, ceil = case
    _, _, _, out, names = _pool_run(case, c, FP16)
    assert _launch(names, "maxpool", "pool") is not None, names
    conv, pool = out["conv"], out["pool"]
    assert (conv < 0).any()
    want = maxpool_ref(conv, k, s, p, ceil)
    assert pool.shape == want.shape
    np.testing.assert_array_equal(pool, want)
    assert (want < 0).any()   # windows with no positive value: the max starts from -inf, never from 0


# ------------------------------------------------------------------------------------------------------------------
# c. global average pool, FC, softmax and the fused tail
# ------------------------------------------------------------------------------------------------------------------
def _tail_id(t):
    return f"n{t[0]}-hw{t[1]}-c{t[2]}-cout{t[3]}"


@functools.lru_cache(maxsize=None)
def tail_graph(case):
    n, hw, c, cout = case
    net = tail_net(hw, c, cout)
    wts = weights.random_weights(net, 5)
    return net, wts, graph.lower(net, wts), _inputs((n, 64, hw, hw), 6)


def run_tail(case, fused, precision=FP16):
    """-> (outputs, launch names).  Unfused: taps conv, pool, fc and prob.  Fused: conv, pool and prob (a tapped fc
    keeps the tail apart)."""
    _, _, low, x = tail_graph(case)
    taps = ["conv", "pool", "prob"] if fused else ["conv", "pool", "fc", "prob"]
    out = helpers.run_engine(low, x, precision, None if fused else {"fuse_tail": 0}, outputs=taps)
    return out, list(helpers.LAST_LAUNCH_NAMES)


def tail_applies(case):
    """kernels.cu tail_f16_applies(N, HW, C_phys, Cout)"""
    c_phys = builder.phys_channels(case[2], FP16)
    return c_phys % 256 == 0 and c_phys <= 2048


@functools.lru_cache(maxsize=None)
def _tail_fused(case):
    return run_tail(case, fused=True)


@pytest.mark.parametrize("case", TAIL_CASES, ids=_tail_id)
def test_pool_fc_softmax_on_their_own_inputs(gpu, case):
    n, hw, c, cout = case
    out, names = run_tail(case, fused=False)
    assert not any(nm.startswith("tail_pool_fc_softmax") for nm in names), names
    for kind, op in (("avgpool", "pool"), ("fc", "fc"), ("softmax", "prob")):
        assert _launch(names, kind, op) is not None, names
    # pool: within one fp16 ulp of the float64 mean of the tapped convolution
    mean = mean_ref(out["conv"])
    pooled = out["pool"].reshape(n, c).astype(np.float64)
    assert (np.abs(pooled - mean) <= fp16_ulp(mean)).all(), np.abs(pooled - mean).max()
    # FC: the tapped pooled vector times the plan's fp16 weights, within the fp32 summation bound
    _, wts, low, _ = tail_graph(case)
    W16 = wts["fc"]["W"].astype(np.float16)
    want, mag = fc_ref(pooled, W16, wts["fc"]["b"])
    logits = out["fc"].astype(np.float64)
    assert (np.abs(logits - want) <= fc_bound(c, mag)).all(), np.abs(logits - want).max()
    # softmax: float64 softmax of the tapped fp32 logits
    ref = softmax_ref(logits)
    assert (np.abs(out["prob"] - ref) <= softmax_rel_bound(logits) * ref).all()


@pytest.mark.parametrize("case", TAIL_CASES, ids=_tail_id)
def test_fused_tail_is_bit_identical_where_it_applies(gpu, case):
    fused, names = _tail_fused(case)
    plain, _ = run_tail(case, fused=False)
    tail = [nm for nm in names if nm.startswith("tail_pool_fc_softmax:")]
    assert len(tail) == (1 if tail_applies(case) else 0), names
    if not tail:
        assert _launch(names, "fc", "fc") is not None, names
    # the fused kernel's pooled vector is judged on its own input too, then every bit against the unfused operators
    mean = mean_ref(fused["conv"])
    pooled = fused["pool"].reshape(case[0], case[2]).astype(np.float64)
    assert (np.abs(pooled - mean) <= fp16_ulp(mean)).all(), np.abs(pooled - mean).max()
    np.testing.assert_array_equal(fused["pool"], plain["pool"])
    np.testing.assert_array_equal(fused["prob"], plain["prob"])


_TAIL_SCRIPT = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from tests import test_gpu_geometry as T
np.savez(sys.argv[2], *[T.run_tail(case, fused=True)[0]["prob"] for case in T.TAIL_CASES])
"""


@pytest.mark.parametrize("ctas", [1, 5])
def test_fused_tail_on_other_grid_sizes(gpu, tmp_path, ctas):
    """B2_TAIL_CTAS is read once per process: a child process runs every tail case on a grid of `ctas` CTAs (one CTA
    takes every pool, FC and softmax item in turn) and must reproduce this process's bits."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = tmp_path / "prob.npz"
    env = dict(os.environ, B2_TAIL_CTAS=str(ctas))
    r = subprocess.run([sys.executable, "-c", _TAIL_SCRIPT, root, str(out)], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    got = np.load(out)
    for case, key in zip(TAIL_CASES, got.files):
        np.testing.assert_array_equal(got[key], _tail_fused(case)[0]["prob"], err_msg=_tail_id(case))


@pytest.mark.parametrize("case", FC_CASES, ids=lambda t: f"{t[0]}x{t[1]}x{t[2]}-{t[3]}")
def test_fc_on_a_spatial_tensor(gpu, case):
    """K = H * W * C_phys: the plan permutes Caffe's (C, H, W) weight order to the engine's (H, W, C_phys) and zero-fills
    the padded channels; the reference uses the Caffe order on the tapped convolution output."""
    h, w, c, cout = case
    net = fc_net(h, w, c, cout)
    wts = weights.random_weights(net, 7)
    low = graph.lower(net, wts)
    x = _inputs((5, 16, h, w), 8)
    out = helpers.run_engine(low, x, FP16, outputs=["conv", "fc"])
    assert _launch(helpers.LAST_LAUNCH_NAMES, "fc", "fc") is not None, helpers.LAST_LAUNCH_NAMES
    want, mag = fc_ref(out["conv"], wts["fc"]["W"].astype(np.float16), wts["fc"]["b"])
    got = out["fc"].astype(np.float64)
    assert (np.abs(got - want) <= fc_bound(h * w * c, mag)).all(), np.abs(got - want).max()


# ------------------------------------------------------------------------------------------------------------------
# d. input cast
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w", CAST_WIDTHS, ids=["even_w", "odd_w"])
@pytest.mark.parametrize("c", CAST_CHANNELS)
def test_input_cast_f16_binding_matches_f32_binding(gpu, c, w):
    case = (c, 20, w, 64, 7, 2, 3, False, 3)
    net = conv_net(case, relu=False)
    low = graph.lower(net, weights.random_weights(net, 9))
    x = _fp16_exact(_inputs((3, c, 20, w), 10))
    a, names = _run_blob(builder.build_plan(low, FP16, 3), x)
    b, _ = _run_blob(builder.build_plan(low, FP16, 3, input_dtype="f16"), x)
    assert f" kb={_expected_kb(case)} " in _launch(names, "conv_tcgen05", "conv"), names
    a, b = list(a.values())[0], list(b.values())[0]
    np.testing.assert_array_equal(a, b)
    assert helpers.rel_err(a.reshape(3, -1), lowered_forward_f16emu(low, x)) <= TOL


# ------------------------------------------------------------------------------------------------------------------
# e. INT8, bit-exact against oracle.int8_forward
# ------------------------------------------------------------------------------------------------------------------
def i8_graph(cin, h, w, cout, k, s, p, relu=True, residual=False, seed=0):
    net = builder.single_conv_net(cin, h, w, cout, k, s, p, relu=relu, residual=residual)
    return graph.lower(net, weights.random_weights(net, seed))


def _i8_check(low, x, options=None, outputs=None):
    lq = quantize.quantize_lowered(low, x)
    out = helpers.run_engine(lq, x, INT8, options, outputs=outputs)
    names = list(helpers.LAST_LAUNCH_NAMES)
    assert _launch(names, "conv_i8_tcgen05", "conv") is not None, names
    want = int8_forward(lq, x)
    got = out[lq["output"]].reshape(x.shape[0], -1)
    np.testing.assert_array_equal(got, want.astype(np.float32))
    return lq, out, names


@pytest.fixture(scope="module")
def i8_deep():
    cin, h, w, cout, k, s, p = I8_DEEP
    low = i8_graph(cin, h, w, cout, k, s, p, relu=False, seed=11)
    x = _fp16_exact(_inputs((3, cin, h, w), 12))
    lq = quantize.quantize_lowered(low, x)
    return lq, x, int8_forward(lq, x).astype(np.float32)


@pytest.mark.parametrize("bn,st", I8_TILES)
def test_int8_every_tile_and_ring_depth(gpu, i8_deep, bn, st):
    lq, x, want = i8_deep
    out = helpers.run_engine(lq, x, INT8, {"i8_bn": bn, "i8_stages": st})
    name = _launch(helpers.LAST_LAUNCH_NAMES, "conv_i8_tcgen05", "conv")
    assert f" bn={bn} st={st} " in name and " kblk=18" in name, name
    np.testing.assert_array_equal(out[lq["output"]].reshape(3, -1), want)


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("cin,cout", I8_CHANNELS)
def test_int8_partial_channel_blocks(gpu, cin, cout, bn):
    """Cin 192 / 320: the last 128-channel K block is half full.  Cout 320 pads to 384: N tile 256 does not divide it and
    falls back to 128, whose last tile holds 64 real channels.  The output binding is an INT8 tensor tap."""
    low = i8_graph(cin, 14, 14, cout, 3, 1, 1, relu=False, seed=13)
    x = _fp16_exact(_inputs((3, cin, 14, 14), 14))
    _, _, names = _i8_check(low, x, {"i8_bn": bn})
    used = bn if (cout + 127) // 128 * 128 % bn == 0 else 128
    assert f" bn={used} " in _launch(names, "conv_i8_tcgen05", "conv"), names
    assert _launch(names, "output_cast_i8", "cast:conv") is not None, names


@pytest.mark.parametrize("residual", [False, True], ids=["plain", "res"])
@pytest.mark.parametrize("geom", I8_GEOMS, ids=lambda g: f"{g[0]}x{g[1]}x{g[2]}-{g[3]}-k{g[4]}s{g[5]}p{g[6]}")
def test_int8_geometry(gpu, geom, residual):
    cin, h, w, cout, k, s, p = geom
    low = i8_graph(cin, h, w, cout, k, s, p, relu=not residual, residual=residual, seed=15)
    _i8_check(low, _fp16_exact(_inputs((3, cin, h, w), 16)))


# fp16 input -> quantized value at s = 2 (inv_s = 0.5): ties go to the even neighbour, |q| <= 127
_TIES = {0: 0, 1: 0, -1: 0, 2: 1, -2: -1, 3: 2, -3: -2, 4: 2, 5: 2, -5: -2, 7: 4, -7: -4, 9: 4, -9: -4, 253: 126, -253: -126,
         254: 127, -254: -127, 255: 127, -255: -127, 256: 127, 300: 127, -300: -127}


def test_int8_quantize_rounds_half_to_even_on_the_gpu(gpu):
    low = i8_graph(64, 4, 6, 64, 1, 1, 0, relu=False, seed=17)
    vals = np.array(sorted(_TIES), np.float32)
    x = vals[np.random.default_rng(18).integers(0, len(vals), size=(2, 64, 4, 6))]
    x.reshape(-1)[:len(vals)] = vals   # every value at least once
    amax = quantize.calibrate(low, x)
    amax["data"] = 254.0               # s = 254 / 127 = 2 exactly
    lq = quantize.quantize_lowered(low, x, amax=amax)
    assert lq["tensor_scales"]["data_q"] == 2.0 and lq["ops"][0]["inv_scale"] == np.float32(0.5)
    out = helpers.run_engine(lq, x, INT8, outputs=["data_q", "conv"])
    assert _launch(helpers.LAST_LAUNCH_NAMES, "quantize", "quantize:data") is not None, helpers.LAST_LAUNCH_NAMES
    want = np.vectorize(_TIES.get)(x.astype(np.int64))
    np.testing.assert_array_equal(out["data_q"], want * 2.0)
    _, snaps = int8_forward(lq, x, keep=["data_q"])
    np.testing.assert_array_equal(snaps["data_q"], want)
    np.testing.assert_array_equal(out["conv"].reshape(2, -1), int8_forward(lq, x).astype(np.float32))


@pytest.mark.parametrize("hw", I8_POOL_HW)
def test_int8_global_average_pool(gpu, hw):
    net = builder.single_conv_net(64, hw, hw, 320, 1, 1, 0, relu=False)
    net["layers"].append(dict(name="pool", type="Pooling", bottoms=["conv"], tops=["pool"], pool="AVE", kernel_size=hw, stride=1, pad=0))
    low = graph.lower(net, weights.random_weights(net, 19))
    x = _fp16_exact(_inputs((3, 64, hw, hw), 20))
    lq = quantize.quantize_lowered(low, x)
    out = helpers.run_engine(lq, x, INT8)
    assert _launch(helpers.LAST_LAUNCH_NAMES, "avgpool_i8", "pool") is not None, helpers.LAST_LAUNCH_NAMES
    np.testing.assert_array_equal(out["pool"].reshape(3, -1), int8_forward(lq, x).astype(np.float32))


# ------------------------------------------------------------------------------------------------------------------
# f. ResNet-50 at 200x264
# ------------------------------------------------------------------------------------------------------------------
WIDE_TAPS = ["conv1", "pool1", "res2c", "res3d", "res4f", "res5c"]


@pytest.fixture(scope="module")
def wide(gpu):
    net = resnet50_200x264()
    wts = weights.random_weights(net, 0)
    low = graph.lower(net, wts)
    x = weights.synthetic_input(3, chw=(3, 200, 264), seed=21)
    blob = builder.build_plan(low, FP16, 3, outputs=WIDE_TAPS)
    out, names = _run_blob(blob, x)
    return dict(low=low, x=x, blob=blob, out=out, names=names)


def test_resnet50_200x264_fp16_taps(wide):
    names = wide["names"]
    assert sum(n.startswith("conv_tcgen05:") for n in names) == 53, names
    assert " kb=32 " in _launch(names, "conv_tcgen05", "conv1") and _launch(names, "maxpool", "pool1") is not None
    _, snaps = lowered_forward_f16emu(wide["low"], wide["x"], keep=WIDE_TAPS)
    for t in WIDE_TAPS:
        assert wide["out"][t].shape == snaps[t].shape, t
        assert helpers.rel_err(wide["out"][t].reshape(3, -1), snaps[t].reshape(3, -1)) <= 4e-3, t
    assert wide["out"]["res5c"].shape == (3, 2048, 7, 9)


def test_resnet50_200x264_batch_position_invariance(wide):
    eng = capi.Engine(wide["blob"])
    sess = capi.Session(eng)
    try:
        perm = np.array([2, 0, 1])
        got = sess.infer(wide["x"][perm])
        for t in WIDE_TAPS:
            np.testing.assert_array_equal(got[t], wide["out"][t][perm], err_msg=t)
        for b in (1, 2):
            got = sess.infer(wide["x"][:b])
            np.testing.assert_array_equal(got["res5c"], wide["out"]["res5c"][:b])
    finally:
        sess.close()
        eng.destroy()


def test_resnet50_200x264_tuned_tactics_change_no_bit(wide):
    eng = capi.Engine(wide["blob"])
    try:
        assert eng.tune(streams=2) == 53
        sess = capi.Session(eng)
        try:
            got = sess.infer(wide["x"])
        finally:
            sess.close()
    finally:
        eng.destroy()
    for t in WIDE_TAPS:
        np.testing.assert_array_equal(got[t], wide["out"][t], err_msg=t)


def test_resnet50_200x264_int8(wide):
    """The _full_net_check scheme of tests/test_int8.py: the fp16 stem within fp16 tolerance, everything INT8 downstream of
    the GPU's own pool1 bit for bit."""
    lq = quantize.quantize_lowered(wide["low"], weights.synthetic_input(4, chw=(3, 200, 264), seed=4321))
    x = wide["x"][:2]
    last = [o for o in lq["ops"] if o.get("int8")][-1]["output"]
    taps = ["pool1", "res3d", last]
    out = helpers.run_engine(lq, x, INT8, outputs=taps)
    n_i8 = sum(1 for o in lq["ops"] if o.get("int8"))
    assert sum(n.startswith("conv_i8_tcgen05:") for n in helpers.LAST_LAUNCH_NAMES) == n_i8
    stem = int8_forward(dict(lq, ops=lq["ops"][:2], output="pool1"), x)   # conv1 + pool1 only
    assert helpers.rel_err(out["pool1"].reshape(2, -1), stem) <= 4e-3
    _, snaps = int8_forward(lq, x, keep=["res3d", last], start_from={"pool1": out["pool1"].astype(np.float64)})
    for t in ("res3d", last):
        np.testing.assert_array_equal(out[t], snaps[t].astype(np.float32) * np.float32(lq["tensor_scales"][t]), err_msg=t)


# ------------------------------------------------------------------------------------------------------------------
# g. the fp32 engine: SIMT convolution, generic max pool / average pool / FC on unpadded channels
# ------------------------------------------------------------------------------------------------------------------
FP32_CONV_CASES = [CONV_CASES[i] for i in (0, 3, 4, 6, 7, 10, 12, 13, 14)]
FP32_TAIL_CASES = [TAIL_CASES[i] for i in (1, 3, 5)]


@pytest.mark.parametrize("case", FP32_CONV_CASES, ids=_case_id)
def test_fp32_engine_conv(gpu, case):
    net = conv_net(case, relu=False)
    wts = weights.random_weights(net, 0)
    x = _inputs((case[-1],) + tuple(net["input_dims"][1:]), 1)
    got = list(helpers.run_engine(graph.lower(net, wts), x, FP32).values())[0].reshape(x.shape[0], -1)
    assert _launch(helpers.LAST_LAUNCH_NAMES, "conv_simt", "conv") is not None, helpers.LAST_LAUNCH_NAMES
    assert helpers.rel_err(got, caffe_forward(net, wts, x, dtype=torch.float64)) < 1e-5


@pytest.mark.parametrize("case", POOL_CASES[1:5], ids=lambda t: f"{t[0]}x{t[1]}-k{t[2]}s{t[3]}p{t[4]}-{'ceil' if t[5] else 'floor'}")
def test_fp32_engine_maxpool(gpu, case):
    h, w, k, s, p, ceil = case
    net, _, x, out, names = _pool_run(case, 5, FP32)
    assert _launch(names, "maxpool", "pool") is not None, names
    np.testing.assert_array_equal(out["pool"], maxpool_ref(out["conv"], k, s, p, ceil))
    _, snaps = caffe_forward(net, weights.random_weights(net, 2), x, dtype=torch.float64, keep=["conv"])
    assert helpers.rel_err(out["conv"], snaps["conv"]) < 1e-5


@pytest.mark.parametrize("case", FP32_TAIL_CASES, ids=_tail_id)
def test_fp32_engine_pool_fc_softmax(gpu, case):
    net, wts, low, x = tail_graph(case)
    out, names = run_tail(case, fused=False, precision=FP32)
    ref, snaps = caffe_forward(net, wts, x, dtype=torch.float64, keep=["pool", "fc"])
    n = x.shape[0]
    for t in ("pool", "fc"):
        assert helpers.rel_err(out[t].reshape(n, -1), snaps[t].reshape(n, -1)) < 1e-5, t
    assert helpers.rel_err(out["prob"], ref) < 1e-5
