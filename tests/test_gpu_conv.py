"""GPU parity of the tcgen05 implicit-GEMM convolution, one layer at a time, THROUGH THE C ABI
(single-conv plans: b2_engine_deserialize -> b2_context_enqueue), against the CPU oracle that emulates
the engine's fp16 rounding points.  Bit-level agreement is not expected (fp32 accumulation order differs
between the tensor core and the oracle); the bar is 2 fp16 ulp of the tensor's max magnitude."""
import numpy as np
import pytest

from oracle.caffe_forward import lowered_forward_f16emu
from tensorrt_laboratory_b200 import builder
from tests import helpers

pytestmark = pytest.mark.gpu

TOL = 2.0 ** -9  # 2 ulp of fp16 at the top binade, relative to max|ref|

# the 20 unique ResNet-50 convolution shapes (Cin, H_in, Cout, k, stride) -- SURVEY.md 8(d)
RN50_CONVS = [
    (3, 224, 64, 7, 2), (64, 56, 64, 1, 1), (64, 56, 64, 3, 1), (64, 56, 256, 1, 1), (256, 56, 64, 1, 1),
    (256, 56, 128, 1, 2), (256, 56, 512, 1, 2), (128, 28, 128, 3, 1), (128, 28, 512, 1, 1), (512, 28, 128, 1, 1),
    (512, 28, 256, 1, 2), (512, 28, 1024, 1, 2), (256, 14, 256, 3, 1), (256, 14, 1024, 1, 1), (1024, 14, 256, 1, 1),
    (1024, 14, 512, 1, 2), (1024, 14, 2048, 1, 2), (512, 7, 512, 3, 1), (512, 7, 2048, 1, 1), (2048, 7, 512, 1, 1),
]


def _check(cin, h, cout, k, stride, batch, relu=True, residual=False, options=None, seed=0):
    pad = {1: 0, 3: 1, 5: 2, 7: 3}[k]
    net, wts, low = helpers.conv_case(cin, h, h, cout, k, stride, pad, relu=relu, residual=residual, seed=seed)
    x = np.random.default_rng(seed + 1).standard_normal((batch, cin, h, h), dtype=np.float32)
    ref = lowered_forward_f16emu(low, x)
    out = helpers.run_engine(low, x, builder.PREC_FP16, options)
    got = list(out.values())[0].reshape(batch, -1)
    assert got.shape == ref.shape
    assert np.isfinite(got).all()
    err = helpers.rel_err(got, ref)
    assert err <= TOL, f"rel err {err:.3e} > {TOL:.3e}"
    return got


@pytest.mark.parametrize("cin,h,cout,k,stride", RN50_CONVS)
def test_resnet50_conv_shapes(gpu, cin, h, cout, k, stride):
    _check(cin, h, cout, k, stride, batch=2)


@pytest.mark.parametrize("cin,h,cout,k,stride", [(64, 56, 256, 1, 1), (128, 28, 512, 1, 1), (512, 7, 2048, 1, 1), (64, 56, 64, 3, 1)])
def test_fused_residual_and_relu(gpu, cin, h, cout, k, stride):
    _check(cin, h, cout, k, stride, batch=2, relu=True, residual=True)


def test_no_relu_keeps_negative_values(gpu):
    got = _check(64, 28, 64, 1, 1, batch=1, relu=False)
    assert (got < 0).any()


@pytest.mark.parametrize("bn", [32, 64, 128, 256])
def test_every_n_tile(gpu, bn):
    _check(64, 28, 256, 1, 1, batch=2, options={"bn": bn})
    _check(128, 14, 256, 3, 1, batch=2, residual=True, options={"bn": bn, "stages": 2})
    if bn <= 128:
        _check(3, 64, 128, 7, 2, batch=1, options={"bn": bn, "stages": 4})  # row-folded stem path


@pytest.mark.parametrize("stages", [1, 2, 4, 8])
def test_every_pipeline_depth(gpu, stages):
    # 18 k-blocks through a ring of `stages` slots: exercises phase wrap-around of the full/empty barriers
    _check(128, 28, 128, 3, 1, batch=2, options={"bn": 64, "stages": stages})


@pytest.mark.parametrize("bn,stages", [(32, 2), (64, 2), (64, 4), (128, 2), (256, 2)])
def test_double_width_pipeline_stages(gpu, bn, stages):
    # 128 K-elements per mbarrier round trip; 9 (odd) and 18 K-blocks exercise the half-filled last stage
    a = _check(64, 28, 256, 3, 1, batch=2, options={"bn": bn, "stages": stages, "sps": 2})
    b = _check(64, 28, 256, 3, 1, batch=2, options={"bn": bn, "stages": stages, "sps": 1})
    np.testing.assert_array_equal(a, b)
    _check(128, 14, 256, 3, 1, batch=2, residual=True, options={"bn": bn, "stages": stages, "sps": 2})
    if bn == 64:
        _check(512, 7, 512, 3, 1, batch=2, options={"bn": 64, "stages": 2, "sps": 2, "splits": 3})


@pytest.mark.parametrize("bn,stages,sps", [(32, 4, 1), (64, 2, 1), (64, 4, 2), (128, 2, 1), (128, 2, 2), (256, 2, 1)])
def test_persistent_warp_specialised_tactic(gpu, bn, stages, sps):
    """conv_f16_tcgen05_ws: persistent CTAs, producers running ahead across tiles, double-buffered staging.  Same K order as the
    one-tile-per-CTA kernel -> bit-identical results."""
    opts = {"bn": bn, "stages": stages, "sps": sps}
    # many tiles per CTA (M = 4*56*56 = 12544 -> 98 m-tiles x n-tiles on <= one CTA per SM), 1x1 tiled A, fused residual
    a = _check(64, 56, 256, 1, 1, batch=4, residual=True, options=dict(opts, ws=1))
    b = _check(64, 56, 256, 1, 1, batch=4, residual=True, options=dict(opts, ws=-1))
    np.testing.assert_array_equal(a, b)
    # im2col 3x3 with a ragged last tile and 18 K-blocks
    a = _check(128, 14, 256, 3, 1, batch=3, options=dict(opts, ws=1))
    b = _check(128, 14, 256, 3, 1, batch=3, options=dict(opts, ws=-1))
    np.testing.assert_array_equal(a, b)
    # forced small grid: every CTA walks several tiles, both staging buffers and barrier phases wrap many times
    _check(256, 28, 256, 1, 2, batch=4, relu=False, options=dict(opts, ws=7))


@pytest.mark.parametrize("cin,h,cout,bn", [(64, 56, 64, 64), (128, 28, 128, 128), (256, 14, 256, 64), (256, 14, 256, 256),
                                            (512, 7, 512, 128), (64, 20, 128, 64), (64, 126, 64, 64)])
def test_halo_3x3_tactic(gpu, cin, h, cout, bn):
    """conv3x3_halo_tcgen05: the input block of a tile is loaded once and the nine taps are shifted views of it.  Covers
    every ResNet 3x3 geometry (R = 2, 4, 8, 7 rows per tile; 1, 2, 4, 8 resident channel blocks), ragged last row-tiles (14 = 8 + 6, 20 = 5*4), the widest
    row the tile holds (W + 2 = 128) and every N tile."""
    batch = 1 if h > 100 else 3
    a = _check(cin, h, cout, 3, 1, batch=batch, options={"bn": bn, "halo": 1})
    assert any(" halo" in n for n in helpers.LAST_LAUNCH_NAMES), helpers.LAST_LAUNCH_NAMES
    b = _check(cin, h, cout, 3, 1, batch=batch, options={"bn": bn, "halo": -1})
    assert not any(" halo" in n for n in helpers.LAST_LAUNCH_NAMES)
    np.testing.assert_array_equal(a, b)  # same K order as the im2col kernel: bit-identical
    _check(cin, h, cout, 3, 1, batch=batch, relu=False, options={"bn": bn, "halo": 1}, seed=3)


@pytest.mark.parametrize("cn,bn,stages,sps", [(2, 64, 2, 1), (4, 64, 4, 2), (2, 128, 2, 1), (4, 32, 4, 1), (2, 64, 1, 1)])
def test_cluster_multicast_tactic(gpu, cn, bn, stages, sps):
    """Clusters of `cn` CTAs along N: every CTA fetches 1/cn of each activation sub-block and multicasts it; stage
    release is multicast back.  The MMAs are the same as without clusters -> bit-identical results."""
    opts = {"bn": bn, "stages": stages, "sps": sps}
    # 1x1 tiled A, fused residual, ragged last m-tile (M = 3*28*28 = 2352 = 18.4 tiles)
    a = _check(128, 28, 512, 1, 1, batch=3, residual=True, options=dict(opts, cn=cn))
    assert any(f" cn={cn}" in n for n in helpers.LAST_LAUNCH_NAMES), helpers.LAST_LAUNCH_NAMES
    b = _check(128, 28, 512, 1, 1, batch=3, residual=True, options=dict(opts, cn=-1))
    assert not any(" cn=" in n for n in helpers.LAST_LAUNCH_NAMES)
    np.testing.assert_array_equal(a, b)
    # im2col 3x3, 18 K-blocks (barrier phases wrap), last tile has slices that start past the final pixel
    a = _check(128, 14, 256, 3, 1, batch=2, options=dict(opts, cn=cn))
    b = _check(128, 14, 256, 3, 1, batch=2, options=dict(opts, cn=-1))
    np.testing.assert_array_equal(a, b)
    # strided 1x1 through im2col mode + split-K inside a cluster
    _check(256, 14, 512, 1, 2, batch=2, relu=False, options=dict(opts, cn=cn))
    if bn == 64 and sps == 1 and stages == 2:
        _check(512, 7, 512, 3, 1, batch=2, options=dict(opts, cn=cn, splits=2))


@pytest.mark.parametrize("splits", [2, 3, 4, 8])  # 8: bn 64 keeps tiles*splits within the workspace bound
def test_split_k_matches_oracle_and_is_deterministic(gpu, splits):
    # res5-like: M = 2*7*7 = 98 (one ragged tile), K = 4608 -> 72 k-blocks
    opts = {"bn": 64, "stages": 4, "splits": splits}
    a = _check(512, 7, 512, 3, 1, batch=2, options=opts)
    b = _check(512, 7, 512, 3, 1, batch=2, options=opts)
    np.testing.assert_array_equal(a, b)  # fixed-order reduction: bitwise repeatable
    if splits <= 4:  # 5 m-tiles x 8 n-tiles x splits must stay within the 160-CTA split budget
        _check(1024, 14, 256, 1, 1, batch=3, residual=False, options={"bn": 32, "stages": 2, "splits": splits})


def test_split_k_with_fused_residual(gpu):
    _check(512, 7, 2048, 1, 1, batch=2, relu=True, residual=True, options={"bn": 128, "stages": 2, "splits": 2})


@pytest.mark.parametrize("pdl,trigger", [(0, 1), (1, 0), (1, 1)])
def test_programmatic_dependent_launch_modes(gpu, pdl, trigger):
    try:
        _check(64, 56, 256, 1, 1, batch=2, residual=True, options={"pdl": pdl, "pdl_trigger": trigger})
        _check(64, 56, 256, 1, 1, batch=2, residual=True, options={"pdl": pdl, "pdl_trigger": trigger, "graph": 0})
    finally:
        from tensorrt_laboratory_b200 import capi
        eng = None  # restore the process-wide default
        import ctypes as C
        # any context can flip the process-wide switch back
        _check(64, 14, 64, 1, 1, batch=1, options={"pdl": 1})


def test_row_folded_stem_equals_generic_tap_path(gpu):
    # same plan, two A-operand strategies: one 64-byte TMA "pixel" per filter row (KB=32, SWIZZLE_64B) vs one
    # 16-byte im2col load per tap (KB=8, no swizzle); K order is identical -> bit identical
    a = _check(3, 64, 64, 7, 2, batch=2, options={"no_fold": 0})
    b = _check(3, 64, 64, 7, 2, batch=2, options={"no_fold": 1})
    np.testing.assert_array_equal(a, b)
    _check(3, 30, 64, 3, 2, batch=1)   # 3x3/s2 stem variant: kw2 = 2 -> not foldable, generic path
    _check(1, 28, 64, 5, 2, batch=3)   # single-channel input


def test_im2col_tma_equals_tiled_tma_on_pointwise(gpu):
    a = _check(256, 28, 128, 1, 1, batch=2, options={"im2col": 0})
    b = _check(256, 28, 128, 1, 1, batch=2, options={"im2col": 1})
    np.testing.assert_array_equal(a, b)  # same MMA order -> bit identical


@pytest.mark.parametrize("batch,h", [(1, 7), (3, 7), (1, 14), (5, 28), (8, 7)])
def test_ragged_m_tails(gpu, batch, h):
    # M = batch*h*h is not a multiple of the 128-row tile: TMA zero-fills, the epilogue predicates stores
    _check(512 if h == 7 else 128, h, 512 if h == 7 else 128, 3, 1, batch=batch)


def test_tcgen05_agrees_with_simt_kernel(gpu):
    a = _check(128, 28, 128, 3, 1, batch=2, options={"simt": 0})
    b = _check(128, 28, 128, 3, 1, batch=2, options={"simt": 1})
    assert helpers.rel_err(a, b) <= TOL


def test_fp32_engine_conv_matches_fp32_oracle(gpu):
    import torch
    from oracle.caffe_forward import caffe_forward
    net, wts, low = helpers.conv_case(16, 20, 20, 24, 3, 2, 1, relu=True, residual=False)
    x = np.random.default_rng(3).standard_normal((3, 16, 20, 20), dtype=np.float32)
    ref = caffe_forward(net, wts, x, dtype=torch.float64)
    got = list(helpers.run_engine(low, x, builder.PREC_FP32).values())[0].reshape(3, -1)
    assert helpers.rel_err(got, ref) < 1e-6
