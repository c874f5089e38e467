"""GPU: how many convolution CTAs share an SM, and that sharing changes no bits.

The one-tile-per-CTA kernel and the 3x3 halo kernel run 320 threads (two consumer warpgroups and two producer warps), so
at <= 96 registers per thread two 128-wide CTAs fit in an SM's register file, and three 64-wide ones at <= 64.  Shared
memory then decides: a 2-stage 128-wide ring with a residual tile fits twice, a 4-stage one once.
`b2_debug_conv_residency` reports the occupancy calculator's count, the one the cost model uses."""
import ctypes as C
import functools

import numpy as np
import pytest

from tensorrt_laboratory_b200 import builder, capi, graph, weights
from tests import helpers

pytestmark = pytest.mark.gpu

FP16 = builder.PREC_FP16


def _residency(bn, kb=64, stages=2, sps=1, residual=True, halo=(0, 0, 0)):
    lib = capi.load()
    fn = lib.b2_debug_conv_residency
    fn.restype = C.c_int
    fn.argtypes = [C.c_int] * 8 + [C.POINTER(C.c_int)]
    n = C.c_int(0)
    capi.check(fn(bn, kb, stages, sps, int(residual), *halo, C.byref(n)))
    return n.value


@pytest.mark.parametrize("bn,stages,residual,want", [
    (128, 2, True, 2),   # 97.8 KiB: two share an SM
    (128, 2, False, 2),
    (128, 4, True, 1),   # 162 KiB: alone
    (64, 2, True, 3),    # 65.5 KiB and <= 64 registers: three
    (64, 4, False, 2),   # 97.5 KiB: shared memory holds two
    (64, 4, True, 1),    # 113.5 KiB: one
    (256, 2, True, 1),   # 128 accumulators per thread: one
])
def test_tile_kernel_residency(gpu, bn, stages, residual, want):
    assert _residency(bn, stages=stages, residual=residual) == want


def test_halo_kernel_residency(gpu):
    # res2 (56 x 56, one channel block, 2 rows per tile): 64.5 KiB at BN 64 -> three; res5 (7 x 7, eight blocks) at BN 128
    assert _residency(64, halo=(56, 2, 1)) == 3
    assert _residency(128, halo=(7, 7, 8)) == 1
    assert _residency(128, halo=(14, 8, 4)) >= 1


def test_residency_of_a_missing_instantiation_is_an_error(gpu):
    with pytest.raises(capi.B2Error):
        _residency(128, stages=8)


@functools.lru_cache(maxsize=None)
def _resnet50(batch):
    net = graph.resnet_caffe(50)
    low = graph.lower(net, weights.random_weights(net, 0))
    return low, weights.synthetic_input(batch, seed=5)


TAPS = ["conv1", "res2c", "res3d", "res4f", "res5c", "prob"]


def test_resnet50_shared_sm_ring_equals_the_deep_ring(gpu):
    """Every 128-wide layer on a 2-stage ring (two CTAs per SM) against a 4-stage one (one per SM): the same MMAs in the
    same order, so the same bits in every tap."""
    batch = 8
    low, x = _resnet50(batch)
    runs = []
    for st in (2, 4):
        out = helpers.run_engine(low, x, FP16, {"bn": 128, "stages": st}, outputs=TAPS)
        names = [n for n in helpers.LAST_LAUNCH_NAMES if n.startswith("conv_tcgen05:")]
        assert sum(f" bn=128 kb=64 st={st}x1 " in n for n in names) >= 30, names
        runs.append(out)
    two, four = runs
    for k in TAPS:
        assert (two[k] != 0).any(), k
        np.testing.assert_array_equal(two[k], four[k], err_msg=k)


@pytest.mark.parametrize("cin,h,bn", [(64, 56, 64), (128, 28, 128), (256, 14, 128), (512, 7, 128)])
def test_halo_kernel_equals_the_tile_kernel_at_batch_8(gpu, cin, h, bn):
    """Every ResNet 3x3 geometry at the benchmark's batch: the halo kernel against the im2col tile kernel on a 2-stage
    (SM-sharing) ring, bit for bit."""
    batch = 8
    _, _, low = helpers.conv_case(cin, h, h, cin, 3, 1, 1, relu=True, seed=2)
    x = np.random.default_rng(3).standard_normal((batch, cin, h, h), dtype=np.float32)
    got = helpers.run_engine(low, x, FP16, {"bn": bn, "halo": 1})
    assert any(" halo" in n and f" bn={bn} " in n for n in helpers.LAST_LAUNCH_NAMES), helpers.LAST_LAUNCH_NAMES
    want = helpers.run_engine(low, x, FP16, {"bn": bn, "stages": 2, "halo": -1})
    assert any(" halo" not in n and f" bn={bn} kb=64 st=2x1 im2col" in n for n in helpers.LAST_LAUNCH_NAMES), helpers.LAST_LAUNCH_NAMES
    (g,), (w,) = got.values(), want.values()
    assert (w > 0).any()
    np.testing.assert_array_equal(g, w)
