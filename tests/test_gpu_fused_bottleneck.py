"""GPU: a bottleneck's 3x3 and the 1x1 after it as one launch (conv3x3_halo_1x1_tcgen05).

The fused kernel keeps the 3x3's fp16 output in shared memory and runs the 1x1 with bias, residual and ReLU on it, adding
the same products in the same order as the two separate launches.  Every case compares it bit for bit against the
unfused pair (option fuse = -1) and checks from the launch names that the fusion did or did not happen."""
import functools

import numpy as np
import pytest

from tensorrt_laboratory_b200 import builder, capi, graph, weights
from tests import helpers
from tests.test_gpu_tactic_table import _check_refused

pytestmark = pytest.mark.gpu

FP16 = builder.PREC_FP16


def _bottleneck(c, h, w, seed=0):
    """x (4c channels) -> 1x1 c -> 3x3 c -> 1x1 4c, + x, ReLU: a ResNet bottleneck with an identity shortcut."""
    n2 = 4 * c
    L = [
        dict(name="a", type="Convolution", bottoms=["data"], tops=["a"], num_output=c, kernel_size=1, pad=0, stride=1, bias_term=True),
        dict(name="a_relu", type="ReLU", bottoms=["a"], tops=["a"]),
        dict(name="b", type="Convolution", bottoms=["a"], tops=["b"], num_output=c, kernel_size=3, pad=1, stride=1, bias_term=True),
        dict(name="b_relu", type="ReLU", bottoms=["b"], tops=["b"]),
        dict(name="c", type="Convolution", bottoms=["b"], tops=["c"], num_output=n2, kernel_size=1, pad=0, stride=1, bias_term=True),
        dict(name="sum", type="Eltwise", bottoms=["data", "c"], tops=["sum"], operation="SUM"),
        dict(name="sum_relu", type="ReLU", bottoms=["sum"], tops=["sum"]),
    ]
    net = {"name": f"bottleneck_{c}x{h}x{w}", "input": "data", "input_dims": [1, n2, h, w], "layers": L}
    return graph.lower(net, weights.random_weights(net, seed))


def _fused_names():
    return [n for n in helpers.LAST_LAUNCH_NAMES if " fused" in n]


def _check_pair(c, h, w, batch, seed=0):
    low = _bottleneck(c, h, w, seed)
    x = np.random.default_rng(seed + 1).standard_normal((batch, 4 * c, h, w), dtype=np.float32)
    got = helpers.run_engine(low, x, FP16, {"fuse": 1})
    fused = _fused_names()
    assert len(fused) == 1 and "b+c" in fused[0] and f" bn={c} " in fused[0], helpers.LAST_LAUNCH_NAMES
    n_fused = len(helpers.LAST_LAUNCH_NAMES)
    want = helpers.run_engine(low, x, FP16, {"fuse": -1})
    assert not _fused_names() and len(helpers.LAST_LAUNCH_NAMES) == n_fused + 1, helpers.LAST_LAUNCH_NAMES
    assert any(n.startswith("conv_tcgen05:b ") for n in helpers.LAST_LAUNCH_NAMES), helpers.LAST_LAUNCH_NAMES
    assert any(n.startswith("conv_tcgen05:c ") for n in helpers.LAST_LAUNCH_NAMES), helpers.LAST_LAUNCH_NAMES
    (g,), (wv,) = got.values(), want.values()
    assert (wv > 0).any()
    np.testing.assert_array_equal(g, wv)


@pytest.mark.parametrize("c,h", [(64, 56), (128, 28), (256, 14)])
def test_resnet50_geometries_at_batch_8(gpu, c, h):
    _check_pair(c, h, h, 8)


@pytest.mark.parametrize("batch", [1, 3])
def test_small_batches(gpu, batch):
    _check_pair(64, 56, 56, batch, seed=batch)


def test_sixty_wide_image_two_rows_per_tile(gpu):
    _check_pair(64, 60, 60, 2, seed=7)


@pytest.mark.parametrize("c,h,w", [(256, 14, 14), (128, 30, 14), (64, 7, 9), (64, 9, 7)])
def test_last_tile_of_an_image_is_partial(gpu, c, h, w):
    _check_pair(c, h, w, 2, seed=11)


def test_a_tapped_3x3_output_does_not_fuse(gpu):
    low = _bottleneck(64, 28, 28, 3)
    x = np.random.default_rng(4).standard_normal((2, 256, 28, 28), dtype=np.float32)
    got = helpers.run_engine(low, x, FP16, {"fuse": 1}, outputs=["b", "sum"])
    assert not _fused_names(), helpers.LAST_LAUNCH_NAMES
    want = helpers.run_engine(low, x, FP16, {"fuse": -1}, outputs=["b", "sum"])
    for k in ("b", "sum"):
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)


@functools.lru_cache(maxsize=None)
def _resnet50():
    net = graph.resnet_caffe(50)
    low = graph.lower(net, weights.random_weights(net, 0))
    return low, weights.synthetic_input(8, seed=5)


def test_resnet50_fused_equals_unfused(gpu):
    low, x = _resnet50()
    got = helpers.run_engine(low, x, FP16, {"fuse": 1}, outputs=["prob"])
    fused = _fused_names()
    # res2 (64), res3 (128) and res4 (256): 13 blocks; res5's 512-channel 3x3 has no halo kernel
    assert len(fused) == 13, helpers.LAST_LAUNCH_NAMES
    want = helpers.run_engine(low, x, FP16, {"fuse": -1}, outputs=["prob"])
    assert not _fused_names()
    assert got["prob"].tobytes() == want["prob"].tobytes()


@pytest.mark.parametrize("op_name,bn", [("res5a_branch2b", 512), ("res4a_branch2c", 128), ("res2a_branch2a", 64)])
def test_a_fused_table_entry_on_an_op_that_cannot_fuse_is_refused(gpu, op_name, bn):
    """res5's 512-channel 3x3 (no halo kernel that wide), a 1x1 with a residual and a 1x1 without one, each given the
    fused tactic in the plan's tactic table: the record is ignored, as every refused record is."""
    low, x = _resnet50()
    blob = builder.build_plan(low, FP16, 4)
    _check_refused(blob, x[:4], op_name, bn=bn, stages=2, halo=2)


def test_an_untuned_engine_stays_unfused(gpu):
    low, x = _resnet50()
    helpers.run_engine(low, x[:2], FP16, {"autotune": 0})
    assert not _fused_names(), helpers.LAST_LAUNCH_NAMES


@pytest.mark.parametrize("fuse,launches", [(-1, 56), (1, 43)])
def test_device_throughput_harness_counts_fused_launches(gpu, monkeypatch, fuse, launches):
    """The tuned harness counts the launches of a step: 56 for ResNet-50 unfused, 13 fewer with every res2-res4
    bottleneck fused.  (Which blocks the timing fuses depends on the device, so the count is pinned at both ends.)"""
    low, _ = _resnet50()
    monkeypatch.setenv("B2_FORCE_FUSE", str(fuse))
    blob = builder.build_plan(low, FP16, 8)
    ms, n = capi.device_throughput(blob, contexts=2, batch=8, steps=8, warmup=4, ring=weights.synthetic_input(8, ring=2))
    assert ms > 0 and n == launches
