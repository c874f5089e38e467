"""CPU: the oracle against the reference's in-tree golden vectors, and its internal consistency."""
import os

import numpy as np
import pytest
import torch

from oracle.caffe_forward import caffe_forward, lowered_forward_f16emu
from tensorrt_laboratory_b200 import graph, weights
from tests import helpers

# reference examples/30_PyTensorRT/server.py:31: np.testing.assert_almost_equal(result, expected, decimal=3)
DECIMAL3 = 1.5e-3


def test_mnist_golden_vectors_fp32_and_fp64():
    net, w, xs, ys = helpers.load_mnist_golden()
    expect_argmax = [2, 0, 9]  # SURVEY.md 8(c)
    for x, y, am in zip(xs, ys, expect_argmax):
        for dt in (torch.float32, torch.float64):
            got = caffe_forward(net, w, x, dtype=dt)
            assert got.shape == (1, 10)
            assert np.abs(got - y).max() < DECIMAL3
            assert int(got.argmax()) == am == int(y.argmax())


def test_mnist_golden_known_values():
    _, _, _, ys = helpers.load_mnist_golden()
    # first test vector, as transcribed in SURVEY.md 8(c)
    np.testing.assert_allclose(ys[0][0, :4], [975.67, -618.72, 6574.57, 668.03], atol=0.01)


def test_mnist_batched_equals_single():
    net, w, xs, ys = helpers.load_mnist_golden()
    got = caffe_forward(net, w, np.concatenate(xs, 0), dtype=torch.float64)
    np.testing.assert_allclose(got, np.concatenate(ys, 0), atol=DECIMAL3)


def test_folding_is_exact_on_resnet_block():
    """BN+Scale folding / residual fusion (graph.lower) == unfused Caffe semantics, exactly (fp64)."""
    net = graph.resnet_caffe(50)
    # first 2 bottlenecks only, small image, to keep the CPU cost low
    cut = [i for i, L in enumerate(net["layers"]) if L["name"] == "res2b_relu"][0] + 1
    small = dict(net, layers=net["layers"][:cut], input_dims=[1, 3, 64, 64])
    w = weights.random_weights(small, 3)
    x = np.random.default_rng(0).standard_normal((2, 3, 64, 64), dtype=np.float32)
    ref = caffe_forward(small, w, x, dtype=torch.float64)
    low = graph.lower(small, w)
    got = lowered_forward_f16emu(low, x, round16=False)
    assert helpers.rel_err(got, ref) < 1e-6  # weights are folded in fp64 then stored as fp32


def test_f16_emulation_is_close_to_fp32():
    net, w, low = helpers.conv_case(64, 14, 14, 64, 3, 1, 1, relu=True, residual=True)
    x = np.random.default_rng(5).standard_normal((2, 64, 14, 14), dtype=np.float32)
    ref = caffe_forward(net, w, x, dtype=torch.float64)
    emu = lowered_forward_f16emu(low, x)
    assert 0 < helpers.rel_err(emu, ref) < 5e-3


def test_f16_emulation_refuses_a_grouped_conv():
    """The emulation restates dense convolutions only; a grouped one raises instead of running as if dense."""
    _, _, low = helpers.conv_case(64, 8, 8, 64, 3, 1, 1, relu=True)
    op = low["ops"][0]
    grouped = dict(low, ops=[dict(op, groups=2, W=op["W"][..., :32])])
    with pytest.raises(ValueError, match="has 2 groups"):
        lowered_forward_f16emu(grouped, np.zeros((1, 64, 8, 8), np.float32))


def test_caffe_ceil_pooling_matches_definition():
    net = {"name": "p", "input": "data", "input_dims": [1, 1, 6, 6],
           "layers": [dict(name="pool", type="Pooling", bottoms=["data"], tops=["pool"], pool="MAX",
                           kernel_size=3, stride=2, pad=0)]}
    x = np.arange(36, dtype=np.float32).reshape(1, 1, 6, 6)
    got = caffe_forward(net, {}, x).reshape(3, 3)  # ceil((6-3)/2)+1 = 3, last window clipped
    want = np.array([[14, 16, 17], [26, 28, 29], [32, 34, 35]], dtype=np.float64)
    np.testing.assert_array_equal(got, want)
    assert graph.infer_shapes(net)["pool"] == (1, 3, 3)


def test_softmax_rows_sum_to_one():
    net = graph.resnet_caffe(50)
    tail = dict(net, layers=net["layers"][-3:], input="res5c", input_dims=[1, 2048, 7, 7])
    w = weights.random_weights(tail, 1)
    x = np.abs(np.random.default_rng(2).standard_normal((3, 2048, 7, 7), dtype=np.float32))
    p = caffe_forward(tail, w, x)
    np.testing.assert_allclose(p.sum(1), 1.0, atol=1e-6)
