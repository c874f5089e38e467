"""CPU side of tests/test_gpu_geometry.py: its own-input references against torch in float64, and every one of its
geometries built into a plan that the engine accepts, so a builder or engine refusal shows up here and not on a GPU."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tensorrt_laboratory_b200 import builder, capi, graph, quantize, weights
from tests import test_gpu_geometry as G

FP16, FP32, INT8 = builder.PREC_FP16, builder.PREC_FP32, builder.PREC_INT8


def _accepts(blob):
    eng = capi.Engine(blob, inspect_only=True)
    eng.destroy()


# ------------------------------------------------------------------------------------------------------------------
# references
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", G.POOL_CASES)
def test_maxpool_reference_matches_torch(case):
    h, w, k, s, p, ceil = case
    x = np.random.default_rng(0).standard_normal((2, 3, h, w))
    want = F.max_pool2d(torch.from_numpy(x), k, s, padding=p, ceil_mode=ceil).numpy()   # implicit padding acts as -inf
    np.testing.assert_array_equal(G.maxpool_ref(x, k, s, p, ceil), want)
    np.testing.assert_array_equal(G.maxpool_ref(-np.abs(x), k, s, p, ceil), F.max_pool2d(torch.from_numpy(-np.abs(x)), k, s, padding=p, ceil_mode=ceil).numpy())
    for n in (h, w):
        assert G.pool_size(n, k, s, p, ceil) == graph.pool_out_ceil(n, k, p, s, ceil)


def test_pool_cases_cover_the_window_rules():
    sizes = {c: (G.pool_size(c[0], c[2], c[3], c[4], c[5]), G.pool_size(c[1], c[2], c[3], c[4], c[5])) for c in G.POOL_CASES}
    # a partial last window (ceil mode reads past the far edge) ...
    assert any(c[5] and ((ho - 1) * c[3] + c[2] - c[4] > c[0]) for c, (ho, _) in sizes.items())
    # ... a ceil-mode window that would start in the far padding and is dropped (14 + 2 - 3 = 13 -> ceil(13 / 3) + 1 = 6 -> 5)
    assert sizes[(14, 18, 3, 3, 1, True)][0] == 5 and -(-(14 + 2 - 3) // 3) + 1 == 6
    # ... and floor mode, which never reads the last row / column of 15 x 21
    assert sizes[(15, 21, 2, 2, 0, False)] == (7, 10)


def test_mean_fc_and_softmax_references_match_torch():
    rng = np.random.default_rng(1)
    x = rng.standard_normal((3, 24, 4, 5))
    np.testing.assert_allclose(G.mean_ref(x), torch.from_numpy(x).mean(dim=(2, 3)).numpy(), rtol=1e-14, atol=1e-15)
    W, b = rng.standard_normal((7, 24 * 4 * 5)), rng.standard_normal(7)
    y, mag = G.fc_ref(x, W, b)
    np.testing.assert_allclose(y, F.linear(torch.from_numpy(x).flatten(1), torch.from_numpy(W), torch.from_numpy(b)).numpy(), rtol=1e-13, atol=1e-13)
    assert (mag >= np.abs(y)).all()
    logits = rng.standard_normal((4, 2100)) * 4
    np.testing.assert_allclose(G.softmax_ref(logits), torch.softmax(torch.from_numpy(logits), 1).numpy(), rtol=1e-13, atol=0)
    # an fp32 softmax (torch's, on the CPU) lies within the bound the GPU test applies to the engine's
    l32 = logits.astype(np.float32)
    ref = G.softmax_ref(l32)
    got = torch.softmax(torch.from_numpy(l32), 1).numpy().astype(np.float64)
    assert (np.abs(got - ref) <= G.softmax_rel_bound(l32) * ref).all()


@pytest.mark.parametrize("case", G.FC_CASES)
def test_fc_reference_uses_the_order_the_plan_permutes_to(case):
    """The GPU test holds the engine's FC to the Caffe (C, H, W) flattening of the raw weights; the lowered op carries
    them in the engine's (H, W, C) order.  Both give the same product."""
    h, w, c, cout = case
    net = G.fc_net(h, w, c, cout)
    wts = weights.random_weights(net, 7)
    op = [o for o in graph.lower(net, wts)["ops"] if o["type"] == graph.OP_FC][0]
    x = np.random.default_rng(2).standard_normal((2, c, h, w))
    want, _ = G.fc_ref(x, wts["fc"]["W"], wts["fc"]["b"])
    got = x.transpose(0, 2, 3, 1).reshape(2, -1) @ op["W"].astype(np.float64).T + op["bias"]
    np.testing.assert_allclose(got, want, rtol=1e-6, atol=1e-6)


def test_fp16_ulp_and_fc_bound():
    assert G.fp16_ulp(1.0) == 2.0 ** -10 and G.fp16_ulp(-0.75) == 2.0 ** -11
    assert G.fc_bound(2048, 1.0) == 2049 * 2.0 ** -24


# ------------------------------------------------------------------------------------------------------------------
# every geometry of the GPU file builds, and the engine accepts the plan
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", G.CONV_CASES + [G.COUT320], ids=G._case_id)
def test_conv_cases_build(case):
    cin, h, w, cout, k, s, p, res, batch = case
    ho, wo = graph.conv_out(h, k, p, s), graph.conv_out(w, k, p, s)
    assert (batch * ho * wo) % 128, "the batch must leave a ragged last M tile"
    for relu in (True, False):
        low = graph.lower(G.conv_net(case, relu), weights.random_weights(G.conv_net(case, relu), 0))
        for prec in (FP16, FP32):
            _accepts(builder.build_plan(low, prec, batch))
    if cin <= 4:
        _accepts(builder.build_plan(low, FP16, batch, input_dtype="f16"))


def test_edge_cases_end_on_the_far_edge():
    """The stride-2 cases whose (size + 2 pad - k) divides by the stride: the last window ends exactly on the edge."""
    for cin, h, w, cout, k, s, p, res, batch in G.EDGE_CASES + [G.CONV_CASES[1]]:
        assert s == 2 and (h + 2 * p - k) % s == 0 and (w + 2 * p - k) % s == 0


@pytest.mark.parametrize("c", [64, 3, 5])
@pytest.mark.parametrize("case", G.POOL_CASES)
def test_maxpool_cases_build(case, c):
    net = G.conv_pool_net(c, *case)
    low = graph.lower(net, weights.random_weights(net, 2))
    h, w, k, s, p, ceil = case
    assert low["tensors"]["pool"] == (c, G.pool_size(h, k, s, p, ceil), G.pool_size(w, k, s, p, ceil))
    for prec in (FP16, FP32):
        _accepts(builder.build_plan(low, prec, 3, outputs=["conv", "pool"]))


@pytest.mark.parametrize("case", G.TAIL_CASES)
def test_tail_cases_build(case):
    net, wts, low, x = G.tail_graph(case)
    for prec in (FP16, FP32):
        _accepts(builder.build_plan(low, prec, case[0], outputs=["conv", "pool", "fc", "prob"]))
        _accepts(builder.build_plan(low, prec, case[0], outputs=["conv", "pool", "prob"]))
    assert G.tail_applies(case) == (case[2] not in (100, 2560))


@pytest.mark.parametrize("case", G.FC_CASES)
def test_fc_cases_build(case):
    h, w, c, cout = case
    net = G.fc_net(h, w, c, cout)
    low = graph.lower(net, weights.random_weights(net, 7))
    for prec in (FP16, FP32):
        _accepts(builder.build_plan(low, prec, 5, outputs=["conv", "fc"]))
    k = h * w * builder.phys_channels(c, FP16)
    assert (k % 256 == 0 and k <= 2048) == (h * w != 49)   # fc_h8 for 4x5, the generic kernel for 7x7


@pytest.mark.parametrize("w", G.CAST_WIDTHS)
@pytest.mark.parametrize("c", G.CAST_CHANNELS)
def test_input_cast_cases_build(c, w):
    net = G.conv_net((c, 20, w, 64, 7, 2, 3, False, 3), relu=False)
    low = graph.lower(net, weights.random_weights(net, 9))
    for dt in ("f32", "f16"):
        _accepts(builder.build_plan(low, FP16, 3, input_dtype=dt))


def _i8_accepts(low, x, outputs=None):
    lq = quantize.quantize_lowered(low, x)
    assert all(o.get("int8") for o in lq["ops"] if o["type"] == graph.OP_CONV)
    _accepts(builder.build_plan(lq, INT8, x.shape[0], outputs=outputs))
    return lq


def test_int8_cases_build():
    rng = np.random.default_rng(3)
    cin, h, w, cout, k, s, p = G.I8_DEEP
    lq = _i8_accepts(G.i8_graph(cin, h, w, cout, k, s, p), rng.standard_normal((3, cin, h, w)).astype(np.float32))
    assert k * k * cin // 128 == 18
    for cin, cout in G.I8_CHANNELS:
        _i8_accepts(G.i8_graph(cin, 14, 14, cout, 3, 1, 1), rng.standard_normal((3, cin, 14, 14)).astype(np.float32))
    for cin, h, w, cout, k, s, p in G.I8_GEOMS:
        for res in (False, True):
            _i8_accepts(G.i8_graph(cin, h, w, cout, k, s, p, residual=res), rng.standard_normal((3, cin, h, w)).astype(np.float32))
    low = G.i8_graph(64, 4, 6, 64, 1, 1, 0, relu=False)
    _i8_accepts(low, rng.standard_normal((2, 64, 4, 6)).astype(np.float32), outputs=["data_q", "conv"])
    for hw in G.I8_POOL_HW:
        net = builder.single_conv_net(64, hw, hw, 320, 1, 1, 0, relu=False)
        net["layers"].append(dict(name="pool", type="Pooling", bottoms=["conv"], tops=["pool"], pool="AVE", kernel_size=hw, stride=1, pad=0))
        lq = _i8_accepts(graph.lower(net, weights.random_weights(net, 19)), rng.standard_normal((3, 64, hw, hw)).astype(np.float32))
        assert lq["ops"][-1]["type"] == graph.OP_AVGPOOL and "k_scale" in lq["ops"][-1]


def test_int8_quantize_ties_table_is_round_half_even():
    for v, q in G._TIES.items():
        assert q == int(np.clip(np.rint(np.float32(v) * np.float32(0.5)), -127, 127)), v


def test_resnet50_200x264_builds():
    net = G.resnet50_200x264()
    low = graph.lower(net, weights.random_weights(net, 0))
    t = low["tensors"]
    assert t["conv1"] == (64, 100, 132) and t["pool1"] == (64, 50, 66)
    assert t["res3a"] == (512, 25, 33) and t["res4a"] == (1024, 13, 17) and t["res5c"] == (2048, 7, 9)
    # the halo tile rows R = 128 // (W + 2) of the four stages' 3x3 convolutions
    assert [min(128 // (t[f"res{s}a"][2] + 2), t[f"res{s}a"][1]) for s in (2, 3, 4, 5)] == [1, 3, 6, 7]
    _accepts(builder.build_plan(low, FP16, 3, outputs=G.WIDE_TAPS))
    lq = quantize.quantize_lowered(low, weights.synthetic_input(1, chw=(3, 200, 264), seed=4321))
    _accepts(builder.build_plan(lq, INT8, 2, outputs=["pool1", "res3d", "res5c"]))
    # the full classifier does not lower: a global AVE pool needs a square map
    full = graph.resnet_caffe(50)
    full["input_dims"] = [1, 3, 200, 264]
    with pytest.raises(ValueError, match="global AVE"):
        graph.lower(full, weights.random_weights(full, 0))
