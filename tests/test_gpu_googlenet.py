"""GoogLeNet on the H100: convolutions that store into their channel slice of a concatenated tensor, under every tactic
the rule admits; lrn_h8_kernel against float64; the whole fp16 network against the fp32 and fp16-emulating oracles; and
the invariances every plan keeps (batch position, partial batch, replay, contexts, tuning, InferenceManager)."""
from __future__ import annotations

import copy
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle.caffe_forward import lrn_f16emu
from oracle.numpy_ops import lrn as lrn_numpy
from tensorrt_laboratory_b200 import builder, capi, graph, weights
from tests.cnn_nets import inception_net

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(blob, x, options=None):
    eng = capi.Engine(blob)
    s = capi.Session(eng, options)
    try:
        out = s.infer(x)
        names = [s._lib.b2_context_launch_name(s.ctx, x.shape[0], i).decode() for i in range(s.nb_launches(x.shape[0]))]
    finally:
        s.close()
        eng.destroy()
    return out, names


def _ulp16(v):
    a = np.maximum(np.abs(np.asarray(v, np.float64)), 2.0 ** -14)
    return 2.0 ** (np.floor(np.log2(a)) - 10)


def _split_net(net):
    """The same net with the Concat removed: its inputs become separate outputs."""
    n2 = copy.deepcopy(net)
    cat = next(L for L in n2["layers"] if L["type"] == "Concat")
    n2["layers"].remove(cat)
    return n2, cat["bottoms"]


# ---- concatenation geometry ----------------------------------------------------------------------------------------
# branch widths: offsets multiples of 8 but not of 64, with and without a tail pad (c_phys > c)
WIDTHS = [(16, 32, 48, 96), (16, 32, 48, 112), (112, 208, 48, 16), (96, 208, 16, 32)]
GEOMS = [(1, 3), (7, 5), (13, 2), (14, 4), (28, 1)]  # (plane, batch)
OPTIONS = [None, {"bn": 64}, {"bn": 128}, {"stages": 2}, {"bn": 64, "halo": 1}, {"splits": 2}, {"ws": 1}]


def _emu_conv(op, a):
    """One lowered convolution with the fp16 engine's rounding points on its (fp16) input a (NCHW) -> (result, bound): the
    bound is 2 fp16 ulp of the result plus the worst case of K fp32 additions, K 2^-24 sum |w x| (a sum that cancels to
    almost nothing, at a ReLU's edge, has an error relative to its terms, not to itself)."""
    import torch
    import torch.nn.functional as F
    w = torch.from_numpy(op["W"]).double().to(torch.float16).double().permute(0, 3, 1, 2)
    xa = torch.from_numpy(np.asarray(a, np.float64))
    b = torch.from_numpy(op["bias"]).double().view(1, -1, 1, 1)
    y = F.conv2d(xa, w, None, stride=op["stride"], padding=op["pad"]) + b
    y = (torch.relu(y) if op["relu"] else y).to(torch.float16).double().numpy()
    terms = (F.conv2d(xa.abs(), w.abs(), None, stride=op["stride"], padding=op["pad"]) + b.abs()).numpy()
    return y, 2 * _ulp16(y) + w[0].numel() * 2.0 ** -24 * terms


@pytest.mark.parametrize("widths", WIDTHS, ids=lambda w: "-".join(map(str, w)))
@pytest.mark.parametrize("hw, batch", GEOMS, ids=lambda v: str(v))
def test_slices_equal_the_host_concatenation(gpu, widths, hw, batch):
    net = inception_net(cin=64, hw=hw, widths=widths)
    wts = weights.random_weights(net, seed=hw + batch)
    low = graph.lower(net, wts)
    split, branches = _split_net(net)
    low_split = graph.lower(split, wts)
    x = np.random.default_rng(hw).standard_normal((batch, 64, hw, hw)).astype(np.float32)
    blob = builder.build_plan(low, builder.PREC_FP16, max_batch=batch + 1)  # (a partial batch of its plan)
    inputs = {"b/1x1": "data", "b/3x3": "b/3x3_reduce", "b/5x5": "b/5x5_reduce", "b/pool_proj": "b/pool"}
    blob_split = builder.build_plan(low_split, builder.PREC_FP16, max_batch=batch + 1, outputs=branches + ["b/3x3_reduce", "b/5x5_reduce",
                                                                                                              "b/pool"])
    ops = {o["name"]: o for o in low["ops"]}
    for opt in OPTIONS:
        out, names = _run(blob, x, opt)
        parts, _ = _run(blob_split, x, opt)
        cat = out["b/output"]
        assert np.array_equal(cat, np.concatenate([parts[b] for b in branches], axis=1)), (opt, names)
        slices = [n for n in names if " c0=" in n]
        assert len(slices) == 4 and all(n.startswith("conv_tcgen05:") for n in slices), names
        # each convolution against the emulation on its own (engine-computed) input
        parts["data"] = x.astype(np.float16).astype(np.float64)
        for b in branches:
            c0 = ops[b]["out_c0"]
            ref, bound = _emu_conv(ops[b], parts[inputs[b]])
            got = cat[:, c0:c0 + ops[b]["cout"]]
            assert np.all(np.abs(got - ref) <= bound), (opt, b, float((np.abs(got - ref) / bound).max()))


def test_slice_launch_names_and_tactics(gpu):
    net = inception_net(cin=64, hw=14, widths=(16, 32, 48, 112))
    low = graph.lower(net, weights.random_weights(net, 3))
    x = np.random.default_rng(0).standard_normal((2, 64, 14, 14)).astype(np.float32)
    blob = builder.build_plan(low, builder.PREC_FP16, max_batch=2)
    _, names = _run(blob, x)
    cw = {n.split(":")[1].split(" ")[0]: n.split(" c0=")[1] for n in names if " c0=" in n}
    assert cw == {"b/1x1": "0 cw=16", "b/3x3": "16 cw=32", "b/5x5": "48 cw=48", "b/pool_proj": "96 cw=160"}, names
    _, halo = _run(blob, x, {"bn": 64, "halo": 1})
    assert any(n.startswith("conv_tcgen05:b/3x3 ") and " halo" in n for n in halo), halo
    _, ws = _run(blob, x, {"ws": 1})
    assert any(" ws=" in n for n in ws if " c0=" in n), ws  # (where a persistent configuration exists for the N tile)
    with pytest.raises(capi.B2Error, match="only the tensor-core kernels"):
        _run(blob, x, {"simt": 1})


def test_refused_table_entry_falls_back_to_the_cost_model(gpu):
    net = inception_net(cin=64, hw=14, widths=(16, 32, 48, 112))
    low = graph.lower(net, weights.random_weights(net, 5))
    x = np.random.default_rng(1).standard_normal((2, 64, 14, 14)).astype(np.float32)
    blob = builder.build_plan(low, builder.PREC_FP16, max_batch=2)
    want, _ = _run(blob, x, {"autotune": 0})
    ops = [o["name"] for o in low["ops"]]
    k3 = 1 + ops.index("b/3x3")  # plan op index (op 0 is the input cast)
    # {op, batch, bn, stages, splits, sps, ws, cn, halo, 0}: the fused 3x3 + 1x1 record, and an N tile wider than the slice's rows
    table = np.array([[k3, 2, 64, 2, 1, 1, 0, 1, 2, 0], [k3 + 2, 2, 256, 2, 1, 1, 0, 1, 0, 0]], np.uint32)
    got, names = _run(builder.attach_tactics(blob, table), x)
    assert np.array_equal(got["b/output"], want["b/output"])
    assert not any("halo fused" in n for n in names), names


def test_tail_padding_is_rewritten_every_pass(gpu):
    """c = 208, c_phys = 256: a consumer reads the padding channels 208 ... 255 (with zero weights).  An overflowing request
    leaves NaN there (0 x inf); the next request must rewrite them, or the consumer's sums stay NaN."""
    net = inception_net(cin=64, hw=7, widths=(16, 32, 48, 112))
    net["layers"].append(dict(name="after", type="Convolution", bottoms=["b/output"], tops=["after"], num_output=64, kernel_size=1,
                              pad=0, stride=1, bias_term=True))
    low = graph.lower(net, weights.random_weights(net, 9))
    blob = builder.build_plan(low, builder.PREC_FP16, max_batch=2)
    x = np.random.default_rng(2).standard_normal((2, 64, 7, 7)).astype(np.float32)
    fresh, _ = _run(blob, x)
    eng = capi.Engine(blob)
    s = capi.Session(eng)
    try:
        hot = s.infer(x * 6e4)["after"]
        assert not np.all(np.isfinite(hot))  # the overflow reached the tensor
        again = s.infer(x)
    finally:
        s.close()
        eng.destroy()
    assert np.array_equal(again["after"], fresh["after"])
    assert np.all(np.isfinite(fresh["after"]))


# ---- LRN ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", [64, 100, 192])
@pytest.mark.parametrize("n", [3, 5, 7])
@pytest.mark.parametrize("k", [1.0, 2.0])
@pytest.mark.parametrize("beta", [0.75, 0.5])
def test_lrn_against_float64(gpu, c, n, k, beta):
    alpha = 0.05
    net = {"name": "lrn", "input": "data", "input_dims": [1, c, 5, 6],
           "layers": [dict(name="norm", type="LRN", bottoms=["data"], tops=["norm"], local_size=n, alpha=alpha, beta=beta, k=k)]}
    low = graph.lower(net, {})
    x = (np.random.default_rng(c + n).standard_normal((3, c, 5, 6)) * 4).astype(np.float32)
    x[:, :, 0, 0] = 40.0  # a pixel where the normalisation dominates
    out, names = _run(builder.build_plan(low, builder.PREC_FP16, max_batch=3), x)
    y = out["norm"]
    assert any(nm.startswith("lrn:norm") for nm in names), names
    x16 = x.astype(np.float16).astype(np.float64)
    ref = lrn_numpy(x16, n, alpha, beta, k)
    assert float(np.abs(ref - x16).max()) > 1.0  # the normalisation changes the values
    # fp16 output rounding (2^-11) plus the fp32 sum and powf: within 1.5 fp16 ulp of the float64 value, edges included
    err = np.abs(y - ref) / _ulp16(ref)
    assert float(err.max()) <= 1.5, float(err.max())
    emu = lrn_f16emu(__import__("torch").from_numpy(x16), n, alpha, beta, k).numpy()
    assert float((np.abs(y - emu) / _ulp16(emu)).max()) <= 1.0


# ---- whole GoogLeNet --------------------------------------------------------------------------------------------------
def _googlenet_oracles(tmp_path):
    """The fp32 oracle and the fp16 emulation of the fixture's network and images, run in a child process: the two forward
    passes hold several GB of float64 activations and start torch's CPU thread pool, none of which should stay in the
    process that goes on to time the engine."""
    code = ("import sys, numpy as np; sys.path.insert(0, sys.argv[1]);"
            "from tensorrt_laboratory_b200 import graph, weights; from oracle.caffe_forward import caffe_forward, lowered_forward_f16emu;"
            "net = graph.googlenet_caffe(); wts = weights.random_weights(net, 0); x = weights.synthetic_input(8, seed=77);"
            "np.savez(sys.argv[2], ref=caffe_forward(net, wts, x), emu=lowered_forward_f16emu(graph.lower(net, wts), x))")
    out = tmp_path / "oracles.npz"
    subprocess.run([sys.executable, "-c", code, ROOT, str(out)], check=True, timeout=900)
    z = np.load(out)
    return z["ref"], z["emu"]


@pytest.fixture(scope="module")
def googlenet(gpu):
    net = graph.googlenet_caffe()
    wts = weights.random_weights(net, 0)
    low = graph.lower(net, wts)
    blob = builder.build_plan(low, builder.PREC_FP16, max_batch=8)
    x = weights.synthetic_input(8, seed=77)
    return net, wts, low, blob, x


def test_googlenet_against_the_oracles(googlenet, tmp_path):
    net, wts, low, blob, x = googlenet
    out, names = _run(blob, x)
    prob = out["prob"].reshape(8, -1)
    ref, emu = _googlenet_oracles(tmp_path)
    rel = float(np.abs(prob - ref).max() / np.abs(ref).max())
    rel_emu = float(np.abs(prob - emu).max() / np.abs(emu).max())
    # fp16 storage alone (the emulation) is this far from fp32 on the seeded net; the engine's fp32 sums are ordered
    # differently from the emulation's exact ones, so it drifts from the emulation by about as much again
    floor = float(np.abs(emu - ref).max() / np.abs(ref).max())
    top = np.sort(ref, axis=1)
    margin = (top[:, -1] - top[:, -2]) / top[:, -1]
    clear = margin > 4 * rel
    print(f"GoogLeNet fp16: rel {rel:.2e} vs fp32 (emulation {floor:.2e} vs fp32), {rel_emu:.2e} vs fp16 emulation; "
          f"top-1 margins {np.round(margin, 4)}")
    assert rel <= 2 * floor + 1e-3, (rel, floor)
    assert rel_emu <= floor + 1e-3, (rel_emu, floor)
    assert np.array_equal(prob.argmax(1)[clear], ref.argmax(1)[clear])
    assert sum(n.startswith("lrn:") for n in names) == 2
    assert sum(" c0=" in n for n in names) == 36, names
    assert any(n.startswith("conv_tcgen05:conv1/7x7_s2 ") for n in names)
    assert names[0].startswith("input_cast:"), names[0]
    assert not any(n.startswith("conv_simt") for n in names)


def test_googlenet_space_to_depth_stem(googlenet):
    _, _, _, blob, _ = googlenet
    eng = capi.Engine(blob, inspect_only=True)
    try:
        assert eng.flops(1) == pytest.approx(graph.conv_flops(googlenet[2]))
    finally:
        eng.destroy()
    # the stem reads the space-to-depth input: an 8-channel tensor and a row-folded (kb=32) convolution
    _, names = _run(blob, googlenet[4][:1])
    stem = next(n for n in names if n.startswith("conv_tcgen05:conv1/7x7_s2 "))
    assert " kb=32" in stem, stem


def test_googlenet_invariance(googlenet):
    _, _, _, blob, x = googlenet
    eng = capi.Engine(blob)
    s = capi.Session(eng)
    try:
        full = s.infer(x)["prob"]
        again = s.infer(x)["prob"]
        perm = np.array([3, 1, 7, 0, 5, 2, 6, 4])
        permuted = s.infer(x[perm])["prob"]
        part = s.infer(x[:5])["prob"]
    finally:
        s.close()
    s2 = capi.Session(eng)
    try:
        other = s2.infer(x)["prob"]
    finally:
        s2.close()
    assert eng.tune(4) > 0
    tuned_blob = builder.attach_tactics(blob, eng.tactics())
    eng.destroy()
    tuned, _ = _run(tuned_blob, x)
    assert np.array_equal(again, full)
    assert np.array_equal(permuted, full[perm])
    assert np.array_equal(part, full[:5])
    assert np.array_equal(other, full)
    assert np.array_equal(tuned["prob"], full)
    m = capi.InferenceManager(max_exec_concurrency=1)
    try:
        m.register_model("googlenet", blob)
        m.update_resources()
        for batch in (x, x[:5]):
            got = m.infer("googlenet", batch)
            assert np.array_equal(np.asarray(got).reshape(batch.shape[0], -1), full[:batch.shape[0]].reshape(batch.shape[0], -1))
    finally:
        m.close()
