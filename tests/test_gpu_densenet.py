"""DenseNet on the H100: the BatchNorm + ReLU prologue 1x1 against its emulation under every admitted tactic, prefix reads
that never see a later layer's channels, the prologue average pools and the pitched max pool bit for bit, and the whole
fp16 networks against the float64 oracle and the fp16 emulation, with the invariances every plan keeps."""
from __future__ import annotations

import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle.caffe_forward import avgpool_pre_ref, conv_pre_emu, prologue_f32, r16
from tensorrt_laboratory_b200 import builder, capi, graph, weights
from tests.cnn_nets import dense_net

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def _one_torch_thread():
    """The per-op references run on one CPU thread: torch's thread pool would otherwise stay behind in this process and
    disturb the host latencies that later GPU tests measure."""
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    yield
    torch.set_num_threads(n)


def _run(blob, x, options=None, passes=1):
    eng = capi.Engine(blob)
    s = capi.Session(eng, options)
    try:
        outs = [s.infer(x) for _ in range(passes)]
        names = [s._lib.b2_context_launch_name(s.ctx, x.shape[0], i).decode() for i in range(s.nb_launches(x.shape[0]))]
    finally:
        s.close()
        eng.destroy()
    return (outs if passes > 1 else outs[0]), names


def _ulp16(v):
    a = np.maximum(np.abs(np.asarray(v, np.float64)), 2.0 ** -14)
    return 2.0 ** (np.floor(np.log2(a)) - 10)


def _terms(op, a):
    """sum |w| |a'| + |bias| of a prologue 1x1 on fp16 values a: the scale of its fp32 accumulation error."""
    pa = r16(prologue_f32(a[:, :op["cin"]], op["pre_scale"], op["pre_shift"]))
    w = r16(torch.from_numpy(op["W"]).double()).permute(0, 3, 1, 2).abs()
    return (torch.nn.functional.conv2d(pa.abs(), w) + torch.from_numpy(op["bias"]).double().abs().view(1, -1, 1, 1)).numpy()


OPTIONS = [None, {"bn": 64}, {"bn": 128}, {"bn": 32, "stages": 2}, {"sps": 2}, {"stages": 8}, {"bn": 64, "halo": 1}, {"splits": 2},
           {"ws": 1}]


# (stem width, dense layers, plane, batch): block-2 prefixes 64, 96, 128, 160 / 960, 992; M = batch * (plane / 2)^2 = 192 /
# 180 rows, ragged against the 128-row tile
@pytest.mark.parametrize("cin, layers, hw, batch", [(64, 4, 16, 3), (960, 2, 12, 5)])
def test_prologue_conv_against_the_emulation(gpu, cin, layers, hw, batch):
    net = dense_net(cin=cin, hw=hw, layers=layers)
    low = graph.lower(net, weights.random_weights(net, cin + layers))
    block = f"concat_2_{layers}"
    x1 = [o for o in low["ops"] if o.get("pre") and o["type"] == graph.OP_CONV and o["input"] == block]
    assert [o["cin"] for o in x1] == [cin + 32 * l for l in range(layers)]
    taps = [block] + [o["output"] for o in x1]
    blob = builder.build_plan(low, builder.PREC_FP16, max_batch=batch + 1, outputs=["prob"] + taps)
    x = weights.synthetic_input(batch, chw=(3, hw, hw), seed=hw)
    for opt in OPTIONS:
        out, names = _run(blob, x, opt)
        a = torch.from_numpy(out[block].astype(np.float64))
        for op in x1:
            ref = conv_pre_emu(op, a).numpy()
            got = out[op["output"]]
            # 2 fp16 ulp of the result plus the worst case of K fp32 additions, K 2^-24 sum |w a| (a sum that cancels to
            # almost nothing has an error relative to its terms, not to itself)
            err = np.abs(got - ref) / (2 * _ulp16(ref) + op["cin"] * 2.0 ** -24 * _terms(op, a))
            assert float(err.max()) <= 1, (opt, op["name"], float(err.max()))
            launch = next(n for n in names if n.startswith(f"conv_tcgen05:{op['name']} "))
            assert " pre" in launch and " tiled" in launch and " ws=" not in launch and " halo" not in launch, (opt, launch)
            assert launch.split("grid=")[1].split()[0].endswith("x1"), (opt, launch)  # no split-K


def test_stale_channels_never_leak_into_a_prefix_read(gpu):
    # conv2_2/x1 reads [0, 96) of the block tensor (cin_phys 128); conv2_2/x2 writes [96, 128) after it.  With that slice's
    # weights overflowing to +-Inf, the second pass finds non-finite values in the channels the reader's 64-channel block
    # spans.
    net = dense_net(cin=64, hw=16, layers=3)
    wts = weights.random_weights(net, 3)
    hot = {k: dict(v) for k, v in wts.items()}
    hot["conv2_2/x2"]["W"] = wts["conv2_2/x2"]["W"] * 1e6
    x = weights.synthetic_input(2, chw=(3, 16, 16), seed=4)
    outs = []
    for w in (wts, hot):
        low = graph.lower(net, w)
        reader = next(o for o in low["ops"] if o["name"] == "conv2_2/x1")
        assert reader["cin"] == 96
        blob = builder.build_plan(low, builder.PREC_FP16, max_batch=2, outputs=["prob", reader["output"], "concat_2_3"])
        (first, second), _ = _run(blob, x, passes=2)
        outs.append((first[reader["output"]], second[reader["output"]], second["concat_2_3"]))
    assert not np.isfinite(outs[1][2][:, 96:128]).all()  # the overflow happened (+-Inf, and NaN where Infs met)
    assert np.array_equal(outs[1][0], outs[1][1])
    assert np.array_equal(outs[1][0], outs[0][0])
    assert np.array_equal(outs[0][0], outs[0][1])


@pytest.mark.parametrize("cin, layers, hw, pool, c", [(64, 3, 16, "conv2_blk/pool", 160), (128, 2, 28, "pool5", 160)])
def test_prologue_pools_are_bit_exact(gpu, cin, layers, hw, pool, c):
    net = dense_net(cin=cin, hw=hw, layers=layers)
    low = graph.lower(net, weights.random_weights(net, 7))
    op = next(o for o in low["ops"] if o["output"] == pool)
    assert op["type"] == graph.OP_AVGPOOL and op.get("pre") and low["tensors"][op["input"]][0] == c and c % 64 == 32
    blob = builder.build_plan(low, builder.PREC_FP16, max_batch=3, outputs=["prob", op["input"], pool])
    x = weights.synthetic_input(3, chw=(3, hw, hw), seed=11)
    out, names = _run(blob, x)
    src = torch.from_numpy(out[op["input"]].astype(np.float64))
    k = op["k"] if pool != "pool5" else src.shape[2]
    ref = avgpool_pre_ref(src, op["pre_scale"], op["pre_shift"], k).numpy()
    assert np.array_equal(out[pool].reshape(ref.shape), ref)
    assert any(n.startswith(f"avgpool_bnrelu:{op['name']}") for n in names), names
    assert not any(n.startswith("tail_pool_fc_softmax") for n in names)


def test_pitched_max_pool_equals_the_unpitched_one(gpu):
    net = dense_net(cin=64, hw=20, layers=2)
    wts = weights.random_weights(net, 5)
    low = graph.lower(net, wts)
    blob = builder.build_plan(low, builder.PREC_FP16, max_batch=2, outputs=["prob", "concat_2_2"])
    stem = dict(net, layers=[L for L in net["layers"] if L["name"] in ("conv1", "conv1/bn", "conv1/scale", "relu1", "pool1")])
    blob_stem = builder.build_plan(graph.lower(stem, wts), builder.PREC_FP16, max_batch=2, outputs=["pool1"])
    x = weights.synthetic_input(2, chw=(3, 20, 20), seed=6)
    out, names = _run(blob, x)
    plain, plain_names = _run(blob_stem, x)
    assert plain["pool1"].shape[1:] == (64, 10, 10)
    assert np.array_equal(out["concat_2_2"][:, :64], plain["pool1"])
    assert any(n.startswith("maxpool:pool1") for n in names) and any(n.startswith("maxpool:pool1") for n in plain_names)


# ---- whole DenseNets --------------------------------------------------------------------------------------------------
def _oracles(tmp_path, depth, batch):
    """float64 oracle and fp16 emulation (probabilities) of the seeded DenseNet, in a child process: their
    activations and torch's CPU thread pool should not stay in the process that times the engine later."""
    code = ("import sys, numpy as np; sys.path.insert(0, sys.argv[1]);"
            "from tensorrt_laboratory_b200 import graph, weights; import torch; from oracle.caffe_forward import caffe_forward, lowered_forward_f16emu;"
            "d, b = int(sys.argv[3]), int(sys.argv[4]); net = graph.densenet_caffe(d); wts = weights.random_weights(net, 0);"
            "x = weights.synthetic_input(b, seed=77); low = graph.lower(net, wts);"
            "np.savez(sys.argv[2], ref=caffe_forward(net, wts, x, dtype=torch.float64), emu=lowered_forward_f16emu(low, x))")
    out = tmp_path / f"oracles{depth}.npz"
    subprocess.run([sys.executable, "-c", code, ROOT, str(out), str(depth), str(batch)], check=True, timeout=1800)
    z = np.load(out)
    return z["ref"], z["emu"]


@pytest.fixture(scope="module")
def densenet121(gpu):
    blob = builder.build_densenet_plan(121, max_batch=8)
    x = weights.synthetic_input(8, seed=77)
    return blob, x


def test_densenet121_against_the_oracles(densenet121, tmp_path):
    blob, x = densenet121
    out, names = _run(blob, x)
    prob = out["prob"].reshape(8, -1)
    ref, emu = _oracles(tmp_path, 121, 8)
    rel = float(np.abs(prob - ref).max() / np.abs(ref).max())
    rel_emu = float(np.abs(prob - emu).max() / np.abs(emu).max())
    floor = float(np.abs(emu - ref).max() / np.abs(ref).max())
    print(f"DenseNet-121 fp16: prob rel {rel:.2e} vs float64 (emulation {floor:.2e}), {rel_emu:.2e} vs the emulation")
    assert float(np.abs(prob - ref).max()) <= 1e-3
    assert np.array_equal(prob.argmax(1), ref.argmax(1))
    assert rel_emu <= floor + 1e-3, (rel_emu, floor)
    assert sum(" pre" in n for n in names) == 58
    assert sum(n.startswith("avgpool_bnrelu:") for n in names) == 4
    assert sum(" c0=" in n for n in names) == 58 + 3
    assert any(n.startswith("maxpool:pool1") for n in names)
    assert not any(n.startswith(("conv_simt", "tail_pool_fc_softmax")) for n in names)


def test_densenet121_invariance(densenet121):
    blob, x = densenet121
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
    tuned, names = _run(tuned_blob, x)
    assert np.array_equal(again, full)
    assert np.array_equal(permuted, full[perm])
    assert np.array_equal(part, full[:5])
    assert np.array_equal(other, full)
    assert np.array_equal(tuned["prob"], full)
    assert sum(" pre" in n for n in names) == 58
    m = capi.InferenceManager(max_exec_concurrency=1)
    try:
        m.register_model("densenet121", blob)
        m.update_resources()
        for batch in (x, x[:5]):
            got = m.infer("densenet121", batch)
            assert np.array_equal(np.asarray(got).reshape(batch.shape[0], -1), full[:batch.shape[0]].reshape(batch.shape[0], -1))
    finally:
        m.close()


@pytest.mark.parametrize("depth", [169, 201])
def test_deeper_densenets_against_the_oracle(gpu, depth, tmp_path):
    blob = builder.build_densenet_plan(depth, max_batch=2)
    x = weights.synthetic_input(2, seed=77)
    out, names = _run(blob, x)
    prob = out["prob"].reshape(2, -1)
    ref, _ = _oracles(tmp_path, depth, 2)
    print(f"DenseNet-{depth} fp16: prob max abs error {float(np.abs(prob - ref).max()):.2e} vs float64")
    assert float(np.abs(prob - ref).max()) <= 1e-3
    assert np.array_equal(prob.argmax(1), ref.argmax(1))
    assert sum(" pre" in n for n in names) == sum(graph._DENSENET_BLOCKS[depth])
