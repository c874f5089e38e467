"""VGG on the H100: the streaming split-K FC kernel one op at a time against a float64 product of its fp16 operands, its
plan refusals on a real engine, and VGG-16 / VGG-19 end to end against the float64 oracle and the fp16 emulation, with the
invariances every plan keeps."""
from __future__ import annotations

import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle.caffe_forward import fc_ref
from tensorrt_laboratory_b200 import builder, capi, graph, weights
from tests.cnn_nets import fc_net

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def _one_torch_thread():
    """The references run on one CPU thread: torch's thread pool would otherwise stay behind in this process and disturb
    the host latencies that later GPU tests measure."""
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    yield
    torch.set_num_threads(n)


def _ulp16(v):
    a = np.maximum(np.abs(np.asarray(v, np.float64)), 2.0 ** -14)
    return 2.0 ** (np.floor(np.log2(a)) - 10)


def _names(s, batch):
    return [s._lib.b2_context_launch_name(s.ctx, batch, i).decode() for i in range(s.nb_launches(batch))]


def _check_fc(op, x16, got, hidden):
    """got within 2 fp16 ulp plus the fp32 accumulation bound K 2^-23 sum |w| |x| of the float64 reference."""
    ref, terms = fc_ref(op, x16)
    err = np.abs(got - ref) / (2 * _ulp16(ref) + x16.shape[1] * 2.0 ** -23 * terms)
    assert float(err.max()) <= 1, (op["name"], float(err.max()))
    if hidden:  # fp16 values
        assert np.array_equal(got.astype(np.float16).astype(np.float64), got)


def _flat16(x):
    """fp32 NCHW input -> fp16 values in the engine's (h, w, c) K order, [N, K]"""
    return np.ascontiguousarray(x.astype(np.float16).astype(np.float64).transpose(0, 2, 3, 1)).reshape(x.shape[0], -1)


# (input C, H, W), first FC's Cout: K = H W C in {64, 576, 4096, 25088}, Cout in {1, 100, 1000, 4096}
CASES = [((64, 1, 1), 4096), ((64, 3, 3), 1), ((4096, 1, 1), 100), ((512, 7, 7), 1000), ((256, 4, 4), 4096), ((512, 7, 7), 100)]
BATCHES = [1, 3, 8, 17, 32, 64]


@pytest.mark.parametrize("chw, cout", CASES, ids=[f"K{c * h * w}_C{o}" for (c, h, w), o in CASES])
@pytest.mark.parametrize("relu", [True, False], ids=["relu", "linear"])
def test_fc_stream_against_float64(gpu, chw, cout, relu):
    """Two-FC plan: fc1 (hidden, fp16 out, ReLU on or off) -> fc2 (fp32 logits, 64 neurons); single-FC plan with a ReLU
    (fp32 out).  Every batch size from one engine of max batch 64, the same bits at each batch position."""
    k = int(np.prod(chw))
    net2 = fc_net(chw, [cout, 64], [relu, False])
    low2 = graph.lower(net2, weights.random_weights(net2, k + cout))
    fc1, fc2 = low2["ops"]
    assert fc1["hidden"] and not fc2["hidden"]
    blobs = [(builder.build_plan(low2, builder.PREC_FP16, max_batch=64, outputs=["fc1", "fc2"]), True)]
    if relu:
        net1 = fc_net(chw, [cout], [True])
        low1 = graph.lower(net1, weights.random_weights(net1, k + cout))
        blobs.append((builder.build_plan(low1, builder.PREC_FP16, max_batch=64, outputs=["fc1"]), False))
    x = weights.synthetic_input(64, chw=chw, seed=k % 97)
    x16 = _flat16(x)
    for blob, two in blobs:
        eng = capi.Engine(blob)
        s = capi.Session(eng)
        try:
            full = s.infer(x)
            names = _names(s, 64)
            fcs = [n for n in names if n.startswith("fc_stream_f16_wgmma:")]
            assert len(fcs) == (2 if two else 1) and all(re.search(r" splits=\d+ nb=64$", n) for n in fcs), names
            for b in BATCHES:
                part = s.infer(x[:b])
                for key in part:
                    assert np.array_equal(part[key], full[key][:b]), (b, key)
            perm = np.random.default_rng(k).permutation(64)
            permuted = s.infer(x[perm])
            again = s.infer(x)
        finally:
            s.close()
        s2 = capi.Session(eng)
        try:
            other = s2.infer(x)
        finally:
            s2.close()
            eng.destroy()
        for key in full:
            assert np.array_equal(permuted[key], full[key][perm]) and np.array_equal(again[key], full[key])
            assert np.array_equal(other[key], full[key])
        if two:
            h = full["fc1"].reshape(64, -1)
            _check_fc(fc1, x16, h, hidden=True)
            _check_fc(fc2, h, full["fc2"].reshape(64, -1), hidden=False)
        else:
            _check_fc(low1["ops"][0], x16, full["fc1"].reshape(64, -1), hidden=False)


def test_fc_stream_beyond_64_columns(gpu):
    """max batch 80: NB = 64 columns per CTA and a second column chunk along the grid; every batch gives the bits of the
    full one."""
    net = fc_net((512, 7, 7), [1000, 100], [True, False])
    low = graph.lower(net, weights.random_weights(net, 5))
    blob = builder.build_plan(low, builder.PREC_FP16, max_batch=80, outputs=["fc1", "fc2"])
    x = weights.synthetic_input(80, chw=(512, 7, 7), seed=9)
    eng = capi.Engine(blob)
    s = capi.Session(eng)
    try:
        full = s.infer(x)
        assert all(" nb=64" in n for n in _names(s, 80) if n.startswith("fc_stream"))
        for b in (1, 17, 64, 65, 79):
            part = s.infer(x[:b])
            for key in part:
                assert np.array_equal(part[key], full[key][:b]), (b, key)
    finally:
        s.close()
        eng.destroy()
    h = full["fc1"].reshape(80, -1)
    _check_fc(low["ops"][0], _flat16(x), h, hidden=True)
    _check_fc(low["ops"][1], h, full["fc2"].reshape(80, -1), hidden=False)


def test_fc_stream_refusals_on_a_real_engine(gpu):
    from tests.test_vgg_cpu import fc_mutations
    blob, muts = fc_mutations()
    capi.Engine(blob).destroy()
    for what, bad, msg in muts:
        with pytest.raises(capi.B2Error) as ei:
            capi.Engine(bad)
        assert ei.value.code == 1 and re.search(msg, str(ei.value)), (what, str(ei.value))


# ---- whole VGGs -----------------------------------------------------------------------------------------------------------
def _oracles(tmp_path, depth, batch):
    """float64 oracle and fp16 emulation (probabilities) of the seeded VGG, in a child process: their activations and
    torch's CPU thread pool should not stay in the process that times the engine later."""
    code = ("import sys, numpy as np; sys.path.insert(0, sys.argv[1]);"
            "from tensorrt_laboratory_b200 import graph, weights; import torch; from oracle.caffe_forward import caffe_forward, lowered_forward_f16emu;"
            "d, b = int(sys.argv[3]), int(sys.argv[4]); net = graph.vgg_caffe(d); wts = weights.random_weights(net, 0);"
            "x = weights.synthetic_input(b, seed=77); low = graph.lower(net, wts);"
            "np.savez(sys.argv[2], ref=caffe_forward(net, wts, x, dtype=torch.float64), emu=lowered_forward_f16emu(low, x))")
    out = tmp_path / f"oracles{depth}.npz"
    subprocess.run([sys.executable, "-c", code, ROOT, str(out), str(depth), str(batch)], check=True, timeout=1800)
    z = np.load(out)
    return z["ref"], z["emu"]


def _check_net(prob, ref, emu, names, label):
    rel = float(np.abs(prob - ref).max() / np.abs(ref).max())
    rel_emu = float(np.abs(prob - emu).max() / np.abs(emu).max())
    floor = float(np.abs(emu - ref).max() / np.abs(ref).max())
    print(f"{label} fp16: prob rel {rel:.2e} vs float64 (emulation {floor:.2e}), {rel_emu:.2e} vs the emulation")
    # the engine and the emulation are two fp16 computations whose roundings differ wherever fp32 accumulation lands on the
    # other side of an fp16 rounding boundary, so each is its own distance from float64: the engine within twice the
    # emulation's, and within the emulation's of the emulation (+ 1e-3 of the largest probability)
    assert rel <= 2 * floor + 1e-3, (rel, floor)
    assert rel_emu <= floor + 1e-3, (rel_emu, floor)
    assert np.array_equal(prob.argmax(1), ref.argmax(1))
    fcs = [n for n in names if n.startswith("fc_stream_f16_wgmma:")]
    assert [n.split(":")[1].split()[0] for n in fcs] == ["fc6", "fc7", "fc8"], names
    conv1 = next(n for n in names if n.startswith(("conv_tcgen05:conv1_1 ", "conv_simt:conv1_1")))
    assert conv1.startswith("conv_tcgen05:conv1_1 ") and " kb=8 " in conv1, conv1  # thin-input wgmma path (cin_phys 8)
    assert not any(n.startswith(("conv_simt", "fc:", "tail_pool_fc_softmax")) for n in names), names


@pytest.fixture(scope="module")
def vgg16(gpu):
    blob = builder.build_vgg_plan(16, max_batch=8)
    x = weights.synthetic_input(8, seed=77)
    return blob, x


def test_vgg16_against_the_oracles(vgg16, tmp_path):
    blob, x = vgg16
    eng = capi.Engine(blob)
    s = capi.Session(eng)
    try:
        prob = s.infer(x)["prob"].reshape(8, -1)
        names = _names(s, 8)
    finally:
        s.close()
        eng.destroy()
    ref, emu = _oracles(tmp_path, 16, 8)
    _check_net(prob, ref, emu, names, "VGG-16")


def test_vgg16_invariance(vgg16):
    blob, x = vgg16
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
    eng = capi.Engine(tuned_blob)
    s = capi.Session(eng)
    try:
        tuned = s.infer(x)["prob"]
    finally:
        s.close()
        eng.destroy()
    assert np.array_equal(again, full)
    assert np.array_equal(permuted, full[perm])
    assert np.array_equal(part, full[:5])
    assert np.array_equal(other, full)
    assert np.array_equal(tuned, full)
    m = capi.InferenceManager(max_exec_concurrency=1)
    try:
        m.register_model("vgg16", blob)
        m.update_resources()
        for batch in (x, x[:5]):
            got = m.infer("vgg16", batch)
            assert np.array_equal(np.asarray(got).reshape(batch.shape[0], -1), full[:batch.shape[0]].reshape(batch.shape[0], -1))
    finally:
        m.close()


def test_vgg19_against_the_oracles(gpu, tmp_path):
    blob = builder.build_vgg_plan(19, max_batch=2)
    x = weights.synthetic_input(2, seed=77)
    eng = capi.Engine(blob)
    s = capi.Session(eng)
    try:
        prob = s.infer(x)["prob"].reshape(2, -1)
        names = _names(s, 2)
    finally:
        s.close()
        eng.destroy()
    ref, emu = _oracles(tmp_path, 19, 2)
    _check_net(prob, ref, emu, names, "VGG-19")
