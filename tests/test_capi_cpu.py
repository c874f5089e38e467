"""CPU: the C-ABI library loads, exports every symbol the headers declare, and validates plans.
No compute entry point is exercised here (there is no CPU fallback to exercise)."""
import ctypes as C
import os
import re
import struct
import subprocess
import sys

import numpy as np
import pytest

from tensorrt_laboratory_b200 import builder, capi, graph, weights
from tests import helpers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    names = set()
    for hdr in ("b200infer.h", "b200cuda.h", "trtlab_host.h"):
        with open(os.path.join(ROOT, "include", hdr)) as f:
            text = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
        names |= set(re.findall(r"\b((?:b2|trt)_[a-z0-9_]+)\s*\(", text))
    return names


def test_library_exports_every_declared_symbol(lib):
    declared = _declared_symbols()
    assert len(declared) > 55
    missing = [n for n in sorted(declared) if not hasattr(lib, n)]
    assert not missing, missing
    bound = {n for n, _, _ in capi.SYMBOLS}
    assert declared == bound, (declared - bound, bound - declared)
    assert lib.b2_abi_version() == 1


def _small_plan(precision):
    _, _, low = helpers.conv_case(3, 16, 16, 64, 3, 1, 1)
    return builder.build_plan(low, precision, max_batch=4)


def test_plan_roundtrip_metadata(lib):
    blob = builder.build_resnet_plan(50, builder.PREC_FP16, 8)
    eng = capi.Engine(blob, inspect_only=True)
    assert eng.name == "ResNet-50" and eng.max_batch == 8 and eng.precision == builder.PREC_FP16
    assert [(b["name"], b["is_input"], b["shape"]) for b in eng.bindings] == [("data", True, (3, 224, 224)), ("prob", False, (1000,))]
    assert eng.bindings[0]["item_bytes"] * 8 == 4816896 and eng.bindings[1]["item_bytes"] * 8 == 32000  # SURVEY 8(a)
    assert abs(eng.flops(8) - 61.73e9) < 1e7
    assert 50e6 < eng.weights_size < 52e6  # ~51.0 MB of fp16 weights
    assert 20e6 < eng.device_memory_size < 60e6
    assert lib.b2_engine_nb_layers(eng.handle) == 58  # input cast + 57 fused ops
    assert lib.b2_engine_binding_index(eng.handle, b"prob") == 1 and lib.b2_engine_binding_index(eng.handle, b"nope") == -1
    eng.destroy()


def test_fp32_plan_is_twice_the_size(lib):
    a = capi.Engine(_small_plan(builder.PREC_FP16), inspect_only=True)
    b = capi.Engine(_small_plan(builder.PREC_FP32), inspect_only=True)
    assert a.bindings == b.bindings
    assert b.precision == builder.PREC_FP32
    a.destroy(), b.destroy()


def test_malformed_plans_are_rejected(lib):
    blob = bytearray(_small_plan(builder.PREC_FP16))
    for mutate in (lambda b: b.__setitem__(slice(0, 8), b"NOTAPLAN"),
                   lambda b: b.__setitem__(slice(8, 12), struct.pack("<I", 99)),
                   lambda b: b.__delitem__(slice(len(b) - 100, len(b))),
                   lambda b: b.__setitem__(slice(16, 20), struct.pack("<I", 0))):
        bad = bytearray(blob)
        mutate(bad)
        with pytest.raises(capi.B2Error) as ei:
            capi.Engine(bytes(bad), inspect_only=True)
        assert ei.value.code == 1
    with pytest.raises(capi.B2Error):
        capi.Engine(b"short", inspect_only=True)


def test_corrupted_offsets_and_geometry_are_rejected_not_wrapped(lib):
    """Bounds checks must not wrap in uint64, and geometry that would divide by zero or underflow is refused (B2_EINVAL)
    instead of reaching a kernel."""
    blob = bytes(_small_plan(builder.PREC_FP16))
    hdr = builder._HEADER
    n_t, n_o = struct.unpack_from("<II", blob, 20)[0], struct.unpack_from("<II", blob, 24)[0]
    n_t, n_o = struct.unpack_from("<III", blob, 20)[0:2]
    op0 = hdr.size + n_t * builder._TENSOR.size
    conv = next(op0 + i * builder._OP.size for i in range(n_o) if struct.unpack_from("<I", blob, op0 + i * builder._OP.size + 64)[0] == builder.OP_CONV)

    def mutated(offset, fmt, *vals):
        bad = bytearray(blob)
        struct.pack_into(fmt, bad, offset, *vals)
        return bytes(bad)

    cases = {
        "payload offset+bytes wraps": mutated(32, "<QQ", 2 ** 64 - 16, 64),
        "weight offset+bytes wraps": mutated(conv + 64 + 4 + 16 + 4 * 11, "<QQ", 2 ** 64 - 8, 64),
        "conv stride 0": mutated(conv + 64 + 4 + 16 + 4, "<I", 0),
        "conv window larger than the padded input": mutated(conv + 64 + 4 + 16, "<I", 1000),
        "tactic table outside the blob": mutated(112, "<IIQ", 5, 0, 2 ** 63),
    }
    for name, bad in cases.items():
        with pytest.raises(capi.B2Error) as ei:
            capi.Engine(bad, inspect_only=True)
        assert ei.value.code == 1, name


def test_inspect_only_engine_cannot_execute(lib):
    eng = capi.Engine(_small_plan(builder.PREC_FP16), inspect_only=True)
    ctx = C.c_void_p()
    assert lib.b2_context_create(eng.handle, C.byref(ctx)) == 5  # B2_ESTATE
    eng.destroy()


def test_no_device_means_loud_failure_not_fallback(lib):
    if capi.device_count() > 0:
        pytest.skip("a GPU is visible here")
    with pytest.raises(capi.B2Error) as ei:
        capi.Engine(_small_plan(builder.PREC_FP16))
    assert ei.value.code == 2 and "no CPU fallback" in str(ei.value)


def test_builder_layouts():
    net, wts, low = helpers.conv_case(3, 8, 8, 64, 7, 2, 3)
    # plain layout (stem re-expression off): channels padded to 8, taps padded to an even count
    blob = builder.build_plan(low, builder.PREC_FP16, 2, stem_s2d=False)
    hdr = struct.unpack_from("<8sIIIIIIQQ", blob, 0)
    assert hdr[0] == b"B2ENGINE" and hdr[2] == builder.PREC_FP16 and hdr[3] == 2
    n_t, n_o, n_b = hdr[4], hdr[5], hdr[6]
    assert (n_t, n_o, n_b) == (2, 3, 2)  # data, conv | cast, conv, cast | data, conv
    op_off = 128 + n_t * 96 + 176  # second op record = the conv
    fmt = "<64sIiiiiIIIIIIIIIIIQQQQIIII"
    rec = struct.unpack_from(fmt, blob, op_off)
    assert rec[1] == builder.OP_CONV
    k, cin, cout, cin_p, cout_p, taps, taps_p = rec[6], rec[11], rec[12], rec[13], rec[14], rec[15], rec[16]
    assert (k, cin, cout, cin_p, cout_p, taps, taps_p) == (7, 3, 64, 8, 64, 49, 50)
    w_off, w_bytes = rec[17], rec[18]
    assert w_bytes == 64 * 50 * 8 * 2 and rec[21:25] == (0, 0, 0, 0)
    payload = hdr[7]
    W = np.frombuffer(blob, np.float16, 64 * 50 * 8, payload + w_off).reshape(64, 50, 8)
    assert np.all(W[:, 49, :] == 0) and np.all(W[:, :, 3:] == 0)
    np.testing.assert_array_equal(W[:, :49, :3], low["ops"][0]["W"].reshape(64, 49, 3).astype(np.float16))
    # default fp16 layout: the stride-2 stem runs on a horizontally space-to-depth packed input (7x4 taps x 8 ch)
    blob = builder.build_plan(low, builder.PREC_FP16, 2)
    cast = struct.unpack_from(fmt, blob, 128 + n_t * 96)
    rec = struct.unpack_from(fmt, blob, op_off)
    assert cast[1] == builder.OP_INPUT_CAST and (cast[6], cast[7], cast[8]) == (2, 1, 2)  # s2d, right pad 1, left pad 2
    assert (rec[6], rec[7], rec[8], rec[11], rec[13], rec[15], rec[16]) == (7, 2, 3, 8, 8, 28, 28)
    assert rec[10] == 3 * 49  # algorithmic K of the original conv, for FLOP accounting
    assert rec[21:25] == (4, 1, 0, 0)  # kw, stride_w, pad_w_lo, pad_w_hi (padding is physical)
    t0 = struct.unpack_from("<64sIIIIIi", blob, 128)
    assert t0[2:6] == (8, 4 + 3, 8, 8)  # tensor `data`: h=8, w=2+8/2+1, c=8, c_phys=8
    assert builder.phys_channels(3, builder.PREC_FP16) == 8 and builder.phys_channels(1000, builder.PREC_FP16) == 1024
    assert builder.phys_channels(3, builder.PREC_FP32) == 3


def test_stem_space_to_depth_is_exact():
    """7x7/s2 conv on (N,3,H,W)  ==  7x4/s(2,1) conv on the pixel-pair packed input (N,8,H,W/2)."""
    import torch
    import torch.nn.functional as F
    rng = np.random.default_rng(0)
    for k, pad, w_in in ((7, 3, 16), (3, 1, 12), (5, 2, 10)):
        W = rng.standard_normal((5, k, k, 3)).astype(np.float32)
        x = rng.standard_normal((2, 3, 14, w_in)).astype(np.float32)
        ref = F.conv2d(torch.from_numpy(x), torch.from_numpy(W).permute(0, 3, 1, 2).contiguous(), stride=2, padding=pad).numpy()
        W2, kw2, plo, phi = builder.stem_s2d_transform(W, k, pad, w_in)
        X2 = np.zeros((2, 8, 14, w_in // 2), np.float32)
        for dw in range(2):
            X2[:, dw * 4:dw * 4 + 3] = x[:, :, :, dw::2]
        xp = F.pad(torch.from_numpy(X2), (plo, phi, pad, pad))
        got = F.conv2d(xp, torch.from_numpy(W2).permute(0, 3, 1, 2).contiguous(), stride=(2, 1)).numpy()
        assert got.shape == ref.shape
        np.testing.assert_allclose(got, ref, atol=1e-5)


def test_cpp_core_unit_tests(tmp_path):
    exe = tmp_path / "test_core"
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "test_core.cc"), "-o", str(exe), "-lpthread", "-ldl"], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and "ALL OK" in out.stdout, out.stderr


def test_cuda_sync_policies_against_a_fake_device(tmp_path):
    """cuda_sync<standard_threads | userspace_threads> (include/trtlab/cuda/sync.h; reference trtlab/cuda/sync.h:13-62):
    the polling flavour yields once per not-ready answer through the installable hook and throws on a device error."""
    exe = tmp_path / "test_sync"
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "test_sync.cc"), "-o", str(exe), "-lpthread"], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and "test_sync OK" in out.stdout, out.stderr


def test_fp16_input_binding_is_recorded_in_the_plan():
    """Secondary mode of SURVEY.md 8(d): the input binding of an fp16 engine may be declared fp16."""
    import struct
    net = builder.single_conv_net(64, 8, 8, 64, 1, 1, 0)
    from tensorrt_laboratory_b200 import graph, weights
    low = graph.lower(net, weights.random_weights(net, 0))
    blob32 = builder.build_plan(low, builder.PREC_FP16, 2)
    blob16 = builder.build_plan(low, builder.PREC_FP16, 2, input_dtype="f16")
    assert len(blob32) == len(blob16)
    diff = [i for i in range(len(blob32)) if blob32[i] != blob16[i]]
    assert len(diff) == 1  # exactly the dtype field of the input binding record
    assert blob32[diff[0]] == 0 and blob16[diff[0]] == 1
    with pytest.raises(ValueError):
        builder.build_plan(low, builder.PREC_FP32, 2, input_dtype="f16")
    with pytest.raises(ValueError):
        builder.build_plan(low, builder.PREC_FP16, 2, input_dtype="int8")


def test_prometheus_http_endpoint(lib):
    """GET /metrics on the manager's exposer returns the text exposition (reference metrics.cc:34-60: prometheus::Exposer);
    runs without a GPU: the endpoint only renders counters."""
    import urllib.error
    import urllib.request
    mgr = capi.InferenceManager(max_exec_concurrency=1, max_copy_concurrency=2)
    try:
        port = mgr.serve_metrics(0)
        assert 1024 <= port < 65536
        body = urllib.request.urlopen(f"http://127.0.0.1:{port}/metrics", timeout=5).read().decode()
        assert "# TYPE yais_inference_load_ratio histogram" in body and 'yais_inference_load_ratio_bucket{le="+Inf"} 0' in body
        assert body == mgr.metrics_text() or "yais_gpus_power_usage" in body
        with pytest.raises(urllib.error.HTTPError) as ei:
            urllib.request.urlopen(f"http://127.0.0.1:{port}/nope", timeout=5)
        assert ei.value.code == 404
    finally:
        mgr.close()


def test_per_layer_roofs_of_resnet50():
    """roofs.conv_floors: pure shape arithmetic -- 53 convolutions at batch 8, FLOPs add up to the network's conv FLOPs, the
    wide short-K layers with a residual are memory-bound and the 3x3 layers tensor-bound."""
    from tensorrt_laboratory_b200 import graph, roofs, weights
    net = graph.resnet_caffe(50)
    fl = roofs.conv_floors(graph.lower(net, weights.random_weights(net, 0)), 8, 1429.0, 17.5e12, 7.3e12)
    assert len(fl) == 53
    by = {f["name"]: f for f in fl}
    assert abs(sum(f["flops"] for f in fl) / 61.69e9 - 1) < 0.01
    assert by["res2b_branch2c"]["roof"] == "memory" and by["res4b_branch2b"]["roof"] == "tensor"
    assert abs(by["res2b_branch2c"]["read_bytes"] + by["res2b_branch2c"]["write_bytes"] - 28.9e6) < 0.2e6
    assert all(f["floor_us"] == max(f["tensor_floor_us"], f["memory_floor_us"]) for f in fl)
    assert 55 < sum(f["floor_us"] for f in fl) < 62


_PLAN_FUZZ = r"""
import random, sys
sys.path.insert(0, sys.argv[1])
from tensorrt_laboratory_b200 import builder, capi, graph, weights
net = builder.single_conv_net(64, 8, 8, 64, 3, 1, 1, residual=True)
blob = builder.build_plan(graph.lower(net, weights.random_weights(net, 0)), builder.PREC_FP16, 2)
rnd = random.Random(int(sys.argv[2]))
ok = err = 0
for t in range(int(sys.argv[3])):
    b = bytearray(blob)
    mode = t % 3
    if mode == 0:
        b = b[:rnd.randrange(1, len(b))]
    else:
        for _ in range(rnd.randrange(1, 4)):
            i = rnd.randrange(4096) if mode == 1 else rnd.randrange(len(b))   # mostly the header and the records
            b[i] = rnd.randrange(256)
    try:
        capi.Engine(bytes(b), inspect_only=True).destroy()
        ok += 1
    except capi.B2Error:
        err += 1
print("ok", ok, "rejected", err)
"""


def test_plan_parser_survives_random_corruption():
    """b2_engine_deserialize on 900 randomly truncated / byte-flipped plans (in a child process, so that a crash of the C
    parser is a test failure and not the end of the test run): every one is either accepted or rejected with a B2 error."""
    out = subprocess.run([sys.executable, "-c", _PLAN_FUZZ, ROOT, "7", "900"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, (out.returncode, out.stderr[-1500:])
    ok, rejected = int(out.stdout.split()[1]), int(out.stdout.split()[3])
    assert ok + rejected == 900 and rejected > 200
