"""GPU: a tactic table carried by the plan is input from outside the engine.  A record the tactic rule refuses for its
layer is ignored -- the layer runs the cost model's tactic, exactly as an untuned (autotune=0) session runs it."""
import numpy as np
import pytest

from tensorrt_laboratory_b200 import bert, builder, capi, graph, weights
from tests.test_gpu_bert import SMALL, _inputs

pytestmark = pytest.mark.gpu

BATCH = 4


def _op_index(blob, name):
    _, version, _, _, n_tensors, n_ops, *_ = builder._HEADER.unpack_from(blob, 0)
    size = {builder.VERSION: builder._OP, builder.VERSION_GROUPED: builder._OP_V2, builder.VERSION_TRANSFORMER: builder._OP_V3}[version].size
    base = builder._HEADER.size + n_tensors * builder._TENSOR.size
    return [blob[base + i * size:base + i * size + 64].split(b"\0")[0].decode() for i in range(n_ops)].index(name)


def _run(blob, inputs, options):
    eng = capi.Engine(blob)
    s = capi.Session(eng, options)
    try:
        out = s.infer_bindings(inputs) if isinstance(inputs, dict) else s.infer(inputs)
        names = [s._lib.b2_context_launch_name(s.ctx, BATCH, i).decode() for i in range(s.nb_launches(BATCH))]
    finally:
        s.close()
        eng.destroy()
    return out, names


def _check_refused(blob, inputs, op_name, bn, stages, splits=1, sps=1, ws=0, cn=1, halo=0):
    rec = np.array([[_op_index(blob, op_name), BATCH, bn, stages, splits, sps, ws, cn, halo, 0]], np.uint32)
    want, want_names = _run(blob, inputs, {"autotune": 0})
    got, names = _run(builder.attach_tactics(blob, rec), inputs, None)
    assert names == want_names, [n for n in names if f":{op_name} " in n]
    for k in want:
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)


def _conv(cin, h, cout, k, groups=1):
    net = builder.single_conv_net(cin, h, h, cout, k, 1, k // 2, group=groups)
    blob = builder.build_plan(graph.lower(net, weights.random_weights(net, 0)), builder.PREC_FP16, BATCH)
    return blob, np.random.default_rng(1).standard_normal((BATCH, cin, h, h), dtype=np.float32)


@pytest.mark.parametrize("tactic", [dict(bn=64, stages=2, ws=64), dict(bn=64, stages=2, cn=2)])
def test_gelu_layer_refuses_persistent_and_cluster_records(gpu, tactic):
    cfg = bert.BertConfig(**{**SMALL.__dict__, "layers": 1})
    blob = builder.build_bert_plan(cfg, bert.random_weights(cfg, 7), max_batch=BATCH)
    _check_refused(blob, _inputs(cfg, BATCH), "l0.ffn1", **tactic)


def test_halo_record_on_a_1x1_is_refused(gpu):
    _check_refused(*_conv(256, 14, 256, 1), "conv", bn=64, stages=2, halo=1)


@pytest.mark.parametrize("tactic", [dict(bn=64, stages=2, splits=2), dict(bn=64, stages=2, cn=2), dict(bn=64, stages=2, halo=1)])
def test_grouped_conv_refuses_split_cluster_and_halo_records(gpu, tactic):
    _check_refused(*_conv(256, 14, 256, 3, groups=32), "conv", **tactic)


def test_n_tile_not_dividing_cout_is_refused(gpu):
    _check_refused(*_conv(64, 14, 192, 3), "conv", bn=128, stages=2)  # 192 channels: no padding up to a multiple of 128


@pytest.mark.parametrize("tactic", [dict(bn=256, stages=8), dict(bn=64, stages=3), dict(bn=64, stages=2, splits=0)])
def test_uninstantiated_or_malformed_record_is_refused(gpu, tactic):
    _check_refused(*_conv(64, 14, 256, 3), "conv", **tactic)
