"""GPU: the persistent stem tactic (conv_stem_ws_tcgen05) against the one-tile-per-CTA kernel.

The row-folded 7x7 / stride-2 stem may run as a persistent kernel that keeps its weights in shared memory and reuses the
input-row sub-tiles of one output row for the next.  It issues the tile kernel's MMAs in the tile kernel's order, so its
output must be the tile kernel's bit for bit.  Launch names show which kernel ran: ` ws=N` on the stem's launch is the
persistent kernel with N CTAs."""
import functools

import numpy as np
import pytest

from tensorrt_laboratory_b200 import builder, capi, graph, weights
from tests import helpers
from tests.test_gpu_tactic_table import _op_index

pytestmark = pytest.mark.gpu

FP16 = builder.PREC_FP16

# (h, w, batch, forced CTA count: 1 = one per SM, capped at the output rows); bands are ceil(batch * Ho / CTAs) rows
STEM_CASES = [
    (224, 224, 1, 1),   # ResNet-50 conv1: 112 CTAs, one row each
    (224, 224, 3, 1),   # 132 CTAs, bands of 3 rows
    (224, 224, 8, 1),   # 132 CTAs, bands of 7 rows (the benchmark's shape)
    (224, 224, 8, 66),  # half the SMs: bands of 14 rows
    (224, 224, 1, 10),  # bands of 12 rows: 112 = 9 * 12 + 4, a short last band
    (222, 224, 2, 1),   # Ho = 111: an odd number of rows, bands of 2 with a 1-row band at the end of every image
    (60, 90, 2, 7),     # Wo = 45: 4 bands of 9, 9, 9, 3 rows per image on 7 CTAs, so one CTA runs two bands
    (28, 28, 3, 5),     # Wo = 14: bands of 9 and 5 rows, 6 bands on 5 CTAs
]


def _case_id(case):
    h, w, batch, ws = case
    return f"{h}x{w}-b{batch}-ws{ws}"


def _launch(names, op):
    return next(n for n in names if n.split(" ")[0] == f"conv_tcgen05:{op}")


@functools.lru_cache(maxsize=None)
def _stem(h, w, batch, relu=True, cout=64):
    net = builder.single_conv_net(3, h, w, cout, 7, 2, 3, relu=relu)
    low = graph.lower(net, weights.random_weights(net, 0))
    x = np.random.default_rng(1).standard_normal((batch, 3, h, w), dtype=np.float32)
    return low, x


def _run(low, x, options):
    out = helpers.run_engine(low, x, FP16, options)
    return list(out.values())[0], _launch(helpers.LAST_LAUNCH_NAMES, "conv")


@pytest.mark.parametrize("case", STEM_CASES, ids=_case_id)
def test_stem_tactic_is_bit_identical_to_the_tile_kernel(gpu, case):
    h, w, batch, ws = case
    low, x = _stem(h, w, batch)
    got, name = _run(low, x, {"ws": ws})
    want, want_name = _run(low, x, {"ws": -1})
    rows = batch * ((h - 1) // 2 + 1)
    assert f" ws={min(rows, 132 if ws == 1 else ws)} " in name and " kb=32 " in name and " st=16x1 " in name, name
    assert " ws=" not in want_name and " kb=32 " in want_name, want_name
    assert (want > 0).any() and (want == 0).any()
    np.testing.assert_array_equal(got, want)


def test_stem_tactic_is_batch_position_invariant(gpu):
    low, x = _stem(224, 224, 3)
    blob = builder.build_plan(low, FP16, 3)
    eng = capi.Engine(blob)
    sess = capi.Session(eng, {"ws": 1})
    try:
        names = [capi.load().b2_context_launch_name(sess.ctx, 3, i).decode() for i in range(sess.nb_launches(3))]
        assert " ws=132 " in _launch(names, "conv"), names
        out = sess.infer(x)
        key = list(out)[0]
        full = out[key]
        perm = np.array([2, 0, 1])
        np.testing.assert_array_equal(sess.infer(x[perm])[key], full[perm])
        for b in (1, 2):
            np.testing.assert_array_equal(sess.infer(x[:b])[key], full[:b])
    finally:
        sess.close()
        eng.destroy()


@pytest.mark.parametrize("geometry", ["wide", "linear", "no_fold", "cout128"])
def test_stem_tactic_is_refused_outside_its_geometry(gpu, geometry):
    """Wo = 132 (> 128), no ReLU, the generic 8-channel tap path and 128 output channels keep the tile kernel under ws=1."""
    h, w, relu, cout, opts = 100, 224, True, 64, {}
    if geometry == "wide":
        w = 264
    elif geometry == "linear":
        relu = False
    elif geometry == "no_fold":
        opts = {"no_fold": 1}
    else:
        cout = 128
    low, x = _stem(h, w, 2, relu, cout)
    got, name = _run(low, x, {"ws": 1, **opts})
    want, _ = _run(low, x, {"ws": -1, **opts})
    assert " ws=" not in name and f" kb={8 if geometry == 'no_fold' else 32} " in name, name
    np.testing.assert_array_equal(got, want)


def test_resnet50_with_the_stem_tactic_equals_the_untuned_session(gpu):
    """A plan whose tactic table puts conv1 on the persistent stem gives the untuned session's conv1 and prob bits."""
    batch = 8
    net = graph.resnet_caffe(50)
    low = graph.lower(net, weights.random_weights(net, 0))
    x = weights.synthetic_input(batch, seed=5)
    blob = builder.build_plan(low, FP16, batch, outputs=["conv1", "prob"])
    rec = np.array([[_op_index(blob, "conv1"), batch, 64, 16, 1, 1, 132, 1, 0, 0]], np.uint32)
    runs = []
    for b, opts in ((builder.attach_tactics(blob, rec), None), (blob, {"autotune": 0})):
        eng = capi.Engine(b)
        sess = capi.Session(eng, opts)
        try:
            out = sess.infer(x)
            names = [capi.load().b2_context_launch_name(sess.ctx, batch, i).decode() for i in range(sess.nb_launches(batch))]
        finally:
            sess.close()
            eng.destroy()
        runs.append((out, names))
    (got, names), (want, want_names) = runs
    assert " ws=132 " in _launch(names, "conv1") and " ws=" not in _launch(want_names, "conv1")
    assert len(names) == len(want_names) and [n for n in names if ":conv1 " not in n] == [n for n in want_names if ":conv1 " not in n]
    for k in ("conv1", "prob"):
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)
