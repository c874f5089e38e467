"""GPU: the fused 3x3 + 1x1 bottleneck launch (conv3x3_halo_1x1_tcgen05) at geometries and epilogues ResNet never
produces, judged against a float64 reference.

The fusion rule (engine.cu fuse_partner, and tactic_applies with halo == 2) admits any 3x3 with 64, 128 or 256 output
channels on 1-8 input channel blocks, followed by any 1x1 with a multiple of 64 output channels and a residual that is
not the 3x3's output, with or without ReLU on either convolution, on images up to 126 pixels wide, wherever the kernel's
shared memory fits in 227 KiB.  Every case is one block

    data -> [1x1 "a" -> cin3] -> 3x3 "b" (c3, ReLU optional) -> 1x1 "c" (cout2) + residual -> ReLU optional

with the residual one of: the block input (identity), a 1x1 projection "short" of it, or "a" (the 3x3's own input).
For every case the launch names must agree with the restated rule's prediction of whether the pair fuses; the fused
output must equal the unfused pair bit for bit; each operator of the unfused run is held within TOL of
oracle.caffe_forward.lowered_forward_f16emu on its own (tapped) input; and the whole block is held within TOL of the
emulation from the fp32 input.  Since the fused output equals the unfused one, that holds the fused launch to the
reference operator by operator.  Geometries the rule refuses are asserted refused from the launch names, never forced.
tests/test_fused_geometry_cpu.py builds every case and checks the references without a GPU."""
from typing import NamedTuple, Optional

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.caffe_forward import lowered_forward_f16emu
from tensorrt_laboratory_b200 import builder, capi, graph, weights
from tests import helpers
from tests import test_gpu_geometry as G
from tests.test_gpu_fused_bottleneck import _fused_names
from tests.test_gpu_tactic_table import BATCH, _op_index

pytestmark = pytest.mark.gpu

TOL = G.TOL   # 2 ulp of fp16 at the top binade, relative to max|ref| (tests/test_gpu_conv.py)
FP16 = builder.PREC_FP16


# ------------------------------------------------------------------------------------------------------------------
# the fusion rule, restated
# ------------------------------------------------------------------------------------------------------------------
SMEM_LIMIT = 227 * 1024   # engine.cu kSmemLimit: the dynamic shared memory one CTA may opt in to on sm_90
HALO_MAX_CBLOCKS = 8      # kernels.cu kHaloMaxCBlocks
FUSE_TILE = 128 * 64 * 2  # kernels.cu kFuseTile: one 128-row x 64-channel fp16 residual / output staging buffer


def halo_a_stage_bytes(w, r):
    """kernels.cu halo_a_stage_bytes: one channel block's halo, (R+2)(W+2) pixel rows of 128 B, but never less than the
    farthest tap's 128-row window touches, rounded up to 1 KiB."""
    rows = max((r + 2) * (w + 2), 128 + 2 * (w + 2) + 2)
    return (rows * 128 + 1023) // 1024 * 1024


def halo_fused_smem_bytes(bn, w, r, cblocks, cout2):
    """kernels.cu halo_fused_smem_bytes: halo blocks (the 3x3's output tile reuses them, so at least BN x 256 B), two
    residual / output buffers, the weight ring (halo_b_stages: 3 stages of BN x 128 B at BN = 256, else 4), barriers,
    both bias vectors and the 1 KiB alignment slack."""
    stages = 3 if bn >= 256 else 4
    return max(cblocks * halo_a_stage_bytes(w, r), bn * 256) + 2 * FUSE_TILE + stages * bn * 128 + 256 + (bn + cout2) * 4 + 1024


def halo_rows(h, w):
    """engine.cu conv_halo_rows for a 3x3 / stride 1 / pad 1 on 64-channel blocks: R whole rows per 128-row tile, 0 where
    a padded row does not fit."""
    return min(128 // (w + 2), h) if w + 2 <= 128 else 0


def phys(c):
    return builder.phys_channels(c, FP16)


class Case(NamedTuple):
    cin3: int                # input channels of the 3x3 (output of "a", or the block input without "a")
    c3: int                  # output channels of the 3x3 = K of the 1x1
    cout2: int               # output channels of the 1x1
    h: int
    w: int
    batch: int = 2
    relu3: bool = True       # ReLU after the 3x3
    relu2: bool = True       # ReLU after the residual sum
    res: str = "identity"    # identity (the block input), projection ("short", a 1x1 of the block input), input ("a")
    a: bool = True           # a 1x1 "a" in front of the 3x3
    max_batch: Optional[int] = None
    seed: int = 0

    @property
    def cblocks(self):
        return phys(self.cin3) // 64

    @property
    def chunks(self):
        return phys(self.cout2) // 64

    @property
    def data_channels(self):
        if self.res == "identity":
            return self.cout2 if self.a else self.cin3
        return 64 if self.a else self.cin3

    @property
    def smem(self):
        return halo_fused_smem_bytes(phys(self.c3), self.w, halo_rows(self.h, self.w), self.cblocks, phys(self.cout2))

    @property
    def fused(self):
        """Whether the rule admits the pair: a halo instantiation for the 3x3's channels, at most eight input channel
        blocks, a padded row of at most 128 pixels, a 1x1 of whole 64-channel chunks, and shared memory within the limit."""
        return (phys(self.c3) in (64, 128, 256) and self.cblocks <= HALO_MAX_CBLOCKS and halo_rows(self.h, self.w) > 0 and
                phys(self.cout2) % 64 == 0 and self.smem <= SMEM_LIMIT)


def case_id(c):
    s = f"ci{c.cin3}-c{c.c3}-co{c.cout2}-{c.h}x{c.w}-n{c.batch}"
    if c.max_batch:
        s += f"of{c.max_batch}"
    s += f"-{c.res}" + ("" if c.a else "-noa")
    s += ("" if c.relu3 else "-lin3") + ("" if c.relu2 else "-lin2")
    return s + ("" if c.fused else "-refused")


def block_layers(case, bottom, sfx=""):
    """The layers of one block reading `bottom` -> (layers, top).  The projection shortcut comes first, as in ResNet,
    so that the 1x1 "c" is the op right after the 3x3 "b"."""
    def conv(name, src, cout, k):
        return dict(name=name + sfx, type="Convolution", bottoms=[src], tops=[name + sfx], num_output=cout, kernel_size=k,
                    pad=k // 2, stride=1, bias_term=True)

    def relu(name):
        return dict(name=name + sfx + "_relu", type="ReLU", bottoms=[name + sfx], tops=[name + sfx])

    L = []
    if case.res == "projection":
        L.append(conv("short", bottom, case.cout2, 1))
    x3 = bottom
    if case.a:
        L += [conv("a", bottom, case.cin3, 1), relu("a")]
        x3 = "a" + sfx
    L.append(conv("b", x3, case.c3, 3))
    if case.relu3:
        L.append(relu("b"))
    L.append(conv("c", "b" + sfx, case.cout2, 1))
    residual = {"identity": bottom, "projection": "short" + sfx, "input": x3}[case.res]
    L.append(dict(name="sum" + sfx, type="Eltwise", bottoms=[residual, "c" + sfx], tops=["sum" + sfx], operation="SUM"))
    if case.relu2:
        L.append(relu("sum"))
    return L, "sum" + sfx


def block_net(case):
    if case.res == "input":
        assert case.a and case.cin3 == case.cout2, "the residual is the 3x3's input: cin3 == cout2"
    if case.res == "identity" and not case.a:
        assert case.cin3 == case.cout2
    L, _ = block_layers(case, "data")
    return {"name": "fused_" + case_id(case), "input": "data", "input_dims": [1, case.data_channels, case.h, case.w], "layers": L}


def lowered(net, seed):
    return graph.lower(net, weights.random_weights(net, seed))


def block_input(case):
    return np.random.default_rng(case.seed + 1).standard_normal((case.batch, case.data_channels, case.h, case.w), dtype=np.float32)


def taps(case, sfx=""):
    """The tensors the per-operator checks read back: the 3x3's input and output, the residual and the block output."""
    t = ["b" + sfx, "sum" + sfx]
    if case.a:
        t.insert(0, "a" + sfx)
    if case.res == "projection":
        t.insert(0, "short" + sfx)
    return t


# ------------------------------------------------------------------------------------------------------------------
# own-input references (tests/test_fused_geometry_cpu.py ties them to the emulation and to torch)
# ------------------------------------------------------------------------------------------------------------------
def f16(a):
    return np.asarray(a, np.float32).astype(np.float16).astype(np.float64)


def ref_op(low, name, x):
    """The emulation of the single op `name` of `low` on its input `x` (an op without a residual) -> [N, C*H*W]."""
    op = next(o for o in low["ops"] if o["name"] == name)
    assert op["residual"] is None
    return lowered_forward_f16emu(dict(low, input=op["input"], ops=[op], output=op["output"]), x)


def ref_1x1_residual(op, b, res):
    """A 1x1 op with its residual in the emulation's numerics: fp16 weights, exact sum, + bias + residual (ReLU) -> fp16,
    on the fp16 tensors `b` (its input) and `res` -> [N, C*H*W]."""
    w = torch.from_numpy(op["W"]).double().to(torch.float16).double().permute(0, 3, 1, 2)
    y = F.conv2d(torch.from_numpy(np.asarray(b, np.float64)), w)
    y = y + torch.from_numpy(op["bias"]).double().view(1, -1, 1, 1) + torch.from_numpy(np.asarray(res, np.float64))
    if op["relu"]:
        y = torch.relu(y)
    return y.to(torch.float16).double().reshape(y.shape[0], -1).numpy()


def check_block_ops(low, x, case, out, sfx=""):
    """Every operator of one block against its reference, on the engine's own tapped inputs."""
    n = x.shape[0]
    x3 = out["a" + sfx] if case.a else f16(x)
    err = helpers.rel_err(out["b" + sfx].reshape(n, -1), ref_op(low, "b" + sfx, x3))
    assert err <= TOL, f"3x3 b{sfx}: rel err {err:.3e}"
    res = {"identity": f16(x), "projection": out.get("short" + sfx), "input": x3}[case.res]
    op_c = next(o for o in low["ops"] if o["name"] == "c" + sfx)
    err = helpers.rel_err(out["sum" + sfx].reshape(n, -1), ref_1x1_residual(op_c, out["b" + sfx], res))
    assert err <= TOL, f"1x1 c{sfx} + residual: rel err {err:.3e}"
    if case.res == "projection":
        err = helpers.rel_err(out["short" + sfx].reshape(n, -1), ref_op(low, "short" + sfx, f16(x)))
        assert err <= TOL, f"projection: rel err {err:.3e}"


# ------------------------------------------------------------------------------------------------------------------
# cases (every one builds in tests/test_fused_geometry_cpu.py, which also checks their coverage)
# ------------------------------------------------------------------------------------------------------------------
# channel blocks of the 3x3's input against its N tile: cblocks 1, 3 and 8 below, at and above BN / 64.  10 x 12 has
# R = 9, so its second tile is a single row.
CHANNEL_CASES = [Case(cin3, c3, 4 * c3, 10, 12, seed=cin3 + c3) for cin3 in (64, 192, 512) for c3 in (64, 128, 256)]

# the 1x1's width: one chunk, odd chunk counts (3, 5), 4 * c3 and 32 chunks, through all three residual kinds
WIDTH_CASES = [
    Case(64, 64, 64, 14, 14, res="projection", seed=1),
    Case(192, 64, 192, 14, 14, res="input", seed=2),
    Case(64, 64, 320, 14, 14, seed=3),
    Case(64, 128, 320, 14, 14, res="projection", seed=4),
    Case(128, 128, 512, 14, 14, seed=5),
    Case(64, 64, 2048, 14, 14, seed=6),
]

# padded channel counts: c3 100 -> 128, cout2 200 -> 256, cin3 96 -> 128; zero channels flow through both phases
PADDED_CASES = [
    Case(96, 100, 200, 14, 14, seed=7),
    Case(96, 100, 200, 14, 14, relu3=False, relu2=False, res="projection", seed=8),
    Case(200, 100, 200, 9, 9, res="input", seed=9),
]

# image widths and heights.  R (W+2) = 128 exactly at W = 14, 30, 62 and 126; R = 1 at 63 and 126; W = 1 has R = 42
GEOMETRY_CASES = [
    Case(64, 64, 256, 50, 1, seed=10),           # R = 42: the second tile holds 8 rows
    Case(64, 64, 256, 16, 14, seed=11),          # R = 8: the last tile is full
    Case(64, 64, 256, 15, 14, seed=12),          # ... one row short
    Case(64, 64, 256, 9, 14, seed=13),           # ... a single row
    Case(64, 64, 256, 3, 14, seed=14),           # H < 128 // 16: R = H = 3
    Case(64, 128, 256, 40, 14, seed=15),         # tall
    Case(64, 64, 256, 8, 30, seed=16),           # wide, R = 4
    Case(64, 64, 128, 5, 62, seed=17),           # R = 2: the last tile is a single row
    Case(64, 64, 256, 4, 63, seed=18),           # R = 1: 65 of 128 rows used
    Case(128, 64, 192, 3, 126, batch=1, seed=19),   # R = 1: all 128 rows used
]

# ReLU on either convolution, independently, and the three residual kinds
EPILOGUE_CASES = [
    Case(64, 64, 256, 14, 14, relu3=False, seed=20),
    Case(64, 64, 256, 14, 14, relu2=False, seed=21),
    Case(64, 64, 256, 14, 14, relu3=False, relu2=False, seed=22),
    Case(64, 128, 256, 12, 12, relu2=False, res="projection", seed=23),
    Case(64, 128, 256, 12, 12, relu3=False, relu2=False, res="projection", seed=24),
    Case(192, 128, 192, 12, 12, relu2=False, res="input", seed=25),
    Case(256, 64, 256, 12, 12, relu3=False, a=False, seed=26),   # no "a": the identity residual is the 3x3's input too
]

# batches, and a partial batch through a max-batch-8 plan
BATCH_CASES = [
    Case(64, 64, 256, 14, 14, batch=1, seed=27),
    Case(64, 64, 256, 14, 14, batch=5, relu2=False, seed=28),
    Case(128, 128, 320, 9, 9, batch=5, res="projection", seed=29),
    Case(64, 64, 256, 14, 14, batch=3, max_batch=8, seed=30),
]

# the shared-memory boundary: 232448 B = 227 KiB exactly fuses, 256 B more is refused; 8 channel blocks at 14 x 14 never
# fit, at 16 x 6 (R = 16) up to 2432 channels do; W = 127 has no halo tile at all
BOUNDARY_CASES = [
    Case(256, 256, 3264, 14, 14, batch=1, seed=31),
    Case(256, 256, 3328, 14, 14, batch=1, seed=32),
    Case(512, 64, 256, 14, 14, batch=1, seed=33),
    Case(512, 64, 2432, 16, 6, batch=1, seed=34),
    Case(512, 64, 2496, 16, 6, batch=1, seed=35),
    Case(64, 64, 256, 2, 127, batch=1, seed=36),
]

CASES = CHANNEL_CASES + WIDTH_CASES + PADDED_CASES + GEOMETRY_CASES + EPILOGUE_CASES + BATCH_CASES + BOUNDARY_CASES

# two blocks back to back: the first block's 1x1 output is the second 3x3's input (4 channel blocks under a 64-wide
# N tile) and its residual
CHAIN = (Case(64, 64, 256, 14, 14, batch=2, seed=40), Case(256, 64, 256, 14, 14, batch=2, res="input", a=False, seed=40))

# halo widths of the plain conv3x3_halo_tcgen05 (tests/test_gpu_geometry.py covers W = 60)
HALO_CASES = [(64, 50, 1, 64, 3, 1, 1, False, 3), (64, 5, 62, 64, 3, 1, 1, False, 3), (64, 4, 63, 64, 3, 1, 1, False, 3),
              (64, 3, 126, 64, 3, 1, 1, False, 3)]

# a block outside ResNet for the tactic tables: 3 channel blocks, 5 chunks, a projection shortcut
TABLE_CASE = Case(192, 64, 320, 14, 14, batch=BATCH, res="projection", seed=41)


def chain_net():
    L1, top1 = block_layers(CHAIN[0], "data", "1")
    L2, top2 = block_layers(CHAIN[1], top1, "2")
    return {"name": "fused_chain", "input": "data", "input_dims": [1, CHAIN[0].data_channels, CHAIN[0].h, CHAIN[0].w],
            "layers": L1 + L2}


# ------------------------------------------------------------------------------------------------------------------
# launch names
# ------------------------------------------------------------------------------------------------------------------
def _has(names, op):
    return any(n.startswith(f"conv_tcgen05:{op} ") for n in names)


def assert_fused(names, pairs):
    """Exactly one fused launch per (3x3, 1x1, N tile) in `pairs`, and nothing else fused."""
    fused = [n for n in names if " fused" in n]
    assert len(fused) == len(pairs), names
    for b, c, bn in pairs:
        assert sum(f"{b}+{c}" in n and f" bn={bn} " in n for n in fused) == 1, (b, c, bn, fused)


def assert_unfused(names, ops):
    assert not [n for n in names if " fused" in n], names
    for op in ops:
        assert _has(names, op), (op, names)


# ------------------------------------------------------------------------------------------------------------------
# a. one block
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_fused_block(gpu, case):
    low = lowered(block_net(case), case.seed)
    x = block_input(case)
    n = x.shape[0]
    got = helpers.run_engine(low, x, FP16, {"fuse": 1}, max_batch=case.max_batch)["sum"]
    names = list(helpers.LAST_LAUNCH_NAMES)
    if case.fused:
        assert_fused(names, [("b", "c", phys(case.c3))])
    else:
        assert_unfused(names, ["b", "c"])
        if halo_rows(case.h, case.w) == 0:
            assert not any(" halo" in nm for nm in names), names
    # the unfused pair, every operator read back through a tap (a tapped 3x3 output never fuses)
    out = helpers.run_engine(low, x, FP16, {"fuse": -1}, outputs=taps(case), max_batch=case.max_batch)
    assert_unfused(helpers.LAST_LAUNCH_NAMES, ["b", "c"])
    assert got.tobytes() == out["sum"].tobytes()
    check_block_ops(low, x, case, out)
    err = helpers.rel_err(got.reshape(n, -1), lowered_forward_f16emu(low, x))
    assert err <= TOL, f"block: rel err {err:.3e}"
    if not case.relu2:
        assert (got < 0).any()
    if not case.relu3:
        assert (out["b"] < 0).any()


# ------------------------------------------------------------------------------------------------------------------
# b. two blocks back to back
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def chain():
    net = chain_net()
    low = lowered(net, 42)
    return low, block_input(CHAIN[0])


@pytest.mark.parametrize("tap_first", [False, True], ids=["one_output", "first_block_tapped"])
def test_two_fused_blocks_back_to_back(gpu, chain, tap_first):
    """Block 2's 3x3 reads block 1's 1x1 output, which is also block 2's residual (and, tapped, a network output)."""
    low, x = chain
    outputs = ["sum1", "sum2"] if tap_first else ["sum2"]
    got = helpers.run_engine(low, x, FP16, {"fuse": 1}, outputs=outputs)
    assert_fused(helpers.LAST_LAUNCH_NAMES, [("b1", "c1", 64), ("b2", "c2", 64)])
    out = helpers.run_engine(low, x, FP16, {"fuse": -1}, outputs=taps(CHAIN[0], "1") + taps(CHAIN[1], "2"))
    assert_unfused(helpers.LAST_LAUNCH_NAMES, ["b1", "c1", "b2", "c2"])
    for t in outputs:
        assert got[t].tobytes() == out[t].tobytes(), t
    check_block_ops(low, x, CHAIN[0], out, "1")
    check_block_ops(low, out["sum1"], CHAIN[1], out, "2")
    n = x.shape[0]
    ref, snaps = lowered_forward_f16emu(low, x, keep=["sum1"])
    assert helpers.rel_err(got["sum2"].reshape(n, -1), ref) <= TOL
    if tap_first:
        assert helpers.rel_err(got["sum1"].reshape(n, -1), snaps["sum1"].reshape(n, -1)) <= TOL


# ------------------------------------------------------------------------------------------------------------------
# c. tactic tables
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def table_block():
    low = lowered(block_net(TABLE_CASE), TABLE_CASE.seed)
    assert TABLE_CASE.fused
    return builder.build_plan(low, FP16, BATCH), block_input(TABLE_CASE)


def _tuned_tactics(blob, streams):
    eng = capi.Engine(blob)
    try:
        eng.tune(streams=streams)
        return eng.tactics()
    finally:
        eng.destroy()


def test_tuned_table_runs_what_the_tuner_chose(gpu, table_block):
    """Tuned for four streams, the fused tactic is timed against the pair; whichever won, the plan carrying the table
    runs it, with the bits of the untuned engine."""
    blob, x = table_block
    tac = _tuned_tactics(blob, 4)
    b = _op_index(blob, "b")
    rec = tac[(tac[:, 0] == b) & (tac[:, 1] == BATCH)]
    assert len(rec) == 1, tac
    want, _ = G._run_blob(blob, x, {"autotune": 0})
    got, names = G._run_blob(builder.attach_tactics(blob, tac), x)
    if rec[0, 8] == 2:
        assert_fused(names, [("b", "c", 64)])
    else:
        assert_unfused(names, ["b", "c"])
    assert got["sum"].tobytes() == want["sum"].tobytes()


def test_two_stream_tuning_never_records_the_fused_tactic(gpu, table_block):
    blob, _ = table_block
    tac = _tuned_tactics(blob, 2)
    assert len(tac) and not (tac[:, 8] == 2).any(), tac


@pytest.mark.parametrize("batch", [BATCH, 2])
def test_a_fused_table_entry_on_an_admissible_op_is_accepted(gpu, table_block, batch):
    """A hand-written max-batch record {bn = 64, halo = 2} for the 3x3: the engine runs the fused launch at the max batch
    and, through the max-batch record, at a smaller one -- with the untuned engine's bits."""
    blob, x = table_block
    x = x[:batch]
    rec = np.array([[_op_index(blob, "b"), BATCH, 64, 2, 1, 1, 0, 1, 2, 0]], np.uint32)
    want, want_names = G._run_blob(blob, x, {"autotune": 0})
    assert_unfused(want_names, ["b", "c"])
    got, names = G._run_blob(builder.attach_tactics(blob, rec), x)
    assert_fused(names, [("b", "c", 64)])
    assert got["sum"].tobytes() == want["sum"].tobytes()


# ------------------------------------------------------------------------------------------------------------------
# d. the plain halo kernel at the new widths
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("relu", [True, False], ids=["relu", "linear"])
@pytest.mark.parametrize("case", HALO_CASES, ids=G._case_id)
def test_plain_halo_kernel_at_new_widths(gpu, case, relu):
    a, names_a, err_a = G._conv(case, relu, {"bn": 64, "halo": 1})
    assert " halo" in G._launch(names_a, "conv_tcgen05", "conv"), names_a
    b, names_b, err_b = G._conv(case, relu, {"bn": 64, "halo": -1})
    assert " halo" not in G._launch(names_b, "conv_tcgen05", "conv"), names_b
    assert max(err_a, err_b) <= TOL, (err_a, err_b)
    np.testing.assert_array_equal(a, b)
    if not relu:
        assert (a < 0).any()
