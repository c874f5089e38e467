"""CPU side of tests/test_gpu_fused_geometry.py: the restated shared-memory formula against DESIGN.md's figures and the
227 KiB boundary, the coverage of its case list, its references against torch in float64, and every one of its blocks
built into a plan that the engine accepts, so a builder or plan refusal shows up here and not on a GPU."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.caffe_forward import lowered_forward_f16emu
from tensorrt_laboratory_b200 import builder, capi, graph
from tests import test_gpu_fused_geometry as FG

FP16 = builder.PREC_FP16
KIB = 1024


def _accepts(blob):
    eng = capi.Engine(blob, inspect_only=True)
    eng.destroy()


# ------------------------------------------------------------------------------------------------------------------
# the restated rule
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bn,hw,cblocks,cout2,kib", [(64, 56, 1, 256, 97.5), (128, 28, 2, 512, 147.75), (256, 14, 4, 1024, 218.25)])
def test_fused_smem_matches_the_resnet_figures(bn, hw, cblocks, cout2, kib):
    """DESIGN.md: 97.5, 147.75 and 218.25 KiB at res2, res3 and res4."""
    assert FG.halo_fused_smem_bytes(bn, hw, FG.halo_rows(hw, hw), cblocks, cout2) == kib * KIB


def test_fused_smem_boundary():
    limit = FG.SMEM_LIMIT
    assert limit == 232448
    # 256 channels on 4 blocks at 14 x 14: 3264 output channels fill 227 KiB exactly, one more chunk does not fit
    assert FG.halo_fused_smem_bytes(256, 14, 8, 4, 3264) == limit
    assert FG.halo_fused_smem_bytes(256, 14, 8, 4, 3328) > limit
    # 8 channel blocks under a 64-wide tile: never at 14 x 14, up to 2432 channels at 16 x 6 (R = 16)
    assert FG.halo_fused_smem_bytes(64, 14, 8, 8, 64) > limit
    assert FG.halo_rows(16, 6) == 16
    assert FG.halo_fused_smem_bytes(64, 6, 16, 8, 2432) == limit
    assert FG.halo_fused_smem_bytes(64, 6, 16, 8, 2496) > limit
    assert FG.halo_rows(2, 127) == 0


def test_halo_rows_at_the_case_widths():
    # R (W + 2) = 128 exactly at 14, 30, 62 and 126; R = 1 at 63 and 126; H < 128 // (W + 2) caps R at H
    for w, r in [(1, 42), (14, 8), (30, 4), (62, 2), (63, 1), (126, 1)]:
        assert FG.halo_rows(1000, w) == r
    assert [w for w in (1, 14, 30, 62, 63, 126) if FG.halo_rows(1000, w) * (w + 2) == 128] == [14, 30, 62, 126]
    assert FG.halo_rows(3, 14) == 3


def test_case_list_covers_the_rule():
    cases = FG.CASES
    fused = [c for c in cases if c.fused]
    assert {c.cblocks for c in fused} >= {1, 3, 8}
    assert any(c.cblocks < FG.phys(c.c3) // 64 for c in fused) and any(c.cblocks > FG.phys(c.c3) // 64 for c in fused)
    assert {c.chunks for c in fused} >= {1, 3, 5, 32}
    assert any(c.cout2 == 4 * c.c3 for c in fused)
    assert {c.w for c in fused} >= {1, 14, 30, 62, 63, 126}
    assert {c.res for c in fused} == {"identity", "projection", "input"}
    assert any(not c.relu3 for c in fused) and any(not c.relu2 for c in fused)
    assert any(not c.relu3 and not c.relu2 for c in fused)
    assert {c.batch for c in fused} >= {1, 2, 5} and any(c.max_batch and c.batch < c.max_batch for c in fused)
    assert any(c.c3 % 64 for c in fused) and any(c.cout2 % 64 for c in fused) and any(c.cin3 % 64 for c in fused)
    assert any(c.h > c.w for c in fused) and any(c.h < c.w for c in fused)
    # the last tile of an image full, one row short, a single row; and an image shorter than 128 // (W + 2)
    last_tile = {(c.h % FG.halo_rows(c.h, c.w), FG.halo_rows(c.h, c.w)) for c in fused if c.h > FG.halo_rows(c.h, c.w) > 2}
    assert {rows for rows, _ in last_tile} >= {0, 1} and any(rows == r - 1 for rows, r in last_tile)
    assert any(c.h < 128 // (c.w + 2) for c in fused)
    # both sides of the 227 KiB boundary, and 8 channel blocks refused by shared memory alone
    assert any(c.smem == FG.SMEM_LIMIT and c.fused for c in cases)
    assert any(c.smem == FG.SMEM_LIMIT + 256 and not c.fused for c in cases)
    assert any(c.cblocks == 8 and not c.fused and FG.halo_rows(c.h, c.w) for c in cases)
    assert any(FG.halo_rows(c.h, c.w) == 0 for c in cases)
    assert all(c.fused for c in FG.CHAIN) and FG.TABLE_CASE.fused


# ------------------------------------------------------------------------------------------------------------------
# every block builds, and the engine accepts the plan
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", FG.CASES, ids=FG.case_id)
def test_block_builds(case):
    net = FG.block_net(case)
    low = graph.lower(net, None)
    names = [op["name"] for op in low["ops"]]
    assert names[names.index("b") + 1] == "c"   # the fusion rule needs the 1x1 right after the 3x3
    c = low["ops"][names.index("c")]
    assert c["residual"] == {"identity": "data", "projection": "short", "input": "a"}[case.res]
    assert c["relu"] == case.relu2 and low["ops"][names.index("b")]["relu"] == case.relu3
    low = FG.lowered(net, case.seed)
    mb = case.max_batch or case.batch
    _accepts(builder.build_plan(low, FP16, mb))
    _accepts(builder.build_plan(low, FP16, mb, outputs=FG.taps(case)))


def test_chain_and_table_blocks_build():
    low = FG.lowered(FG.chain_net(), 42)
    names = [op["name"] for op in low["ops"]]
    assert names == ["a1", "b1", "c1", "b2", "c2"]
    assert low["ops"][4]["residual"] == "sum1" and low["ops"][3]["input"] == "sum1"
    for outputs in (["sum2"], ["sum1", "sum2"], FG.taps(FG.CHAIN[0], "1") + FG.taps(FG.CHAIN[1], "2")):
        _accepts(builder.build_plan(low, FP16, 2, outputs=outputs))
    _accepts(builder.build_plan(FG.lowered(FG.block_net(FG.TABLE_CASE), FG.TABLE_CASE.seed), FP16, FG.BATCH))


# ------------------------------------------------------------------------------------------------------------------
# references
# ------------------------------------------------------------------------------------------------------------------
REF_CASES = [FG.Case(cin3, 100, 200, 6, 7, res=res, relu3=r3, relu2=r2, seed=3)
             for cin3, res, r3, r2 in [(96, "identity", True, True), (96, "projection", False, True), (200, "input", True, False)]]


def _torch_block(low, x):
    """float64 torch: [short] [a -> ReLU] -> 3x3 b (ReLU) -> 1x1 c + residual (ReLU), from the lowered (folded) weights."""
    ops = {o["name"]: o for o in low["ops"]}

    def conv(name, t):
        o = ops[name]
        w = torch.from_numpy(o["W"]).double().permute(0, 3, 1, 2)
        y = F.conv2d(t, w, torch.from_numpy(o["bias"]).double(), padding=o["pad"])
        return y

    x = torch.from_numpy(x).double()
    t = {"data": x}
    if "short" in ops:
        t["short"] = conv("short", x)
    t["a"] = torch.relu(conv("a", x))
    b = conv("b", t["a"])
    if ops["b"]["relu"]:
        b = torch.relu(b)
    y = conv("c", b) + t[ops["c"]["residual"]]
    if ops["c"]["relu"]:
        y = torch.relu(y)
    return y.reshape(y.shape[0], -1).numpy()


@pytest.mark.parametrize("case", REF_CASES, ids=FG.case_id)
def test_emulation_without_rounding_is_the_block(case):
    low = FG.lowered(FG.block_net(case), case.seed)
    x = np.random.default_rng(4).standard_normal((2, case.data_channels, case.h, case.w))
    want = _torch_block(low, x)
    got = lowered_forward_f16emu(low, x, round16=False)
    assert np.abs(got - want).max() <= 1e-10 * max(1.0, np.abs(want).max())


@pytest.mark.parametrize("case", REF_CASES, ids=FG.case_id)
def test_own_input_references_reproduce_the_emulation(case):
    """Fed the emulation's own intermediate tensors, the per-operator references give its bits: the 3x3 on its input,
    the 1x1 with its residual on the 3x3's output."""
    low = FG.lowered(FG.block_net(case), case.seed)
    x = np.random.default_rng(5).standard_normal((2, case.data_channels, case.h, case.w)).astype(np.float32)
    keep = [t for t in ("short", "a", "b") if t in low["tensors"]]
    out, snaps = lowered_forward_f16emu(low, x, keep=keep)
    np.testing.assert_array_equal(FG.ref_op(low, "b", snaps["a"]), snaps["b"].reshape(2, -1))
    res = {"identity": FG.f16(x), "projection": snaps.get("short"), "input": snaps["a"]}[case.res]
    op_c = next(o for o in low["ops"] if o["name"] == "c")
    np.testing.assert_array_equal(FG.ref_1x1_residual(op_c, snaps["b"], res), out)
    if case.res == "projection":
        np.testing.assert_array_equal(FG.ref_op(low, "short", FG.f16(x)), snaps["short"].reshape(2, -1))
    # a wrong epilogue is visible: the 1x1's ReLU applied where the block has none, or the residual left out
    if not case.relu2:
        wrong = FG.ref_1x1_residual(dict(op_c, relu=True), snaps["b"], res)
        assert np.abs(wrong - out).max() > FG.TOL * np.abs(out).max()
    wrong = FG.ref_1x1_residual(op_c, snaps["b"], np.zeros_like(res))
    assert np.abs(wrong - out).max() > FG.TOL * np.abs(out).max()
