"""Tile layouts of the fused tc32 DCN (vps_deform_conv_tc32): the plan covers all output channels of the UPSNet head's
layers in one N tile at the P2 / P3 shapes (each input sampled once), every layout it picks matches the oracle DCNv1, and
the layout does not change a single output bit: a 256 -> 256 layer run in one launch equals its two 128-channel weight
halves run as separate launches."""
import pytest
import torch

pytestmark = pytest.mark.gpu

HEAD_LAYERS = [(256, 256), (256, 128), (128, 128)]     # cin, cout of the three DCNs per level


def to_nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous().cuda()


def inputs(g, n, c, h, w):
    x = torch.randn(n, c, h, w, generator=g)
    off = torch.randn(n, 18, h, w, generator=g) * 3.0
    off[:, :, 0, :] -= 4.0                           # some samples fall outside the image
    return x, off


def kind(plan):
    if plan["n_tiles"] > 1:
        return "multi_n"
    return plan["layout"]


@pytest.mark.parametrize("hw", [(256, 512), (128, 256)], ids=["P2", "P3"])
def test_production_levels_one_n_tile(cuda, hw):
    from vps_b200 import ops
    h, w = hw
    for ci, co in HEAD_LAYERS:
        x = torch.empty(1, h, w, ci, dtype=torch.float32, device="cuda")
        pk = ops.PackedConv(torch.zeros(co, ci, 3, 3, device="cuda"), None)
        plan = ops.deform_conv_tc32_plan(x, pk)
        assert plan["n_tiles"] == 1, (hw, ci, co, plan)
        assert plan["bn"] * (2 if plan["layout"] == "split_n" else 1) == co, plan


def test_layouts_match_oracle(cuda):
    from oracle import ops as O
    from vps_b200 import ops
    g = torch.Generator().manual_seed(21)
    seen = set()
    old = ops.F32_TC[0]
    ops.F32_TC[0] = True
    try:
        # ragged tiles and two images; split-N over 256 channels, split-M, narrow tiles over several N tiles
        for (n, ci, co, h, w) in [(2, 256, 256, 61, 99), (2, 256, 128, 60, 100), (1, 256, 256, 48, 80), (1, 128, 128, 19, 37)]:
            x, off = inputs(g, n, ci, h, w)
            wt = torch.randn(co, ci, 3, 3, generator=g) / (ci * 9) ** 0.5
            ref = O.deform_conv(x, off, wt)
            pk = ops.PackedConv(wt.cuda(), None)
            xd = to_nhwc(x)
            seen.add(kind(ops.deform_conv_tc32_plan(xd, pk)))
            y = torch.full((n, h, w, co), float("nan"), dtype=torch.float32, device="cuda")
            ops.deform_conv_tc32(xd, to_nhwc(off), pk, y)
            torch.cuda.synchronize()
            got = y.permute(0, 3, 1, 2).cpu()
            assert not torch.isnan(got).any()
            assert float((got - ref).abs().max()) <= 1e-5 * max(1.0, float(ref.abs().max())), (n, ci, co, h, w)
        assert ops.tc32_overflow() == 0
    finally:
        ops.F32_TC[0] = old
    assert {"split_n", "split_m", "multi_n"} <= seen, seen


@pytest.mark.parametrize("shape", [(2, 60, 100), (1, 48, 80), (1, 16, 32)])
def test_full_width_equals_halves(cuda, shape):
    from vps_b200 import ops
    n, h, w = shape
    g = torch.Generator().manual_seed(22)
    x, off = inputs(g, n, 256, h, w)
    wt = torch.randn(256, 256, 3, 3, generator=g) / (256 * 9) ** 0.5
    xd, offd = to_nhwc(x), to_nhwc(off)
    full = ops.PackedConv(wt.cuda(), None)
    halves = [ops.PackedConv(wt[:128].contiguous().cuda(), None), ops.PackedConv(wt[128:].contiguous().cuda(), None)]
    plans = [ops.deform_conv_tc32_plan(xd, full)] + [ops.deform_conv_tc32_plan(xd, pk) for pk in halves]
    old = ops.F32_TC[0]
    ops.F32_TC[0] = True
    try:
        y = torch.full((n, h, w, 256), float("nan"), dtype=torch.float32, device="cuda")
        ops.deform_conv_tc32(xd, offd, full, y)
        y2 = torch.full((n, h, w, 256), float("nan"), dtype=torch.float32, device="cuda")
        ops.deform_conv_tc32(xd, offd, halves[0], y2[..., :128])
        ops.deform_conv_tc32(xd, offd, halves[1], y2[..., 128:])
        torch.cuda.synchronize()
    finally:
        ops.F32_TC[0] = old
    assert not torch.isnan(y).any()
    assert torch.equal(y, y2), plans
