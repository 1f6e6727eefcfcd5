"""Channel-split layouts of the tc32 convolution (vps_conv2d_tc32_plan plan[6] = Q): a tile of 64 P pixels x block_n
channels, consumer warpgroup w taking pixels 64 (w / Q).. and channels (block_n / Q) (w % Q).. of it.  The layout does not
change a single output bit: each layer runs once at its full cout, in a layout with Q > 1, and once as 16-channel weight
slices, which have one channel group (Q = 1), each writing its channel slice of the output; the two must be equal, and both
within the componentwise bound of tests/tc32_model.py against fp64.  The production shapes of tools/diag_tc32.py select
every layout the planner offers."""
import importlib.util
import os

import pytest
import torch
import torch.nn.functional as F

from tests import tc32_model as M

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SLICE = 16
LAYOUTS = {(2, 1), (4, 1), (2, 2), (1, 4)}      # (P, Q) the planner may pick


@pytest.fixture()
def tc32(cuda):
    from vps_b200 import ops
    old = ops.F32_TC[0]
    ops.F32_TC[0] = True
    yield ops
    ops.F32_TC[0] = old


def dev_nhwc(t):
    from vps_b200.layers import empty_nhwc
    n, c, h, w = t.shape
    x = empty_nhwc(n, h, w, c, torch.float32, t.device)
    x.copy_(t.permute(0, 2, 3, 1))
    return x


# kind, n, cin, cout, (H, W) input, k, stride, residual.  Full-size grids, so that the planner picks Q > 1 on the H100's
# 132 SMs; odd sizes give partial edge tiles, cout 120 a last channel group that is partly padding.
CASES = {
    "halo_3x3": ("conv", 1, 256, 256, (100, 260), 3, 1, False),
    "halo_3x3_cout120": ("conv", 1, 96, 120, (131, 257), 3, 1, False),
    "flat_3x3_s2": ("conv", 1, 128, 256, (254, 510), 3, 2, False),
    "flat_1x1_res_tma": ("conv", 2, 64, 256, (126, 250), 1, 1, True),
    "flat_1x1_res_tma_cout120": ("conv", 2, 256, 120, (126, 250), 1, 1, True),
    "deconv4x4_s2": ("deconv", 1, 256, 128, (62, 126), 4, 2, False),
}


def make(name, g):
    kind, n, cin, cout, (h, w), k, s, resk = CASES[name]
    x = M.fat((n, cin, h, w), g)
    wshape = (cin, cout, k, k) if kind == "deconv" else (cout, cin, k, k)
    wt = M.fat(wshape, g) * 2.0 ** -round(0.5 * (cin * k * k).bit_length())
    b = M.fat((cout,), g)
    if kind == "deconv":
        oh, ow = 2 * h, 2 * w
    else:
        oh, ow = (h + 2 * (k // 2) - k) // s + 1, (w + 2 * (k // 2) - k) // s + 1
    res = M.fat((n, cout, oh, ow), g) if resk else None
    return x, wt, b, res


def run(ops, name, xd, wt, b, y, rd):
    """the layer with weights wt (OIHW, IOHW for the deconvolution) into y; returns its plan"""
    from vps_b200.layers import deconv4x4_s2
    kind, _, _, _, _, k, s, _ = CASES[name]
    if kind == "deconv":
        layer = deconv4x4_s2(wt, b)
        pws, pads = [ph[3] for ph in layer.phases], [ph[2] for ph in layer.phases]
        plan = ops.conv2d_tc32_plan(xd, pws, pads=pads, oh=xd.shape[1], ow=xd.shape[2], y=y,
                                    omaps=[(2, ph[0], 2, ph[1]) for ph in layer.phases])
        layer(xd, y, act=ops.ACT_RELU)
        return plan
    pk = ops.PackedConv(wt, b)
    plan = ops.conv2d_tc32_plan(xd, pk, stride=s, pad=k // 2, y=y, res=rd)
    ops.conv2d(xd, pk, y, stride=s, pad=k // 2, act=ops.ACT_RELU, res=rd, use_tc=True)
    return plan


def reference(name, x, wt, b, res):
    """(fp64 result, componentwise bound) of the layer with ReLU and the residual added before it"""
    kind, _, cin, _, _, k, s, _ = CASES[name]
    if kind == "deconv":
        lin = lambda u, v: F.conv_transpose2d(u, v, stride=2, padding=1)
        sum_w = wt.double().abs().sum((0, 2, 3)).view(1, -1, 1, 1)
        ones = torch.ones((cin, 1, k, k), dtype=torch.float64, device=x.device)
        steps = M.steps(cin, (k // 2) ** 2)
    else:
        lin = lambda u, v: F.conv2d(u, v, stride=s, padding=k // 2)
        sum_w = wt.double().abs().sum((1, 2, 3)).view(1, -1, 1, 1)
        ones = torch.ones((1, cin, k, k), dtype=torch.float64, device=x.device)
        steps = M.steps(cin, k * k)
    x64, w64 = x.double(), wt.double()
    pre = lin(x64, w64) + b.double().view(1, -1, 1, 1)
    if res is not None:
        pre = pre + res.double()
    ref = pre.clamp_min(0)
    bnd = M.bound(lin(x64.abs(), w64.abs()), sum_w, lin(x64.abs(), ones), M.gamma(steps), bias=b.double().view(1, -1, 1, 1),
                  res=0.0 if res is None else res.double(), out=ref, pre=pre, act="relu")
    return ref, bnd


@pytest.mark.parametrize("name", sorted(CASES))
def test_split_n_equals_slices_and_fp64(tc32, name):
    ops = tc32
    kind, n, cin, cout, _, k, s, _ = CASES[name]
    g = torch.Generator(device="cuda").manual_seed(31 + cin + cout)
    x, wt, b, res = make(name, g)
    xd = dev_nhwc(x)
    rd = dev_nhwc(res) if res is not None else None
    oh, ow = (res.shape[2:] if res is not None else
              ((2 * x.shape[2], 2 * x.shape[3]) if kind == "deconv"
               else ((x.shape[2] + 2 * (k // 2) - k) // s + 1, (x.shape[3] + 2 * (k // 2) - k) // s + 1)))
    y = torch.full((n, oh, ow, cout), float("nan"), dtype=torch.float32, device="cuda")
    plan = run(ops, name, xd, wt, b, y, rd)
    assert plan["wg_n"] > 1, plan
    if name.startswith("flat_1x1_res_tma"):
        assert plan["epilogue"] == "tma", plan
    y2 = torch.full_like(y, float("nan"))
    for c0 in range(0, cout, SLICE):
        c1 = min(cout, c0 + SLICE)
        ws = (wt[:, c0:c1] if kind == "deconv" else wt[c0:c1]).contiguous()
        sp = run(ops, name, xd, ws, b[c0:c1].contiguous(), y2[..., c0:c1], None if rd is None else rd[..., c0:c1])
        assert sp["wg_n"] == 1 and sp["block_n"] == 16, sp
    torch.cuda.synchronize()
    assert not torch.isnan(y).any()
    assert torch.equal(y, y2), plan
    ref, bnd = reference(name, x, wt, b, res)
    err = (y.permute(0, 3, 1, 2).double() - ref).abs()
    assert bool((err <= bnd).all()), "%s: worst err / bound %g" % (name, float((err / bnd).max()))
    assert ops.tc32_overflow() == 0


def _diag_shapes():
    spec = importlib.util.spec_from_file_location("diag_tc32", os.path.join(ROOT, "tools", "diag_tc32.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.SHAPES, mod.DECONVS


def test_production_shapes_pick_every_layout(tc32):
    ops = tc32
    from vps_b200.layers import deconv4x4_s2, empty_nhwc
    shapes, deconvs = _diag_shapes()
    seen = set()
    for (n, cin, cout, oh, ow, k, s, r, _) in shapes:
        x = empty_nhwc(n, oh * s, ow * s, cin, torch.float32, "cuda")
        y = empty_nhwc(n, oh, ow, cout, torch.float32, "cuda")
        pk = ops.PackedConv(torch.zeros(cout, cin, k, k, device="cuda"), None)
        pad = k // 2 if s == 1 or k % 2 else 1
        plan = ops.conv2d_tc32_plan(x, pk, stride=s, pad=pad, oh=oh, ow=ow, y=y, res=y if r else None)
        assert plan["layout"][0] * plan["layout"][1] == plan["nwg"], plan
        seen.add(plan["layout"])
    for (n, cin, cout, h, w, _) in deconvs:
        x = empty_nhwc(n, h, w, cin, torch.float32, "cuda")
        y = empty_nhwc(n, 2 * h, 2 * w, cout, torch.float32, "cuda")
        layer = deconv4x4_s2(torch.zeros(cin, cout, 4, 4, device="cuda"), None)
        plan = ops.conv2d_tc32_plan(x, [ph[3] for ph in layer.phases], pads=[ph[2] for ph in layer.phases], oh=h, ow=w, y=y,
                                    omaps=[(2, ph[0], 2, ph[1]) for ph in layer.phases])
        seen.add(plan["layout"])
    assert seen == LAYOUTS, seen
