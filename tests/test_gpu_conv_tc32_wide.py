"""Four consumer warpgroups in the tc32 convolution (256-pixel tiles at block_n <= 64, vps_conv2d_tc32_plan).  The plan
depends on the grid size, so the same layer runs with four warpgroups on a large input and with two on a crop of it: the
outputs away from the crop border must be bit-identical (the tiling does not change any element's K order) and both must
hold the 2e-5 fp64 tolerance of test_gpu_conv_tc32.py."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = 2e-5


@pytest.fixture()
def tc32():
    from vps_b200 import ops
    old = ops.F32_TC[0]
    ops.F32_TC[0] = True
    yield ops
    ops.F32_TC[0] = old


def _dev_nhwc(t, cuda):
    from vps_b200.layers import empty_nhwc
    n, c, h, w = t.shape
    x = empty_nhwc(n, h, w, c, torch.float32, cuda)
    x.copy_(t.permute(0, 2, 3, 1).to(cuda))
    return x


def _check_fp64(got_nhwc, ref):
    got = got_nhwc.cpu().permute(0, 3, 1, 2).double()
    assert got.shape == ref.shape
    err = (got - ref).abs().max().item()
    assert err <= TOL * max(1.0, ref.abs().max().item()), "max err %g" % err


CONVS = [
    # cin, cout, (H, W) large, k, stride, (y0, x0, h, w) crop of the input
    (82, 16, (256, 512), 3, 1, (40, 72, 48, 96)),       # FlowNetFusion conv0-like halo layer, N = 16
    (162, 32, (128, 256), 3, 1, (16, 40, 40, 64)),      # halo, N = 32
    (11, 64, (256, 512), 3, 1, (8, 16, 40, 64)),        # thin-cin halo, N = 64
    (256, 64, (128, 256), 1, 1, (16, 40, 24, 64)),      # flat (one box per K step), 1x1
    (64, 64, (256, 512), 3, 2, (32, 64, 40, 64)),       # flat, stride 2 (TMA element strides)
]


@pytest.mark.parametrize("case", CONVS)
def test_wide_conv_matches_narrow_and_fp64(cuda, tc32, case):
    ops = tc32
    cin, cout, (H, W), k, s, (y0, x0, h, w) = case
    p = k // 2
    g = torch.Generator().manual_seed(cin * 1000 + cout)
    x = torch.randn(1, cin, H, W, generator=g)
    wt = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, generator=g)
    pk = ops.PackedConv(wt.to(cuda), b.to(cuda))
    outs = []
    for xi, nwg in ((x, 4), (x[:, :, y0:y0 + h, x0:x0 + w].contiguous(), 2)):
        xd = _dev_nhwc(xi, cuda)
        assert ops.conv2d_tc32_plan(xd, pk, stride=s, pad=p)["nwg"] == nwg
        ref = F.leaky_relu(F.conv2d(xi.double(), wt.double(), b.double(), stride=s, padding=p), 0.1)
        y = torch.full((1, ref.shape[2], ref.shape[3], cout), float("nan"), dtype=torch.float32, device=cuda)
        ops.conv2d(xd, pk, y, stride=s, pad=p, act=ops.ACT_LRELU, slope=0.1, use_tc=True)
        torch.cuda.synchronize()
        _check_fp64(y, ref)
        outs.append(y)
    big, crop = outs
    m = p                                           # output pixels of the crop that see no crop-border padding
    ho, wo = crop.shape[1:3]
    oy, ox = y0 // s, x0 // s                       # crop offsets are multiples of the stride
    assert torch.equal(crop[:, m:ho - m, m:wo - m], big[:, oy + m:oy + ho - m, ox + m:ox + wo - m])


DECONVS = [
    # cin, cout, (H, W) large input, (y0, x0, h, w) crop
    (162, 16, (128, 256), (24, 40, 24, 48)),            # FlowNetFusion deconv: four 2x2 stride phases, N = 16
    (128, 32, (128, 256), (8, 8, 24, 40)),
]


@pytest.mark.parametrize("case", DECONVS)
def test_wide_deconv_phases_match_narrow_and_fp64(cuda, tc32, case):
    ops = tc32
    from vps_b200.layers import deconv4x4_s2
    cin, cout, (H, W), (y0, x0, h, w) = case
    g = torch.Generator().manual_seed(cin * 7 + cout)
    x = torch.randn(1, cin, H, W, generator=g)
    wt = torch.randn(cin, cout, 4, 4, generator=g) / (cin * 4) ** 0.5
    b = torch.randn(cout, generator=g)
    layer = deconv4x4_s2(wt.to(cuda), b.to(cuda))
    pws, pads = [ph[3] for ph in layer.phases], [ph[2] for ph in layer.phases]
    outs = []
    for xi, nwg in ((x, 4), (x[:, :, y0:y0 + h, x0:x0 + w].contiguous(), 2)):
        xd = _dev_nhwc(xi, cuda)
        plan = ops.conv2d_tc32_plan(xd, pws, pads=pads, oh=xi.shape[2], ow=xi.shape[3])
        assert plan["nwg"] == nwg and plan["halo"] == 1, plan
        ref = F.leaky_relu(F.conv_transpose2d(xi.double(), wt.double(), b.double(), stride=2, padding=1), 0.1)
        y = torch.full((1, 2 * xi.shape[2], 2 * xi.shape[3], cout), float("nan"), dtype=torch.float32, device=cuda)
        layer(xd, y, act=ops.ACT_LRELU)
        torch.cuda.synchronize()
        _check_fp64(y, ref)
        outs.append(y)
    big, crop = outs
    inner = crop[:, 2:2 * h - 2, 2:2 * w - 2]       # one input pixel of crop border = two output pixels
    assert torch.equal(inner, big[:, 2 * y0 + 2:2 * (y0 + h) - 2, 2 * x0 + 2:2 * (x0 + w) - 2])
