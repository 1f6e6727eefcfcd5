"""GPU parity: convolution kernels (wgmma implicit GEMM and CUDA-core fp32) vs the oracle conv
(torch CPU fp32 F.conv2d / conv_transpose2d on the same seeded inputs)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _nhwc(t, dtype):
    """NCHW cpu tensor -> NHWC view whose pixel stride is padded to a multiple of 8 (TMA alignment)."""
    n, c, h, w = t.shape
    cs = (c + 7) // 8 * 8
    buf = torch.zeros(n, h, w, cs, dtype=dtype)
    buf[..., :c] = t.permute(0, 2, 3, 1).to(dtype)
    return buf


CASES = [
    # n, cin, cout, h, w, k, stride, pad
    (1, 64, 64, 16, 32, 3, 1, 1),
    (2, 128, 256, 24, 40, 3, 1, 1),
    (1, 256, 64, 32, 32, 1, 1, 0),
    (1, 64, 128, 33, 47, 3, 2, 1),
    (1, 128, 512, 20, 28, 1, 2, 0),
    (1, 473, 256, 16, 24, 3, 1, 1),      # FlowNetC conv3_1: ragged cin (TMA OOB zero fill on channels)
    (1, 64, 2, 16, 32, 3, 1, 1),         # predict_flow: cout 2 -> padded N=16
    (1, 128, 128, 24, 24, 5, 2, 2),      # FlowNet 5x5 s2
    (3, 256, 256, 14, 14, 3, 1, 1),      # mask-head shape (batch of RoIs)
    (1, 192, 1024, 1, 300, 1, 1, 0),     # Linear as 1x1 over a row of "pixels"
    (1, 1026, 2, 8, 16, 3, 1, 1),        # predict_flow5: ragged cin, cout 2
    (1, 194, 2, 32, 48, 3, 1, 1),        # predict_flow2
    (1, 16, 2, 40, 56, 3, 1, 1),         # FlowNetFusion predict_flow0 (bk=16 path)
    (1, 12, 64, 32, 64, 7, 2, 3),        # FlowNetS conv1 stem (cin 12): bk=16 implicit GEMM without s2d
    (1, 48, 32, 20, 36, 3, 1, 1),        # cin < 64
    (1, 256, 256, 128, 256, 3, 1, 1),    # N = 256 halo layer, 256 tiles (two per CTA)
    (1, 256, 256, 120, 248, 3, 1, 1),    # same, ragged tiles (240 tiles)
]


@pytest.mark.parametrize("case", CASES)
def test_conv_tc_vs_oracle(cuda, case):
    from vps_b200 import ops
    n, cin, cout, h, w, k, s, p = case
    g = torch.Generator().manual_seed(hash(case) % (2 ** 31))
    x = torch.randn(n, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, generator=g)
    # oracle on bf16-representable operands, fp32 accumulation
    xq, wq = x.bfloat16().float(), wt.bfloat16().float()
    ref = F.leaky_relu(F.conv2d(xq, wq, b, stride=s, padding=p), 0.1)
    pk = ops.PackedConv(wt.to(cuda), b.to(cuda))
    xd = _nhwc(x, torch.bfloat16).to(cuda)[..., :cin]
    oh, ow = ref.shape[2:]
    y = torch.full((n, oh, ow, cout), float("nan"), dtype=torch.float32, device=cuda)
    ops.conv2d(xd, pk, y, stride=s, pad=p, act=ops.ACT_LRELU, slope=0.1)
    torch.cuda.synchronize()
    got = y.cpu().permute(0, 3, 1, 2)
    err = (got - ref).abs().max().item()
    assert err <= 1e-3 * max(1.0, ref.abs().max().item()), "max err %g" % err


@pytest.mark.parametrize("case", CASES[:6])
def test_conv_simt_vs_oracle(cuda, case):
    from vps_b200 import ops
    n, cin, cout, h, w, k, s, p = case
    g = torch.Generator().manual_seed(1 + hash(case) % (2 ** 31))
    x = torch.randn(n, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, generator=g)
    res = torch.randn(n, cout, (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1, generator=g)
    ref = F.relu(F.conv2d(x, wt, b, stride=s, padding=p) + res)
    pk = ops.PackedConv(wt.to(cuda), b.to(cuda))
    xd = _nhwc(x, torch.float32).to(cuda)[..., :cin]
    rd = _nhwc(res, torch.float32).to(cuda)
    y = torch.empty_like(rd)
    ops.conv2d(xd, pk, y, stride=s, pad=p, act=ops.ACT_RELU, res=rd)
    torch.cuda.synchronize()
    got = y.cpu().permute(0, 3, 1, 2)
    err = (got - ref).abs().max().item()
    assert err <= 1e-4 * max(1.0, ref.abs().max().item()), "max err %g" % err


def test_conv_tc_residual_bf16_out_and_slice(cuda):
    """bf16 output written into a channel slice of a concat buffer, residual add before ReLU."""
    from vps_b200 import ops
    g = torch.Generator().manual_seed(7)
    n, cin, cout, h, w = 1, 64, 256, 24, 40
    x = torch.randn(n, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, 1, 1, generator=g) / cin ** 0.5
    res = torch.randn(n, cout, h, w, generator=g)
    xq, wq, rq = x.bfloat16().float(), wt.bfloat16().float(), res.bfloat16().float()
    ref = F.relu(F.conv2d(xq, wq) + rq)
    pk = ops.PackedConv(wt.to(cuda))
    buf = torch.zeros(n, h, w, cout + 64, dtype=torch.bfloat16, device=cuda)
    ops.conv2d(_nhwc(x, torch.bfloat16).to(cuda), pk, buf[..., 64:], act=ops.ACT_RELU,
               res=_nhwc(res, torch.bfloat16).to(cuda))
    torch.cuda.synchronize()
    got = buf[..., 64:].float().cpu().permute(0, 3, 1, 2)
    assert (buf[..., :64] == 0).all()
    err = (got - ref).abs().max().item()
    assert err <= 2e-2 * max(1.0, ref.abs().max().item())   # one bf16 rounding of the output
    assert (got - ref).abs().mean().item() < 3e-3


def test_deconv4x4_as_phase_convs(cuda):
    """ConvTranspose2d(k=4,s=2,p=1) (submodules.py:33-37) as four 2x2 stride-phase convolutions."""
    from vps_b200 import ops
    from vps_b200.layers import deconv4x4_s2
    g = torch.Generator().manual_seed(11)
    cin, cout, h, w = 128, 64, 12, 20
    x = torch.randn(1, cin, h, w, generator=g)
    wt = torch.randn(cin, cout, 4, 4, generator=g) / (cin * 4) ** 0.5
    b = torch.randn(cout, generator=g)
    for dtype, tol in ((torch.float32, 1e-4), (torch.bfloat16, 1e-3)):
        xq = x.to(dtype).float()
        wq = wt.to(dtype).float()
        ref = F.leaky_relu(F.conv_transpose2d(xq, wq, b, stride=2, padding=1), 0.1)
        layer = deconv4x4_s2(wt.to(cuda), b.to(cuda))
        y = torch.empty(1, 2 * h, 2 * w, cout, dtype=torch.float32, device=cuda)
        layer(_nhwc(x, dtype).to(cuda), y, act=ops.ACT_LRELU)
        torch.cuda.synchronize()
        got = y.cpu().permute(0, 3, 1, 2)
        err = (got - ref).abs().max().item()
        assert err <= tol * max(1.0, ref.abs().max().item()), (dtype, err)


@pytest.mark.parametrize("cin,h,w", [(3, 33, 47), (12, 32, 64), (6, 17, 30)])
def test_stem_7x7s2_space_to_depth(cuda, cin, h, w):
    """StemConv7x7s2 (space-to-depth + 4x4 stride-1 tensor-core conv) == the 7x7 / stride 2 / pad 3 convolution it replaces
    (resnet.py conv1, FlowNetC/S conv1), odd and even sizes."""
    from vps_b200 import ops
    from vps_b200.layers import StemConv7x7s2
    g = torch.Generator().manual_seed(100 + cin)
    x = torch.randn(1, cin, h, w, generator=g)
    wt = torch.randn(64, cin, 7, 7, generator=g) / (cin * 49) ** 0.5
    b = torch.randn(64, generator=g)
    ref = F.relu(F.conv2d(x.bfloat16().float(), wt.bfloat16().float(), b, stride=2, padding=3))
    stem = StemConv7x7s2(wt.to(cuda), b.to(cuda), act=ops.ACT_RELU)
    xd = _nhwc(x, torch.bfloat16).to(cuda)[..., :cin]
    y = stem(xd, out_dtype=torch.float32)
    torch.cuda.synchronize()
    got = y.cpu().permute(0, 3, 1, 2)
    assert got.shape == ref.shape
    err = (got - ref).abs().max().item()
    assert err <= 1e-3 * max(1.0, ref.abs().max().item()), "max err %g" % err


BF16_OUT_CASES = [
    # n, cin, cout, h, w, k, stride, pad, with_residual
    (1, 64, 256, 37, 53, 1, 1, 0, True),      # bottleneck expand + residual, ragged tiles
    (2, 128, 128, 24, 40, 3, 1, 1, False),    # halo mode, N = 128
    (1, 96, 64, 33, 20, 3, 2, 1, False),      # flat stride 2, N = 64
    (1, 256, 320, 16, 24, 1, 1, 0, True),     # several N tiles
    (1, 64, 48, 16, 16, 3, 1, 1, False),      # partial 32-column chunk (16-byte store groups)
]


@pytest.mark.parametrize("case", BF16_OUT_CASES)
def test_conv_tc_bf16_output_epilogues(cuda, case):
    """bf16 outputs (the production dtype) with bias, ReLU and a residual added before the activation
    (resnet.py:236-258), written into a channel slice of a wider buffer whose other channels must stay untouched."""
    from vps_b200 import ops
    n, cin, cout, h, w, k, s, p, with_res = case
    g = torch.Generator().manual_seed(hash(case) % (2 ** 31))
    x = torch.randn(n, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, generator=g)
    xq, wq = x.bfloat16().float(), wt.bfloat16().float()
    pre = F.conv2d(xq, wq, b, stride=s, padding=p)
    oh, ow = pre.shape[2:]
    res = torch.randn(n, cout, oh, ow, generator=g).bfloat16().float() if with_res else None
    ref = F.relu(pre + res) if with_res else F.relu(pre)
    pk = ops.PackedConv(wt.to(cuda), b.to(cuda))
    xd = _nhwc(x, torch.bfloat16).to(cuda)[..., :cin]
    wide = torch.full((n, oh, ow, cout + 32), 7.0, dtype=torch.bfloat16, device=cuda)     # slice [16, 16 + cout)
    y = wide[..., 16:16 + cout]
    rd = _nhwc(res, torch.bfloat16).to(cuda)[..., :cout] if with_res else None
    ops.conv2d(xd, pk, y, stride=s, pad=p, act=ops.ACT_RELU, res=rd)
    torch.cuda.synchronize()
    got = y.float().cpu().permute(0, 3, 1, 2)
    err = (got - ref).abs().max().item()
    assert err <= 2.0 ** -7 * max(1.0, ref.abs().max().item()), "max err %g" % err
    assert float((wide[..., :16].float() - 7.0).abs().max()) == 0.0 and float((wide[..., 16 + cout:].float() - 7.0).abs().max()) == 0.0
