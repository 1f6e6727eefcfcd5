"""GPU parity: correlation / resample2d / channelnorm kernels vs the oracle restatements."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _nhwc(t, dtype=torch.float32):
    return t.permute(0, 2, 3, 1).contiguous().to(dtype)


@pytest.mark.parametrize("cfg", [(20, 2, 64, 24, 40), (4, 1, 48, 20, 36), (20, 2, 256, 16, 70), (4, 1, 256, 33, 31)])
def test_correlation(cuda, cfg):
    from oracle import ops as O
    from vps_b200 import ops
    md, s2, C, H, W = cfg
    g = torch.Generator().manual_seed(3)
    f1 = torch.randn(1, C, H, W, generator=g)
    f2 = torch.randn(1, C, H, W, generator=g)
    ref = O.correlation(f1, f2, md, 1, md, 1, s2)
    D = 2 * (md // s2) + 1
    out = torch.empty(1, H, W, D * D, device=cuda)
    ops.correlation(_nhwc(f1).to(cuda), _nhwc(f2).to(cuda), out, md, md, 1, s2)
    torch.cuda.synchronize()
    got = out.cpu().permute(0, 3, 1, 2)
    assert (got - ref).abs().max().item() <= 1e-5


def test_resample2d_and_channelnorm(cuda):
    from oracle import ops as O
    from vps_b200 import ops
    g = torch.Generator().manual_seed(5)
    src = torch.randn(2, 3, 40, 56, generator=g)
    flow = (torch.rand(2, 2, 40, 56, generator=g) - 0.5) * 30
    ref = O.resample2d(src, flow)
    out = torch.empty(2, 40, 56, 3, device=cuda)
    ops.resample2d(_nhwc(src).to(cuda), _nhwc(flow).to(cuda), out)
    nrm = torch.empty(2, 40, 56, 1, device=cuda)
    ops.channelnorm(_nhwc(src).to(cuda), nrm, b=out)
    torch.cuda.synchronize()
    assert (out.cpu().permute(0, 3, 1, 2) - ref).abs().max().item() <= 1e-5
    refn = O.channelnorm(src - ref)
    assert (nrm.cpu().permute(0, 3, 1, 2) - refn).abs().max().item() <= 1e-5


@pytest.mark.parametrize("cfg", [(20, 2, 256, 128, 256), (20, 2, 64, 37, 53), (4, 1, 256, 64, 96), (4, 1, 128, 21, 50),
                                 (20, 2, 192, 9, 11), (4, 1, 64, 3, 5)])
def test_correlation_tensor_core(cuda, cfg):
    """banded-GEMM correlation on wgmma vs the oracle on bf16-representable features (fp32 accumulation both)."""
    from oracle import ops as O
    from vps_b200 import ops
    md, s2, C, H, W = cfg
    g = torch.Generator().manual_seed(17)
    f1 = torch.randn(1, C, H, W, generator=g).bfloat16().float()
    f2 = torch.randn(1, C, H, W, generator=g).bfloat16().float()
    ref = torch.nn.functional.leaky_relu(O.correlation(f1, f2, md, 1, md, 1, s2), 0.1)
    D = 2 * (md // s2) + 1
    cs = (D * D + 7) // 8 * 8
    for odt, tol in ((torch.float32, 2e-5), (torch.bfloat16, 1e-2)):
        buf = torch.full((1, H, W, cs + 8), 7.0, dtype=odt, device=cuda)
        out = buf[..., 8:8 + D * D]
        ops.correlation(_nhwc(f1, torch.bfloat16).to(cuda), _nhwc(f2, torch.bfloat16).to(cuda), out, md, md, 1, s2,
                        act=ops.ACT_LRELU, slope=0.1, impl="tc")
        torch.cuda.synchronize()
        got = out.float().cpu().permute(0, 3, 1, 2)
        assert (got - ref).abs().max().item() <= tol * max(1.0, ref.abs().max().item()), (cfg, odt)
        assert (buf[..., :8] == 7.0).all() and (buf[..., 8 + D * D:] == 7.0).all()     # neighbours of the slice untouched


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_flownet_glue_fused_equals_separate_ops(cuda, dtype):
    """vps_flownet_stage / vps_flownet_cat3 (one kernel per concat input of FlowNet2, flownet2.py:142-153, 176-189) are
    bit-identical to the chains of resize / axpby / resample2d / channelnorm launches they replace."""
    from vps_b200 import ops
    from vps_b200.layers import empty_nhwc
    g = torch.Generator().manual_seed(77)
    n, H, W = 1, 64, 96
    dev = torch.device("cuda:0")
    x6 = empty_nhwc(n, H, W, 6, dtype, dev)
    x6.copy_(torch.randn(n, H, W, 6, generator=g).to(dev))
    x6[0, 0, 0, 0] = -0.0
    img0, img1 = x6[..., 0:3], x6[..., 3:6]
    flow2 = (torch.randn(n, H // 4, W // 4, 2, generator=g) * 3).to(dev)
    sd2 = (torch.randn(n, H // 4, W // 4, 2, generator=g) * 40).to(dev)
    div = 20.0
    f32 = lambda c: torch.empty(n, H, W, c, dtype=torch.float32, device=dev)
    # ---- stage
    ref = empty_nhwc(n, H, W, 12, dtype, dev)
    flow = f32(2)
    ops.resize_bilinear(flow2, flow, mul=div)
    ops.copy_scale(x6, ref[..., 0:6])
    ops.resample2d(img1, flow, ref[..., 6:9])
    ops.copy_scale(flow, ref[..., 9:11], 1.0 / div)
    ops.channelnorm(img0, ref[..., 11:12], b=ref[..., 6:9])
    got = empty_nhwc(n, H, W, 12, dtype, dev)
    ops.flownet_stage(x6, flow2, div, 1.0 / div, got)
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int16 if dtype == torch.bfloat16 else torch.int32),
                       ref.view(torch.int16 if dtype == torch.bfloat16 else torch.int32))
    # ---- concat3
    ref3 = empty_nhwc(n, H, W, 11, dtype, dev)
    s2f, sdf = f32(2), f32(2)
    ops.resize_nearest(flow2, s2f, mul=div)
    ops.resize_nearest(sd2, sdf, mul=1.0 / div)
    ops.copy_scale(img0, ref3[..., 0:3])
    ops.copy_scale(sdf, ref3[..., 3:5])
    ops.copy_scale(s2f, ref3[..., 5:7])
    ops.channelnorm(sdf, ref3[..., 7:8])
    ops.channelnorm(s2f, ref3[..., 8:9])
    warped = empty_nhwc(n, H, W, 3, dtype, dev)
    ops.resample2d(img1, sdf, warped)
    ops.channelnorm(img0, ref3[..., 9:10], b=warped)
    ops.resample2d(img1, s2f, warped)
    ops.channelnorm(img0, ref3[..., 10:11], b=warped)
    got3 = empty_nhwc(n, H, W, 11, dtype, dev)
    ops.flownet_cat3(x6, flow2, sd2, div, 1.0 / div, got3)
    torch.cuda.synchronize()
    assert torch.equal(got3.view(torch.int16 if dtype == torch.bfloat16 else torch.int32),
                       ref3.view(torch.int16 if dtype == torch.bfloat16 else torch.int32))


@pytest.mark.parametrize("cfg", [(20, 2, 256, 40, 72), (4, 1, 256, 33, 31), (20, 2, 64, 37, 53), (4, 1, 128, 21, 50)])
def test_correlation_tc32(cuda, cfg):
    """fp32 features on the tensor cores (split fp16 planes, three banded-GEMM passes) vs the fp32 oracle: fp32-class error
    (the single bf16 pass on the same features is off by ~1e-2), slice neighbours untouched, no saturation"""
    from oracle import ops as O
    from vps_b200 import ops
    md, s2, C, H, W = cfg
    g = torch.Generator().manual_seed(23)
    f1 = torch.randn(1, C, H, W, generator=g)
    f2 = torch.randn(1, C, H, W, generator=g)
    ref = torch.nn.functional.leaky_relu(O.correlation(f1, f2, md, 1, md, 1, s2), 0.1)
    D = 2 * (md // s2) + 1
    cs = (D * D + 7) // 8 * 8
    buf = torch.full((1, H, W, cs + 8), 7.0, dtype=torch.float32, device=cuda)
    out = buf[..., 8:8 + D * D]
    old = ops.F32_TC[0]
    ops.F32_TC[0] = True
    try:
        n0 = ops.launch_count()
        ops.correlation(_nhwc(f1).to(cuda), _nhwc(f2).to(cuda), out, md, md, 1, s2, act=ops.ACT_LRELU, slope=0.1, impl="tc32")
        assert ops.launch_count() - n0 == 5          # 2 operand splits + 3 tensor-core passes
    finally:
        ops.F32_TC[0] = old
    torch.cuda.synchronize()
    got = out.cpu().permute(0, 3, 1, 2)
    assert (got - ref).abs().max().item() <= 2e-6 * max(1.0, ref.abs().max().item()), cfg
    assert (buf[..., :8] == 7.0).all() and (buf[..., 8 + D * D:] == 7.0).all()
    assert ops.tc32_overflow() == 0
