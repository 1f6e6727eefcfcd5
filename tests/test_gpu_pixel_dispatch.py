"""GPU: the launch arms of the memory-bound pixel kernels.

Each vector-capable launcher runs V channels per thread (V = 4 fp32 / 8 bf16) when every tensor has channels a multiple of
V, a 16-byte aligned base and a 16-byte multiple pixel stride, and V = 1 otherwise.  Both arms run here on the same values,
in fp32 and bf16: once on dense NHWC tensors, once on channel slices starting at channel 1 of a wider buffer.  The
per-element arithmetic does not depend on V, so the outputs must be bit-identical.  The mixed-dtype arms (bf16 flow or
offsets, fp32 <-> bf16 input / output) run once each against torch references."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BF16_TOL = 1e-2          # bf16 outputs: one bf16 rounding of the fp32 result


def dense(t, dtype):
    """NCHW -> dense NHWC CUDA tensor: a vector-eligible layout"""
    return t.permute(0, 2, 3, 1).contiguous().to(dtype).cuda()


def sliced(t, dtype):
    """NCHW -> the same values at channels 1..c of a c+1 channel NHWC buffer: base and pixel stride unaligned, V = 1"""
    n, c, h, w = t.shape
    buf = torch.zeros(n, h, w, c + 1, dtype=dtype, device="cuda")
    buf[..., 1:] = t.permute(0, 2, 3, 1).to(dtype).cuda()
    return buf[..., 1:]


def out_nhwc(shape, dtype, layout):
    n, h, w, c = shape
    return layout(torch.full((n, c, h, w), float("nan")), dtype)


def nchw(t):
    return t.float().permute(0, 3, 1, 2).cpu()


def bits(t):
    t = t.contiguous()
    return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32).cpu()


def close(got, ref, tol):
    return float((got - ref).abs().max()) <= tol * max(1.0, float(ref.abs().max()))


def rnd(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g) * scale


# Each case: (NCHW inputs whose layout is varied, NHWC output shape, launch(out, *inputs), torch reference(*inputs) NCHW,
# fp32 tolerance, vector / scalar tolerance or None for bit-identical).
def case_axpby(g):
    return ([rnd(g, 2, 16, 9, 13), rnd(g, 2, 16, 9, 13)], (2, 9, 13, 16),
            lambda o, a, b: ops().axpby(a, o, 0.75, b, -1.5), lambda a, b: 0.75 * a - 1.5 * b, 1e-5, None)


def case_resize_bilinear(g):
    return ([rnd(g, 1, 16, 9, 13)], (1, 20, 27, 16), lambda o, x: ops().resize_bilinear(x, o, mul=0.5),
            lambda x: F.interpolate(x, size=(20, 27), mode="bilinear", align_corners=False) * 0.5, 1e-5, None)


def case_resize_nearest(g):
    return ([rnd(g, 1, 16, 9, 13)], (1, 20, 27, 16), lambda o, x: ops().resize_nearest(x, o, mul=2.0),
            lambda x: F.interpolate(x, size=(20, 27), mode="nearest") * 2.0, 1e-5, None)


def case_pool2d_max(g):
    return ([rnd(g, 1, 16, 15, 22)], (1, 8, 11, 16), lambda o, x: ops().pool2d(x, o, 3, 2, 1, False),
            lambda x: F.max_pool2d(x, 3, 2, 1), 1e-5, None)


def case_pool2d_avg(g):
    return ([rnd(g, 1, 16, 15, 22)], (1, 8, 11, 16), lambda o, x: ops().pool2d(x, o, 3, 2, 1, True),
            lambda x: F.avg_pool2d(x, 3, 2, 1), 1e-5, None)


def case_groupnorm(g):
    # 128 channels in 16 groups: the dense layout takes gn_stats_vec in both dtypes, the slice takes gn_stats, which sums in
    # another order -- the statistics, and so the outputs, agree only to rounding
    gamma, beta = (torch.rand(128, generator=g) + 0.5).cuda(), torch.randn(128, generator=g).cuda()
    return ([rnd(g, 2, 128, 10, 13, scale=2.0) + 0.5], (2, 10, 13, 128),
            lambda o, x: ops().groupnorm(x, o, gamma, beta, 16, 1e-5, relu=True),
            lambda x: F.relu(F.group_norm(x, 16, gamma.cpu(), beta.cpu(), 1e-5)), 2e-5, 2e-5)


def case_bfp_gather(g):
    sizes = [(12, 20), (6, 10), (3, 5)]
    return ([rnd(g, 1, 16, h, w) for h, w in sizes], (1, 12, 20, 16), lambda o, *lv: ops().bfp_gather(list(lv), o),
            lambda *lv: sum(F.interpolate(t, size=sizes[0], mode="nearest") for t in lv) / len(lv), 1e-5, None)


def case_bfp_scatter(g):
    return ([rnd(g, 1, 16, 12, 20), rnd(g, 1, 16, 6, 10)], (1, 6, 10, 16), lambda o, bsf, t: ops().bfp_scatter(bsf, t, o),
            lambda bsf, t: F.adaptive_max_pool2d(bsf, (6, 10)) + t, 1e-5, None)


def case_flow_warp(g):
    from oracle import ops as O
    flow = (torch.rand(1, 2, 12, 20, generator=g) - 0.5) * 12
    fd = dense(flow, torch.float32)
    return ([rnd(g, 1, 16, 12, 20)], (1, 12, 20, 16), lambda o, x: ops().flow_warp(x, fd, o),
            lambda x: O.flow_warp(x, flow), 2e-5, None)


def case_resample2d(g):
    from oracle import ops as O
    flow = (torch.rand(1, 2, 12, 20, generator=g) - 0.5) * 30
    fd = dense(flow, torch.float32)
    return ([rnd(g, 1, 16, 12, 20)], (1, 12, 20, 16), lambda o, x: ops().resample2d(x, fd, o),
            lambda x: O.resample2d(x, flow), 1e-5, None)


def case_tcea_temporal(g):
    # a lane sums channels lane*V + 32*V*k, so V changes the order of the embedding dot products: equal to rounding
    def ref(f0, f1, e0, e1, er):
        return torch.cat([f0 * torch.sigmoid((e0 * er).sum(1, keepdim=True)), f1 * torch.sigmoid((e1 * er).sum(1, keepdim=True))], 1)
    return ([rnd(g, 1, 64, 10, 14, scale=0.3) for _ in range(5)], (1, 10, 14, 128),
            lambda o, *t: ops().tcea_temporal(*t, o), ref, 2e-5, 2e-5)


def case_tcea_combine(g):
    return ([rnd(g, 1, 16, 10, 14) for _ in range(3)], (1, 10, 14, 16), lambda o, f, a, d: ops().tcea_combine(f, a, d, o),
            lambda f, a, d: f * torch.sigmoid(a) * 2 + d, 2e-5, None)


def case_roi_align(g):
    from oracle.model import roi_extract
    n = 40
    xy = torch.rand(n, 2, generator=g) * torch.tensor([128.0, 64.0])
    wh = torch.exp(torch.rand(n, 2, generator=g) * 4.5)
    rois = torch.cat([torch.zeros(n, 1), xy - wh / 2, xy + wh / 2], 1)
    rd = rois.cuda()
    feats = [rnd(g, 1, 16, 64 // s, 128 // s) for s in (4, 8, 16, 32)]
    return (feats, (n, 7, 7, 16), lambda o, *f: ops().roi_align(list(f), [4, 8, 16, 32], rd, n, o, 2),
            lambda *f: roi_extract(list(f), rois, 7), 2e-5, None)


CASES = {k[5:]: v for k, v in globals().items() if k.startswith("case_")}


def ops():
    from vps_b200 import ops as _ops
    return _ops


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_vector_and_scalar_arms_agree(cuda, name, dtype):
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    ins, oshape, launch, ref_fn, tol, vs_tol = CASES[name](g)
    ins = [t.to(dtype).float() for t in ins]           # the values both layouts hold
    outs = []
    for layout in (dense, sliced):
        o = out_nhwc(oshape, dtype, layout)
        launch(o, *[layout(t, dtype) for t in ins])
        outs.append(o)
    torch.cuda.synchronize()
    vec, sca = outs
    if vs_tol is None:
        assert torch.equal(bits(vec), bits(sca)), name
    else:
        assert close(nchw(vec), nchw(sca), vs_tol if dtype == torch.float32 else BF16_TOL), name
    ref = ref_fn(*ins)
    assert close(nchw(vec), ref, tol if dtype == torch.float32 else BF16_TOL), name


def test_axpby_mixed_dtypes(cuda):
    g = torch.Generator().manual_seed(11)
    a, b = rnd(g, 1, 16, 9, 13), rnd(g, 1, 16, 9, 13)
    for ti, to, tol in ((torch.float32, torch.bfloat16, BF16_TOL), (torch.bfloat16, torch.float32, 1e-5)):
        ai, bi = a.to(ti).float(), b.to(ti).float()
        o = out_nhwc((1, 9, 13, 16), to, dense)
        ops().axpby(dense(ai, ti), o, 0.75, dense(bi, ti), -1.5)
        torch.cuda.synchronize()
        assert close(nchw(o), 0.75 * ai - 1.5 * bi, tol), (ti, to)


@pytest.mark.parametrize("op", ["resample2d", "flow_warp"])
def test_bf16_flow(cuda, op):
    from oracle import ops as O
    g = torch.Generator().manual_seed(12)
    flow = ((torch.rand(1, 2, 12, 20, generator=g) - 0.5) * 12).bfloat16().float()
    src = rnd(g, 1, 16, 12, 20)
    for dt, tol in ((torch.float32, 2e-5), (torch.bfloat16, BF16_TOL)):
        s = src.to(dt).float()
        o = out_nhwc((1, 12, 20, 16), dt, dense)
        getattr(ops(), op)(dense(s, dt), dense(flow, torch.bfloat16), o)
        torch.cuda.synchronize()
        assert close(nchw(o), getattr(O, op)(s, flow), tol), dt


def test_channelnorm_bf16_out(cuda):
    g = torch.Generator().manual_seed(13)
    a, b = rnd(g, 2, 3, 12, 20), rnd(g, 2, 3, 12, 20)
    o = out_nhwc((2, 12, 20, 1), torch.bfloat16, dense)
    ops().channelnorm(dense(a, torch.float32), o, b=dense(b, torch.float32))
    torch.cuda.synchronize()
    assert close(nchw(o), ((a - b) ** 2).sum(1, keepdim=True).sqrt(), BF16_TOL)


def test_deform_im2col_bf16_offsets(cuda):
    """fp32 data (generic kernel) and bf16 data with 8-channel chunks (the bf16x8 kernel), both with bf16 offsets"""
    from oracle import ops as O
    g = torch.Generator().manual_seed(14)
    C, H, W = 16, 11, 15
    off = (rnd(g, 1, 18, H, W) * 2.5).bfloat16().float()
    x = rnd(g, 1, C, H, W)
    for dt, tol in ((torch.float32, 1e-5), (torch.bfloat16, BF16_TOL)):
        xi = x.to(dt).float()
        cols = out_nhwc((1, H, W, 9 * C), dt, dense)
        ops().deform_im2col(dense(xi, dt), dense(off, torch.bfloat16), cols)
        torch.cuda.synchronize()
        ref = O.deform_im2col(xi, off).view(1, C, 9, H, W).permute(0, 2, 1, 3, 4).reshape(1, 9 * C, H, W)   # tap-major
        assert close(nchw(cols), ref, tol), dt


def test_flow_deconv_dtype_pairs(cuda):
    g = torch.Generator().manual_seed(15)
    x = rnd(g, 1, 2, 6, 9)
    w, b = rnd(g, 2, 2, 4, 4, scale=0.3), rnd(g, 2)
    for ti in (torch.float32, torch.bfloat16):
        for to in (torch.float32, torch.bfloat16):
            xi = x.to(ti).float()
            y = out_nhwc((1, 12, 18, 2), to, dense)
            ops().flow_deconv(dense(xi, ti), w.flatten().tolist(), b.tolist(), y)
            torch.cuda.synchronize()
            ref = F.conv_transpose2d(xi, w, b, stride=2, padding=1)
            assert close(nchw(y), ref, 1e-5 if to == torch.float32 else BF16_TOL), (ti, to)
