"""TMA epilogue of the tc32 convolution (results staged in shared-memory output boxes, residual loaded by TMA, TMA store).
Every case runs twice into a wider concat buffer: once into a 16-byte aligned channel slice, where the plan reports the TMA
epilogue for flat tiles, and once into a slice one channel further, which TMA cannot address, so the same convolution stores from the
accumulator fragments.  The two outputs must be bit-identical, both within the 2e-5 fp64 tolerance of
test_gpu_conv_tc32.py, and the channels around the slice untouched."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = 2e-5
FILL = 3.0


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


def _ref(ops, x, wt, b, s, p, act, res, after, scale):
    v = F.conv2d(x.double(), wt.double(), b.double(), stride=s, padding=p)
    r = None if res is None else res.double()
    if r is not None and not after:
        v = v + r
    if act == ops.ACT_RELU:
        v = v.clamp_min(0)
    elif act == ops.ACT_LRELU:
        v = F.leaky_relu(v, 0.1)
    elif act == ops.ACT_SIGMOID:
        v = torch.sigmoid(v)
    v = v * scale
    if r is not None and after:
        v = v + r
    return v


# n, cin, cout, (H, W) input, k, stride, act, residual (None / "before" / "after" the activation), out_scale, (nwg, halo).
# Flat tiles (1x1, strided) take the TMA epilogue; halo tiles keep the fragment epilogue, so their two runs compare the
# fragment path with itself at two slice offsets.
CASES = [
    (2, 64, 256, (128, 128), 1, 1, "relu", "before", 1.0, (4, 0)),        # R50 conv3 + identity: 512 tiles, 4 per CTA
    (2, 64, 256, (64, 96), 1, 1, "lrelu", "after", 0.5, (4, 0)),
    (1, 64, 48, (40, 56), 1, 1, "lrelu", "after", 1.0, (2, 0)),           # cout 48: block_n 16
    (1, 48, 40, (37, 53), 1, 1, "sigmoid", "before", 0.5, (2, 0)),        # odd output, cout 40: not a multiple of 16
    (1, 32, 64, (130, 98), 3, 2, "sigmoid", None, 2.0, None),             # stride 2: flat, partial tiles
    (2, 32, 40, (37, 53), 3, 1, "sigmoid", "before", 0.5, (2, 1)),        # halo
    (1, 64, 16, (251, 317), 3, 1, "relu", None, 1.0, (4, 1)),             # halo, partial tiles
]


@pytest.mark.parametrize("case", CASES)
def test_tma_epilogue_matches_fragment_path_and_fp64(cuda, tc32, case):
    ops = tc32
    n, cin, cout, (H, W), k, s, act, resk, scale, shape = case
    act = {"relu": ops.ACT_RELU, "lrelu": ops.ACT_LRELU, "sigmoid": ops.ACT_SIGMOID}[act]
    p = k // 2
    g = torch.Generator().manual_seed(cin * 1000 + cout + k)
    x = torch.randn(n, cin, H, W, generator=g)
    wt = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, generator=g)
    oh, ow = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    res = torch.randn(n, cout, oh, ow, generator=g) if resk else None
    ref = _ref(ops, x, wt, b, s, p, act, res, resk == "after", scale)
    pk = ops.PackedConv(wt.to(cuda), b.to(cuda))
    xd = _dev_nhwc(x, cuda)
    rd = _dev_nhwc(res, cuda) if res is not None else None
    ctot = (cout + 8 + 7) // 8 * 8
    outs = []
    for off, epi in ((4, "frag" if shape is not None and shape[1] else "tma"), (1, "frag")):
        buf = torch.full((n, oh, ow, ctot), FILL, dtype=torch.float32, device=cuda)
        y = buf[..., off:off + cout]
        plan = ops.conv2d_tc32_plan(xd, pk, stride=s, pad=p, y=y, res=rd)
        assert plan["epilogue"] == epi, plan
        if shape is not None:
            assert (plan["nwg"], plan["halo"]) == shape, plan
        ops.conv2d(xd, pk, y, stride=s, pad=p, act=act, slope=0.1, res=rd, res_after_act=resk == "after",
                   out_scale=scale, use_tc=True)
        torch.cuda.synchronize()
        got = y.cpu().permute(0, 3, 1, 2).double()
        err = (got - ref).abs().max().item()
        assert err <= TOL * max(1.0, ref.abs().max().item()), "%s: max err %g" % (epi, err)
        assert bool((buf[..., :off] == FILL).all()) and bool((buf[..., off + cout:] == FILL).all()), epi
        outs.append(y)
    assert torch.equal(outs[0], outs[1])


def test_deconv_phases_keep_fragment_epilogue(cuda, tc32):
    """The stride phases of a transposed convolution write every second output pixel: no tensor map expresses that."""
    ops = tc32
    from vps_b200.layers import deconv4x4_s2
    cin, cout, H, W = 64, 32, 48, 80
    g = torch.Generator().manual_seed(5)
    x = torch.randn(1, cin, H, W, generator=g)
    wt = torch.randn(cin, cout, 4, 4, generator=g) / (cin * 4) ** 0.5
    b = torch.randn(cout, generator=g)
    layer = deconv4x4_s2(wt.to(cuda), b.to(cuda))
    xd = _dev_nhwc(x, cuda)
    y = torch.full((1, 2 * H, 2 * W, cout), float("nan"), dtype=torch.float32, device=cuda)
    pws, pads = [ph[3] for ph in layer.phases], [ph[2] for ph in layer.phases]
    omaps = [(2, ph[0], 2, ph[1]) for ph in layer.phases]
    plan = ops.conv2d_tc32_plan(xd, pws, pads=pads, oh=H, ow=W, y=y, omaps=omaps)
    assert plan["epilogue"] == "frag", plan
    layer(xd, y, act=ops.ACT_LRELU)
    torch.cuda.synchronize()
    ref = F.leaky_relu(F.conv_transpose2d(x.double(), wt.double(), b.double(), stride=2, padding=1), 0.1)
    got = y.cpu().permute(0, 3, 1, 2).double()
    assert (got - ref).abs().max().item() <= TOL * max(1.0, ref.abs().max().item())
