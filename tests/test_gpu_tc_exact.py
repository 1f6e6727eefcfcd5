"""The bf16 tensor-core kernels checked bit for bit against exact references.

Operands are small integers ({+-1 .. +-4}, no zeros), so every product and every partial sum is exact in fp32 whatever order
the kernel adds them in and whether or not the tensor core truncates: the correct output is one bit pattern, and any
dropped, duplicated or misplaced K term, wrong pixel, wrong tap or wrong output address changes it.  The contraction is
computed in fp64 on the device, the epilogue in fp32 in the kernels' operation order (epi_math in conv_tc_common.cuh: bias,
residual before the activation, activation, out_scale, residual after the activation), and bf16 outputs are rounded to
nearest even as __float2bfloat16_rn does.

  * vps_conv2d_tc / vps_conv2d_tc_multi over shapes whose plans (ops.conv2d_tc_plan) together cover both modes, both K step
    widths, every N tile width, filter-row weight slots, grouped flat slots with a partial last slot, every ragged last
    chunk, the stride phases of both transposed convolutions and several tiles per CTA, so that the rings wrap across tiles;
    the same operands through the CUDA-core and tc32 kernels (fp32 activations), which must give the same bits.
  * vps_deform_conv_tc with offsets on a 1/4 grid (bilinear weights on a 1/16 grid: every sampled value is exact in bf16),
    samples exactly on and beyond the image edges, against the reference kernel's deformable_im2col (oracle.ops).
  * vps_correlation_tc at both call sites, two images, odd and tiny maps, against the exact channel sum times the kernel's
    fp32 1/C.

Inputs are channel slices whose padding channels hold NaN; outputs are slices of wider buffers whose other channels hold a
sentinel that must survive.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import tc32_model as M

pytestmark = pytest.mark.gpu

SENTINEL = 12288.0          # exact in bf16 as well
SLOPE = 0.1


def _act(ops, name):
    return {"none": ops.ACT_NONE, "relu": ops.ACT_RELU, "lrelu": ops.ACT_LRELU, "sigmoid": ops.ACT_SIGMOID}[name]


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def ints(shape, g, lo=1, hi=4, positive=False):
    """integers of magnitude lo .. hi, random signs unless `positive`, as fp64 on the device"""
    v = torch.randint(lo, hi + 1, shape, generator=g, device="cuda").double()
    if not positive:
        v = v * (torch.randint(0, 2, shape, generator=g, device="cuda").double() * 2 - 1)
    return v


def quarters(shape, g, mag):
    """multiples of 1/4 in [-mag, mag]"""
    return torch.randint(-4 * mag, 4 * mag + 1, shape, generator=g, device="cuda").double() / 4


def nhwc_in(t, dtype):
    """NCHW -> NHWC channel slice of a buffer with at least 8 padding channels, which hold NaN"""
    n, c, h, w = t.shape
    buf = torch.full((n, h, w, (c + 7) // 8 * 8 + 8), float("nan"), dtype=dtype, device="cuda")
    buf[..., :c] = t.permute(0, 2, 3, 1).to(dtype)
    return buf[..., :c]


def slice_out(shape, dtype, vec, fill=SENTINEL):
    """(wide buffer, channel slice, offset) for an NHWC tensor of `shape`: vec 2 = 32-byte aligned slice and pixel stride,
    1 = 16-byte aligned slice, 0 = channel offset 1 (element stores)"""
    n, h, w, c = shape
    esz = torch.tensor([], dtype=dtype).element_size()
    off = {2: 0, 1: 16 // esz, 0: 1}[vec]
    cs = (off + c + 1 + 15) // 16 * 16
    wide = torch.full((n, h, w, cs), fill, dtype=dtype, device="cuda")
    return wide, wide[..., off:off + c], off


def check_sentinel(wide, off, c):
    assert bool((wide[..., :off].float() == SENTINEL).all()), "channels below the slice were written"
    assert bool((wide[..., off + c:].float() == SENTINEL).all()), "channels above the slice were written"


def assert_bits(got, ref, what):
    """got (NHWC, fp32 or bf16) equals the fp32 reference ref (NCHW) rounded to got's dtype, bit for bit"""
    want = ref.permute(0, 2, 3, 1).to(got.dtype).contiguous()
    g = got.contiguous()
    assert not bool(torch.isnan(g.float()).any()), "%s: NaN in the output" % what
    bad = g.view(torch.int16 if g.dtype == torch.bfloat16 else torch.int32) != want.view(
        torch.int16 if want.dtype == torch.bfloat16 else torch.int32)
    nbad = int(bad.sum())
    if nbad:
        idx = bad.nonzero()[:4].tolist()
        pairs = [(i, float(g[tuple(i)]), float(want[tuple(i)])) for i in idx]
        raise AssertionError("%s: %d of %d outputs differ, e.g. [n, y, x, c] got / want %s" % (what, nbad, bad.numel(), pairs))


def epilogue32(s, bias, act, res, after, scale):
    """the kernels' epilogue in fp32 on the exact contraction s (fp64, NCHW): returns the fp32 result"""
    v = s.float()
    if bias is not None:
        v = v + bias.float().view(1, -1, 1, 1)
    if res is not None and not after:
        v = v + res.float()
    if act == "relu":
        v = torch.clamp_min(v, 0.0)
    elif act == "lrelu":
        v = torch.where(v > 0, v, v * torch.tensor(SLOPE, dtype=torch.float32, device=v.device))
    v = v * torch.tensor(scale, dtype=torch.float32, device=v.device)
    if res is not None and after:
        v = v + res.float()
    return v


# ------------------------------------------------------------------------------------------------ convolutions
# name -> (kind, n, cin, cout, (h, w) input, k, stride, pad, variant).  The plan each shape gives on 132 SMs is noted; the
# coverage test checks that the plans together cover the plan space, whichever case lands where.
# variant: act, res ("bf16" / "f32" / None), after (residual after the activation), scale, out dtype, yv / rv (store / load
# width of the output / residual slice, see slice_out), pos (all-positive operands: sums above 2^17).
V = dict(act="none", res=None, after=False, scale=1.0, out="f32", yv=2, rv=2, pos=False)
CONV_CASES = {
    # halo, block_n 256, 4 chunks on a 3-slot A ring, ~7.8 tiles per CTA
    "fpn_3x3_256": ("conv", 1, 256, 256, (256, 512), 3, 1, 1, dict(V, act="relu", res="bf16", out="bf16")),
    # flat, block_n 128, ~3.9 tiles per CTA, two images
    "s2_3x3_128": ("conv", 2, 128, 128, (256, 512), 3, 2, 1, dict(V, act="relu", out="bf16", yv=1)),
    # flat, block_n 256, ~15.5 tiles per CTA
    "1x1_64_256": ("conv", 2, 64, 256, (256, 512), 1, 1, 0, dict(V, res="f32", after=True, scale=0.5)),
    # flat, block_n 128, ~2.9 tiles per CTA
    "1x1_256_512": ("conv", 2, 256, 512, (64, 96), 1, 1, 0, dict(V, act="lrelu", res="bf16", after=True, out="bf16", yv=1, rv=1)),
    # flat, gsub 2, ragged chunk of 63 channels (nk_last 4)
    "1x1_127_128": ("conv", 2, 127, 128, (96, 96), 1, 1, 0, dict(V, act="sigmoid")),
    # halo, bk 16, ~7.8 tiles per CTA; element stores of fp32
    "3x3_11_64": ("conv", 1, 11, 64, (256, 512), 3, 1, 1, dict(V, act="lrelu", res="f32", yv=0, rv=0)),
    # flat, bk 16, gsub 4 with a partial last slot; element stores of bf16
    "7x7s2_12_64": ("conv", 1, 12, 64, (256, 512), 7, 2, 3, dict(V, act="relu", scale=0.5, out="bf16", yv=0)),
    # halo, block_n 32, nk_last 3
    "3x3_162_32": ("conv", 1, 162, 32, (128, 256), 3, 1, 1, dict(V, res="bf16", out="bf16", rv=0)),
    # halo, block_n 64, nk_last 2
    "3x3_473_64": ("conv", 1, 473, 64, (96, 160), 3, 1, 1, dict(V, act="lrelu", scale=0.5, yv=1)),
    # halo, block_n 128, filter-row weight slots (rowg)
    "3x3_128_128": ("conv", 1, 128, 128, (96, 160), 3, 1, 1, dict(V, act="sigmoid", out="bf16")),
    # 4 stride phases of 2x2 taps in halo mode, nk_last 1
    "deconv4x4_386_64": ("deconv", 1, 386, 64, (64, 128), 4, 2, 1, dict(V, act="lrelu", out="bf16", yv=1)),
    # 4 stride phases of one tap in flat mode; element stores into interleaved pixels
    "deconv2x2_256_256": ("deconv", 2, 256, 256, (28, 28), 2, 2, 0, dict(V, act="relu", yv=0)),
    # flat, gsub 2 with a partial last slot, ragged tiles
    "3x3s2_64_128": ("conv", 1, 64, 128, (33, 47), 3, 2, 1, dict(V, act="relu", res="f32", rv=1, yv=1)),
    # block_n 16, nk_last 1, cout 2
    "3x3_1026_2": ("conv", 1, 1026, 2, (8, 16), 3, 1, 1, dict(V, yv=0)),
    # all-positive operands: sums above 2^17; cout 3
    "3x3_2000_3_pos": ("conv", 1, 2000, 3, (8, 16), 3, 1, 1, dict(V, pos=True)),
    # odd cout (the single-channel tail of the last pair), two images, ragged tiles in x and y, residual after the activation
    "3x3_48_47": ("conv", 2, 48, 47, (37, 29), 3, 1, 1, dict(V, act="relu", res="bf16", after=True, out="bf16", yv=0, rv=2)),
    # StemConv7x7s2: space-to-depth of a 3-channel input + the 4x4 bk-16 halo convolution
    "stem_3ch": ("stem", 1, 3, 64, (67, 131), 7, 2, 3, dict(V, act="relu", out="bf16")),
}


def out_hw(name):
    kind, n, cin, cout, (h, w), k, s, p, _ = CONV_CASES[name]
    if kind == "deconv":
        return 2 * h, 2 * w
    return (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1


def build_layer(ops, name, w, b):
    """the packed layer of case `name`: PackedConv, a stride-phase deconvolution or StemConv7x7s2"""
    from vps_b200.layers import StemConv7x7s2, deconv2x2_s2, deconv4x4_s2
    kind, _, _, _, _, k, _, _, v = CONV_CASES[name]
    if kind == "deconv":
        return (deconv4x4_s2 if k == 4 else deconv2x2_s2)(w, b)
    if kind == "stem":
        return StemConv7x7s2(w, b, act=_act(ops, v["act"]))
    return ops.PackedConv(w, b)


def case_plan(ops, name, x, layer, y=None, res=None):
    """(the plan ops.conv2d_tc_plan reports for case `name` on input x, geometry of the launch: nprob, K steps per tile,
    output size)"""
    from vps_b200.layers import empty_nhwc
    kind, n, cin, cout, (h, w), k, s, p, _ = CONV_CASES[name]
    if kind == "deconv":
        pws, pads = [ph[3] for ph in layer.phases], [ph[2] for ph in layer.phases]
        plan = ops.conv2d_tc_plan(x, pws, pads=pads, oh=h, ow=w, y=y, omaps=[(2, ph[0], 2, ph[1]) for ph in layer.phases])
        geo = dict(nprob=4, cin=cin, taps=(k // 2) ** 2, oh=h, ow=w)
    elif kind == "stem":
        oh, ow = out_hw(name)
        xs = empty_nhwc(n, (h + 1) // 2, (w + 1) // 2, 4 * cin, torch.bfloat16, x.device)
        plan = ops.conv2d_tc_plan(xs, layer.s2d.pk, stride=1, pad=2, oh=oh, ow=ow)
        geo = dict(nprob=1, cin=4 * cin, taps=16, oh=oh, ow=ow)
    else:
        plan = ops.conv2d_tc_plan(x, layer, stride=s, pad=p, y=y, res=res)
        oh, ow = out_hw(name)
        geo = dict(nprob=1, cin=cin, taps=k * k, oh=oh, ow=ow)
    geo["steps"] = math.ceil(geo["cin"] / plan["bk"]) * geo["taps"]
    return plan, geo


def conv_operands(name, seed):
    """x (NCHW), w (OIHW, IOHW for a deconvolution), bias, residual (NCHW or None) as fp64 on the device"""
    kind, n, cin, cout, (h, w), k, s, p, v = CONV_CASES[name]
    g = gen(seed)
    x = ints((n, cin, h, w), g, lo=2 if v["pos"] else 1, positive=v["pos"])
    wt = ints((cin, cout, k, k) if kind == "deconv" else (cout, cin, k, k), g, lo=2 if v["pos"] else 1, positive=v["pos"])
    b = quarters((cout,), g, 4)
    oh, ow = out_hw(name)
    res = quarters((n, cout, oh, ow), g, 8) if v["res"] else None
    return x, wt, b, res


def contraction(name, x, wt):
    kind, _, _, _, _, k, s, p, _ = CONV_CASES[name]
    if kind == "deconv":
        return F.conv_transpose2d(x, wt, stride=s, padding=p)
    return F.conv2d(x, wt, stride=s, padding=p)


def conv_reference(name, x, wt, b, res):
    """(exact contraction, fp32 result of the epilogue or None for the sigmoid, and the precondition checked)"""
    v = CONV_CASES[name][-1]
    s = contraction(name, x, wt)
    absprod = contraction(name, x.abs(), wt.abs())
    # bias and residual are quarter-integers: every sum stays exact in fp32 while it is below 2^22
    mag = absprod + b.abs().view(1, -1, 1, 1) + (res.abs() if res is not None else 0)
    assert float(mag.max()) < 2.0 ** 22, "operands too large for an exact test"
    if v["pos"]:
        assert float(s.max()) > 2.0 ** 17, "the all-positive case must exceed 2^17"
    ref = None if v["act"] == "sigmoid" else epilogue32(s, b, v["act"], res, v["after"], v["scale"])
    return s, ref


def check_sigmoid(got, s, b, res, v):
    """the sigmoid goes through __expf: within tc32_model.bound with an exact pre-activation (+ one bf16 rounding)"""
    pre = s + b.view(1, -1, 1, 1) + (res if res is not None and not v["after"] else 0)
    ref = torch.sigmoid(pre) * v["scale"] + (res if res is not None and v["after"] else 0)
    zero = torch.zeros_like(pre)
    e = M.bound(zero, 0.0, 0.0, 0.0, bias=b.view(1, -1, 1, 1), res=res if res is not None else 0.0, out=ref, pre=pre,
                act="sigmoid", res_after_act=v["after"], scale=v["scale"])
    # below t = -88.7 __expf(-t) overflows and the kernel returns 0 for a sigmoid under 2^-127, which fp32 with flushed
    # subnormals could not hold anyway
    e = e + 2.0 ** -126
    if got.dtype == torch.bfloat16:
        e = e + 2.0 ** -8 * ref.abs()
    g = got.permute(0, 3, 1, 2).double()
    assert not bool(torch.isnan(g).any())
    err = (g - ref).abs()
    assert bool((err <= e).all()), "sigmoid: max err %g, worst ratio %g" % (float(err.max()), float((err / e).max()))


def run_conv(ops, name, x_dt, layer, y, res_dt, act, after, scale, use_tc=True):
    kind, n, cin, cout, (h, w), k, s, p, _ = CONV_CASES[name]
    a = _act(ops, act)
    if kind == "deconv":
        layer(x_dt, y, act=a, out_scale=scale)
    elif kind == "stem":
        layer(x_dt, y=y)
    else:
        ops.conv2d(x_dt, layer, y, stride=s, pad=p, act=a, slope=SLOPE, res=res_dt, res_after_act=after, out_scale=scale,
                   use_tc=use_tc)


@pytest.mark.parametrize("name", list(CONV_CASES))
def test_conv_tc_exact(cuda, name):
    """vps_conv2d_tc / vps_conv2d_tc_multi == the exact reference, bit for bit"""
    from vps_b200 import ops
    n, cout, v = CONV_CASES[name][1], CONV_CASES[name][3], CONV_CASES[name][-1]
    x, wt, b, res = conv_operands(name, 1000 + sorted(CONV_CASES).index(name))
    exact, ref = conv_reference(name, x, wt, b, res)
    odt = torch.bfloat16 if v["out"] == "bf16" else torch.float32
    xd = nhwc_in(x, torch.bfloat16)
    rd = None
    if res is not None:
        rdt = torch.bfloat16 if v["res"] == "bf16" else torch.float32
        _, rd, _ = slice_out(res.permute(0, 2, 3, 1).shape, rdt, v["rv"], fill=float("nan"))
        rd.copy_(res.permute(0, 2, 3, 1).to(rdt))
    oh, ow = out_hw(name)
    wide, y, off = slice_out((n, oh, ow, cout), odt, v["yv"])
    layer = build_layer(ops, name, wt.float(), b.float())
    plan, _ = case_plan(ops, name, xd, layer, y=y, res=rd)
    print(name, plan)
    run_conv(ops, name, xd, layer, y, rd, v["act"], v["after"], v["scale"])
    torch.cuda.synchronize()
    check_sentinel(wide, off, cout)
    if ref is None:
        check_sigmoid(y, exact, b, res, v)
    else:
        assert_bits(y, ref, "%s %s" % (name, plan))


@pytest.mark.parametrize("name", [nm for nm, c in CONV_CASES.items() if c[0] == "conv" and c[-1]["act"] != "sigmoid"])
@pytest.mark.parametrize("impl", ["simt", "tc32"])
def test_conv_fp32_kernels_exact(cuda, name, impl):
    """the CUDA-core kernel and the tc32 kernel on the same integer operands as fp32 activations: integers up to 2^11
    split into an fp16 main plane and a zero correction, so both give the exact reference's bits as well"""
    from vps_b200 import ops
    n, cout, v = CONV_CASES[name][1], CONV_CASES[name][3], CONV_CASES[name][-1]
    x, wt, b, res = conv_operands(name, 1000 + sorted(CONV_CASES).index(name))
    _, ref = conv_reference(name, x, wt, b, res)
    xd = nhwc_in(x, torch.float32)
    rd = None
    if res is not None:
        rdt = torch.bfloat16 if v["res"] == "bf16" else torch.float32
        _, rd, _ = slice_out(res.permute(0, 2, 3, 1).shape, rdt, v["rv"], fill=float("nan"))
        rd.copy_(res.permute(0, 2, 3, 1).to(rdt))
    oh, ow = out_hw(name)
    wide, y, off = slice_out((n, oh, ow, cout), torch.float32, v["yv"])
    layer = ops.PackedConv(wt.float(), b.float())
    ops.tc32_overflow()
    run_conv(ops, name, xd, layer, y, rd, v["act"], v["after"], v["scale"], use_tc=impl == "tc32")
    torch.cuda.synchronize()
    assert ops.tc32_overflow() == 0
    check_sentinel(wide, off, cout)
    assert_bits(y, ref, "%s %s" % (impl, name))


def plan_features(name, plan, geo, sms):
    """the coverage items one case's plan contributes"""
    n = CONV_CASES[name][1]
    mode = "halo" if plan["halo"] else "flat"
    per_cta = plan["total_tiles"] / min(plan["total_tiles"], sms)
    chunks = math.ceil(geo["cin"] / plan["bk"])
    f = {(mode, "bk", plan["bk"]), ("block_n", plan["block_n"]), (mode, "block_n", plan["block_n"]),
         ("nprob", geo["nprob"], mode), ("gsub", plan["gsub"])}
    if plan["halo"]:
        f.add(("rowg", plan["rowg"]))
    else:
        f.add(("rowg", 0))
        if geo["steps"] % plan["gsub"]:
            f.add(("gsub_partial", plan["gsub"]))
    if plan["bk"] == 64:
        f.add(("nk_last", math.ceil((geo["cin"] - (chunks - 1) * 64) / 16)))
    if per_cta >= 3:
        f.add((mode, "wrap"))
        if plan["halo"] and chunks % plan["a_stages"]:
            f.add(("halo", "wrap_mid_tile"))
    if n == 2:
        f.add(("batch", 2))
    if geo["ow"] % plan["tw"]:
        f.add(("ragged", "x"))
    if geo["oh"] % plan["th"]:
        f.add(("ragged", "y"))
    return f


COVERAGE = ({(m, "bk", bk) for m in ("halo", "flat") for bk in (16, 64)}
            | {("block_n", bn) for bn in (16, 32, 64, 128, 256)}
            | {(m, "block_n", bn) for m in ("halo", "flat") for bn in (128, 256)}
            | {("rowg", 0), ("rowg", 1), ("gsub", 1), ("gsub", 2), ("gsub", 4), ("gsub_partial", 2), ("gsub_partial", 4)}
            | {("nk_last", k) for k in (1, 2, 3, 4)}
            | {("nprob", 1, "halo"), ("nprob", 1, "flat"), ("nprob", 4, "halo"), ("nprob", 4, "flat")}
            | {("halo", "wrap"), ("flat", "wrap"), ("halo", "wrap_mid_tile")}
            | {("batch", 2), ("ragged", "x"), ("ragged", "y")})


def test_conv_tc_plan_coverage(cuda):
    """the plans of the exact cases cover the bf16 convolution's plan space (the shapes are chosen for 132 SMs)"""
    from vps_b200 import ops
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if sms != 132:
        pytest.skip("the case shapes are chosen for 132 SMs, this device has %d" % sms)
    seen = set()
    for name, (kind, n, cin, cout, (h, w), k, s, p, v) in CONV_CASES.items():
        x = torch.empty(n, h, w, (cin + 7) // 8 * 8, dtype=torch.bfloat16, device="cuda")[..., :cin]
        wshape = (cin, cout, k, k) if kind == "deconv" else (cout, cin, k, k)
        layer = build_layer(ops, name, torch.zeros(wshape, device="cuda"), None)
        plan, geo = case_plan(ops, name, x, layer)
        seen |= plan_features(name, plan, geo, sms)
    missing = COVERAGE - seen
    assert not missing, "plan items no case reaches: %s" % sorted(missing, key=str)


# ------------------------------------------------------------------------------------------------ fused DCN
# n, C, cout, H, W, output dtype, output slice (yv), all-positive
DCN_CASES = [
    (1, 64, 48, 19, 37, torch.float32, 0, False),       # block_n 64: weight rows 48 .. 63 are TMA zero fill
    (2, 128, 192, 12, 20, torch.bfloat16, 1, False),    # two N tiles of 128, channels 192 .. 255 do not exist
    (1, 256, 256, 16, 24, torch.float32, 2, True),      # all-positive: sums above 2^17
    (2, 256, 256, 96, 160, torch.bfloat16, 2, False),   # ~3.6 tiles per CTA: the set-up table is rewritten between tiles
]


def dcn_offsets(n, H, W, g):
    """(dy, dx) per tap on a 1/4 grid in [-3.5, 3.5]; about one sample in six is moved exactly onto an image edge
    (-1, H - 1, H - 0.75) or wholly outside, independently in y and in x"""
    off = torch.randint(-14, 15, (n, 18, H, W), generator=g, device="cuda").double() / 4
    yo = torch.arange(H, device="cuda").double().view(1, 1, H, 1)
    xo = torch.arange(W, device="cuda").double().view(1, 1, 1, W)
    k = torch.arange(9, device="cuda").double().view(1, 9, 1, 1)
    base_h, base_w = yo - 1 + torch.div(k, 3, rounding_mode="floor"), xo - 1 + torch.remainder(k, 3)
    for comp, base, size in ((0, base_h, H), (1, base_w, W)):
        targets = torch.tensor([-1.0, -0.75, size - 1.0, size - 1.5, size - 0.75, float(size), -2.0, size + 0.25],
                               device="cuda").double()
        pick = targets[torch.randint(0, len(targets), (n, 9, H, W), generator=g, device="cuda")]
        hit = torch.rand((n, 9, H, W), generator=g, device="cuda") < 1.0 / 6
        off[:, comp::2] = torch.where(hit, pick - base, off[:, comp::2])
    return off


@pytest.mark.parametrize("case", DCN_CASES, ids=["n%d_C%d_cout%d_%dx%d" % c[:5] for c in DCN_CASES])
def test_deform_conv_tc_exact(cuda, case):
    """vps_deform_conv_tc == the reference kernel's columns (oracle.ops.deform_im2col) times the weights, bit for bit"""
    from oracle import ops as O
    from vps_b200 import ops
    n, C, cout, H, W, odt, yv, pos = case
    g = gen(2000 + DCN_CASES.index(case))
    x = ints((n, C, H, W), g, positive=pos)
    w = ints((cout, C, 3, 3), g, lo=48, hi=64, positive=True) if pos else ints((cout, C, 3, 3), g)
    off = dcn_offsets(n, H, W, g)
    cols = O.deform_im2col(x.float().cpu(), off.float().cpu()).to("cuda")
    assert torch.equal(cols.bfloat16().float(), cols), "sampled columns are not exact in bf16"
    cols = cols.double().view(n, C * 9, H * W)
    s = (w.view(cout, C * 9) @ cols).view(n, cout, H, W)
    absprod = (w.abs().view(cout, C * 9) @ cols.abs()).view(n, cout, H, W)
    # products lie on the 1/16 grid: sums are exact in fp32 below 2^20
    assert float(absprod.max()) < 2.0 ** 20
    if pos:
        assert float(s.max()) > 2.0 ** 17
    wide, y, yoff = slice_out((n, H, W, cout), odt, yv)
    ops.deform_conv_tc(nhwc_in(x, torch.bfloat16), off.float().permute(0, 2, 3, 1).contiguous(),
                       ops.PackedConv(w.float(), None), y)
    torch.cuda.synchronize()
    check_sentinel(wide, yoff, cout)
    assert_bits(y, s.float(), "dcn %s" % (case,))


# ------------------------------------------------------------------------------------------------ correlation
# max displacement (= pad), stride2, C, n, H, W, output dtype, output slice offset, activation, all-positive
CORR_CASES = [
    (20, 2, 64, 2, 37, 53, torch.float32, 8, "lrelu", False),
    (4, 1, 128, 2, 3, 5, torch.bfloat16, 1, "none", False),        # smaller than one tile
    (20, 2, 256, 1, 128, 256, torch.bfloat16, 8, "lrelu", False),  # 352 tiles: more than one per CTA
    (4, 1, 192, 2, 21, 50, torch.float32, 1, "lrelu", False),
    (20, 2, 192, 1, 9, 11, torch.bfloat16, 8, "none", False),
    (4, 1, 256, 2, 33, 31, torch.float32, 8, "none", True),        # all-positive: sums above 2^17
    (4, 1, 64, 2, 64, 96, torch.bfloat16, 1, "lrelu", False),
    (20, 2, 128, 2, 17, 23, torch.float32, 1, "none", False),
]


def corr_sum(f1, f2, md, s2):
    """sum_c f1[y, x] * f2[y + tj s2, x + ti s2] (zero outside), channel (tj + R) D + (ti + R); fp64 NCHW"""
    R = md // s2
    D = 2 * R + 1
    n, C, H, W = f1.shape
    p2 = F.pad(f2, (md,) * 4)
    out = f1.new_zeros(n, D * D, H, W)
    for tj in range(-R, R + 1):
        for ti in range(-R, R + 1):
            y0, x0 = md + tj * s2, md + ti * s2
            out[:, (tj + R) * D + ti + R] = (f1 * p2[:, :, y0:y0 + H, x0:x0 + W]).sum(1)
    return out


@pytest.mark.parametrize("case", CORR_CASES, ids=["d%d_s%d_C%d_n%d_%dx%d" % c[:6] for c in CORR_CASES])
def test_correlation_tc_exact(cuda, case):
    """vps_correlation_tc on bf16 features == the exact channel sum times fp32 1/C, then the activation, as the kernel
    computes it (corr_consumer)"""
    from oracle import ops as O
    from vps_b200 import ops
    md, s2, C, n, H, W, odt, off, act, pos = case
    g = gen(3000 + CORR_CASES.index(case))
    f1 = ints((n, C, H, W), g, lo=32 if pos else 1, hi=64 if pos else 4, positive=pos)
    f2 = ints((n, C, H, W), g, lo=32 if pos else 1, hi=64 if pos else 4, positive=pos)
    s = corr_sum(f1, f2, md, s2)
    assert float(corr_sum(f1.abs(), f2.abs(), md, s2).max()) < 2.0 ** 24
    if pos:
        assert float(s.max()) > 2.0 ** 17
    inv_c = torch.tensor(np.float32(1) / np.float32(C), device="cuda")       # the kernel's scale: 1.0f / (float)C
    ref = s.float() * inv_c
    if C & (C - 1) == 0:
        # a power of two: the reciprocal is exact, and the result is the reference's sum / C bit for bit.  For C = 192 (not
        # a production width) the kernel's reciprocal multiply may differ from that division by one rounding; the test pins
        # the kernel's arithmetic there.
        assert torch.equal(ref, O.correlation(f1.float(), f2.float(), md, 1, md, 1, s2))
    if act == "lrelu":
        ref = torch.where(ref > 0, ref, ref * torch.tensor(SLOPE, dtype=torch.float32, device="cuda"))
    D2 = (2 * (md // s2) + 1) ** 2
    cs = (off + D2 + 1 + 15) // 16 * 16
    wide = torch.full((n, H, W, cs), SENTINEL, dtype=odt, device="cuda")
    out = wide[..., off:off + D2]
    ops.correlation(nhwc_in(f1, torch.bfloat16), nhwc_in(f2, torch.bfloat16), out, md, md, 1, s2, act=_act(ops, act),
                    slope=SLOPE, impl="tc")
    torch.cuda.synchronize()
    check_sentinel(wide, off, D2)
    assert_bits(out, ref, "correlation %s" % (case,))
