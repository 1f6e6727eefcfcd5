"""The tc32 tensor-core kernels against their documented error model (tests/tc32_model.py), element by element:

  * K-position probes: one-hot weights, so every output is one product of fat operands (tc32_model.fat) and must be within
    2^-20 of it; a wrong tap shift, a swizzled channel or a lost correction product is off by 2^-14 or more.  The probes of
    each plan kind together cover every tap, every 32-channel chunk, every channel residue mod 32 (each converter task and
    swizzle position), both K16 halves and the first and last channel of a ragged last chunk.
  * The componentwise bound on dense data with per-channel scales (folded-BN-like weights 2^-12 .. 2^6, activations
    2^-6 .. 2^6), bias, activations and residuals.
  * Dynamic range: bit-exact power-of-two equivariance, tiny operands through the 2^-36 floor, large ones below 2^15.
  * The saturation counter at each of its counting sites, and its reset.
  * NaN in the padding channels of every padded operand changes nothing.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from tests import tc32_model as M

pytestmark = pytest.mark.gpu

ACTS = ("none", "relu", "lrelu", "sigmoid")
SENTINEL = 12288.0          # exact in bf16 as well


@pytest.fixture()
def tc32(cuda):
    from vps_b200 import ops
    old = ops.F32_TC[0]
    ops.F32_TC[0] = True
    yield ops
    ops.F32_TC[0] = old


@pytest.fixture()
def unsaturated(tc32):
    """the counter starts at zero and no test but the saturation tests may leave it set"""
    tc32.tc32_overflow()
    yield tc32
    torch.cuda.synchronize()
    assert tc32.tc32_overflow() == 0


def _act(ops, name):
    return {"none": ops.ACT_NONE, "relu": ops.ACT_RELU, "lrelu": ops.ACT_LRELU, "sigmoid": ops.ACT_SIGMOID}[name]


def dev_nhwc(t, fill=0.0, extra=0, dtype=torch.float32, c_align=8):
    """NCHW tensor -> NHWC device channel slice of a buffer whose pixel stride is padded (empty_nhwc's rounding, plus
    `extra` channels) and whose padding channels hold `fill`"""
    n, c, h, w = t.shape
    cs = (c + c_align - 1) // c_align * c_align + extra
    buf = torch.full((n, h, w, cs), fill, dtype=dtype, device="cuda")
    buf[..., :c] = t.permute(0, 2, 3, 1).to(device="cuda", dtype=dtype)
    return buf[..., :c]


def nchw(y):
    return y.permute(0, 3, 1, 2).double()


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ------------------------------------------------------------------------------------------------ the plan set
# name -> kind, n, cin, cout, (h, w), k, stride, pad, expected plan.  The shapes give each plan on the H100's 132 SMs.
CASES = {
    "halo_nwg2_bn128": ("conv", 1, 473, 256, (16, 320), 3, 1, 1, dict(nwg=2, block_n=128, halo=1)),
    "halo_nwg4": ("conv", 1, 82, 16, (256, 512), 3, 1, 1, dict(nwg=4, halo=1)),
    "flat_1x1_tma_nwg4": ("conv", 2, 64, 256, (128, 128), 1, 1, 0, dict(nwg=4, halo=0, epilogue="tma")),
    "flat_3x3_s2": ("conv", 1, 48, 64, (40, 56), 3, 2, 1, dict(halo=0)),
    "flat_5x5_s2": ("conv", 1, 128, 128, (24, 28), 5, 2, 2, dict(halo=0)),
    "flat_7x7_s2_cin12": ("conv", 1, 12, 64, (32, 64), 7, 2, 3, dict(halo=0)),
    "stem_s2d_4x4": ("stem", 1, 12, 64, (32, 64), 7, 2, 3, dict(halo=1)),
    "deconv4x4_s2": ("deconv", 1, 128, 64, (12, 20), 4, 2, 1, dict(halo=1)),
    "deconv2x2_s2": ("deconv", 1, 128, 64, (12, 20), 2, 2, 0, dict(halo=0)),
    "thin_tap_major": ("thin", 1, 194, 2, (24, 40), 3, 1, 1, dict(halo=0)),
}


def ntaps_of(kind, k):
    return k * k


def steps_of(kind, cin, k):
    """K steps of the kernel behind one output element (the thin layer: its 1x1's steps per tap, plus the gather's 9
    round-to-nearest adds, bounded by the 3x3 implicit GEMM's count)"""
    if kind == "deconv":
        return M.steps(cin, (k // 2) ** 2)
    if kind == "stem":
        return M.steps(4 * cin, 16)
    return M.steps(cin, k * k)


def lin(kind, x, w, k, s, p):
    """the contraction of the layer in fp64 (x NCHW, w OIHW or, for a deconvolution, IOHW)"""
    if kind == "deconv":
        return F.conv_transpose2d(x, w, stride=s, padding=p)
    return F.conv2d(x, w, stride=s, padding=p)


def weights_like(kind, cin, cout, k):
    return (cin, cout, k, k) if kind == "deconv" else (cout, cin, k, k)


def run_layer(ops, name, x, w, b=None, act="none", res=None, after=False, scale=1.0, check_plan=True, y=None, want=None):
    """run case `name` on device tensors x (NHWC slice), w (layout as lin()), b; returns the NHWC output"""
    from vps_b200.layers import Conv, StemConv7x7s2, deconv2x2_s2, deconv4x4_s2, empty_nhwc
    kind, n, cin, cout, _, k, s, p, case_want = CASES[name]
    want = case_want if want is None else want
    h, wd = x.shape[1:3]
    a = _act(ops, act)
    if kind == "conv":
        oh, ow = (h + 2 * p - k) // s + 1, (wd + 2 * p - k) // s + 1
        y = y if y is not None else torch.full((n, oh, ow, cout), float("nan"), device="cuda")
        pk = ops.PackedConv(w, b)
        plan = ops.conv2d_tc32_plan(x, pk, stride=s, pad=p, y=y, res=res)
        ops.conv2d(x, pk, y, stride=s, pad=p, act=a, slope=0.1, res=res, res_after_act=after, out_scale=scale, use_tc=True)
    elif kind == "deconv":
        layer = (deconv4x4_s2 if k == 4 else deconv2x2_s2)(w, b)
        y = y if y is not None else torch.full((n, 2 * h, 2 * wd, cout), float("nan"), device="cuda")
        pws, pads = [ph[3] for ph in layer.phases], [ph[2] for ph in layer.phases]
        plan = ops.conv2d_tc32_plan(x, pws, pads=pads, oh=h, ow=wd, y=y, omaps=[(2, ph[0], 2, ph[1]) for ph in layer.phases])
        layer(x, y, act=a, out_scale=scale)
    elif kind == "stem":
        stem = StemConv7x7s2(w, b, act=a)
        oh, ow = (h - 1) // 2 + 1, (wd - 1) // 2 + 1
        xs = empty_nhwc(n, (h + 1) // 2, (wd + 1) // 2, 4 * cin, torch.float32, x.device)
        ops.space_to_depth2(x, xs)
        plan = ops.conv2d_tc32_plan(xs, stem.s2d.pk, stride=1, pad=2, oh=oh, ow=ow)
        y = stem(x, y=y)
    else:
        layer = Conv(w, b, stride=1, pad=1, act=a)
        assert layer.pk_tap is not None
        y = y if y is not None else torch.full((n, h, wd, cout), float("nan"), device="cuda")
        plan = ops.conv2d_tc32_plan(x, layer.pk_tap)
        layer.pk_tap.tc32()                          # packs the weights
        n0 = ops.launch_count()
        layer(x, y, out_scale=scale)
        assert ops.launch_count() - n0 == 2          # the tap-major 1x1 tensor-core GEMM + the gather
    if check_plan:
        assert {key: plan[key] for key in want} == want, (name, plan)
    return y


def epilogue(v, b, act, res, after, scale):
    """fp64 epilogue of the kernels: returns (out, pre-activation)"""
    pre = v if b is None else v + b.view(1, -1, 1, 1)
    if res is not None and not after:
        pre = pre + res
    t = {"none": lambda u: u, "relu": lambda u: u.clamp_min(0), "lrelu": lambda u: F.leaky_relu(u, 0.1),
         "sigmoid": torch.sigmoid}[act](pre)
    out = t * scale
    if res is not None and after:
        out = out + res
    return out, pre


# ------------------------------------------------------------------------------------------------ part 1: probes
def probe_list(cin, ntaps):
    """(ci, tap) probes that together cover every tap, chunk, residue mod 32, K16 half and the edges of a ragged last
    chunk: the last chunk's first and last channel, then residue k in chunk k mod nch (chunk 0 where that channel does
    not exist), taps round-robin"""
    nch = math.ceil(cin / M.STEP_K)
    cis = [(nch - 1) * M.STEP_K, cin - 1]
    for kk in range(max(M.STEP_K, nch)):
        r, ch = kk % M.STEP_K, kk % nch
        ci = ch * M.STEP_K + r
        if ci >= cin:
            ci = r
        if ci < cin:
            cis.append(ci)
    count = max(len(cis), ntaps)
    return [(cis[j % len(cis)], j % ntaps) for j in range(count)]


def coverage(probes, cin, ntaps):
    got = dict(taps=set(), chunks=set(), residues=set(), halves=set(), ragged_edges=set())
    nch = math.ceil(cin / M.STEP_K)
    edges = {(nch - 1) * M.STEP_K, cin - 1} if cin % M.STEP_K else set()
    for ci, t in probes:
        got["taps"].add(t)
        got["chunks"].add(ci // M.STEP_K)
        got["residues"].add(ci % M.STEP_K)
        got["halves"].add(ci % M.STEP_K // M.SLAB)
        if ci in edges:
            got["ragged_edges"].add(ci)
    want = dict(taps=set(range(ntaps)), chunks=set(range(nch)), residues=set(range(min(cin, M.STEP_K))),
                halves=set(range(min(2, math.ceil(min(cin, M.STEP_K) / M.SLAB)))), ragged_edges=edges)
    return got, want


def probe_launches(probes, cout):
    return [probes[i:i + cout] for i in range(0, len(probes), cout)]


def check_probe(got, ref, extra=0.0):
    """per element: |got - ref| <= 2^-20 |ref| (+ extra)"""
    err = (got - ref).abs()
    lim = 2.0 ** -20 * ref.abs() + extra
    bad = ~(err <= lim)
    assert not bool(bad.any()), "probe: %d elements off, worst err / |ref| %g" % (
        int(bad.sum()), float((err / ref.abs().clamp_min(1e-300))[bad].max()))
    return float((err / lim.clamp_min(1e-300)).max())


def one_hot(kind, cin, cout, k, probes, wvals):
    w = torch.zeros(weights_like(kind, cin, cout, k), dtype=torch.float32, device="cuda")
    for co, (ci, t) in enumerate(probes):
        r, s = divmod(t, k)
        if kind == "deconv":
            w[ci, co, r, s] = wvals[co]
        else:
            w[co, ci, r, s] = wvals[co]
    return w


@pytest.mark.parametrize("name", sorted(CASES))
def test_probes_conv(unsaturated, name):
    ops = unsaturated
    kind, n, cin, cout, (h, wd), k, s, p, _ = CASES[name]
    g = gen(sum(map(ord, name)))
    x = M.fat((n, cin, h, wd), g)
    xd = dev_nhwc(x)
    probes = probe_list(cin, ntaps_of(kind, k))
    if kind == "stem":      # all 12 x 49 (channel, tap) pairs: every K position of the 4x4 space-to-depth form
        probes = [(ci, t) for t in range(49) for ci in range(cin)]
    got_cov, want_cov = coverage(probes, cin, ntaps_of(kind, k))
    assert got_cov == want_cov, (name, got_cov, want_cov)
    worst = 0.0
    launches = probe_launches(probes, cout)
    for i, pr in enumerate(launches):
        wv = M.fat((cout,), g)
        w = one_hot(kind, cin, cout, k, pr, wv)
        y = run_layer(ops, name, xd, w, check_plan=i == 0)
        ref = lin(kind, x.double(), w.double(), k, s, p)
        torch.cuda.synchronize()
        worst = max(worst, check_probe(nchw(y)[:, :len(pr)], ref[:, :len(pr)]))
    print("%s: %d probes in %d launches, worst err / probe bound %.3f" % (name, len(probes), len(launches), worst))


# DCN layouts (their plans on 132 SMs): split-M, split-N with one N tile, split-N over several N tiles
DCN_CASES = {
    "split_m": ((1, 64, 64, 96, 128), dict(layout="split_m", n_tiles=1)),
    "split_n": ((1, 64, 128, 64, 96), dict(layout="split_n", n_tiles=1)),
    "multi_n": ((1, 64, 128, 24, 40), dict(layout="split_n", n_tiles=4)),
}


def dcn_offsets(g, n, h, w, integer=False):
    off = torch.randn(n, 18, h, w, generator=g, device="cuda") * 3.0
    off[:, :, 0, :] -= 4.0                     # some samples fall outside the image
    return off.round() if integer else off


def dcn_cols(x, off):
    """the oracle's deform_im2col: fp32 samples [n, C, 9, h, w] as float64, and the same with |x| (the corner terms' size)"""
    from oracle import ops as O
    n, c, h, w = x.shape
    xc, oc = x.cpu(), off.cpu()
    cols = O.deform_im2col(xc, oc).view(n, c, 9, h, w)
    acols = O.deform_im2col(xc.abs(), oc).view(n, c, 9, h, w)
    return cols.double().cuda(), acols.double().cuda()


def run_dcn(ops, x, off, w, want=None, y=None):
    xd, od = dev_nhwc(x), dev_nhwc(off, extra=0)
    return run_dcn_dev(ops, xd, od, w, want, y)


def run_dcn_dev(ops, xd, od, w, want=None, y=None):
    pk = ops.PackedConv(w, None)
    if want is not None:
        plan = ops.deform_conv_tc32_plan(xd, pk)
        assert {key: plan[key] for key in want} == want, plan
    n, h, wd, _ = xd.shape
    y = y if y is not None else torch.full((n, h, wd, pk.cout), float("nan"), device="cuda")
    ops.deform_conv_tc32(xd, od, pk, y)
    return y


@pytest.mark.parametrize("name", sorted(DCN_CASES))
def test_probes_dcn(unsaturated, name):
    """one product of a weight and an fp32 bilinear sample per output; the sample is the oracle's, which the kernel's need
    not match to the bit: both sum four corner terms in fp32 (4 fused and 7 separate roundings), 11 * 2^-24 of their size"""
    ops = unsaturated
    (n, cin, cout, h, wd), want = DCN_CASES[name]
    g = gen(31 + cout)
    x = M.fat((n, cin, h, wd), g)
    off = dcn_offsets(g, n, h, wd)
    cols, acols = dcn_cols(x, off)
    probes = probe_list(cin, 9)
    got_cov, want_cov = coverage(probes, cin, 9)
    assert got_cov == want_cov, got_cov
    worst = 0.0
    for i, pr in enumerate(probe_launches(probes, cout)):
        wv = M.fat((cout,), g)
        w = one_hot("conv", cin, cout, 3, pr, wv)
        y = run_dcn(ops, x, off, w, want if i == 0 else None)
        ci = torch.tensor([c for c, _ in pr], device="cuda")
        tp = torch.tensor([t for _, t in pr], device="cuda")
        wv64 = wv[:len(pr)].double().view(1, -1, 1, 1)
        ref = wv64 * cols[:, ci, tp]
        extra = 11 * 2.0 ** -24 * wv64.abs() * acols[:, ci, tp] + 2.0 ** -36 * wv64.abs()
        torch.cuda.synchronize()
        worst = max(worst, check_probe(nchw(y)[:, :len(pr)], ref, extra))
    print("dcn %s: worst err / probe bound %.3f" % (name, worst))


CORR_CASES = [(20, 2, 64, 24, 40), (4, 1, 256, 20, 24)]      # max_disp, stride2, C, H, W


def corr_ref(f1, f2, md, s2):
    """fp64 correlation on the device: out[n, (tj + R) D + ti + R, y, x] = sum_c f1[y, x] f2[y + tj s2, x + ti s2] / C"""
    n, c, h, w = f1.shape
    R = md // s2
    D = 2 * R + 1
    p2 = F.pad(f2, (md, md, md, md))
    out = torch.empty(n, D * D, h, w, dtype=f1.dtype, device=f1.device)
    for tj in range(-R, R + 1):
        for ti in range(-R, R + 1):
            y0, x0 = md + tj * s2, md + ti * s2
            out[:, (tj + R) * D + ti + R] = (f1 * p2[:, :, y0:y0 + h, x0:x0 + w]).sum(1) / c
    return out


def run_corr(ops, f1d, f2d, md, s2, act="none", impl="tc32", out=None):
    D = 2 * (md // s2) + 1
    n, h, w, _ = f1d.shape
    out = out if out is not None else torch.full((n, h, w, D * D), float("nan"), device="cuda")
    ops.correlation(f1d, f2d, out, md, md, 1, s2, act=_act(ops, act), slope=0.1, impl=impl)
    return out


@pytest.mark.parametrize("cfg", CORR_CASES)
def test_probes_correlation(unsaturated, cfg):
    """f1 is non-zero in one channel per pixel, the channel running over all C: every output is one product / C"""
    ops = unsaturated
    md, s2, C, H, W = cfg
    g = gen(41 + C)
    f2 = M.fat((1, C, H, W), g)
    f1 = torch.zeros(1, C, H, W, device="cuda")
    ch = torch.arange(H * W, device="cuda") % C
    assert set(ch.tolist()) == set(range(C))
    f1.view(C, H * W)[ch, torch.arange(H * W, device="cuda")] = M.fat((H * W,), g)
    out = run_corr(ops, dev_nhwc(f1), dev_nhwc(f2), md, s2)
    ref = corr_ref(f1.double(), f2.double(), md, s2)
    torch.cuda.synchronize()
    print("correlation d%d s%d C%d: worst err / probe bound %.3f" % (md, s2, C, check_probe(nchw(out), ref)))


# ------------------------------------------------------------------------------------------------ part 2: dense bound
# per case: activation, residual (None / "before" / "after"), out_scale
DENSE_EPI = {
    "halo_nwg2_bn128": ("sigmoid", "before", 1.0),
    "halo_nwg4": ("lrelu", None, 1.0),
    "flat_1x1_tma_nwg4": ("relu", "before", 1.0),
    "flat_3x3_s2": ("lrelu", "after", 0.5),
    "flat_5x5_s2": ("sigmoid", "after", 1.0),
    "flat_7x7_s2_cin12": ("relu", None, 1.0),
    "stem_s2d_4x4": ("relu", None, 1.0),
    "deconv4x4_s2": ("lrelu", None, 0.5),
    "deconv2x2_s2": ("sigmoid", None, 1.0),
    "thin_tap_major": ("lrelu", None, 0.5),
}


def dense_conv_data(name, g, xscale=None):
    kind, n, cin, cout, (h, wd), k, s, p, _ = CASES[name]
    xs = M.pow2_scales(cin, -6, 6, g) if xscale is None else torch.full((cin,), xscale, dtype=torch.float64, device="cuda")
    ws = M.pow2_scales(cout, -12, 6, g)
    x = (M.fat((n, cin, h, wd), g).double() * xs.view(1, -1, 1, 1)).float()
    wshape = weights_like(kind, cin, cout, k)
    wsv = ws.view(1, -1, 1, 1) if kind == "deconv" else ws.view(-1, 1, 1, 1)
    w = (M.fat(wshape, g).double() * wsv).float()
    b = (M.fat((cout,), g).double() * ws * 4).float()
    return x, w, b, ws


def dense_bound(name, x, w, b, act, res, after, scale):
    """(ref, bound) of case `name` in fp64 on the device"""
    kind, n, cin, cout, _, k, s, p, _ = CASES[name]
    x64, w64 = x.double(), w.double()
    ref, pre = epilogue(lin(kind, x64, w64, k, s, p), None if b is None else b.double(), act, res, after, scale)
    absprod = lin(kind, x64.abs(), w64.abs(), k, s, p)
    sum_w = w64.abs().sum((0, 2, 3) if kind == "deconv" else (1, 2, 3)).view(1, -1, 1, 1)
    ones = torch.ones((cin, 1, k, k) if kind == "deconv" else (1, cin, k, k), dtype=torch.float64, device="cuda")
    sum_x = lin(kind, x64.abs(), ones, k, s, p)
    bb = 0.0 if b is None else b.double().view(1, -1, 1, 1)
    bnd = M.bound(absprod, sum_w, sum_x, M.gamma(steps_of(kind, cin, k)), bias=bb, res=0.0 if res is None else res,
                  out=ref, pre=pre, act=act, res_after_act=after, scale=scale)
    return ref, bnd


def check_bound(got, ref, bnd, label):
    err = (got - ref).abs()
    ratio = err / bnd
    bad = ~(err <= bnd)
    assert not bool(bad.any()), "%s: %d of %d elements outside the bound, worst err / bound %g" % (
        label, int(bad.sum()), bad.numel(), float(ratio[bad].max()))
    r = float(ratio.max())
    print("%s: worst err / bound %.4f" % (label, r))
    return r


@pytest.mark.parametrize("name", sorted(CASES))
def test_dense_componentwise_bound(unsaturated, name):
    ops = unsaturated
    kind, n, cin, cout, (h, wd), k, s, p, _ = CASES[name]
    act, resk, scale = DENSE_EPI[name]
    g = gen(7 + cin + cout)
    x, w, b, ws = dense_conv_data(name, g)
    oh, ow = ((2 * h, 2 * wd) if kind == "deconv" else ((h + 2 * p - k) // s + 1, (wd + 2 * p - k) // s + 1))
    res = (M.fat((n, cout, oh, ow), g).double() * ws.view(1, -1, 1, 1) * 8).float() if resk else None
    y = run_layer(ops, name, dev_nhwc(x), w, b, act=act, res=dev_nhwc(res) if resk else None, after=resk == "after",
                  scale=scale)
    ref, bnd = dense_bound(name, x, w, b, act, None if res is None else res.double(), resk == "after", scale)
    torch.cuda.synchronize()
    check_bound(nchw(y), ref, bnd, "%s %s res=%s" % (name, act, resk))


@pytest.mark.parametrize("name", sorted(DCN_CASES))
def test_dense_bound_dcn(unsaturated, name):
    ops = unsaturated
    (n, cin, cout, h, wd), want = DCN_CASES[name]
    g = gen(53 + cout)
    xs, ws = M.pow2_scales(cin, -6, 6, g), M.pow2_scales(cout, -12, 6, g)
    x = (M.fat((n, cin, h, wd), g).double() * xs.view(1, -1, 1, 1)).float()
    w = (M.fat((cout, cin, 3, 3), g).double() * ws.view(-1, 1, 1, 1)).float()
    off = dcn_offsets(g, n, h, wd)
    cols, acols = dcn_cols(x, off)
    y = run_dcn(ops, x, off, w, want)
    w64 = w.double().view(cout, cin, 9)
    ref = torch.einsum("nckhw,ock->nohw", cols, w64)
    absprod = torch.einsum("nckhw,ock->nohw", acols, w64.abs())      # |sample| <= the sum of its corner terms' sizes
    bnd = M.bound(absprod, w64.abs().sum((1, 2)).view(1, -1, 1, 1), acols.sum((1, 2)).unsqueeze(1),
                  M.gamma(M.steps(cin, 9)) + 11 * 2.0 ** -24, out=ref)
    torch.cuda.synchronize()
    check_bound(nchw(y), ref, bnd, "dcn " + name)


@pytest.mark.parametrize("cfg", CORR_CASES)
@pytest.mark.parametrize("act", ["none", "lrelu"])
def test_dense_bound_correlation(unsaturated, cfg, act):
    ops = unsaturated
    md, s2, C, H, W = cfg
    g = gen(59 + C)
    f1 = (M.fat((1, C, H, W), g).double() * M.pow2_scales(C, -6, 6, g).view(1, -1, 1, 1)).float()
    f2 = (M.fat((1, C, H, W), g).double() * M.pow2_scales(C, -6, 6, g).view(1, -1, 1, 1)).float()
    out = run_corr(ops, dev_nhwc(f1), dev_nhwc(f2), md, s2, act)
    ref = corr_ref(f1.double(), f2.double(), md, s2)
    if act == "lrelu":
        ref = F.leaky_relu(ref, 0.1)
    absprod = corr_ref(f1.double().abs(), f2.double().abs(), md, s2)
    s1 = f1.double().abs().sum(1, keepdim=True) / C
    sx = corr_ref(torch.ones_like(f1, dtype=torch.float64), f2.double().abs(), md, s2)
    bnd = M.bound(absprod, s1, sx, M.gamma_chain(C // 16), out=ref)
    torch.cuda.synchronize()
    check_bound(nchw(out), ref, bnd, "correlation d%d s%d C%d %s" % (md, s2, C, act))


# ------------------------------------------------------------------------------------------------ part 3: dynamic range
EQUI_CASES = {
    # name -> case of CASES to run at a smaller size, (h, w), the plan it must take there
    "halo": ("halo_nwg4", (64, 96), dict(halo=1)),
    "flat_tma": ("flat_1x1_tma_nwg4", (96, 128), dict(halo=0, epilogue="tma")),
    "deconv_phases": ("deconv4x4_s2", (12, 20), dict(halo=1)),
}


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("act", ["none", "relu", "lrelu"])
@pytest.mark.parametrize("name", sorted(EQUI_CASES))
def test_pow2_equivariance_conv(unsaturated, name, act, bias):
    """out(2^k x) == 2^k out(x) bit for bit (the bias scaled as well), k = -8, 8: both planes of fat data stay normal fp16
    at every scale, so an absolute threshold, a flush to zero or a saturation inside the normal range would show"""
    ops = unsaturated
    base, (h, wd), want = EQUI_CASES[name]
    kind, n, cin, cout, _, k, s, p, _ = CASES[base]
    g = gen(61)
    x = M.fat((n, cin, h, wd), g)
    w = M.fat(weights_like(kind, cin, cout, k), g)
    b = M.fat((cout,), g) if bias else None
    outs = {}
    for e in (-8, 0, 8):
        f = 2.0 ** e
        outs[e] = run_layer(ops, base, dev_nhwc(x * f), w, None if b is None else b * f, act=act, want=want)
    torch.cuda.synchronize()
    for e in (-8, 8):
        assert torch.equal(outs[e], outs[0] * 2.0 ** e), (name, act, e)


def test_pow2_equivariance_correlation(unsaturated):
    ops = unsaturated
    for md, s2, C, H, W in CORR_CASES:
        g = gen(67)
        f1, f2 = M.fat((1, C, H, W), g), M.fat((1, C, H, W), g)
        outs = {e: run_corr(ops, dev_nhwc(f1 * 2.0 ** e), dev_nhwc(f2 * 2.0 ** e), md, s2, "lrelu") for e in (-8, 0, 8)}
        torch.cuda.synchronize()
        for e in (-8, 8):
            assert torch.equal(outs[e], outs[0] * 2.0 ** (2 * e)), (md, e)


def test_pow2_equivariance_dcn(unsaturated):
    """integer offsets: every sample is one of the constructed values"""
    ops = unsaturated
    for name, ((n, cin, cout, h, wd), want) in sorted(DCN_CASES.items()):
        g = gen(71)
        x, w = M.fat((n, cin, h, wd), g), M.fat((cout, cin, 3, 3), g)
        off = dcn_offsets(g, n, h, wd, integer=True)
        outs = {e: run_dcn(ops, x * 2.0 ** e, off, w) for e in (-8, 0, 8)}
        torch.cuda.synchronize()
        for e in (-8, 8):
            assert torch.equal(outs[e], outs[0] * 2.0 ** e), (name, e)


@pytest.mark.parametrize("xscale", [2.0 ** -20, 2.0 ** -30, 2.0 ** 14])
@pytest.mark.parametrize("name", ["halo_nwg4", "flat_1x1_tma_nwg4"])
def test_operand_range(unsaturated, name, xscale):
    """Tiny activations (2^-20, 2^-30) hold the bound through its 2^-36 floor term: the relative accuracy is not promised
    there and the printed worst relative error shows it degrade.  Activations up to 2^15 hold the relative bound and do not
    touch the saturation counter."""
    ops = unsaturated
    g = gen(73)
    x, w, b, ws = dense_conv_data(name, g, xscale=xscale)
    y = run_layer(ops, name, dev_nhwc(x), w, None, check_plan=False)
    ref, bnd = dense_bound(name, x, w, None, "none", None, False, 1.0)
    torch.cuda.synchronize()
    got = nchw(y)
    check_bound(got, ref, bnd, "%s x * 2^%d" % (name, round(math.log2(xscale))))
    absprod = dense_bound(name, x.abs(), w.abs(), None, "none", None, False, 1.0)[0]
    print("   worst |err| / (|W| * |X|): %.3g" % float(((got - ref).abs() / absprod.clamp_min(1e-300)).max()))


# ------------------------------------------------------------------------------------------------ part 4: saturation
SITES = ["halo_converter", "flat_converter", "weight_packing", "dcn_sampler", "correlation_f1", "correlation_f2"]


def _site_run(ops, site, val):
    """one run with `val` planted (None: clean); returns (got, ref) of the probe outputs"""
    g = gen(79)
    if site.startswith("correlation"):
        C, H, W = 64, 16, 24
        f1 = torch.zeros(1, C, H, W, device="cuda")
        ch = torch.arange(H * W, device="cuda") % C
        f1.view(C, H * W)[ch, torch.arange(H * W, device="cuda")] = M.fat((H * W,), g)
        f2 = M.fat((1, C, H, W), g)
        if val is not None:
            pix = 5 * W + 7
            (f1 if site == "correlation_f1" else f2).view(C, H * W)[int(ch[pix]), pix] = val
        out = run_corr(ops, dev_nhwc(f1), dev_nhwc(f2), 4, 1)
        return nchw(out), corr_ref(f1.double(), f2.double(), 4, 1)
    cin, cout, h, wd = 64, 16, 16, 24
    x = M.fat((1, cin, h, wd), g)
    wv = M.fat((cout,), g)
    probes = [(co * 4 % cin, 4) for co in range(cout)]       # centre tap: output (y, x) reads x[y, x]
    if site == "dcn_sampler":
        w = one_hot("conv", cin, cout, 3, probes, wv)
        off = torch.zeros(1, 18, h, wd, device="cuda")
        if val is not None:
            x[0, 8, 7, 9] = val
        y = run_dcn(ops, x, off, w)
        ref = F.conv2d(x.double(), w.double(), padding=1)
        return nchw(y), ref
    k = 3 if site == "halo_converter" else 1
    w = one_hot("conv", cin, cout, k, [(ci, k * k // 2) for ci, _ in probes], wv)
    if val is not None:
        if site == "weight_packing":
            w[2, probes[2][0], k // 2, k // 2] = val
        else:
            x[0, 8, 7, 9] = val
    pk = ops.PackedConv(w, None)
    plan = ops.conv2d_tc32_plan(dev_nhwc(x), pk, pad=k // 2)
    assert plan["halo"] == (k == 3), plan
    y = torch.full((1, h, wd, cout), float("nan"), device="cuda")
    ops.conv2d(dev_nhwc(x), pk, y, pad=k // 2, use_tc=True)
    return nchw(y), F.conv2d(x.double(), w.double(), padding=k // 2)


@pytest.mark.parametrize("site", SITES)
def test_saturation_counter(tc32, site):
    """every output is one product (one-hot weights, or one f1 channel per pixel): clean and at exactly 65504 the counter
    stays 0 and the outputs hold the probe bound; 65505, NaN and +Inf set it; reading with reset clears it"""
    ops = tc32
    ops.tc32_overflow()
    got, ref_clean = _site_run(ops, site, None)
    torch.cuda.synchronize()
    assert ops.tc32_overflow(reset=False) == 0, "clean run"
    check_probe(got, ref_clean)
    got, ref = _site_run(ops, site, 65504.0)
    torch.cuda.synchronize()
    assert ops.tc32_overflow(reset=False) == 0, "65504 is in range"
    assert not torch.equal(ref, ref_clean)                   # the planted element reaches an output
    check_probe(got, ref)
    for val in (65505.0, float("nan"), float("inf")):
        _site_run(ops, site, val)
        torch.cuda.synchronize()
        assert ops.tc32_overflow(reset=False) > 0, (site, val)
        assert ops.tc32_overflow(reset=True) > 0
        assert ops.tc32_overflow(reset=False) == 0, "reset"


def test_dcn_unreached_large_input_does_not_count(tc32):
    """out-of-image corners read pixel (0, 0) of the input with weight 0: a 70000 there counts only when an in-image sample
    reaches it"""
    ops = tc32
    ops.tc32_overflow()
    g = gen(83)
    cin, cout, h, wd = 64, 64, 16, 24
    x = M.fat((2, cin, h, wd), g)
    x[0, :, 0, 0] = 70000.0
    w = M.fat((cout, cin, 3, 3), g)
    off = torch.full((2, 18, h, wd), 2.0, device="cuda")      # sample (y + i + 1, x + j + 1): never (0, 0)
    y = run_dcn(ops, x, off, w)
    torch.cuda.synchronize()
    assert ops.tc32_overflow() == 0
    assert not bool(torch.isnan(y).any())
    run_dcn(ops, x, torch.zeros_like(off), w)                 # tap (0, 0) of output (1, 1) samples it
    torch.cuda.synchronize()
    assert ops.tc32_overflow() > 0


# ------------------------------------------------------------------------------------------------ part 5: NaN padding
def _padded_pair(run):
    """run(fill) with zero and with NaN padding channels: bit-identical outputs, sentinels kept"""
    outs = [run(fill) for fill in (0.0, float("nan"))]
    torch.cuda.synchronize()
    (y0, buf0), (y1, buf1) = outs
    assert torch.equal(y0.view(torch.int32) if y0.dtype == torch.float32 else y0.view(torch.int16),
                       y1.view(torch.int32) if y1.dtype == torch.float32 else y1.view(torch.int16))
    assert not bool(torch.isnan(y1.float()).any())
    for buf, y in ((buf0, y0), (buf1, y1)):
        c0 = (y.data_ptr() - buf.data_ptr()) // buf.element_size()
        assert bool((buf[..., :c0].float() == SENTINEL).all()) and bool((buf[..., c0 + y.shape[-1]:].float() == SENTINEL).all())


def _out_slice(shape, c, dtype=torch.float32):
    n, h, w = shape
    buf = torch.full((n, h, w, 8 + c + 12), SENTINEL, dtype=dtype, device="cuda")
    return buf[..., 8:8 + c], buf


@pytest.mark.parametrize("what", ["halo", "flat_tma_residual", "deconv_phases", "dcn", "correlation",
                                  "bf16_conv", "bf16_dcn", "bf16_correlation"])
def test_nan_padding_channels(unsaturated, what):
    ops = unsaturated
    g = gen(89)
    bf = what.startswith("bf16")
    dt = torch.bfloat16 if bf else torch.float32
    if what in ("halo", "flat_tma_residual", "bf16_conv"):
        k = 1 if what == "flat_tma_residual" else 3
        cin, cout, h, wd = (64, 64, 96, 128) if k == 1 else (82, 40, 40, 64)
        x = M.fat((1, cin, h, wd), g)
        w = M.fat((cout, cin, k, k), g) / (cin * k * k)
        b = M.fat((cout,), g)
        res = M.fat((1, cout, h, wd), g) if k == 1 else None
        pk = ops.PackedConv(w, b)

        def run(fill):
            xd = dev_nhwc(x, fill, extra=8, dtype=dt)
            rd = dev_nhwc(res, fill, extra=8) if res is not None else None
            y, buf = _out_slice((1, h, wd), cout, dt)
            if k == 1:
                assert ops.conv2d_tc32_plan(xd, pk, y=y, res=rd)["epilogue"] == "tma"
            ops.conv2d(xd, pk, y, pad=k // 2, act=ops.ACT_LRELU, res=rd, use_tc=True)
            return y, buf
    elif what == "deconv_phases":
        from vps_b200.layers import deconv4x4_s2
        x = M.fat((1, 128, 12, 20), g)
        layer = deconv4x4_s2(M.fat((128, 32, 4, 4), g) / 512, M.fat((32,), g))

        def run(fill):
            y, buf = _out_slice((1, 24, 40), 32)
            layer(dev_nhwc(x, fill, extra=8), y, act=ops.ACT_LRELU)
            return y, buf
    elif what in ("dcn", "bf16_dcn"):
        x = M.fat((1, 64, 24, 40), g)
        w = M.fat((48, 64, 3, 3), g) / 576
        off = dcn_offsets(g, 1, 24, 40)
        pk = ops.PackedConv(w, None)

        def run(fill):
            xd = dev_nhwc(x, fill, extra=8 if not bf else 16, dtype=dt)
            od = dev_nhwc(off, fill)                       # 18 of 24 channels
            assert od.stride(2) == 24
            y, buf = _out_slice((1, 24, 40), 48, dt)
            (ops.deform_conv_tc if bf else ops.deform_conv_tc32)(xd, od, pk, y)
            return y, buf
    else:
        C, H, W = 64, 24, 40
        f1, f2 = M.fat((1, C, H, W), g), M.fat((1, C, H, W), g)

        def run(fill):
            y, buf = _out_slice((1, H, W), 441)
            run_corr(ops, dev_nhwc(f1, fill, extra=8, dtype=dt), dev_nhwc(f2, fill, extra=8, dtype=dt), 20, 2, "lrelu",
                     impl="tc" if bf else "tc32", out=y)
            return y, buf
    _padded_pair(run)
