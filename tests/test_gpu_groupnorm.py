"""GPU: vps_groupnorm against an fp64 reference on every launch arm, at the UPSNet head's shapes and on ill-conditioned groups.

The reference is F.group_norm in float64 on the values the kernel reads (bf16 inputs upcast), then ReLU where the call uses
it.  An fp32 output must satisfy, element by element,

    |got - ref| <= 2e-5 * max(1, max|ref|) + 2^-23 * |gamma_c| * |mean_g| * rstd_g

where the second term is the unavoidable error of forming x - mean in fp32 with mean rounded to fp32.  A bf16 output may
also carry one bf16 rounding of the result.

Launch arms (vps_b200/csrc/pointwise.cu, V = 4 fp32 / 8 bf16 channels per thread):
  statistics  vector when the input is 16-byte accessible, C / V divides 256 and cg % V == 0 (one group per chunk) or
              V == 2 * cg (two groups per chunk); scalar otherwise
  apply       vector when input and output share a dtype and both are 16-byte accessible; scalar otherwise
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

EPS = 1e-5


def ops():
    from vps_b200 import ops as _ops
    return _ops


def vec_width(dtype):
    return 4 if dtype == torch.float32 else 8


def dense(x, dtype):
    """NCHW (CPU) -> dense NHWC CUDA tensor"""
    return x.permute(0, 2, 3, 1).to(dtype).contiguous().cuda()


def sliced(x, dtype):
    """NCHW (CPU) -> the same values at channels 1..C of a C+1 channel NHWC buffer: base and pixel stride unaligned"""
    n, c, h, w = x.shape
    buf = torch.zeros(n, h, w, c + 1, dtype=dtype, device="cuda")
    buf[..., 1:] = x.permute(0, 2, 3, 1).to(dtype).cuda()
    return buf[..., 1:]


LAYOUTS = {"dense": dense, "sliced": sliced}


def empty_out(shape_nchw, dtype, layout):
    return LAYOUTS[layout](torch.full(shape_nchw, float("nan")), dtype)


def nchw(t):
    return t.permute(0, 3, 1, 2).double().cpu()


def bits(t):
    t = t.contiguous()
    return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32).cpu()


def stored(x, dtype):
    """the values a tensor of `dtype` holds"""
    return x.to(dtype).float()


def groupnorm(x, y, gamma, beta, groups, relu):
    ops().groupnorm(x, y, gamma.cuda(), beta.cuda(), groups, EPS, relu=relu)


def reference(x, groups, gamma, beta, relu):
    """fp64 GroupNorm (+ ReLU) of the NCHW values x, and the per-element fp32 mean-rounding term of the bound"""
    xd = x.double()
    n, c = xd.shape[:2]
    ref = F.group_norm(xd, groups, gamma.double(), beta.double(), EPS)
    if relu:
        ref = ref.clamp_min(0.0)
    xg = xd.reshape(n, groups, -1)
    mean = xg.mean(-1)
    rstd = 1.0 / torch.sqrt(xg.var(-1, unbiased=False) + EPS)
    per_c = (mean.abs() * rstd).repeat_interleave(c // groups, 1)          # [n, c]
    term = 2.0 ** -23 * gamma.double().abs().view(1, c) * per_c
    return ref, term.view(n, c, 1, 1)


def assert_close(got, x, groups, gamma, beta, relu, what=""):
    """got: the NHWC output; x: the NCHW values the kernel read"""
    ref, term = reference(x, groups, gamma, beta, relu)
    g = nchw(got)
    assert torch.isfinite(g).all(), "%s: non-finite outputs" % what
    bound = 2e-5 * max(1.0, float(ref.abs().max())) + term
    if got.dtype == torch.bfloat16:
        bound = bound + 2.0 ** -8 * (ref.abs() + bound)
    ratio = (g - ref).abs() / bound
    worst = float(ratio.max())
    if worst > 1.0:
        idx = np.unravel_index(int(ratio.argmax()), tuple(ratio.shape))
        raise AssertionError("%s: error / bound %.3g at (n, c, y, x) = %s: got %r ref %r (channel group %d)"
                             % (what, worst, idx, float(g[idx]), float(ref[idx]), idx[1] // (x.shape[1] // groups)))


def grouped_input(gen, n, c, h, w, groups, mean, std):
    """NCHW values with mean[n, g] and std[n, g] per (image, group)"""
    z = torch.randn(n, c, h, w, generator=gen)
    m = mean.repeat_interleave(c // groups, 1).view(n, c, 1, 1)
    s = std.repeat_interleave(c // groups, 1).view(n, c, 1, 1)
    return z * s + m


def affine(gen, c):
    return torch.rand(c, generator=gen) + 0.5, torch.randn(c, generator=gen)


def run_case(gen, n, c, h, w, groups, dtype, relu, layout="dense", mean=None, std=None):
    if mean is None:
        mean = torch.rand(n, groups, generator=gen) * 6 - 3
    if std is None:
        std = torch.rand(n, groups, generator=gen) * 2.5 + 0.5
    x = stored(grouped_input(gen, n, c, h, w, groups, mean, std), dtype)
    gamma, beta = affine(gen, c)
    xd = LAYOUTS[layout](x, dtype)
    y = empty_out((n, c, h, w), dtype, layout)
    groupnorm(xd, y, gamma, beta, groups, relu)
    torch.cuda.synchronize()
    return x, y, gamma, beta


DTYPES = {"f32": torch.float32, "bf16": torch.bfloat16}


# ---------------------------------------------------------------- group-index probes
@pytest.mark.parametrize("layout", ["dense", "sliced"])
@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("cg", [1, 2, 3, 4, 5, 6, 7, 8, 12, 16, 32])
def test_group_index_probe(cuda, cg, dt, layout):
    """every group has its own mean (g*10 + noise) and its own gamma / beta: a channel normalised with another group's
    statistics or affine parameters is off by O(1)"""
    dtype, groups = DTYPES[dt], 32
    c = cg * groups
    gen = torch.Generator().manual_seed(100 + cg)
    gidx = torch.arange(c) // cg
    x = torch.randn(1, c, 6, 10, generator=gen) + (gidx * 10.0).view(1, c, 1, 1)
    x = stored(x, dtype)
    gamma = 1.0 + 0.25 * (gidx % 5).float() + 0.05 * torch.rand(c, generator=gen)
    beta = 0.5 * gidx.float() - 8.0 + 0.1 * torch.randn(c, generator=gen)
    y = empty_out((1, c, 6, 10), dtype, layout)
    groupnorm(LAYOUTS[layout](x, dtype), y, gamma, beta, groups, relu=False)
    torch.cuda.synchronize()
    assert_close(y, x, groups, gamma, beta, False, "cg=%d %s %s" % (cg, dt, layout))


# ---------------------------------------------------------------- launch arms
def _aligned(t, v):
    c, cs = t.shape[-1], (t.stride(2) if t.shape[2] > 1 else t.shape[-1])
    return c % v == 0 and cs % v == 0 and t.data_ptr() % 16 == 0


def expected_kernels(x, y, groups):
    """the statistics and apply kernels the launcher picks for these tensors, as in vps_groupnorm"""
    v = vec_width(x.dtype)
    c = x.shape[-1]
    cg = c // groups
    tname = {torch.float32: "float", torch.bfloat16: "__nv_bfloat16"}
    chunks = c // v
    if _aligned(x, v) and chunks <= 256 and 256 % chunks == 0 and (cg % v == 0 or v == 2 * cg):
        stats = "gn_stats_vec_kernel<%s, %d" % (tname[x.dtype], v)
    else:
        stats = "gn_stats_kernel<%s>" % tname[x.dtype]
    va = v if x.dtype == y.dtype and _aligned(x, v) and _aligned(y, v) else 1
    return stats, "gn_apply_kernel<%s, %s, %d>" % (tname[x.dtype], tname[y.dtype], va)


def launched_kernels(fn, attempts=3):
    """names of the device activities fn causes, from torch.profiler; a session that recorded no device activity at all
    (the profiler occasionally misses every kernel of a session) is repeated"""
    from torch.profiler import ProfilerActivity, profile
    names = []
    for _ in range(attempts):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
        if names:
            break
    return names


# arm: (channels, groups, input layout, output layout, vector statistics, vector apply when the dtypes match)
ARMS = {
    "vec_one_group": (256, 32, "dense", "dense", True, True),       # cg = 8: cg % V == 0 in both dtypes
    "vec_two_groups": (None, 32, "dense", "dense", True, True),     # V == 2 * cg: C = 64 (fp32), 128 (bf16)
    "scalar_stats": (96, 32, "dense", "dense", False, True),        # cg = 3
    "scalar_both": (256, 32, "sliced", "sliced", False, False),     # unaligned input
    "scalar_apply": (256, 32, "dense", "sliced", True, False),      # unaligned output
}
PAIRS = {"f32_f32": (torch.float32, torch.float32), "bf16_bf16": (torch.bfloat16, torch.bfloat16),
         "f32_bf16": (torch.float32, torch.bfloat16), "bf16_f32": (torch.bfloat16, torch.float32)}


@pytest.mark.parametrize("pair", sorted(PAIRS))
@pytest.mark.parametrize("arm", sorted(ARMS))
def test_launch_arms(cuda, arm, pair):
    ti, to = PAIRS[pair]
    c, groups, lin, lout, vec_stats, vec_apply = ARMS[arm]
    v = vec_width(ti)
    if c is None:
        c = groups * v // 2
    gen = torch.Generator().manual_seed(7)
    x = stored(grouped_input(gen, 1, c, 19, 37, groups, torch.rand(1, groups, generator=gen) * 4 - 2,
                             torch.rand(1, groups, generator=gen) + 0.5), ti)
    gamma, beta = affine(gen, c)
    xd = LAYOUTS[lin](x, ti)
    y = empty_out((1, c, 19, 37), to, lout)
    stats, apply = expected_kernels(xd, y, groups)
    assert ("vec" in stats) == vec_stats, stats
    assert apply.endswith(", %d>" % v) == (vec_apply and ti == to), apply
    names = launched_kernels(lambda: groupnorm(xd, y, gamma, beta, groups, True))
    for k in (stats, apply):
        assert any(k in nm for nm in names), "%s not launched; kernels: %s" % (k, names)
    assert_close(y, x, groups, gamma, beta, True, "%s %s" % (arm, pair))


# ---------------------------------------------------------------- shapes
# (n, C, H, W, groups, relu): the UPSNet head's GroupNorm(32, 256 / 128) on P2..P5 of a 1024x2048 frame and one level of a
# 1088x1920 frame, a map long enough that every vector-arm thread strides over many pixels, edge sizes, two images, the
# extreme group counts and the widest C
SHAPES = {
    "P2_c256": (1, 256, 256, 512, 32, True), "P2_c128": (1, 128, 256, 512, 32, True),
    "P3_c256": (1, 256, 128, 256, 32, True), "P3_c128": (1, 128, 128, 256, 32, True),
    "P4_c256": (1, 256, 64, 128, 32, True), "P4_c128": (1, 128, 64, 128, 32, True),
    "P5_c256": (1, 256, 32, 64, 32, True), "P5_c128": (1, 128, 32, 64, 32, True),
    "1088x1920_c256": (1, 256, 272, 480, 32, True),
    "640x640_c128": (1, 128, 640, 640, 32, True),
    "1x1": (1, 256, 1, 1, 32, False), "1xW": (1, 128, 1, 77, 32, True), "Hx1": (1, 128, 53, 1, 32, False),
    "odd": (1, 256, 33, 47, 32, False),
    "two_images": (2, 128, 48, 80, 32, True),
    "groups1": (1, 256, 40, 64, 1, False), "groups64": (1, 256, 40, 64, 64, True),
    "c1024": (1, 1024, 24, 40, 32, False), "c1024_groups64": (1, 1024, 24, 40, 64, True),
}


@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("shape", list(SHAPES))
def test_shapes(cuda, shape, dt):
    n, c, h, w, groups, relu = SHAPES[shape]
    gen = torch.Generator().manual_seed(sum(map(ord, shape)))
    mean = std = None
    if n == 2:                                                 # images with very different statistics
        mean = torch.stack([torch.zeros(groups), torch.full((groups,), 40.0)])
        std = torch.stack([torch.full((groups,), 0.25), torch.full((groups,), 6.0)])
    x, y, gamma, beta = run_case(gen, n, c, h, w, groups, DTYPES[dt], relu, mean=mean, std=std)
    assert_close(y, x, groups, gamma, beta, relu, "%s %s" % (shape, dt))


@pytest.mark.parametrize("offset", [0, 128])
@pytest.mark.parametrize("dt", sorted(DTYPES))
def test_channel_slice_output(cuda, dt, offset):
    """the last GroupNorm of level 0 writes feat[..., :128] of the 512-channel concat buffer: input and output are channel
    slices of 512-channel buffers, and the channels outside the slice keep their contents"""
    dtype, c, groups = DTYPES[dt], 128, 32
    gen = torch.Generator().manual_seed(20 + offset)
    x = stored(grouped_input(gen, 1, c, 64, 128, groups, torch.rand(1, groups, generator=gen) * 4 - 2,
                             torch.rand(1, groups, generator=gen) + 0.5), dtype)
    gamma, beta = affine(gen, c)
    src = torch.randn(1, 64, 128, 512, generator=gen).to(dtype).cuda()
    src[..., offset:offset + c] = x.permute(0, 2, 3, 1).to(dtype).cuda()
    buf = torch.full((1, 64, 128, 512), -1234.5, dtype=dtype, device="cuda")
    before = bits(buf)
    y = buf[..., offset:offset + c]
    groupnorm(src[..., offset:offset + c], y, gamma, beta, groups, True)
    torch.cuda.synchronize()
    assert_close(y, x, groups, gamma, beta, True, "slice at %d %s" % (offset, dt))
    after = bits(buf)
    keep = torch.ones(512, dtype=torch.bool)
    keep[offset:offset + c] = False
    assert torch.equal(after[..., keep], before[..., keep])


# ---------------------------------------------------------------- ill-conditioned groups
@pytest.mark.parametrize("layout", ["dense", "sliced"])
@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("ratio", [1e2, 1e3, 1e4])
def test_large_mean_over_std(cuda, ratio, dt, layout):
    """every group's mean is `ratio` times its standard deviation (of either sign): E[x^2] - E[x]^2 loses log10(ratio^2)
    digits; the error allowed for the fp32 mean is the bound's second term"""
    dtype, c, groups = DTYPES[dt], 128, 32
    gen = torch.Generator().manual_seed(int(ratio))
    std = torch.rand(1, groups, generator=gen) * 1.5 + 0.5
    sign = torch.where(torch.rand(1, groups, generator=gen) < 0.5, -1.0, 1.0)
    mean = sign * ratio * std * (1 + 0.5 * torch.rand(1, groups, generator=gen))
    x, y, gamma, beta = run_case(gen, 1, c, 64, 128, groups, dtype, False, layout, mean=mean, std=std)
    assert_close(y, x, groups, gamma, beta, False, "mean/std %g %s %s" % (ratio, dt, layout))


@pytest.mark.parametrize("layout", ["dense", "sliced"])
@pytest.mark.parametrize("dt", sorted(DTYPES))
def test_outliers(cuda, dt, layout):
    """single elements 1e3 and 1e5 standard deviations away from the rest of their groups"""
    dtype, c, groups = DTYPES[dt], 128, 32
    gen = torch.Generator().manual_seed(31)
    x = grouped_input(gen, 1, c, 64, 128, groups, torch.rand(1, groups, generator=gen) * 4 - 2, torch.ones(1, groups))
    x[0, 3 * 4 + 1, 17, 99] = 1e3
    x[0, 21 * 4 + 3, 0, 0] = -1e5
    x[0, 30 * 4, 63, 127] = 3e4
    x = stored(x, dtype)
    gamma, beta = affine(gen, c)
    y = empty_out((1, c, 64, 128), dtype, layout)
    groupnorm(LAYOUTS[layout](x, dtype), y, gamma, beta, groups, False)
    torch.cuda.synchronize()
    assert_close(y, x, groups, gamma, beta, False, "outliers %s %s" % (dt, layout))


CONST_VALUES = np.concatenate([np.geomspace(0.5, 100.0, 16), -np.geomspace(0.5, 100.0, 16)])


@pytest.mark.parametrize("size", ["64x128", "256x512"])
@pytest.mark.parametrize("relu", [True, False], ids=["relu", "norelu"])
@pytest.mark.parametrize("layout", ["dense", "sliced"])
@pytest.mark.parametrize("cg", [4, 8])
@pytest.mark.parametrize("dt", sorted(DTYPES))
def test_constant_groups(cuda, dt, cg, layout, relu, size):
    """32 constant groups (values +-[0.5, 100]) between 32 normal ones: a constant group has variance 0, so its output is
    exactly relu(beta) -- a negative variance estimate gives NaN (0 after the ReLU), a positive one moves the output"""
    if size != "64x128" and layout != "dense":
        pytest.skip("the long map runs on the production layout only")
    dtype, groups = DTYPES[dt], 64
    c = cg * groups
    h, w = map(int, size.split("x"))
    gen = torch.Generator().manual_seed(cg * 7 + h)
    x = grouped_input(gen, 1, c, h, w, groups, torch.rand(1, groups, generator=gen) * 20 - 10,
                      torch.rand(1, groups, generator=gen) * 2 + 0.5)
    const = torch.zeros(groups, dtype=torch.bool)
    const[0::2] = True
    for i, g in enumerate(range(0, groups, 2)):
        x[0, g * cg:(g + 1) * cg] = float(CONST_VALUES[i])
    x = stored(x, dtype)
    gamma, beta = affine(gen, c)
    y = empty_out((1, c, h, w), dtype, layout)
    groupnorm(LAYOUTS[layout](x, dtype), y, gamma, beta, groups, relu)
    torch.cuda.synchronize()
    ch_const = const.repeat_interleave(cg)
    got = y.permute(0, 3, 1, 2).cpu()[:, ch_const]
    want = (beta.clamp_min(0.0) if relu else beta)[ch_const].to(dtype).view(1, -1, 1, 1).expand_as(got)
    bad = (bits(got) != bits(want)).nonzero()
    assert bad.numel() == 0, "constant groups not equal to relu(beta): %d elements, first at channel %d: got %r want %r" % (
        bad.shape[0], int(bad[0, 1]), float(got[tuple(bad[0])]), float(want[tuple(bad[0])]))
    ch_norm = ~ch_const
    assert_close(y[..., ch_norm.cuda()], x[:, ch_norm], groups // 2, gamma[ch_norm], beta[ch_norm], relu,
                 "normal groups next to constant ones")


# ---------------------------------------------------------------- statistics slots, determinism
def _calls(k, c=256, h=128, w=256, groups=32):
    gen = torch.Generator().manual_seed(1000 + k)
    out = []
    for i in range(k):
        dtype = torch.float32 if i % 2 == 0 else torch.bfloat16
        x = stored(grouped_input(gen, 1, c, h, w, groups, torch.rand(1, groups, generator=gen) * 10 - 5,
                                 torch.rand(1, groups, generator=gen) * 3 + 0.25), dtype)
        gamma, beta = affine(gen, c)
        out.append((x, dense(x, dtype), torch.full((1, h, w, c), float("nan"), dtype=dtype, device="cuda"),
                    gamma.cuda(), beta.cuda()))
    return out


def test_back_to_back_calls(cuda):
    """20 calls on one stream without a synchronise -- more than the 16 statistics slots -- each with its own input"""
    calls = _calls(20)
    torch.cuda.synchronize()
    for _, xd, y, gamma, beta in calls:
        ops().groupnorm(xd, y, gamma, beta, 32, EPS, relu=True)
    torch.cuda.synchronize()
    for i, (x, _, y, gamma, beta) in enumerate(calls):
        assert_close(y, x, 32, gamma.cpu(), beta.cpu(), True, "call %d" % i)


def test_two_streams_equal_serial(cuda):
    """8 calls on each of two streams, interleaved as they are enqueued: bit-equal to the same 16 calls run one after the
    other"""
    calls = _calls(16)
    torch.cuda.synchronize()
    for _, xd, y, gamma, beta in calls:
        ops().groupnorm(xd, y, gamma, beta, 32, EPS, relu=True)
    torch.cuda.synchronize()
    serial = [bits(y) for _, _, y, _, _ in calls]
    for _, _, y, _, _ in calls:
        y.fill_(float("nan"))
    main = torch.cuda.current_stream()
    side = [torch.cuda.Stream(), torch.cuda.Stream()]
    for s in side:
        s.wait_stream(main)
    for i in range(8):
        for j, s in enumerate(side):
            _, xd, y, gamma, beta = calls[j * 8 + i]
            with torch.cuda.stream(s):
                ops().groupnorm(xd, y, gamma, beta, 32, EPS, relu=True)
    for s in side:
        main.wait_stream(s)
    torch.cuda.synchronize()
    for i, (_, _, y, _, _) in enumerate(calls):
        assert torch.equal(bits(y), serial[i]), "call %d" % i


@pytest.mark.parametrize("layout", ["dense", "sliced"])
@pytest.mark.parametrize("dt", sorted(DTYPES))
def test_reproducible(cuda, dt, layout):
    """the statistics are merged in a fixed order: the same input gives the same bits, run after run"""
    dtype = DTYPES[dt]
    gen = torch.Generator().manual_seed(5)
    x = stored(grouped_input(gen, 1, 256, 256, 512, 32, torch.rand(1, 32, generator=gen) * 200 - 100,
                             torch.rand(1, 32, generator=gen) + 0.1), dtype)
    gamma, beta = affine(gen, 256)
    xd = LAYOUTS[layout](x, dtype)
    outs = []
    for _ in range(3):
        y = empty_out((1, 256, 256, 512), dtype, layout)
        groupnorm(xd, y, gamma, beta, 32, True)
        torch.cuda.synchronize()
        outs.append(bits(y))
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


# ---------------------------------------------------------------- argument errors
BAD_ARGS = {              # (n, C, groups)
    "groups0": (1, 64, 0),
    "groups65": (1, 130, 65),
    "c_not_multiple_of_groups": (1, 100, 32),
    "c_over_1024": (1, 1056, 32),
    "n_groups_over_2048": (33, 64, 64),
}


@pytest.mark.parametrize("case", sorted(BAD_ARGS))
def test_argument_errors(cuda, case):
    """rejected on the host with VpsError before anything is launched: the output keeps its contents"""
    from vps_b200._lib import VpsError
    n, c, groups = BAD_ARGS[case]
    x = torch.randn(n, 3, 5, c, device="cuda")
    y = torch.full((n, 3, 5, c), 7.0, device="cuda")
    gamma, beta = torch.ones(c, device="cuda"), torch.zeros(c, device="cuda")
    torch.cuda.synchronize()
    n0 = ops().launch_count()
    with pytest.raises(VpsError):
        ops().groupnorm(x, y, gamma, beta, groups, EPS, relu=True)
    torch.cuda.synchronize()
    assert ops().launch_count() == n0
    assert bool((y == 7.0).all())
