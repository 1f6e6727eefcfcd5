"""CPU model of the tc32 ("parity") precision: the fp16 operand split, fat operands whose correction planes are large and
exact, the componentwise error bound the tc32 kernels are held to, and an emulation of the documented arithmetic.

The split (vps_b200/csrc/conv_tc32.cu, header and split_pair_f16; the same in pack_weights_tc32_kernel and
split_f16_planes_kernel of corr_tc.cu):

    A = fp16_satfinite(v)  (round to nearest),   A2 = fp16_satfinite(2^11 * (v - A))  (the difference taken in fp32),
    v ~ A + 2^-11 * A2,   a*b ~ A*B + 2^-11 * (A2*B + A*B2).

Error bound, output element i of a contraction over k (a = activation, b = weight):

  * One operand.  v - A is exact in fp32 and |v - A| <= 2^-11 |v|.  A2 rounds it to fp16: a relative error of 2^-11 of
    2^11 |v - A| while A2 is normal, i.e. <= 2^-22 |v| in units of v; while A2 is subnormal it lies on the 2^-24 grid, an
    absolute error <= 2^-25, i.e. 2^-36 in units of v (this also covers |v| < 2^-14, where A is subnormal or 0 and A2
    carries the rest).  So each operand is carried with error <= 2^-22 |v| + 2^-36.
  * One product.  The two carried operands give <= 2 * 2^-22 |ab| + 2^-36 (|a| + |b|) (the cross term is below 2^-43 |ab|),
    and the dropped 2^-22 * A2*B2 (|A2| <= |a|, |B2| <= |b|) adds <= 2^-22 |ab|: 3 * 2^-22 |ab| + 2^-36 (|a| + |b|).
  * One K step (32 channels of one tap, two K16 slabs).  The correction chain (up to four MMAs, scaled by 2^-11) and the main
    chain (two MMAs) accumulate in fp32 inside the tensor core, which is not guaranteed to round to nearest: allow
    2^-22 * sum|ab| per main-chain MMA (a truncated alignment and a truncated result), 2^-33 for the correction chain.
    3 * 2^-22 + 2 * 2^-22 + 2^-33 < 2^-19, so the step result is within 2^-19 * sum_step |ab| (plus the 2^-36 terms).
  * S steps are promoted into a register sum with round-to-nearest fp32 adds: each <= 2^-24 of a partial sum, which is at
    most sum |ab| (plus the step errors): S * 2^-24.
  * The epilogue adds bias and residual and applies the activation in fp32, round to nearest: 2^-24 per operation, taken
    as 2^-23 of |bias|, |residual| and |out|.  ReLU and leaky ReLU (slope <= 1) are 1-Lipschitz.  The sigmoid is
    1 / (1 + __expf(-t)): the error e of t moves it by at most (s(1-s) + e) e, and __expf has at most
    2 + 1.173 |t| ulp of error (CUDA C Programming Guide, intrinsic functions), which moves s by s(1-s) times that
    relative error.

    err_i <= gamma_S * (|W| * |X|)_i + 2^-36 (sum|w| + sum|x|)_i + 2^-23 (|bias| + |res| + |out|)_i,
    gamma_S = 2^-19 + S * 2^-24,

where (|W| * |X|)_i is the contraction of the absolute values, sum|w| the absolute weights of output channel i and sum|x|
the absolute activations it reads.

The correlation (vps_correlation_tc32) does not promote: each of its three passes is one chain of C / 16 MMAs, and the
passes are added in the fp32 output.  Its gamma is gamma_chain(C / 16) = 2^-19 + (C / 16) * 2^-22.

Relative accuracy is only promised while the operands are well inside the fp16 range: below 2^-14 the 2^-36 floor
dominates, and above 65504 the main plane saturates (the kernels count that in the saturation counter).
"""
import math

import torch

LO = 2.0 ** 11
F16_MAX = 65504.0
STEP_K = 32                     # channels per K step
SLAB = 16                       # channels per MMA (K16)


def split16(v):
    """(A, A2) as fp16 tensors, bit for bit as the kernels compute them"""
    v = torch.as_tensor(v, dtype=torch.float32)
    a = v.clamp(-F16_MAX, F16_MAX).to(torch.float16)          # satfinite: |v| > 65504 and +-Inf -> +-65504, NaN stays
    r = (v - a.float()) * LO                                   # fp32, exact while v is in range
    return a, r.clamp(-F16_MAX, F16_MAX).to(torch.float16)


def carried(v):
    """the value the two planes carry, A + 2^-11 A2, in fp64"""
    a, a2 = split16(v)
    return a.double() + a2.double() / LO


def fat(shape, gen):
    """fp32 values v = A + 2^-11 A2 with A a random fp16, |A| in [0.5, 2), random sign, and A2 a random fp16 with
    |A2| in [0.25, 0.75] * 2^10 * ulp(A): the correction plane is large and exact, so dropping either correction product
    changes a product by at least 2^-14 of its size.  The value spans at most 24 significant bits: the cast is exact."""
    dev = gen.device
    e = torch.randint(-1, 1, shape, generator=gen, device=dev).double()        # |A| in [2^e, 2^(e+1))
    m = torch.randint(0, 1024, shape, generator=gen, device=dev).double()
    sa = torch.randint(0, 2, shape, generator=gen, device=dev).double() * 2 - 1
    a = sa * torch.pow(2.0, e) * (1 + m / 1024)
    lo, hi = 0.25 * torch.pow(2.0, e), 0.75 * torch.pow(2.0, e)               # 2^10 ulp(A) = 2^e; both ends are fp16
    mag = (lo + (hi - lo) * torch.rand(shape, generator=gen, dtype=torch.float64, device=dev)).half().double()
    mag = torch.minimum(torch.maximum(mag, lo), hi)
    s2 = torch.randint(0, 2, shape, generator=gen, device=dev).double() * 2 - 1
    s2 = torch.where(m == 0, sa, s2)       # at a power of two a correction towards zero would round A into the binade below
    a2 = s2 * mag
    v = (a + a2 / LO).float()
    assert torch.equal(v.double(), a + a2 / LO)
    A, A2 = split16(v)
    assert torch.equal(A.double(), a) and torch.equal(A2.double(), a2)
    return v


def pow2_scales(n, lo, hi, gen):
    """n powers of two spanning 2^lo .. 2^hi (both ends present), shuffled"""
    ex = torch.linspace(lo, hi, n).round() if n > 1 else torch.tensor([float(hi)])
    ex = ex.to(gen.device)[torch.randperm(n, generator=gen, device=gen.device)]
    return torch.pow(2.0, ex).double()


def gamma(steps):
    return 2.0 ** -19 + steps * 2.0 ** -24


def gamma_chain(mmas):
    return 2.0 ** -19 + mmas * 2.0 ** -22


def bound(absprod, sum_w, sum_x, g, bias=0.0, res=0.0, out=0.0, pre=None, act="none", res_after_act=False, scale=1.0):
    """componentwise bound of |got - ref| (broadcasting float64 tensors): absprod = (|W| * |X|)_i, sum_w / sum_x the
    absolute operand sums of the 2^-36 floor, g = gamma(S) (or gamma_chain), pre = the exact pre-activation value"""
    mag = lambda t: torch.as_tensor(t, dtype=torch.float64, device=absprod.device).abs()
    e = g * absprod + 2.0 ** -36 * (sum_w + sum_x) + 2.0 ** -23 * mag(bias)
    if not res_after_act:
        e = e + 2.0 ** -23 * mag(res)
    if act == "sigmoid":
        s = torch.sigmoid(pre)
        d = s * (1 - s)
        e = (d + e) * (e + (2 + 1.173 * (pre.abs() + e)) * 2.0 ** -23)
    e = e * abs(scale)
    e = e + 2.0 ** -23 * mag(out)
    if res_after_act:
        e = e + 2.0 ** -23 * mag(res)
    return e


# ------------------------------------------------------------------------------------------------ emulated arithmetic
def _trunc32(x):
    """fp64 -> fp32 rounded towards zero"""
    t = x.float()
    over = t.double().abs() > x.abs()
    return torch.where(over, torch.nextafter(t, torch.zeros_like(t)), t).double()


def _rn32(x):
    return x.float().double()


def emulate_gemm(x, w, ntaps, drop_cols=None, drop_rows=None, plain=False):
    """The documented tc32 arithmetic on x [P, cin, ntaps] (activation columns) and w [Co, cin, ntaps]: K steps
    chunk-major / tap-minor, per step a fresh correction chain (A2 B, then A B2, one truncating fp32 accumulation per K16
    slab), scaled by 2^-11, the main chain A B on top (truncating), promoted into the sum with round-to-nearest.  Returns
    the fp32 sums [P, Co] as float64.

    Wrong kernels for the negative controls: drop_cols (output channels) / drop_rows (pixels) lose both correction
    products, plain feeds fp16(v) alone."""
    P, cin, _ = x.shape
    xa, xa2 = (t.double() for t in split16(x))
    wb, wb2 = (t.double() for t in split16(w))
    if plain:
        xa2, wb2 = torch.zeros_like(xa2), torch.zeros_like(wb2)
    keep = torch.ones(P, w.shape[0], dtype=torch.float64)
    if drop_cols is not None:
        keep[:, drop_cols] = 0
    if drop_rows is not None:
        keep[drop_rows, :] = 0
    total = torch.zeros(P, w.shape[0], dtype=torch.float64)
    for c0 in range(0, cin, STEP_K):
        slabs = [slice(s, min(s + SLAB, cin)) for s in range(c0, min(c0 + STEP_K, cin), SLAB)]
        for t in range(ntaps):
            acc = torch.zeros_like(total)
            for lhs, rhs in ((xa2, wb), (xa, wb2)):
                for sl in slabs:
                    acc = _trunc32(acc + lhs[:, sl, t] @ rhs[:, sl, t].T)
            acc = acc * keep / LO
            for sl in slabs:
                acc = _trunc32(acc + xa[:, sl, t] @ wb[:, sl, t].T)
            total = _rn32(total + acc)
    return total


def steps(cin, ntaps):
    return math.ceil(cin / STEP_K) * ntaps


# Contraction shapes of the dense componentwise test (test_gpu_tc32_numerics.py): name -> (cin, cout, taps per output, the
# K steps of the kernel that computes it).  The deconvolutions contract 4 (4x4) or 1 (2x2) taps per stride phase, the
# stem runs as a 4x4 convolution over 4 * 12 space-to-depth channels, the thin layer as a 1x1 over 9 tap-major outputs.
DENSE_SHAPES = {
    "halo_nwg2_bn128": (473, 256, 9),
    "halo_nwg4": (82, 16, 9),
    "flat_1x1_tma_nwg4": (64, 256, 1),
    "flat_3x3_s2": (48, 64, 9),
    "flat_5x5_s2": (128, 128, 25),
    "flat_7x7_s2_cin12": (12, 64, 49),
    "stem_s2d_4x4": (48, 64, 16),
    "deconv4x4_s2": (128, 64, 4),
    "deconv2x2_s2": (128, 64, 1),
    "thin_tap_major": (194, 18, 1),
    "dcn": (64, 128, 9),
}


def dense_operands(cin, cout, ntaps, npix, gen):
    """activations (fat x per-input-channel scales 2^-6 .. 2^6) and weights (fat x per-output-channel scales 2^-12 .. 2^6,
    like folded frozen-BN scales): x [npix, cin, ntaps], w [cout, cin, ntaps]"""
    xs = pow2_scales(cin, -6, 6, gen)
    ws = pow2_scales(cout, -12, 6, gen)
    x = (fat((npix, cin, ntaps), gen).double() * xs.view(1, -1, 1)).float()
    w = (fat((cout, cin, ntaps), gen).double() * ws.view(-1, 1, 1)).float()
    return x, w
