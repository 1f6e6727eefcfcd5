"""The CPU model of the tc32 precision (tests/tc32_model.py): the operand split is exact as specified at the edges of the
fp16 range, the emulated arithmetic of the tc32 kernels stays within the componentwise bound on the contraction shapes of
the GPU test, and three emulated wrong kernels (corrections lost for one output channel, for one warpgroup's 64 pixels, or
everywhere) violate it on the same data: the bound is tight enough for the GPU tests to notice such bugs."""
import math

import pytest
import torch

from tests import tc32_model as M


def _bits(h):
    return h.view(torch.int16).item()


@pytest.mark.parametrize("v,a,a2", [
    (1.0, 1.0, 0.0),
    (1.0 + 2.0 ** -11, 1.0, 1.0),                        # half an fp16 ulp above 1: ties to even, A2 carries it
    (1.0 + 3 * 2.0 ** -11, 1.0 + 2.0 ** -9, -1.0),
    (2.0 ** -14, 2.0 ** -14, 0.0),                       # smallest normal fp16
    (2.0 ** -14 + 2.0 ** -30, 2.0 ** -14, 2.0 ** -19),   # below the subnormal grid of A, carried by A2
    (2.0 ** -24, 2.0 ** -24, 0.0),                       # smallest subnormal fp16
    (2.0 ** -25, 0.0, 2.0 ** -14),                       # ties to even: A = 0, A2 = 2^11 v (normal)
    (2.0 ** -25 + 2.0 ** -40, 2.0 ** -24, -(2.0 ** -14)),     # A2 = -2^-14 + 2^-29 rounds onto the 2^-24 grid
    (3 * 2.0 ** -27, 0.0, 3 * 2.0 ** -16),               # A2 subnormal: still exact on the 2^-24 grid
    (2.0 ** -40, 0.0, 0.0),                              # below the 2^-36 floor: lost
    (65504.0, 65504.0, 0.0),
    (65505.0, 65504.0, 2048.0),                          # saturated main plane (counted), A2 still carries the rest
    (65536.0, 65504.0, 65504.0),                         # both planes saturated
    (1e6, 65504.0, 65504.0),
    (-65505.0, -65504.0, -2048.0),
])
def test_split_edges(v, a, a2):
    A, A2 = M.split16(torch.tensor([v]))
    assert A.item() == a and A2.item() == a2, (v, A.item(), A2.item())


def test_split_signed_zero_nan_inf():
    A, A2 = M.split16(torch.tensor([0.0, -0.0, float("nan"), float("inf"), float("-inf")]))
    assert _bits(A[0]) == 0 and _bits(A2[0]) == 0
    assert _bits(A[1]) == -32768 and _bits(A2[1]) == 0      # -0 keeps its sign in A; v - A = +0
    assert math.isnan(A[2].item()) and math.isnan(A2[2].item())
    assert A[3].item() == 65504.0 and A2[3].item() == 65504.0
    assert A[4].item() == -65504.0 and A2[4].item() == -65504.0


def test_split_carries_22_bits_and_floor():
    """|v - (A + 2^-11 A2)| <= 2^-22 |v| + 2^-36 over the whole fp32 range the kernels use without saturation"""
    g = torch.Generator().manual_seed(1)
    v = (torch.randn(200000, generator=g, dtype=torch.float64) * torch.pow(2.0, torch.randint(-40, 16, (200000,), generator=g))).float()
    v = v[v.abs() <= M.F16_MAX]
    err = (M.carried(v) - v.double()).abs()
    assert bool((err <= 2.0 ** -22 * v.double().abs() + 2.0 ** -36).all())
    assert float((err / v.double().abs())[v.abs() >= 2.0 ** -14].max()) > 2.0 ** -24     # and the 2^-22 is not vacuous


def test_fat_operands():
    g = torch.Generator().manual_seed(2)
    v = M.fat((4096,), g)                          # asserts split16(v) == (A, A2) itself
    A, A2 = M.split16(v)
    a, a2 = A.double().abs(), A2.double().abs()
    assert bool((a >= 0.5).all()) and bool((a < 2).all())
    ulp = torch.pow(2.0, torch.floor(torch.log2(a)) - 10)
    assert bool((a2 >= 0.25 * 1024 * ulp).all()) and bool((a2 <= 0.75 * 1024 * ulp).all())
    assert bool((a2 / M.LO >= 2.0 ** -14 * a).all())     # a dropped correction moves a product by >= 2^-14 of its size


def _case(name, npix=256, seed=0):
    cin, cout, ntaps = M.DENSE_SHAPES[name]
    g = torch.Generator().manual_seed(1000 + seed + cin * 7 + cout)
    x, w = M.dense_operands(cin, cout, ntaps, npix, g)
    xd, wd = x.double(), w.double()
    ref = torch.einsum("pct,oct->po", xd, wd)
    absprod = torch.einsum("pct,oct->po", xd.abs(), wd.abs())
    sum_w = wd.abs().sum((1, 2)).view(1, -1)
    sum_x = xd.abs().sum((1, 2)).view(-1, 1)
    b = M.bound(absprod, sum_w, sum_x, M.gamma(M.steps(cin, ntaps)), out=ref)
    return x, w, ntaps, ref, b


@pytest.mark.parametrize("name", sorted(M.DENSE_SHAPES))
def test_emulated_kernel_within_bound_and_wrong_kernels_violate_it(name):
    x, w, ntaps, ref, b = _case(name)
    got = M.emulate_gemm(x, w, ntaps)
    ratio = float(((got - ref).abs() / b).max())
    print("%s: emulated worst err / bound %.3f" % (name, ratio))
    assert ratio <= 1.0
    # one output channel loses both correction products (a slab, tap or chunk of N): caught in that channel
    co = w.shape[0] // 2
    bad = M.emulate_gemm(x, w, ntaps, drop_cols=[co])
    assert float(((bad - ref).abs() / b)[:, co].max()) > 1.0, name
    # one warpgroup's 64 pixels lose them
    bad = M.emulate_gemm(x, w, ntaps, drop_rows=slice(64, 128))
    assert float(((bad - ref).abs() / b)[64:128].max()) > 1.0, name
    # plain fp16 operands
    bad = M.emulate_gemm(x, w, ntaps, plain=True)
    assert float(((bad - ref).abs() / b).max()) > 1.0, name


def test_probe_bound_separates_a_lost_correction():
    """one product of fat operands: the emulated kernel is within 2^-20 of it, a lost correction product is >= 2^-14 off"""
    g = torch.Generator().manual_seed(3)
    x = M.fat((512, 1, 1), g)
    w = M.fat((1, 1, 1), g)
    ref = x.double()[:, 0, 0] * w.double()[0, 0, 0]
    got = M.emulate_gemm(x, w, 1)[:, 0]
    assert bool(((got - ref).abs() <= 2.0 ** -20 * ref.abs()).all())
    A, A2 = (t.double() for t in M.split16(x))
    B, B2 = (t.double() for t in M.split16(w))
    for lost in (A2 * B / M.LO, A * B2 / M.LO):
        assert bool((lost[:, 0, 0].abs() >= 2.0 ** -14 * ref.abs()).all())
