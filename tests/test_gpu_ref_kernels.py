"""The oracle's native-op restatements (oracle/ops.py) against the REFERENCE's OWN CUDA kernels: the extracted `__global__`
bodies of resample2d / channelnorm / correlation / ROIAlign / nms / deformable_im2col with the launch geometry of the
reference's launchers (oracle/ref_kernels/build.py), run on seeded inputs by tests/golden/make_ref_kernels_golden.py and
recorded in tests/golden/ref_kernels.npz.  This pins the oracle to the reference's actual kernels rather than to
transcriptions; the inputs are rebuilt here by the same functions, so no GPU is needed to check against the record."""
import os

import numpy as np
import pytest
import torch

from tests.golden import make_ref_kernels_golden as G

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_kernels.npz")


@pytest.fixture(scope="module")
def ref():
    return np.load(GOLD)


def _check(want, got, tol):
    """`got`: the reference kernel's values at G.sample_idx of the flattened output; `want`: the oracle's full output"""
    w = want.reshape(-1).numpy()[G.sample_idx(want.numel())]
    assert got.shape == w.shape
    assert float(np.abs(got - w).max()) <= tol


def test_resample2d_and_channelnorm(ref):
    from oracle import ops as O
    x, flow = G.resample_inputs()
    _check(O.resample2d(x, flow), ref["resample2d"], 2e-6 * float(x.abs().max()))
    cn = O.channelnorm(x)
    _check(cn, ref["channelnorm"], 1e-6 * float(cn.max()))


@pytest.mark.parametrize("pad,md,s2,C", G.CORR_CASES)
def test_correlation(ref, pad, md, s2, C):
    """both call sites of the path: FlowNetC (pad 20, d 20, s2 2) and LiteFlowNetCorr (pad 4, d 4, s2 1)"""
    from oracle import ops as O
    f1, f2 = G.correlation_inputs(C)
    want = O.correlation(f1, f2, pad, 1, md, 1, s2)
    D, oh, ow = G.correlation_shape(pad, md, s2, f1.shape[2], f1.shape[3])
    assert tuple(want.shape) == (f1.shape[0], D * D, oh, ow)
    _check(want, ref["correlation_%d_%d_%d_%d" % (pad, md, s2, C)], 1e-5 * max(1.0, float(want.abs().max())))


def test_roi_align(ref):
    from oracle import ops as O
    feat, rois = G.roi_inputs()
    for S, scale in G.ROI_CASES:
        want = O.roi_align(feat, rois, S, scale, 2)
        _check(want, ref["roi_align_%d" % S], 1e-5 * max(1.0, float(want.abs().max())))


def test_nms(ref):
    """nms_kernel's bit mask + the host reduction of nms_cuda (nms_kernel.cu:99-121) == oracle.ops.nms, exactly"""
    from oracle import ops as O
    for dets in G.nms_inputs():
        n = dets.shape[0]
        _, want = O.nms(dets, 0.5)
        assert torch.equal(torch.from_numpy(ref["nms_keep_%d" % n]).long(), want.sort()[0]), n


def test_deformable_im2col(ref):
    from oracle import ops as O
    x, off = G.deform_inputs()
    B, C, H, W = x.shape
    want = O.deform_im2col(x, off).reshape(B, C * 9, H * W)            # c-major, tap-minor
    _check(want, ref["deform_im2col"], 1e-5 * max(1.0, float(want.abs().max())))
