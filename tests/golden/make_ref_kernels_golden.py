"""Record the REFERENCE's own CUDA kernels (resample2d / channelnorm / correlation / ROIAlign / nms / deformable_im2col, the
`__global__` bodies extracted by oracle/ref_kernels/build.py into oracle/_ref/libvps_ref_kernels.so) on seeded inputs into
tests/golden/ref_kernels.npz, which tests/test_gpu_ref_kernels.py compares oracle/ops.py against.

The inputs are built by the functions below (CPU torch generators), so the test rebuilds exactly the same tensors.  Outputs
larger than SAMPLE elements are stored at a fixed seeded sample of their flat positions (`sample_idx`) to keep the file small.
Run on a GPU machine after the reference kernels have been built:
    python tests/golden/make_ref_kernels_golden.py [out.npz]"""
import ctypes
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
LIB = os.path.join(ROOT, "oracle", "_ref", "libvps_ref_kernels.so")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_kernels.npz")
SAMPLE = 4096
CORR_CASES = [(20, 20, 2, 64), (4, 4, 1, 96)]        # pad, max displacement, stride2, C: FlowNetC and LiteFlowNetCorr
NMS_SIZES = (5, 64, 65, 700)


def sample_idx(size):
    if size <= SAMPLE:
        return np.arange(size)
    return np.sort(np.random.default_rng(0).choice(size, SAMPLE, replace=False))


def sampled(t):
    a = t.detach().cpu().reshape(-1).numpy()
    return a[sample_idx(a.size)].astype(np.float32)


def resample_inputs():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 5, 19, 27, generator=g)
    flow = (torch.rand(2, 2, 19, 27, generator=g) - 0.5) * 14
    return x, flow


def correlation_inputs(C):
    g = torch.Generator().manual_seed(2)
    B, H, W = 1, 24, 32
    return torch.randn(B, C, H, W, generator=g), torch.randn(B, C, H, W, generator=g)


def correlation_shape(pad, md, s2, H=24, W=32):
    D = 2 * (md // s2) + 1
    return D, H + 2 * pad - 2 * md, W + 2 * pad - 2 * md        # kernel 1, stride1 1


def roi_inputs():
    g = torch.Generator().manual_seed(3)
    feat = torch.randn(1, 16, 40, 56, generator=g)
    n = 37
    xy = torch.rand(n, 2, generator=g) * torch.tensor([200.0, 140.0])
    wh = torch.rand(n, 2, generator=g) * 90 + 1
    rois = torch.cat([torch.zeros(n, 1), xy, xy + wh], 1)
    rois[0, 1:] = torch.tensor([-20.0, -10.0, 5.0, 3.0])             # partly outside
    return feat, rois


ROI_CASES = ((7, 0.25), (14, 0.25))


def nms_inputs():
    g = torch.Generator().manual_seed(4)
    out = []
    for n in NMS_SIZES:
        xy = torch.rand(n, 2, generator=g) * 300
        wh = torch.rand(n, 2, generator=g) * 80 + 2
        out.append(torch.cat([xy, xy + wh, torch.rand(n, 1, generator=g)], 1))
    return out


def deform_inputs():
    g = torch.Generator().manual_seed(5)
    B, C, H, W = 2, 12, 13, 17
    x = torch.randn(B, C, H, W, generator=g)
    off = torch.randn(B, 18, H, W, generator=g) * 2.5
    off[:, :, 0] -= 4.0
    return x, off


def run_reference(ref):
    def P(t):
        return ctypes.c_void_p(t.data_ptr())

    res = {}
    # every device tensor is bound to a name until its kernel has run: a pointer taken from a temporary (`P(x.cuda())`) lets
    # the caching allocator hand the same memory to the next upload before the kernel reads it
    x, flow = resample_inputs()
    xd, fd = x.cuda(), flow.cuda()
    B, C, H, W = x.shape
    out = torch.empty(B, C, H, W, device="cuda")
    assert ref.ref_resample2d(P(xd), P(fd), P(out), B, C, H, W, H, W) == 0
    res["resample2d"] = sampled(out)
    o2 = torch.empty(B, 1, H, W, device="cuda")
    assert ref.ref_channelnorm(P(xd), P(o2), B, C, H, W) == 0
    res["channelnorm"] = sampled(o2)
    for pad, md, s2, C in CORR_CASES:
        f1, f2 = correlation_inputs(C)
        f1d, f2d = f1.cuda(), f2.cuda()
        B, _, H, W = f1.shape
        D, oh, ow = correlation_shape(pad, md, s2, H, W)
        rb1 = torch.empty(B, H + 2 * pad, W + 2 * pad, C, device="cuda")
        rb2 = torch.empty_like(rb1)
        out = torch.empty(B, D * D, oh, ow, device="cuda")
        assert ref.ref_correlation(P(f1d), P(f2d), P(rb1), P(rb2), P(out), B, C, H, W, D * D, oh, ow, pad, 1, md, 1,
                                   s2) == 0
        res["correlation_%d_%d_%d_%d" % (pad, md, s2, C)] = sampled(out)
    feat, rois = roi_inputs()
    featd, roisd = feat.cuda(), rois.cuda()
    n = rois.shape[0]
    for S, scale in ROI_CASES:
        out = torch.empty(n, 16, S, S, device="cuda")
        assert ref.ref_roi_align(P(featd), P(roisd), n, ctypes.c_float(scale), 2, 16, 40, 56, S, S, P(out)) == 0
        res["roi_align_%d" % S] = sampled(out)
    for dets in nms_inputs():
        n = dets.shape[0]
        order = torch.sort(dets[:, 4], descending=True, stable=True)[1]
        bsd = dets[order].contiguous().cuda()
        cb = (n + 63) // 64
        mask = torch.zeros(n * cb, dtype=torch.int64, device="cuda")
        assert ref.ref_nms_mask(P(bsd), n, ctypes.c_float(0.5), P(mask)) == 0
        m = mask.cpu().numpy().view(np.uint64).reshape(n, cb)
        remv = np.zeros(cb, np.uint64)
        keep = []
        for i in range(n):                                            # the reference's host loop (nms_kernel.cu:99-121)
            if not (int(remv[i // 64]) >> (i % 64)) & 1:
                keep.append(i)
                remv |= m[i]
        res["nms_keep_%d" % n] = torch.sort(order[torch.tensor(keep, dtype=torch.long)])[0].numpy().astype(np.int32)
    x, off = deform_inputs()
    xd, offd = x.cuda(), off.cuda()
    B, C, H, W = x.shape
    col = torch.empty(C * 9, B, H, W, device="cuda")
    assert ref.ref_deform_im2col(P(xd), P(offd), B, C, H, W, 3, 1, 1, 1, 1, P(col)) == 0
    res["deform_im2col"] = sampled(col.permute(1, 0, 2, 3).reshape(B, C * 9, H * W))   # [B, C*9, H*W] like the oracle
    return res


if __name__ == "__main__":
    out = sys.argv[1] if len(sys.argv) > 1 else OUT
    np.savez_compressed(out, **run_reference(ctypes.CDLL(LIB)))
    print("wrote", out, os.path.getsize(out) // 1024, "KiB")
