"""Time and error of the tc32 convolution (vps_conv2d_tc32) per layer shape, next to the bf16 tensor-core and the fp32
CUDA-core kernels.

    python tools/bench_tc32.py [--err] [--big]
"""
import os
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vps_b200 import ops                                   # noqa: E402
from vps_b200.layers import empty_nhwc                     # noqa: E402

SHAPES = [
    # cin, cout, h, w, k, stride
    (256, 256, 256, 512, 3, 1),     # FPN P2 / TCEA 3x3
    (64, 64, 256, 512, 3, 1),       # ResNet layer1 conv2
    (64, 256, 256, 512, 1, 1),      # ResNet layer1 conv3
    (256, 64, 256, 512, 1, 1),      # ResNet layer1 conv1
    (128, 128, 128, 256, 3, 1),
    (512, 512, 32, 64, 3, 1),
    (1024, 2048, 32, 64, 1, 1),
    (82, 16, 1024, 2048, 3, 1),     # FlowNetFusion conv0
    (128, 256, 128, 256, 5, 2),     # FlowNet conv3 5x5 s2
]
ERR_SHAPES = [(256, 256, 64, 96, 3, 1), (1026, 2, 8, 16, 3, 1), (2304, 256, 16, 24, 1, 1), (64, 256, 64, 64, 1, 1), (12544, 64, 1, 128, 1, 1)]


def run(shape, dtype, tc, reps=10):
    cin, cout, h, w, k, s = shape
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1, h, w, cin, generator=g).to(dev)
    wt = (torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).to(dev)
    b = torch.randn(cout, generator=g).to(dev)
    pk = ops.PackedConv(wt, b)
    xd = empty_nhwc(1, h, w, cin, dtype, dev)
    xd.copy_(x.to(dtype))
    pad = k // 2
    oh, ow = (h + 2 * pad - k) // s + 1, (w + 2 * pad - k) // s + 1
    y = empty_nhwc(1, oh, ow, cout, dtype, dev)
    ops.F32_TC[0] = tc
    f = lambda: ops.conv2d(xd, pk, y, stride=s, pad=pad, act=ops.ACT_RELU, use_tc=tc)
    for _ in range(3):
        f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        f()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    fl = 2.0 * oh * ow * cout * cin * k * k
    return ms, fl / ms / 1e9, (x, wt, b, y, pad, s)


def main():
    if "--err" in sys.argv:
        for shape in ERR_SHAPES:
            ms, tf, (x, wt, b, y, pad, s) = run(shape, torch.float32, True, reps=2)
            ref = F.relu(F.conv2d(x.cpu().permute(0, 3, 1, 2).double(), wt.cpu().double(), b.cpu().double(), stride=s, padding=pad))
            got = y.cpu().permute(0, 3, 1, 2).double()
            d = got - ref
            ms2, _, (_, _, _, y2, _, _) = run(shape, torch.float32, False, reps=2)
            d2 = y2.cpu().permute(0, 3, 1, 2).double() - ref
            sc = float(ref.abs().max())
            print("err %-28s tc32 max %.3e mean-signed*sign(ref) %.3e | simt max %.3e  (scale %.2f)" %
                  (shape, float(d.abs().max()) / sc, float((d * ref.sign()).mean()) / sc, float(d2.abs().max()) / sc, sc), flush=True)
    shapes = SHAPES if "--big" in sys.argv else SHAPES[:1]
    for shape in shapes:
        r32 = run(shape, torch.float32, True)
        rbf = run(shape, torch.bfloat16, True)
        print("time %-32s tc32 %8.3f ms %7.1f TF/s | bf16 %8.3f ms %7.1f TF/s | ratio %.2f" %
              (shape, r32[0], r32[1], rbf[0], rbf[1], r32[0] / rbf[0]), flush=True)


if __name__ == "__main__":
    main()
