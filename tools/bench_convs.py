"""Time a list of the step's convolution shapes through vps_conv2d_tc (median of N, L2 flushed between runs).
Usage: python tools/bench_convs.py [--iters N] [--set small|all]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from vps_b200 import ops  # noqa: E402
from vps_b200.layers import Conv  # noqa: E402

# cin, cout, h, w, k, stride   (input h, w)
SHAPES = [
    (82, 16, 1024, 2048, 3, 1), (11, 64, 1024, 2048, 3, 1), (6, 64, 1024, 2048, 3, 1), (16, 2, 1024, 2048, 3, 1),
    (162, 32, 512, 1024, 3, 1), (48, 64, 512, 1024, 4, 1), (12, 64, 512, 1024, 4, 1), (64, 128, 512, 1024, 3, 1),
    (64, 64, 256, 512, 3, 1), (194, 2, 256, 512, 3, 1), (194, 64, 256, 512, 3, 1), (128, 128, 256, 512, 3, 1),
    (256, 256, 256, 512, 3, 1), (256, 18, 256, 512, 3, 1), (339, 64, 256, 512, 3, 1),
    (256, 256, 128, 256, 3, 1), (128, 128, 128, 256, 3, 1), (473, 256, 128, 256, 3, 1), (386, 2, 128, 256, 3, 1),
    (256, 256, 64, 128, 3, 1), (512, 512, 64, 128, 3, 1), (512, 512, 32, 64, 3, 1), (1024, 1024, 16, 32, 3, 1),
    (1024, 2, 16, 32, 3, 1), (256, 256, 14, 14, 3, 1),
    # flat mode: 1x1 and strided
    (64, 256, 256, 512, 1, 1), (256, 64, 256, 512, 1, 1), (128, 512, 128, 256, 1, 1), (1024, 256, 64, 128, 1, 1),
    (256, 1024, 64, 128, 1, 1), (512, 2048, 32, 64, 1, 1), (2304, 256, 256, 512, 1, 1), (64, 128, 512, 1024, 5, 2),
    (64, 64, 1024, 2048, 3, 2), (512, 512, 64, 128, 3, 2), (128, 256, 256, 512, 5, 2),
]
iters = int(sys.argv[sys.argv.index("--iters") + 1]) if "--iters" in sys.argv else 7
dev = torch.device("cuda:0")
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
tot = 0.0
for cin, cout, h, w, k, s in SHAPES:
    g = torch.Generator().manual_seed(0)
    n = 100 if h == 14 else 1
    cs = (cin + 7) // 8 * 8
    xb = torch.randn(n, h, w, cs, generator=g).to(dev).bfloat16()
    x = xb[..., :cin]
    conv = Conv((torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).to(dev), torch.zeros(cout, device=dev),
                stride=s, pad=(k - 1) // 2, act=ops.ACT_RELU)
    y = conv(x)
    torch.cuda.synchronize()
    evs = []
    for i in range(iters):
        flush.fill_(i)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        conv(x, y)
        b.record()
        evs.append((a, b))
    torch.cuda.synchronize()
    ms = sorted(a.elapsed_time(b) for a, b in evs)[len(evs) // 2]
    fl = 2.0 * n * y.shape[1] * y.shape[2] * cout * cin * k * k
    tot += ms
    print("conv %dx%d s%d %4d->%4d @%4dx%4d n%3d: %.4f ms  %7.1f TFLOP/s" % (k, k, s, cin, cout, y.shape[1], y.shape[2], n, ms, fl / ms / 1e9))
print("total %.3f ms" % tot)
