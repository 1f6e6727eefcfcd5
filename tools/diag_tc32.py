"""Per-layer diagnosis of the tc32 convolution kernels: median CUDA-event time with an L2 flush between calls, algorithmic
TFLOP/s, and the bytes the layer must move (fp32 in + out + residual) against the HBM copy peak.

    python tools/diag_tc32.py [--dcn] [--only SUBSTR]
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vps_b200 import ops                                   # noqa: E402
from vps_b200.layers import empty_nhwc                     # noqa: E402

HBM_GBPS = 6572.5
# n, cin, cout, out_h, out_w, k, stride, residual, note
SHAPES = [
    (1, 256, 256, 256, 512, 3, 1, 0, "FPN/TCEA 3x3 (fat)"),
    (2, 64, 256, 256, 512, 1, 1, 1, "R50 l1 conv3 + residual"),
    (2, 64, 256, 256, 512, 1, 1, 0, "R50 l1 conv3, no residual"),
    (2, 256, 64, 256, 512, 1, 1, 0, "R50 l1 conv1"),
    (2, 64, 64, 256, 512, 3, 1, 0, "R50 l1 conv2"),
    (2, 128, 512, 128, 256, 1, 1, 1, "R50 l2 conv3 + residual"),
    (2, 256, 1024, 64, 128, 1, 1, 1, "R50 l3 conv3 + residual"),
    (2, 1024, 256, 64, 128, 1, 1, 0, "R50 l3 conv1"),
    (2, 256, 256, 64, 128, 3, 1, 0, "R50 l3 conv2"),
    (1, 128, 256, 128, 256, 5, 2, 0, "FlowNet conv3 5x5 s2"),
    (1, 64, 128, 256, 512, 5, 2, 0, "FlowNet conv2 5x5 s2"),
    (1, 64, 64, 512, 1024, 3, 2, 0, "FlowNetSD 3x3 s2"),
    (1, 82, 16, 1024, 2048, 3, 1, 0, "Fusion conv0"),
    (1, 12, 64, 512, 1024, 4, 1, 0, "stem (s2d form)"),
    (1, 48, 64, 512, 1024, 4, 1, 0, "FlowNetSD stem (s2d form)"),
    (1, 162, 32, 512, 1024, 3, 1, 0, "Fusion conv1 162->32"),
    (1, 6, 64, 1024, 2048, 3, 1, 0, "FlowNetSD conv0 6->64"),
    (1, 11, 64, 1024, 2048, 3, 1, 0, "Fusion 11->64"),
    (1, 256, 18, 256, 512, 3, 1, 0, "tap head 256->18"),
    (1, 16, 2, 1024, 2048, 3, 1, 0, "predict_flow full res"),
    (1, 194, 2, 256, 512, 3, 1, 0, "predict_flow2"),
    (1, 1024, 2, 16, 32, 3, 1, 0, "predict_flow6"),
    (1, 1024, 1024, 16, 32, 3, 1, 0, "conv6_1"),
]
# ConvTranspose2d(4, 2, 1) as four 2x2 stride-phase problems in one launch: n, cin, cout, in_h, in_w, note
DECONVS = [
    (1, 162, 16, 512, 1024, "Fusion deconv 162->16"),
    (1, 386, 64, 128, 256, "FlowNet deconv 386->64"),
    (1, 128, 32, 256, 512, "Fusion deconv 128->32"),
    (1, 770, 128, 64, 128, "FlowNet deconv 770->128"),
]
flush = None


def plan_str(plan):
    """nwg, layout (P pixel groups x Q channel groups), channels per warpgroup, epilogue"""
    return "nwg %d layout %dx%d bn %d/wg %s" % (plan["nwg"], plan["layout"][0], plan["layout"][1], plan["block_n"] // plan["wg_n"],
                                                 plan["epilogue"])


def timeit(fn, iters=5):
    fn()
    torch.cuda.synchronize()
    evs = []
    for i in range(iters):
        flush.fill_(i)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        evs.append((a, b))
    torch.cuda.synchronize()
    return sorted(a.elapsed_time(b) for a, b in evs)[len(evs) // 2]


def main():
    global flush
    dev = torch.device("cuda:0")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    only = sys.argv[sys.argv.index("--only") + 1] if "--only" in sys.argv else None
    ops.F32_TC[0] = True
    for (n, cin, cout, oh, ow, k, s, res, note) in SHAPES:
        if only and only not in note:
            continue
        g = torch.Generator().manual_seed(1)
        h, w = oh * s, ow * s
        x = empty_nhwc(n, h, w, cin, torch.float32, dev)
        x.copy_(torch.randn(n, h, w, cin, generator=g).to(dev))
        wt = (torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).to(dev)
        b = torch.randn(cout, generator=g).to(dev)
        pk = ops.PackedConv(wt, b)
        y = empty_nhwc(n, oh, ow, cout, torch.float32, dev)
        r = None
        if res:
            r = empty_nhwc(n, oh, ow, cout, torch.float32, dev)
            r.copy_(torch.randn(n, oh, ow, cout, generator=g).to(dev))
        pad = k // 2 if s == 1 or k % 2 else 1
        f = lambda: ops.conv2d(x, pk, y, stride=s, pad=pad, act=ops.ACT_RELU, res=r, use_tc=True, oh=oh, ow=ow)
        plan = ops.conv2d_tc32_plan(x, pk, stride=s, pad=pad, oh=oh, ow=ow, y=y, res=r)
        sys.stderr.flush()
        ms = timeit(f)
        fl = 2.0 * n * oh * ow * cout * cin * k * k
        by = 4.0 * n * (h * w * cin + oh * ow * cout * (2 if res else 1))
        print("%-28s %dx%d s%d %4d->%4d @%dx%d n%d: %.4f ms  %6.1f TF/s alg  %6.1f MB  hbm-floor %.4f ms (%.2f of it)  "
              "%s" % (note, k, k, s, cin, cout, oh, ow, n, ms, fl / ms / 1e9, by / 1e6, by / HBM_GBPS / 1e6,
                      by / HBM_GBPS / 1e6 / ms, plan_str(plan)), flush=True)
        del x, y, r, pk
    from vps_b200.layers import deconv4x4_s2
    for (n, cin, cout, h, w, note) in DECONVS:
        if only and only not in note:
            continue
        g = torch.Generator().manual_seed(1)
        x = empty_nhwc(n, h, w, cin, torch.float32, dev)
        x.copy_(torch.randn(n, h, w, cin, generator=g).to(dev))
        layer = deconv4x4_s2((torch.randn(cin, cout, 4, 4, generator=g) / (cin * 4) ** 0.5).to(dev),
                             torch.randn(cout, generator=g).to(dev))
        y = empty_nhwc(n, 2 * h, 2 * w, cout, torch.float32, dev)
        plan = ops.conv2d_tc32_plan(x, [ph[3] for ph in layer.phases], pads=[ph[2] for ph in layer.phases], oh=h, ow=w, y=y,
                                    omaps=[(2, ph[0], 2, ph[1]) for ph in layer.phases])
        ms = timeit(lambda: layer(x, y, act=ops.ACT_LRELU))
        fl = 2.0 * n * h * w * cout * cin * 16
        print("%-28s 2x2 x4 phases %4d->%4d @%dx%d n%d: %.4f ms  %6.1f TF/s alg  %s" % (note, cin, cout, h, w, n, ms, fl / ms / 1e9,
                                                                                       plan_str(plan)), flush=True)
        del x, y, layer
    if "--dcn" in sys.argv:
        for (h, w) in [(256, 512), (128, 256), (64, 128), (32, 64)]:
            for (ci, co) in [(256, 256), (256, 128), (128, 128)]:
                g = torch.Generator().manual_seed(0)
                x = torch.randn(1, h, w, ci, generator=g).to(dev)
                off = (torch.randn(1, h, w, 18, generator=g) * 1.5).to(dev)
                wt = (torch.randn(co, ci, 3, 3, generator=g) / (ci * 9) ** 0.5).to(dev)
                pk = ops.PackedConv(wt, None)
                y = torch.empty(1, h, w, co, dtype=torch.float32, device=dev)
                ms = timeit(lambda: ops.deform_conv_tc32(x, off, pk, y))
                fl = 2.0 * h * w * co * ci * 9
                plan = ops.deform_conv_tc32_plan(x, pk)
                print("dcn32 %3d->%3d @%3dx%3d: %.4f ms  %6.1f TF/s alg  %s %d px bn %d, %d N tiles"
                      % (ci, co, h, w, ms, fl / ms / 1e9, plan["layout"], plan["rows"], plan["bn"], plan["n_tiles"]), flush=True)


if __name__ == "__main__":
    main()
