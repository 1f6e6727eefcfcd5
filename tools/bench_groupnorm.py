"""Time vps_groupnorm (GroupNorm(32) + ReLU) at the UPSNet head's shapes on the GPU, optionally against another build.

    python tools/bench_groupnorm.py [--iters 200] [--warmup 20] [--rounds 5] [--baseline-lib OTHER/libvps_b200.so]

Shapes: C = 256 and 128 on P2..P5 of a 1024x2048 frame (256x512 .. 32x64) and on the 272x480 level of a 1088x1920 frame,
in fp32 and bf16, dense NHWC in and out (the production launch arms).  Device times: --iters calls captured in one CUDA
graph (as the model runs them; no host launch gaps), CUDA events around a replay, per call, median of --rounds replays.
With --baseline-lib (the library another revision's `python -m vps_b200.build` made, copied elsewhere) the two builds
alternate replay by replay on the same seeded inputs, and their outputs are compared: max |this - other| over max |other|.
Each line gives the pass's algorithmic bytes (the map read twice and written once) over the time, and that rate as a share
of the data-sheet 3.35 TB/s.  Then the per-kernel device time of one call at the P2 shapes (torch.profiler), the card and
its power limit, and one JSON line.
"""
import argparse
import ctypes as C
import json
import os
import sys
from collections import defaultdict

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.bench_ipq import card  # noqa: E402

HBM = 3.35e12
SHAPES = [(c, h, w) for h, w in ((256, 512), (128, 256), (64, 128), (32, 64), (272, 480)) for c in (256, 128)]


def graph_of(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    g.replay()
    torch.cuda.synchronize()
    return g


def time_replay(g, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters            # µs per call


def kernel_times(fn, reps=20):
    """average device time per call of each kernel fn launches"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = defaultdict(float)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            nm = e.name.replace("(anonymous namespace)::", "").replace("void ", "").split("(")[0].strip()
            out[nm] += e.device_time_total / reps
    return dict(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--baseline-lib", default=None, help="a libvps_b200.so of another revision to alternate with")
    args = ap.parse_args()
    from vps_b200 import _lib, ops
    libs = {"this": _lib.lib()}
    if args.baseline_lib:
        libs["other"] = C.CDLL(os.path.abspath(args.baseline_lib))
    name, q = card()
    print("card: %s, power limit / max SM clock: %s" % (name, q))
    res, breakdown = {}, {}
    for dtype in (torch.float32, torch.bfloat16):
        for c, h, w in SHAPES:
            g = torch.Generator().manual_seed(c * h + w)
            x = (torch.randn(1, h, w, c, generator=g) * 2 + torch.randn(1, 1, 1, c, generator=g)).to(dtype).cuda()
            gamma = (torch.rand(c, generator=g) + 0.5).cuda()
            beta = torch.randn(c, generator=g).cuda()
            outs = {k: torch.empty_like(x) for k in libs}

            def call(k):
                L = libs[k]
                return lambda: ops.check(L.vps_groupnorm(ops._bt(x), ops._bt(outs[k]), ops._ptr(gamma), ops._ptr(beta), 32,
                                                         C.c_float(1e-5), 1, ops.stream()), "groupnorm")
            graphs = {k: graph_of(call(k), args.iters, args.warmup) for k in libs}
            times = {k: [] for k in libs}
            for _ in range(args.rounds):
                for k in libs:
                    times[k].append(time_replay(graphs[k], args.iters))
            del graphs
            key = "%s_c%d_%dx%d" % ("f32" if dtype == torch.float32 else "bf16", c, h, w)
            nbytes = 3 * x.numel() * x.element_size()
            r = dict(mb=round(nbytes / 1e6, 1))
            line = "%-20s %6.1f MB" % (key, nbytes / 1e6)
            for k in libs:
                us = float(np.median(times[k]))
                r[k] = dict(us=round(us, 2), spread_us=round(max(times[k]) - min(times[k]), 2))
                line += "   %s %7.2f us (spread %5.2f) %5.2f TB/s = %3.0f%% of 3.35" % (
                    k, us, r[k]["spread_us"], nbytes / us / 1e6, 100 * nbytes / us / 1e6 / (HBM / 1e12))
            if "other" in libs:
                a, b = outs["this"].double(), outs["other"].double()
                r["max_diff_rel"] = float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))
                r["time_ratio"] = round(r["this"]["us"] / r["other"]["us"], 4)
                line += "   this/other %.3f   max|diff|/max|other| %.2e" % (r["time_ratio"], r["max_diff_rel"])
            print(line)
            res[key] = r
            if (h, w) == (256, 512):
                breakdown[key] = {k: kernel_times(call(k)) for k in libs}
    for key, per_lib in breakdown.items():
        for k, kt in per_lib.items():
            print("%-20s %-5s per kernel: %s" % (key, k, ", ".join("%s %.2f us" % kv for kv in sorted(kt.items()))))
    print(json.dumps(dict(card=name, limits=q, kernels=breakdown, **res)))


if __name__ == "__main__":
    main()
