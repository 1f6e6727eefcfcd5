"""Time one frame of the tracker (PanopticFuseTrack._track: track-head embedding, match, memory update, the one 4-byte
read-back) at a given number m of remembered tracks, with the full-size track head and k new detections.

    python tools/bench_tracker.py [--m 1024,4096,16384,65536] [--k 100] [--precision tc32] [--iters 30] [--kernels]

The memory is filled by running frames of k new detections (random RoI features, labels no track has, so each one opens
a track) until it holds m tracks; every timed frame then starts from those m tracks again.  Device events around each
frame, after warm-up frames of the same shape.  --kernels adds one torch.profiler run per m with the device time of each
kernel of the frame.  Prints the card and its power limit, then one JSON line per m."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


class _NoWeights(nn.Module):
    def prepare(self, force=False):
        return self


def tracker(precision):
    from vps_b200.default_cfg import fusetrack_cfg
    from vps_b200.detector import PanopticFuseTrack
    from vps_b200.registry import build_head
    det = PanopticFuseTrack.__new__(PanopticFuseTrack)
    nn.Module.__init__(det)
    for name in ("backbone", "neck", "extra_neck", "panopticFPN", "rpn_head", "bbox_head", "mask_head", "flownet2"):
        setattr(det, name, _NoWeights())
    torch.manual_seed(0)
    det.track_head = build_head(dict(fusetrack_cfg()['model']['track_head'])).cuda()
    det.precision = precision
    det._graphs, det._pf_queue, det._tail_done = {}, [], [None, None]
    det.reset_tracker()
    return det


class Detections:
    def __init__(self, k, dtype, roi_shape):
        self.k, self.dtype, self.roi_shape, self.next_label = k, dtype, roi_shape, 0
        self.g = torch.Generator(device="cuda").manual_seed(1)

    def __call__(self, n):
        feats = (torch.randn((n,) + self.roi_shape, generator=self.g, device="cuda") * 0.5).to(self.dtype)
        xy = torch.rand(n, 2, generator=self.g, device="cuda") * 1000
        boxes = torch.cat([xy, xy + 40], 1)
        labels = torch.arange(self.next_label, self.next_label + n, dtype=torch.int32, device="cuda")
        self.next_label += n
        probs = torch.rand(n, generator=self.g, device="cuda") * 0.3 + 0.65
        return feats, boxes, labels, probs


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = "unknown"
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", default="1024,4096,16384,65536")
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--precision", default="tc32", choices=["tc32", "bf16", "fp32"])
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--kernels", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_tracker needs a GPU"
    from vps_b200 import ops
    ops.F32_TC[0] = args.precision == "tc32"
    name, power = card()
    print("card: %s | power.limit, clocks.max.sm: %s" % (name, power), flush=True)
    dtype = torch.bfloat16 if args.precision == "bf16" else torch.float32
    th_cfg = tracker(args.precision).track_head
    roi_shape = (th_cfg.roi_feat_size, th_cfg.roi_feat_size, th_cfg.in_channels)
    k = args.k
    with torch.no_grad():
        for m in [int(v) for v in args.m.split(",")]:
            det = tracker(args.precision)
            dets = Detections(k, dtype, roi_shape)
            first = True
            while det.prev_n < m:
                n = min(k, m - det.prev_n)
                f, b, l, p = dets(n)
                det._track(f, b, l, p, n, first)
                first = False
            assert det.prev_n == m, (det.prev_n, m)
            frame = dets(k)

            def run():
                det.prev_n = m
                det._track(frame[0], frame[1], frame[2], frame[3], k, False)

            for _ in range(args.warmup):
                run()
            torch.cuda.synchronize()
            times = []
            for _ in range(args.iters):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run()
                e1.record()
                e1.synchronize()
                times.append(e0.elapsed_time(e1))
            times.sort()
            out = dict(m=m, k=k, precision=args.precision, ms_median=round(times[len(times) // 2], 4),
                       ms_min=round(times[0], 4), iters=args.iters, card=name, power_limit_and_max_sm_clock=power)
            if args.kernels:
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    run()
                    torch.cuda.synchronize()
                per = {}
                for ev in prof.events():
                    if ev.device_type.name == "CUDA":
                        key = ev.name.replace("(anonymous namespace)::", "").replace("void ", "")
                        key = key.split("(")[0].split("<")[0].split("::")[-1][:48]
                        per[key] = per.get(key, 0.0) + ev.device_time / 1000.0
                out["kernel_ms"] = {kk: round(v, 4) for kk, v in sorted(per.items(), key=lambda kv: -kv[1])}
            print(json.dumps(out), flush=True)
            del det


if __name__ == "__main__":
    main()
