"""Frames per second of the reference's three Cityscapes models -- PanopticFuseTrack, PanopticTrack and PanopticFuse -- at
1024x2048 in tc32 and bf16, through ClipRunner over 30-frame synthetic clips with the frames resident on the device.

Every model carries the synthetic weight set "C" (vps_b200.synth, FuseTrack's tree, restricted to each model's keys).
Each (model, precision) runs one warm-up clip (graph capture, weight packing), then `--clips` timed clips; a clip is
timed with CUDA events around the whole ClipRunner loop, so frames/s includes the per-frame host round trips and the
label-map downloads.  Before timing, the first frame of a clip run through ClipRunner is checked bit for bit against a
direct `simple_test` call.  The card name and its power limit are printed with the numbers.

    python tools/bench_models.py [--frames 30] [--clips 3] [--precisions tc32,bf16]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, W = 1024, 2048


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out


def build_all():
    from vps_b200 import ConfigDict, build_detector, fuse_cfg, fusetrack_cfg, track_cfg
    from vps_b200.synth import make_weights
    dets = {}
    sd = None
    for name, f in (("PanopticFuseTrack", fusetrack_cfg), ("PanopticTrack", track_cfg), ("PanopticFuse", fuse_cfg)):
        c = f()
        det = build_detector(ConfigDict(c["model"]), train_cfg=None, test_cfg=ConfigDict(c["test_cfg"]))
        if sd is None:
            make_weights(det, "C", 0)
            sd = det.state_dict()
        else:
            det.load_state_dict({k: sd[k] for k in det.state_dict()}, strict=True)
        det.label_dtype = torch.uint8
        dets[name] = det.cuda()
    return dets


def clip(n, seed):
    from tests.e2e_util import meta
    g = torch.Generator().manual_seed(seed)
    imgs = [torch.randn(1, 3, H, W, generator=g).cuda() for _ in range(n)]
    metas = [meta(10001 + t, H, W) for t in range(n)]
    return imgs, metas


def pairs_for(det, imgs):
    if det.with_flow:          # the reference frame of frame t is frame t - 1; the first frame references itself
        return [(imgs[t], imgs[max(t - 1, 0)]) for t in range(len(imgs))]
    return [(x, None) for x in imgs]


def check_one_frame(det, imgs, metas):
    """the first frame through ClipRunner == a direct simple_test call, bit for bit"""
    from vps_b200.runner import ClipRunner
    pairs = pairs_for(det, imgs[:2])
    det.reset_tracker()
    r = det.simple_test(pairs[0][0], [metas[0]], ref_img=[pairs[0][1]] if pairs[0][1] is not None else None)
    want = (r[2]["panoptic_outputs"].cpu(), r[2]["fcn_outputs"].cpu(), r[2]["panoptic_cls_inds"].cpu())
    det.reset_tracker()
    got = list(ClipRunner(det, "cuda:0").run(pairs, metas[:2], resident=True))[0]
    ok = torch.equal(want[0], got[2]["panoptic_outputs"]) and torch.equal(want[1], got[2]["fcn_outputs"]) and \
        torch.equal(want[2], got[2]["panoptic_cls_inds"].cpu())
    assert ok, "%s: a ClipRunner frame differs from the direct simple_test call" % type(det).__name__


def time_clip(det, pairs, metas):
    from vps_b200.runner import ClipRunner
    det.reset_tracker()
    runner = ClipRunner(det, "cuda:0")
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    n = sum(1 for _ in runner.run(pairs, metas, resident=True))
    e.record()
    e.synchronize()
    return n / (s.elapsed_time(e) / 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--clips", type=int, default=3)
    ap.add_argument("--precisions", default="tc32,bf16")
    args = ap.parse_args()
    name, plimit = card()
    print("card: %s, power limit %s" % (name, plimit))
    dets = build_all()
    imgs, metas = clip(args.frames, 5)
    results = []
    for precision in args.precisions.split(","):
        for mname, det in dets.items():
            det.precision = precision
            check_one_frame(det, imgs, metas)
            pairs = pairs_for(det, imgs)
            time_clip(det, pairs, metas)                                   # warm-up clip
            fps = [time_clip(det, pairs, metas) for _ in range(args.clips)]
            res = dict(model=mname, precision=precision, frames=args.frames, fps=[round(v, 3) for v in fps],
                       fps_median=round(sorted(fps)[len(fps) // 2], 3))
            results.append(res)
            print("%-18s %-5s %5.2f frames/s  (clips: %s)" % (mname, precision, res["fps_median"],
                                                             " ".join("%.2f" % v for v in fps)), flush=True)
        for det in dets.values():
            det.prepare(force=True)          # free the graphs and packed weights of this precision
        torch.cuda.empty_cache()
    print(json.dumps(dict(card=name, power_limit=plimit, H=H, W=W, results=results)))


if __name__ == "__main__":
    main()
