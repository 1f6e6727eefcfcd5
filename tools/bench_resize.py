"""Time the two ends of the test path for frames of any size on the GPU:

  resize HxW        vps_preprocess_resize_u8: cv2 INTER_LINEAR to the keep-ratio size under img_scale (2048, 1024) +
                    Normalize + Pad(32) + NCHW fp32 write, one pass (1080x1920, 720x1280, 2160x3840)
  identity          vps_preprocess_u8 at 1024x2048 (no Resize), for comparison
  nearest           vps_seg_confusion_nearest: a 1024x1820 uint8 prediction counted against a 1080x1920 gt through
                    Pillow's NEAREST tables (what evaluate_ssegs does for such a prediction)
  host resize       cv2.resize + imnormalize on the host for the same frames, for context (oracle/pipeline.py's numpy
                    normalisation; OpenCV's own thread count)

    python tools/bench_resize.py [--iters 200] [--warmup 20]

Device times: CUDA events around --iters back-to-back calls after --warmup calls, per call.  Each line states its HBM floor:
the bytes the pass must move (source frame read once, fp32 tensor written once; gt + prediction read once for the
confusion) over the data-sheet 3.35 TB/s -- a bound, not a measurement.  Host times: median of repeated perf_counter runs.
Prints the card and its power limit, then one JSON line."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.bench_ipq import card  # noqa: E402

HBM = 3.35e12


def time_calls(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters            # µs per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    from oracle import pipeline as OP
    from vps_b200 import ops
    from vps_b200._lib import lib
    from vps_b200.ipq import nearest_table
    from vps_b200.pipeline import InputStage
    L = lib()
    st = InputStage(resize=True)
    rng = np.random.default_rng(0)
    res = {}
    name, q = card()
    print("card: %s, power limit / max SM clock: %s" % (name, q))
    for h, w in ((1080, 1920), (720, 1280), (2160, 3840), (1024, 2048)):
        img = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
        d = torch.from_numpy(img).cuda()
        oh, ow, hp, wp, _ = st.geometry(h, w)
        out = torch.empty(1, 3, hp, wp, device="cuda")
        if (oh, ow) == (h, w):
            key = "identity_%dx%d" % (h, w)
            fn = lambda: L.vps_preprocess_u8(ops._ptr(d), h, w, st.mean, st.std, 1, ops._ptr(out), hp, wp, ops.stream())  # noqa: E731
        else:
            key = "resize_%dx%d" % (h, w)
            fn = lambda: L.vps_preprocess_resize_u8(ops._ptr(d), h, w, oh, ow, st.mean, st.std, 1, ops._ptr(out), hp, wp,  # noqa: E731
                                                    ops.stream())
        ops.check(fn(), key)
        us = time_calls(fn, args.iters, args.warmup)
        nbytes = h * w * 3 + 3 * hp * wp * 4
        host = []
        for _ in range(5):
            t = time.perf_counter()
            OP.imnormalize(_cv2_resize(img, oh, ow), [123.675, 116.28, 103.53], [58.395, 57.12, 57.375])
            host.append((time.perf_counter() - t) * 1e6)
        res[key] = dict(us=round(us, 2), out=[hp, wp], mb=round(nbytes / 1e6, 1), floor_us=round(nbytes / HBM * 1e6, 1),
                        host_cv2_normalize_us=round(float(np.median(host)), 0))
        print("%-22s %8.2f us/call   moves %5.1f MB -> HBM floor %5.1f us (data sheet)   host cv2.resize + imnormalize %8.0f us"
              % (key, us, nbytes / 1e6, nbytes / HBM * 1e6, np.median(host)))
    # the confusion of a 1024x1820 prediction against a 1080x1920 gt
    gh, gw, ph, pw = 1080, 1920, 1024, 1820
    gt = torch.from_numpy(rng.integers(0, 19, size=(gh // 8, gw // 8)).repeat(8, 0).repeat(8, 1).astype(np.uint8)).cuda()
    pred = torch.from_numpy(rng.integers(0, 19, size=(ph // 4, pw // 4)).repeat(4, 0).repeat(4, 1).astype(np.uint8)).cuda()
    xt, yt = (torch.from_numpy(nearest_table(s, t)).cuda() for s, t in ((pw, gw), (ph, gh)))
    conf = torch.zeros(19 * 19, dtype=torch.int64, device="cuda")
    fn = lambda: L.vps_seg_confusion_nearest(ops._ptr(gt), gh, gw, ops._ptr(pred), 1, ph, pw, ops._ptr(xt), ops._ptr(yt), 19,  # noqa: E731
                                             ops._ptr(conf), ops.stream())
    ops.check(fn(), "seg_confusion_nearest")
    us = time_calls(fn, args.iters, args.warmup)
    nbytes = gh * gw + ph * pw
    res["nearest_1024x1820_to_1080x1920"] = dict(us=round(us, 2), mb=round(nbytes / 1e6, 1), floor_us=round(nbytes / HBM * 1e6, 1))
    print("%-22s %8.2f us/call   moves %5.1f MB -> HBM floor %5.1f us (data sheet)" % ("nearest 1024x1820->1080x1920", us,
                                                                                        nbytes / 1e6, nbytes / HBM * 1e6))
    print(json.dumps(dict(card=name, limits=q, **res)))


def _cv2_resize(img, oh, ow):
    import cv2
    return cv2.resize(img, (ow, oh), interpolation=cv2.INTER_LINEAR) if (oh, ow) != img.shape[:2] else img


if __name__ == "__main__":
    main()
