"""Time the evaluation of one 1024x2048 image of the image panoptic model (vps_b200.ipq) on the GPU, beside the numpy
restatement of the same work on the host (oracle/ipq.py, the reference's arithmetic):

  seg_confusion   vps_seg_confusion (uint8 gt, uint8 and int64 prediction)       -- semantic mIoU, per frame
  image_ids       vps_pan2ch_image_ids                                            -- the image converter's segment key
  pair_table      vps_tube_confusion on one frame (pack, radix sort, run-length encode)
  add_frame       IpqEvaluator.add_frame end to end: rgb_to_id + image ids + pair table + read-back + host bookkeeping
  host_matching   IpqEvaluator.compute on the frame's table (the reference's matching loop)

    python tools/bench_ipq.py [--iters 200] [--warmup 20]

Device times: CUDA events around --iters back-to-back calls after --warmup calls, reported per call (so launch overhead is
included: these kernels are bound by it, not by HBM), and the median of single-call event pairs.  Host times: the median
of repeated perf_counter measurements.  Prints the card and its power limit, then one JSON line."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

H, W = 1024, 2048


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = "unknown"
    return name, q


def frame(rng):
    """a Cityscapes-like frame: blocky stuff, ~30 thing instances; GT = prediction with shifted instances and a VOID band"""
    blocks = lambda hi, b: rng.integers(0, hi, size=(H // b, W // b)).repeat(b, 0).repeat(b, 1)    # noqa: E731
    sem = blocks(11, 64).astype(np.uint8)
    ins = np.zeros((H, W), np.uint8)
    gt_ids = (1000 * sem.astype(np.uint32) + 1)
    for j in range(30):
        h, w = int(rng.integers(20, 200)), int(rng.integers(20, 300))
        y, x = int(rng.integers(0, H - h - 8)), int(rng.integers(0, W - w - 8))
        c = int(rng.integers(11, 19))
        sem[y:y + h, x:x + w] = c
        ins[y:y + h, x:x + w] = j + 1
        gt_ids[y + 4:y + h + 4, x + 4:x + w + 4] = 1000 * c + j + 1
    gt_ids[:16] = 0
    p2 = np.stack([sem, ins, np.zeros_like(sem)], -1)
    fcn = sem.copy()
    trainid = np.where(gt_ids == 0, 255, (gt_ids - 1) // 1000).astype(np.uint8)
    gt_rgb = np.stack([gt_ids % 256, (gt_ids // 256) % 256, gt_ids // 65536], -1).astype(np.uint8)
    return p2, fcn, trainid, gt_ids, gt_rgb


def dev_time(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    loop_us = e0.elapsed_time(e1) * 1000.0 / iters
    single = []
    for _ in range(min(iters, 50)):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        single.append(a.elapsed_time(b) * 1000.0)
    return round(loop_us, 2), round(float(np.median(single)), 2)


def host_time(fn, reps):
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return round(float(np.median(t)) * 1e6, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ipq needs a GPU")
    from oracle import ipq as O
    from vps_b200 import ops
    from vps_b200._lib import lib
    from vps_b200.ipq import IpqEvaluator, SegEvaluator, image_segment_ids
    from vps_b200.vpq import frame_confusion, rgb_to_id
    name, power = card()
    print("card: %s | power.limit, clocks.max.sm: %s" % (name, power), flush=True)
    p2, fcn, trainid, gt_ids, gt_rgb = frame(np.random.default_rng(0))
    categories = {i: {"id": i, "isthing": int(i >= 11)} for i in range(19)}
    d_p2, d_fcn, d_tid, d_rgb = (torch.from_numpy(a).cuda() for a in (p2, fcn, trainid, gt_rgb))
    d_fcn64 = d_fcn.long()
    conf = torch.zeros(19 * 19, dtype=torch.int64, device="cuda")
    n = H * W
    out = dict(shape=[H, W], card=name, power_limit_and_max_sm_clock=power, iters=args.iters,
               unit="us per frame: [per call in a back-to-back loop, median single call]")

    def seg(pred):
        ops.check(lib().vps_seg_confusion(ops._ptr(d_tid), ops._ptr(pred), pred.element_size(), C.c_int64(n), 19,
                                          ops._ptr(conf), ops.stream()), "seg_confusion")
    out["seg_confusion_u8"] = dev_time(lambda: seg(d_fcn), args.iters, args.warmup)
    out["seg_confusion_i64"] = dev_time(lambda: seg(d_fcn64), args.iters, args.warmup)
    out["seg_confusion_hbm_floor_us"] = round((2 * n) / 3.35e12 * 1e6, 2)       # 2 x 2 MB read at the data-sheet 3.35 TB/s
    ids = image_segment_ids(d_p2)
    out["image_ids"] = dev_time(lambda: image_segment_ids(d_p2, 11), args.iters, args.warmup)
    gt = rgb_to_id(d_rgb)
    ws = torch.empty(int(lib().vps_tube_confusion_ws_bytes(C.c_int64(n))), dtype=torch.uint8, device="cuda")
    pairs = torch.empty(n, dtype=torch.int64, device="cuda")
    counts = torch.empty(n, dtype=torch.int32, device="cuda")
    nruns = torch.zeros(1, dtype=torch.int32, device="cuda")

    def table():
        ops.check(lib().vps_tube_confusion(ops._ptr(gt), ops._ptr(ids), C.c_int64(n), C.c_uint64(1 << 24), ops._ptr(pairs),
                                           ops._ptr(counts), ops._ptr(nruns), ops._ptr(ws), C.c_int64(ws.numel()), ops.stream()),
                  "tube_confusion")
    out["pair_table"] = dev_time(table, args.iters, args.warmup)
    gt_segs = [{"id": int(i), "category_id": int((i - 1) // 1000), "iscrowd": 0, "area": int(a)}
               for i, a in zip(*np.unique(gt_ids, return_counts=True)) if i != 0]

    def add():
        ev = IpqEvaluator(categories)
        ev.add_frame(d_rgb, gt_segs, d_p2)
        torch.cuda.synchronize()
        return ev
    for _ in range(3):
        ev = add()
    out["add_frame_host_clock_us"] = host_time(add, args.host_reps * 4)
    out["host_matching_us"] = host_time(ev.compute, args.host_reps * 4)
    tab = frame_confusion(gt, ids)
    out["pair_table_rows"] = int(tab[0].shape[0])
    sev = SegEvaluator()
    sev.add_frame(d_tid, d_fcn)
    assert np.array_equal(sev.confusion_matrix(), O.seg_confusion(trainid, fcn))      # same counts as the restatement
    # the numpy restatement of the same work on the host
    out["numpy_seg_confusion_us"] = host_time(lambda: O.seg_confusion(trainid, fcn), args.host_reps)
    segs, pid = O.convert_image(p2)
    out["numpy_image_convert_us"] = host_time(lambda: O.convert_image(p2), args.host_reps)
    out["numpy_pq_core_us"] = host_time(lambda: O.pq_compute_single_core([(gt_segs, segs, gt_ids, pid)], categories),
                                        args.host_reps)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
