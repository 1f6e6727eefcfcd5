"""Benchmark of the split-level tools (vps_b200.test_vpq, vps_b200.eval_vpq) on one GPU; prints one JSON line.

  writer     per sampled 1024x2048 frame: the previous host writer (device ids + pair table, then last_key_ids,
             find_objects, id2rgb and two serial PNG encodes), PanWriter.add_frame (device segment table, PNGs on writer
             threads; timed over a run of frames up to finish()), the same without PNGs, and vps_pan2ch_segments alone
             (CUDA events over many launches; algorithmic bytes = 6 MB read + 6 MB written)
  eval       vps_b200.vpq.evaluate_split per frame on decoded 1024x2048 frames (PNG decode excluded), 12 frames, 4 windows
  driver     vps_b200.test_vpq.run_split on a synthetic on-disk split (2 clips x 30 frames of 1024x2048, seeded test weights)
             in frames/s, against ClipRunner(unify=True) on the same frames already decoded in memory (the model-only rate)

Every number is a host clock around work that ends in a device synchronise, unless it says CUDA events.  The card name,
power limit and max SM clock are read in the same run and printed with the numbers.
    python tools/bench_split.py [--frames 24] [--precision tc32] [--skip-driver]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def synth_pan2ch(rng, H=1024, W=2048):
    """a unified result with Cityscapes-like structure: 16x16 blocks of stuff (0..10, several track values per class),
    rectangles of things (11..18, tracks 1..40) and VOID"""
    hb, wb = H // 16, W // 16
    sem = rng.choice(np.r_[np.arange(11), 255], size=(hb, wb), p=np.r_[np.full(11, 0.9 / 11), 0.1]).repeat(16, 0).repeat(16, 1)
    trk = (rng.integers(0, 3, size=(hb, wb)) * 7).repeat(16, 0).repeat(16, 1)
    out = np.zeros((H, W, 3), np.uint8)
    out[..., 0], out[..., 2] = sem, trk
    for t in range(30):
        y, x, h, w = rng.integers(0, H - 200), rng.integers(0, W - 300), rng.integers(20, 200), rng.integers(20, 300)
        out[y:y + h, x:x + w, 0] = rng.integers(11, 19)
        out[y:y + h, x:x + w, 1] = t
        out[y:y + h, x:x + w, 2] = t + 1
    return out


def old_add_frame(w, name, pan_2ch):
    """the previous PanWriter.add_frame: device ids and pair table, then the host part with serial PNG encodes"""
    from vps_b200.vpq import segments_from_pan2ch
    from vps_b200.writer import last_key_ids
    ids, segs = segments_from_pan2ch(pan_2ch)
    p2 = pan_2ch.cpu().numpy()
    return w.add_frame_ids(name, ids.cpu().numpy().astype(np.uint32), segs, p2, _counted=True, bbox_ids=last_key_ids(p2))


def bench_writer(frames, tmp):
    from vps_b200.writer import PanWriter, pan2ch_segments
    dev = [torch.from_numpy(f).cuda() for f in frames]
    names = ["frankfurt_%06d_leftImg8bit.png" % i for i in range(len(frames))]
    out = {}
    # warm-up
    old_add_frame(PanWriter(os.path.join(tmp, "w0"), sample=False), names[0], dev[0])
    PanWriter(None, sample=False).add_frame(names[0], dev[0])
    torch.cuda.synchronize()
    w = PanWriter(os.path.join(tmp, "old"), sample=False)
    t = time.perf_counter()
    for n, d in zip(names, dev):
        old_add_frame(w, n, d)
    w.finish()
    out["old_add_frame_ms"] = 1e3 * (time.perf_counter() - t) / len(frames)
    w = PanWriter(os.path.join(tmp, "new"), sample=False)
    t = time.perf_counter()
    for n, d in zip(names, dev):
        w.add_frame(n, d)
    w.finish()
    out["new_add_frame_ms"] = 1e3 * (time.perf_counter() - t) / len(frames)
    w = PanWriter(None, sample=False)
    t = time.perf_counter()
    for n, d in zip(names, dev):
        w.add_frame(n, d)
    torch.cuda.synchronize()
    out["new_add_frame_no_png_ms"] = 1e3 * (time.perf_counter() - t) / len(frames)
    # kernel alone
    from vps_b200 import ops
    from vps_b200._lib import lib
    table = torch.empty(5 * 19 * 256 + 1, dtype=torch.int32, device="cuda")
    rgb = torch.empty_like(dev[0])
    H, W = dev[0].shape[:2]
    call = lambda d: ops.check(lib().vps_pan2ch_segments(ops._ptr(d), H, W, 11, ops._ptr(table), ops._ptr(rgb), ops.stream()), "seg")
    for d in dev[:4]:
        call(d)
    reps = 200
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(reps):
        call(dev[i % len(dev)])
    e1.record()
    torch.cuda.synchronize()
    us = 1e3 * e0.elapsed_time(e1) / reps
    out["kernel_us"] = us
    out["kernel_hbm_floor_us"] = 2 * H * W * 3 / 3.35e12 * 1e6
    pan2ch_segments(dev[0])
    return out


def bench_eval(frames):
    from vps_b200.vpq import evaluate_split
    from vps_b200.writer import PanWriter
    n = 12
    w = PanWriter(None, sample=False)
    rgbs, anns = [], []
    from vps_b200.writer import pan2ch_segments
    for f in frames[:n]:
        d = torch.from_numpy(f).cuda()
        anns.append(w.add_frame("f", d))
        rgbs.append(pan2ch_segments(d)[1].cpu().numpy())
    cats = [{"id": i, "isthing": int(i >= 11)} for i in range(19)]
    gt = {"annotations": anns, "categories": cats}
    pred = {"annotations": anns}
    evaluate_split(dict(gt, annotations=anns[:6]), {"annotations": anns[:6]}, rgbs[:6], rgbs[:6])     # warm-up
    torch.cuda.synchronize()
    t = time.perf_counter()
    res = evaluate_split(gt, pred, rgbs, rgbs)
    torch.cuda.synchronize()
    assert all(r["All"]["pq"] == 1.0 for r in res.values())
    return {"eval_ms_per_frame": 1e3 * (time.perf_counter() - t) / n}


NFR = 30          # frames per clip (one clip = nframes_span_test, as in the Cityscapes-VPS configs)


def write_config(path, root, img_scale=(2048, 1024)):
    """a FuseTrack test config over the synthetic split under root: the default model and the reference's test pipeline
    (configs/cityscapes/fusetrack.py) with Pad(64); the paths say test/ and are rewritten by --mode val"""
    norm = dict(mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], to_rgb=True)
    pipeline = [dict(type="LoadRefImageFromFile"),
                dict(type="MultiScaleFlipAug", img_scale=[tuple(img_scale)], flip=False,
                     transforms=[dict(type="Resize", keep_ratio=True), dict(type="RandomFlip"), dict(type="Normalize", **norm),
                                 dict(type="Pad", size_divisor=64), dict(type="ImageToTensor", keys=["img", "ref_img"]),
                                 dict(type="Collect", keys=["img", "ref_img"])])]
    test = dict(type="CityscapesVPSDataset", data_root=root, ann_file="im_all_info_test_city_vps.json",
                img_prefix="test/img_all/", ref_prefix="test/img_all/", nframes_span_test=NFR, pipeline=pipeline)
    with open(path, "w") as f:
        f.write("from vps_b200.default_cfg import fusetrack_cfg as _fusetrack_cfg\n"
                "_c = _fusetrack_cfg()\nmodel = _c['model']\ntest_cfg = _c['test_cfg']\n"
                "data = dict(test=%r)\n" % (test,))


def bench_driver(tmp, precision):
    import cv2
    from oracle.weights import make_model
    from vps_b200 import test_vpq as T
    from vps_b200.datasets import CityscapesVPSTestSet, rewrite_mode
    from vps_b200.pipeline import InputStage
    from vps_b200.runner import ClipRunner
    H, W = 1024, 2048
    root = os.path.join(tmp, "cityscapes_vps")
    os.makedirs(os.path.join(root, "val", "img_all"))
    rng = np.random.default_rng(1)
    images, decoded = [], []
    for c in range(2):
        base = rng.integers(0, 256, size=(H // 32, W // 32, 3)).repeat(32, 0).repeat(32, 1).astype(np.int16)
        for f in range(NFR):
            img = np.clip(np.roll(base, (4 * f, 8 * f), (0, 1)) + rng.integers(-6, 7, size=(H, W, 3)), 0, 255).astype(np.uint8)
            name = "%04d_%04d_frankfurt_000000_%06d_leftImg8bit.png" % (c, f, 100 + f)
            cv2.imwrite(os.path.join(root, "val", "img_all", name), img)
            images.append({"id": (c + 1) * 10000 + f + 1, "file_name": name})
            decoded.append(img)
    json.dump({"images": images}, open(os.path.join(root, "im_all_info_val_city_vps.json"), "w"))
    write_config(os.path.join(root, "cfg.py"), root, (W, H))
    torch.save({"state_dict": make_model("C", 0).state_dict()}, os.path.join(root, "w.pth"))
    names = sorted(im["file_name"] for im in images)[: len(images[4::5])]
    cfg, model = T.load_model(os.path.join(root, "cfg.py"), os.path.join(root, "w.pth"), "cuda:0", precision)
    test = rewrite_mode(cfg.data.test, "val")
    cfg.data.test.update(test)
    ds = CityscapesVPSTestSet.from_cfg(test)
    out = {}
    # model only: decoded frames in memory, ClipRunner(unify=True), results dropped
    pairs = [(torch.from_numpy(decoded[i]), torch.from_numpy(decoded[i - 1] if i % NFR else decoded[i])) for i in range(len(ds))]
    metas = [ds.img_meta(i) for i in range(len(ds))]
    for rep in range(2):                                             # the first pass captures the CUDA graphs
        runner = ClipRunner(model, "cuda:0", unify=True, input_stage=InputStage.from_pipeline(cfg.data.test.pipeline))
        model.reset_tracker()
        torch.cuda.synchronize()
        t = time.perf_counter()
        for _ in runner.run(pairs, metas):
            pass
        torch.cuda.synchronize()
        out["model_only_fps"] = len(ds) / (time.perf_counter() - t)
    t = time.perf_counter()
    T.run_split(cfg, model, ds, names, os.path.join(root, "out_pans_unified/"))
    torch.cuda.synchronize()
    out["driver_fps"] = len(ds) / (time.perf_counter() - t)
    out["driver_frames"] = len(ds)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=24)
    ap.add_argument("--precision", default="tc32")
    ap.add_argument("--skip-driver", action="store_true")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    rng = np.random.default_rng(0)
    frames = [synth_pan2ch(rng) for _ in range(a.frames)]
    res = {"card": card()}
    with tempfile.TemporaryDirectory() as tmp:
        res.update(bench_writer(frames, tmp))
        res.update(bench_eval(frames))
        if not a.skip_driver:
            res.update(bench_driver(tmp, a.precision))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
