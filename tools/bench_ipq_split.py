"""Benchmark of the image panoptic driver (vps_b200.test_eval_ipq) on one GPU; prints one JSON line.

  converter  per 1024x2048 image: the numpy image converter (oracle.ipq.convert_image: np.unique, then a full-frame mask
             and np.nonzero per key, as the reference's _converter_2ch_single_core), ImageWriter.add_frame (device segment
             table, PNGs on writer threads; timed over a run of images up to finish()), the same without PNGs, and
             vps_pan2ch_image_segments alone (CUDA events over many launches; algorithmic bytes = 6.3 MB read + 6.3 MB
             written)
  scoring    per image, decode excluded: the mIoU counts (SegEvaluator), the GT ids, the converter's ids, the pair table
             and IpqEvaluator.add_frame_table
  driver     vps_b200.test_eval_ipq.run_split on a synthetic on-disk split (1024x2048 images, seeded test weights of the
             image panoptic model) in images/s, against ClipRunner(unify=True) on the same frames already decoded in memory

Every number is a host clock around work that ends in a device synchronise, unless it says CUDA events.  The card name,
power limit and max SM clock are read in the same run and printed with the numbers.
    python tools/bench_ipq_split.py [--images 16] [--precision tc32] [--skip-driver]"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_split import card  # noqa: E402

H, W = 1024, 2048


def synth_image_pan2ch(rng):
    """an image-level unified result: 16x16 blocks of stuff (0..10, instance 0), 30 thing rectangles (11..18, instance
    ranks 1..30) and VOID"""
    hb, wb = H // 16, W // 16
    sem = rng.choice(np.r_[np.arange(11), 255], size=(hb, wb), p=np.r_[np.full(11, 0.9 / 11), 0.1]).repeat(16, 0).repeat(16, 1)
    out = np.zeros((H, W, 3), np.uint8)
    out[..., 0] = sem
    for t in range(30):
        y, x, h, w = rng.integers(0, H - 200), rng.integers(0, W - 300), rng.integers(20, 200), rng.integers(20, 300)
        out[y:y + h, x:x + w, 0] = rng.integers(11, 19)
        out[y:y + h, x:x + w, 1] = t + 1
    return out


def bench_converter(frames, tmp):
    from oracle.ipq import convert_image
    from vps_b200 import ops
    from vps_b200.writer import NKEY, ImageWriter
    dev = [torch.from_numpy(f).cuda() for f in frames]
    names = ["frankfurt_000000_%06d_leftImg8bit.png" % i for i in range(len(frames))]
    out = {}
    n_np = min(3, len(frames))
    t = time.perf_counter()
    for f in frames[:n_np]:
        convert_image(f)
    out["numpy_converter_ms"] = 1e3 * (time.perf_counter() - t) / n_np
    ImageWriter(os.path.join(tmp, "w0")).add_frame(names[0], dev[0])           # warm-up
    torch.cuda.synchronize()
    w = ImageWriter(os.path.join(tmp, "img"))
    t = time.perf_counter()
    for n, d in zip(names, dev):
        w.add_frame(n, d)
    w.finish()
    out["add_frame_ms"] = 1e3 * (time.perf_counter() - t) / len(frames)
    w = ImageWriter(None)
    t = time.perf_counter()
    for n, d in zip(names, dev):
        w.add_frame(n, d)
    torch.cuda.synchronize()
    out["add_frame_no_png_ms"] = 1e3 * (time.perf_counter() - t) / len(frames)
    table = torch.empty(5 * NKEY + 1, dtype=torch.int32, device="cuda")
    rgb = torch.empty_like(dev[0])
    for d in dev[:4]:
        ops.pan2ch_segments(d, 11, table, rgb, image=True)
    reps = 200
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(reps):
        ops.pan2ch_segments(dev[i % len(dev)], 11, table, rgb, image=True)
    e1.record()
    torch.cuda.synchronize()
    out["kernel_us"] = 1e3 * e0.elapsed_time(e1) / reps
    out["kernel_hbm_floor_us"] = 2 * H * W * 3 / 3.35e12 * 1e6
    return out


def bench_scoring(frames):
    from vps_b200.ipq import IpqEvaluator, SegEvaluator, image_segment_ids
    from vps_b200.vpq import frame_confusion, rgb_to_id
    from vps_b200.writer import id2rgb, image_segments_from_table, pan2ch_segments
    cats = {i: {"id": i, "isthing": int(i >= 11)} for i in range(19)}
    dev = [torch.from_numpy(f).cuda() for f in frames]
    gts = []
    for d in dev:                                                    # ground truth = the prediction itself
        table, _ = pan2ch_segments(d, image=True)
        info = image_segments_from_table(table)
        gts.append((d[..., 0].contiguous(), torch.from_numpy(id2rgb(image_segment_ids(d).cpu().numpy())).cuda(), info))
    seg, ipq = SegEvaluator(resize_pred=True), IpqEvaluator(cats)

    def score(d, gt):
        lab, gt_rgb, info = gt
        seg.add_frame(lab, d[..., 0][None])
        pairs, counts = frame_confusion(rgb_to_id(gt_rgb), image_segment_ids(d))
        ipq.add_frame_table(info, info, pairs, counts)
    score(dev[0], gts[0])                                            # warm-up
    torch.cuda.synchronize()
    t = time.perf_counter()
    for d, gt in zip(dev, gts):
        score(d, gt)
    torch.cuda.synchronize()
    ms = 1e3 * (time.perf_counter() - t) / len(dev)
    assert all(s.fp == 0 and s.fn == 0 for s in ipq.compute().values())
    return {"scoring_ms_per_image": ms}


def write_split(root, decoded):
    """images under val/ (fid >= 1) and their previous frames under val_nbr/, the dataset json, a constant ground truth
    (trainId 0 labels, one road segment over the whole panoptic PNG: the timings do not depend on it), a fuse.py-style
    config and weights"""
    import cv2
    from PIL import Image

    from oracle.variants import PanopticFuse, from_fusetrack
    from oracle.weights import make_model
    for d in ("val", "val_nbr", "gt/annotations", "gt/labels", "data/cityscapes/panoptic"):
        os.makedirs(os.path.join(root, d))
    images, pan_images, pan_anns = [], [], []
    zero_lab, road = np.zeros((H, W), np.uint8), np.zeros((H, W, 3), np.uint8)
    road[..., 0] = 1                                                 # id 1
    for i, img in enumerate(decoded):
        n = "frankfurt_000000_%06d_leftImg8bit.png" % (19 + i)
        cv2.imwrite(os.path.join(root, "val", n), img)
        cv2.imwrite(os.path.join(root, "val_nbr", "frankfurt_000000_%06d_leftImg8bit.png" % (18 + i)), np.roll(img, 4, 1))
        Image.fromarray(zero_lab).save(os.path.join(root, "gt", "labels", n.replace("leftImg8bit.png", "gtFine_labelTrainIds.png")))
        Image.fromarray(road).save(os.path.join(root, "data", "cityscapes", "panoptic", n))
        images.append({"id": i + 1, "file_name": n})
        pan_images.append({"id": i + 1, "file_name": n})
        pan_anns.append({"image_id": i + 1, "segments_info": [{"id": 1, "category_id": 0, "iscrowd": 0, "area": H * W}]})
    json.dump({"images": images}, open(os.path.join(root, "ann.json"), "w"))
    json.dump({"images": images}, open(os.path.join(root, "gt", "annotations", "instancesonly_gtFine_val.json"), "w"))
    json.dump({"images": pan_images, "annotations": pan_anns, "categories": [{"id": i, "isthing": int(i >= 11)} for i in range(19)]},
              open(os.path.join(root, "gt", "annotations", "cityscapes_fine_val.json"), "w"))
    norm = dict(mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], to_rgb=True)
    pipeline = [dict(type="LoadRefImageFromFile"),
                dict(type="MultiScaleFlipAug", img_scale=[(W, H)], flip=False,
                     transforms=[dict(type="Resize", keep_ratio=True), dict(type="RandomFlip"), dict(type="Normalize", **norm),
                                 dict(type="Pad", size_divisor=64), dict(type="ImageToTensor", keys=["img", "ref_img"]),
                                 dict(type="Collect", keys=["img", "ref_img"])])]
    test = dict(type="CityscapesDataset", data_root=root, ann_file="ann.json", img_prefix="val/", ref_prefix="val_nbr/",
                pipeline=pipeline)
    with open(os.path.join(root, "cfg.py"), "w") as f:
        f.write("from vps_b200.default_cfg import fuse_cfg as _fuse_cfg\n_c = _fuse_cfg()\nmodel = _c['model']\n"
                "test_cfg = _c['test_cfg']\ndata = dict(test=%r)\n" % (test,))
    torch.save({"state_dict": from_fusetrack(PanopticFuse, make_model("C", 0).state_dict()).state_dict()},
               os.path.join(root, "w.pth"))


def bench_driver(tmp, precision, n):
    from vps_b200 import test_eval_ipq as T
    from vps_b200 import test_vpq as TV
    from vps_b200.datasets import CityscapesTestSet
    from vps_b200.pipeline import InputStage
    from vps_b200.runner import ClipRunner
    root = os.path.join(tmp, "cityscapes")
    rng = np.random.default_rng(1)
    decoded = []
    for _ in range(n):
        base = rng.integers(0, 256, size=(H // 32, W // 32, 3)).repeat(32, 0).repeat(32, 1).astype(np.int16)
        decoded.append(np.clip(base + rng.integers(-6, 7, size=(H, W, 3)), 0, 255).astype(np.uint8))
    write_split(root, decoded)
    cwd = os.getcwd()
    os.chdir(root)                                                   # the panoptic GT is read from data/cityscapes/panoptic
    try:
        cfg, model = TV.load_model(os.path.join(root, "cfg.py"), os.path.join(root, "w.pth"), "cuda:0", precision)
        ds = CityscapesTestSet.from_cfg(cfg.data.test)
        out = {}
        pairs = [(torch.from_numpy(decoded[i]), torch.from_numpy(np.roll(decoded[i], 4, 1))) for i in range(n)]
        metas = [ds.img_meta(i) for i in range(n)]
        for rep in range(2):                                         # the first pass captures the CUDA graphs
            runner = ClipRunner(model, "cuda:0", unify=True, input_stage=InputStage.from_pipeline(cfg.data.test.pipeline))
            torch.cuda.synchronize()
            t = time.perf_counter()
            for _ in runner.run(pairs, metas):
                pass
            torch.cuda.synchronize()
            out["model_only_ips"] = n / (time.perf_counter() - t)
        helper = T.EvalHelper(os.path.join(root, "gt"))
        t = time.perf_counter()
        T.run_split(cfg, model, ds, helper, os.path.join(root, "work", "val.pkl"))
        torch.cuda.synchronize()
        out["driver_ips"] = n / (time.perf_counter() - t)
        out["driver_images"] = n
    finally:
        os.chdir(cwd)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--precision", default="tc32")
    ap.add_argument("--skip-driver", action="store_true")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    rng = np.random.default_rng(0)
    frames = [synth_image_pan2ch(rng) for _ in range(a.images)]
    res = {"card": card()}
    with tempfile.TemporaryDirectory() as tmp:
        res.update(bench_converter(frames, tmp))
        res.update(bench_scoring(frames))
        if not a.skip_driver:
            res.update(bench_driver(tmp, a.precision, a.images))
    print(json.dumps({k: round(v, 3) if isinstance(v, float) else v for k, v in res.items()}))


if __name__ == "__main__":
    main()
