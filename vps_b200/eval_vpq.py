"""Score a Cityscapes-VPS split: the command line of the reference's tools/eval_vpq.py (:249-331).

    python -m vps_b200.eval_vpq --submit_dir <out>_pans_unified/ --truth_dir data/cityscapes_vps/val/panoptic_video/ \\
        --pan_gt_json_file data/cityscapes_vps/panoptic_gt_val_city_vps.json

reads <submit_dir>/pred.json and <submit_dir>/pan_pred/<image id>.png, and writes vpq-0.txt, vpq-5.txt, vpq-10.txt,
vpq-15.txt and vpq-final.txt into submit_dir with the reference's text.  PNGs are decoded on the host by a few threads, a
bounded number of frames ahead; the id decode and each frame's (gt, pred) pair table run on the GPU
(`vps_b200.vpq.evaluate_split`)."""
import argparse
import json
import os
import sys
import time

from .datasets import prefetch_map


def gt_files(gt_json):
    """GT PNG names (eval_vpq.py:287-288): each image's file name mapped to its mask, sorted"""
    files = [im["file_name"].replace("_newImg8bit.png", "_final_mask.png").replace("_leftImg8bit.png", "_gtFine_color.png")
             for im in gt_json["images"]]
    return sorted(files)


def pred_files(gt_json):
    """prediction PNG names (eval_vpq.py:296): pan_pred/<image id>.png in the order of the GT JSON's images"""
    return [os.path.join("pan_pred", im["id"] + ".png") for im in gt_json["images"]]


def read_png(path):
    import numpy as np
    from PIL import Image
    with Image.open(path) as im:
        return np.array(im)


def evaluate_dirs(submit_dir, truth_dir, pan_gt_json_file, output_dir=None, workers=4, depth=8):
    """eval_vpq.py's main: returns evaluate_split's result and writes the five text files into output_dir (default
    submit_dir)"""
    from .vpq import evaluate_split, vpq_final_text, vpq_text
    output_dir = submit_dir if output_dir is None else output_dir
    with open(os.path.join(submit_dir, "pred.json")) as f:
        pred_json = json.load(f)
    with open(pan_gt_json_file) as f:
        gt_json = json.load(f)
    gts, preds = gt_files(gt_json), pred_files(gt_json)
    if len(gts) != len(preds):
        raise AssertionError("number of prediction does not match with the groud truth.")
    paths = [p for pair in zip((os.path.join(truth_dir, g) for g in gts), (os.path.join(submit_dir, p) for p in preds))
             for p in pair]
    images = prefetch_map(read_png, paths, workers=workers, depth=2 * depth)
    results = evaluate_split(gt_json, pred_json, images, images)       # one iterator: gt, pred, gt, pred, ...
    os.makedirs(output_dir, exist_ok=True)
    for k, res in results.items():
        with open(os.path.join(output_dir, "vpq-%d.txt" % k), "w") as f:
            f.write(vpq_text(res))
    with open(os.path.join(output_dir, "vpq-final.txt"), "w") as f:
        f.write(vpq_final_text(results))
    return results


def parse_args(argv=None):
    p = argparse.ArgumentParser(description="Video panoptic quality (VPQ) of a Cityscapes-VPS split, as tools/eval_vpq.py")
    p.add_argument("--submit_dir", type=str, default="work_dirs/cityscapes_vps/fusetrack_vpct/val_pans_unified/",
                   help="directory with pred.json and pan_pred/ (the output of vps_b200.test_vpq); the vpq-*.txt files go here")
    p.add_argument("--truth_dir", type=str, default="data/cityscapes_vps/val/panoptic_video",
                   help="directory of the ground-truth panoptic PNGs")
    p.add_argument("--pan_gt_json_file", type=str, default="data/cityscapes_vps/panpotic_gt_val_city_vps.json",
                   help="ground-truth panoptic JSON")
    p.add_argument("--workers", type=int, default=4, help="PNG decode threads")
    return p.parse_args(argv)


def main(argv=None):
    args = parse_args(argv)
    if not os.path.isdir(args.submit_dir):
        print("%s doesn't exist" % args.submit_dir)
    t0 = time.time()
    res = evaluate_dirs(args.submit_dir, args.truth_dir, args.pan_gt_json_file, workers=args.workers)
    for k in sorted(res):
        print("==> %d-frame vpq:" % k, 100 * res[k]["All"]["pq"], 100 * res[k]["Things"]["pq"], 100 * res[k]["Stuff"]["pq"])
    print("==> All:", time.time() - t0, "sec")
    return 0


if __name__ == "__main__":
    sys.exit(main())
