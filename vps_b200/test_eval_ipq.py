"""Run the image panoptic model over a Cityscapes split and score it as the reference's tools/test_eval_ipq.py does:
semantic mIoU (`Cityscapes.evaluate_ssegs`) and image PQ (`BaseDataset.evaluate_panoptic`).

    python -m vps_b200.test_eval_ipq configs/cityscapes/fuse.py latest.pth --out work_dirs/fuse/val.pkl \\
        --test_config configs/cityscapes/test_cityscapes_1gpu.yaml

The chain: frames decoded on the host (cv2.imread, a few threads ahead of the loop, with the image's ground-truth PNGs) ->
the config's test pipeline on the device (`InputStage.from_pipeline`) -> the model (`ClipRunner`, the image-level unified
result computed per image on the GPU) -> per image, as it finishes:
  * the palette PNG of fcn_outputs in <out>_ssegs/, and its confusion counts against the trainId labels (`SegEvaluator`);
  * the image converter's segment table on the device (`ImageWriter`: pan_2ch/ and pan/ PNGs, segments_info), and the
    image's (GT, prediction) pair table (`IpqEvaluator`).
At the end <out>_pans_unified/ receives gt.json, pred.json and pq.txt, and the reference's texts are printed.

The ground truth is the reference's eval helper dataset: dataset.dataset_path and dataset.test_image_set of the
--test_config yaml give the roidb (<dataset_path>/annotations/instancesonly_gtFine_<set>.json, sorted by image id) whose
label PNGs the mIoU reads, and <dataset_path>/annotations/cityscapes_fine_val.json, whose panoptic PNGs are read from
data/cityscapes/panoptic/ under the working directory, as the reference hard-codes it.

Differences from the reference: no .pkl side files and no --load (--out only names the output directories); the pan/
PNGs are id2rgb of deterministic ids rather than random panopticapi colours; and the predictions must pair with the
panoptic GT json (the reference pairs the sorted predictions with the json's images by position and silently mispairs, or
drops unreadable GT files): a split that does not pair raises ValueError before the model runs."""
import argparse
import itertools
import json
import os
import re
import sys
import time

import numpy as np

_DESC = ("Image panoptic test and evaluation on the GPU: writes <out>_ssegs/ and <out>_pans_unified/ (pan_2ch/, pan/, "
         "gt.json, pred.json, pq.txt) and prints mIoU and PQ.  The reference's .pkl side files and --load are not "
         "implemented; --out only names the output directories.")
ANNO_FILES = {"train": "instancesonly_gtFine_train.json", "val": "instancesonly_gtFine_val.json",
              "test": "image_info_test.json"}                       # tools/dataset/cityscapes.py:40-44
PAN_GT_FOLDER = "data/cityscapes/panoptic"                          # cityscapes.py:49


def parse_args(argv=None):
    p = argparse.ArgumentParser(description=_DESC)
    p.add_argument("config", help="test config file path (configs/cityscapes/fuse.py)")
    p.add_argument("checkpoint", help="checkpoint file (a dict with 'state_dict', or a state dict)")
    p.add_argument("--out", required=True, help="X.pkl: the results go to X_ssegs/ and X_pans_unified/ (no .pkl is written)")
    p.add_argument("--dataset", type=str, default="Cityscapes", choices=["Cityscapes"])
    p.add_argument("--gpus", type=str, default="0", help="the first id is the device used")
    p.add_argument("--test_config", type=str, default="configs/cityscapes/test_cityscapes_1gpu.yaml",
                   help="UPSNet test yaml (must exist): dataset.dataset_path, dataset.test_image_set and "
                        "test.panoptic_stuff_area_limit are read from it")
    p.add_argument("--precision", type=str, default="tc32", choices=["tc32", "fp32", "bf16"])
    p.add_argument("--workers", type=int, default=4, help="host decode / PNG encode threads")
    args = p.parse_args(argv)
    if not args.out.endswith((".pkl", "pickle")):
        raise ValueError("The output file must be a .pkl file.")
    return args


def eval_helper_config(test_config):
    """(dataset_path, test_image_set) of the UPSNet yaml; the file must exist and set dataset.dataset_path (the
    reference's config has no default for it)"""
    import yaml
    if not os.path.isfile(test_config):
        raise FileNotFoundError("--test_config %r not found" % test_config)
    with open(test_config) as f:
        d = (yaml.safe_load(f) or {}).get("dataset") or {}
    if not d.get("dataset_path"):
        raise ValueError("--test_config %r does not set dataset.dataset_path (the ground-truth root, e.g. "
                         "./data/cityscapes/)" % test_config)
    return str(d["dataset_path"]), str(d.get("test_image_set", "val"))


def label_path(image):
    """the trainId label PNG evaluate_ssegs reads for a roidb image path (cityscapes.py:123), replaces as written there"""
    return image.replace('images', 'labels').replace('leftImg8bit.png', 'gtFine_labelTrainIds.png')


def sseg_text(result):
    """what evaluate_ssegs prints (cityscapes.py:153-166), given SegEvaluator.result()"""
    conf = result["confusion_matrix"]
    with np.errstate(divide="ignore", invalid="ignore"):
        norm = conf / conf.sum(axis=1).reshape((-1, 1))
    lines = ["evaluate segmentation:", "IU_array:"] + ["%.5f" % v for v in result["IU_array"]]
    lines += ["meanIU:%.5f" % result["meanIU"], "confusion_matrix:"]
    text = np.array2string(norm, separator='\t', precision=3, suppress_small=True, max_line_width=200)
    return "\n".join(lines + [re.sub(r'[\[\]]', '', text)]) + "\n"


class EvalHelper:
    """The ground truth of the reference's eval helper dataset (`Cityscapes(image_sets=[test_image_set])`,
    tools/dataset/cityscapes.py:29-60): the roidb (the images of the instancesonly json, sorted by id, json_dataset.py:
    64-79) for the mIoU and the panoptic GT json + PNG folder for PQ.  `pair(names)` ties them to the predictions."""

    def __init__(self, dataset_path, image_set="val", pan_gt_folder=PAN_GT_FOLDER):
        from .datasets import coco_images
        sets = image_set.split('+')
        if len(sets) != 1:
            raise ValueError("the eval helper takes one image set, got %r" % image_set)
        images = coco_images(os.path.join(dataset_path, "annotations", ANNO_FILES[sets[0]]))
        image_dir = os.path.join(dataset_path, "images")
        self.roidb = [dict(im, image=os.path.join(image_dir, im["file_name"])) for im in sorted(images, key=lambda im: im["id"])]
        self.panoptic_json_file = os.path.join(dataset_path, "annotations", "cityscapes_fine_val.json")
        self.panoptic_gt_folder = pan_gt_folder
        with open(self.panoptic_json_file) as f:
            self.pan_gt_json = json.load(f)
        self.categories = {el["id"]: el for el in self.pan_gt_json["categories"]}
        self.labels = None

    def pair(self, names):
        """names: the predictions' image basenames in the order they will be produced.  The reference sorts them and pairs
        the i-th with the panoptic GT json's i-th image, so they must be in ascending, unique order, as many as the json's
        images, with equal PNG names (ValueError otherwise).  Each roidb image's label is counted against the prediction
        of the same name; one without a prediction raises FileNotFoundError naming it, and predictions outside the roidb
        are not counted."""
        from .writer import pan_image_name, sseg_path
        names = list(names)
        if names != sorted(set(names)):
            raise ValueError("the dataset's images are not in ascending, unique file-name order: the reference pairs the "
                             "sorted predictions with the panoptic GT json, which this driver does not reorder")
        gt_names = [im["file_name"] for im in self.pan_gt_json["images"]]
        if len(gt_names) != len(names):
            raise ValueError("%d predictions but %s lists %d images" % (len(names), self.panoptic_json_file, len(gt_names)))
        for i, (n, g) in enumerate(zip(names, gt_names)):
            if pan_image_name(n) != pan_image_name(g.split("/")[-1]):
                raise ValueError("prediction %d (%s) does not pair with image %d of %s (%s)" % (i, n, i, self.panoptic_json_file, g))
        index = {os.path.basename(sseg_path("", n)): i for i, n in enumerate(names)}
        self.labels = [[] for _ in names]
        for entry in self.roidb:
            lab = label_path(entry["image"])
            res = os.path.split(lab)[-1][:-len('_gtFine_labelTrainIds.png')] + '.png'
            if res not in index:
                raise FileNotFoundError("no prediction for %s (its semantic PNG would be %s)" % (entry["image"], res))
            self.labels[index[res]].append(lab)

    def load_gt(self, i):
        """host decode of image i's ground truth: ([trainId label maps], panoptic GT RGB image)"""
        from PIL import Image
        labels = [np.array(Image.open(p)) for p in self.labels[i]]
        gt = np.array(Image.open(os.path.join(self.panoptic_gt_folder, self.pan_gt_json["images"][i]["file_name"])))
        return labels, gt


class SplitScorer:
    """The scoring half of the driver: `add` per image in pairing order (the images' device results), `finish()` once."""

    def __init__(self, helper, out, workers=4, num_stuff=11):
        from .ipq import IpqEvaluator, SegEvaluator
        from .writer import ImageWriter
        self.helper, self.num_stuff = helper, num_stuff
        self.pans_dir = out.replace('.pkl', '_pans_unified')
        self.writer = ImageWriter(self.pans_dir, out.replace('.pkl', '_ssegs'), workers=workers)
        self.seg = SegEvaluator(resize_pred=True)
        self.ipq = IpqEvaluator(helper.categories, num_stuff)
        self.count = 0

    def __enter__(self):
        return self

    def __exit__(self, exc_type, exc, tb):
        self.writer.close(raise_errors=exc_type is None)
        return False

    def add(self, name, fcn, pan_2ch, fcn_host=None, pan_2ch_host=None, gt=None):
        """name: the image basename; fcn: device semantic map [1,H,W]; pan_2ch: device image-level unified result [H,W,3];
        fcn_host / pan_2ch_host: host copies of the two, if the caller has them (ClipRunner's fcn_outputs and pan_2ch);
        gt: `helper.load_gt(i)` (read here when None)"""
        import torch

        from .ipq import image_segment_ids
        from .vpq import frame_confusion, rgb_to_id
        i = self.count
        self.count += 1
        labels, gt_rgb = self.helper.load_gt(i) if gt is None else gt
        image = self.helper.pan_gt_json["images"][i]
        if tuple(gt_rgb.shape) != tuple(pan_2ch.shape):          # the reference's PQ core fails on such maps too
            raise ValueError("image %s: prediction %s and panoptic ground truth %s differ in shape"
                             % (image["file_name"], tuple(pan_2ch.shape), tuple(gt_rgb.shape)))
        self.writer.add_sseg(name, (fcn if fcn_host is None else fcn_host).cpu().numpy())
        for lab in labels:
            self.seg.add_frame(torch.from_numpy(lab).to(fcn.device), fcn)
        ann = self.writer.add_frame(image["file_name"], pan_2ch, self.num_stuff, pan_2ch_host)
        gt_ids = rgb_to_id(torch.from_numpy(np.ascontiguousarray(gt_rgb)).to(pan_2ch.device))
        pairs, counts = frame_confusion(gt_ids, image_segment_ids(pan_2ch, self.num_stuff))
        self.ipq.add_frame_table(self.helper.pan_gt_json["annotations"][i]["segments_info"], ann["segments_info"],
                                 pairs, counts)

    def finish(self):
        """write gt.json, pred.json and pq.txt, print the reference's texts; returns {sseg: SegEvaluator.result(), pq:
        IpqEvaluator.write_pq_txt's dict}"""
        self.writer.finish(self.helper.pan_gt_json)
        sseg = self.seg.result()
        pq = self.ipq.write_pq_txt(os.path.join(self.pans_dir, "pq.txt"), self.ipq.compute())
        sys.stdout.write(sseg_text(sseg))
        print("PQ_All:", 100 * pq["All"]["pq"])
        print("PQ_Thing:", 100 * pq["Things"]["pq"])
        print("PQ_Stuff:", 100 * pq["Stuff"]["pq"])
        return {"sseg": sseg, "pq": pq}


def run_split(cfg, model, dataset, helper, out, area_limit=4096, workers=4, device="cuda:0"):
    """single_gpu_test + get_unified_pan_result + evaluate_ssegs + evaluate_panoptic over a whole split"""
    import cv2
    import torch

    from .datasets import prefetch_map
    from .pipeline import InputStage
    from .runner import ClipRunner
    names = [dataset.img_info(i)["filename"].split("/")[-1] for i in range(len(dataset))]
    helper.pair(names)                                          # before the model runs
    stage = InputStage.from_pipeline(cfg.data.test.pipeline, device=device)
    with_ref = model.with_flow

    def read(idx):
        img_path, ref_path = dataset.paths(idx)
        img = cv2.imread(img_path, cv2.IMREAD_COLOR)
        if img is None:
            raise FileNotFoundError(img_path)
        ref = None
        if with_ref:
            ref = cv2.imread(ref_path, cv2.IMREAD_COLOR)
            if ref is None:
                raise FileNotFoundError(ref_path)
        pair = (torch.from_numpy(img), None if ref is None else torch.from_numpy(ref))
        return pair, dataset.img_meta(idx), helper.load_gt(idx)

    a, b, c = itertools.tee(prefetch_map(read, range(len(dataset)), workers=workers, depth=8), 3)
    pairs, metas, gts = (x[0] for x in a), (x[1] for x in b), (x[2] for x in c)
    runner = ClipRunner(model, device, unify=True, input_stage=stage)
    runner.unifier.stuff_area_limit = int(area_limit)
    with SplitScorer(helper, out, workers) as scorer:
        for name, r, gt in zip(names, runner.run(pairs, metas), gts):
            p = r[2]
            scorer.add(name, p["fcn_outputs_device"], p["pan_2ch_device"], p["fcn_outputs"], p["pan_2ch"], gt)
        return scorer.finish()


def main(argv=None):
    args = parse_args(argv)
    import torch

    from .datasets import CityscapesTestSet
    from .test_vpq import load_model, stuff_area_limit
    area_limit = stuff_area_limit(args.test_config)
    dataset_path, image_set = eval_helper_config(args.test_config)
    helper = EvalHelper(dataset_path, image_set)
    device = "cuda:%d" % int(args.gpus.split(",")[0])
    torch.cuda.set_device(device)
    cfg, model = load_model(args.config, args.checkpoint, device, args.precision)
    dataset = CityscapesTestSet.from_cfg(cfg.data.test)
    print("==> Semantic Segmentation PNGs will be saved at:")
    print("---", args.out.split('.pkl')[0] + '_ssegs/')
    print("==> Image Panoptic Segmentation PNGs and PQ.TXT will be saved at:")
    print("---", args.out.split('.pkl')[0] + '_pans_unified/')
    t0 = time.time()
    run_split(cfg, model, dataset, helper, args.out, area_limit, args.workers, device)
    print("==> Done: %d images in %.1f s" % (len(dataset), time.time() - t0))
    return 0


if __name__ == "__main__":
    sys.exit(main())
