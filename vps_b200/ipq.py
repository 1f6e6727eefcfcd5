"""Evaluation of the image panoptic model (PanopticFuse) as the reference's tools/test_eval_ipq.py does it, with the pixel
passes on the GPU:

* semantic mIoU -- `Cityscapes.evaluate_ssegs` (tools/dataset/cityscapes.py:112-166): a C x C confusion matrix of gt
  trainIds against `fcn_outputs`, accumulated over frames on the device (`vps_seg_confusion`; with `resize_pred`, a
  prediction of another shape is read through the reference's Image.NEAREST resize, `vps_seg_confusion_nearest`); applies
  to every model's `fcn_outputs`;
* image PQ -- `BaseDataset.evaluate_panoptic` (tools/dataset/base_dataset.py:104-229): the image converter's segment keying
  (`vps_pan2ch_image_ids`), the frame's (gt, pred) pair table (`vps_tube_confusion`, whose row sums are the predicted
  areas), then `_pq_compute_single_core` (:337-431) on the host in the reference's order, so the IoU sums are identical,
  and its `pq.txt` (:200-211)."""
import ctypes as C
from collections import defaultdict

import numpy as np
import torch

from . import ops
from ._lib import lib
from .vpq import OFFSET, VOID, CatStat, frame_confusion, match_segments, pq_average, recount_pred_areas, rgb_to_id


def nearest_table(src, dst):
    """Pillow's index table of one axis of Image.resize(size, NEAREST) (the affine scaler of a pure scale): a = src / dst,
    xo = a / 2, then per output index int(xo) and xo += a.  The sum is sequential in double, so it is built here, once,
    rather than on the device; -1 marks an index outside the source (the pixel then reads Pillow's fill value 0)."""
    if src == dst:
        return np.arange(dst, dtype=np.int32)                     # Pillow copies an image whose size is unchanged
    a = float(src) / float(dst)
    xo = np.cumsum(np.concatenate([[a * 0.5], np.full(dst - 1, a)]))
    idx = np.where(xo < 0, -1, xo.astype(np.int64))
    return np.where((idx >= 0) & (idx < src), idx, -1).astype(np.int32)


class SegEvaluator:
    """Semantic mIoU of `Cityscapes.evaluate_ssegs`: `add_frame` per frame, `result()` once."""

    def __init__(self, num_classes=19, resize_pred=False):
        self.num_classes = num_classes
        # resize_pred: a prediction of another shape than the gt is resized to it with Image.NEAREST, as evaluate_ssegs does
        # with the PNG it wrote (cityscapes.py:125-126); the index tables are device arrays cached per (pred, gt) shape
        self.resize_pred = bool(resize_pred)
        self._tables = {}
        self._conf = None               # device uint64 [C, C] (held as int64), row = gt

    def _nearest_tables(self, ph, pw, gh, gw, device):
        key = (ph, pw, gh, gw, device)
        if key not in self._tables:
            self._tables[key] = tuple(torch.from_numpy(nearest_table(s, d)).to(device) for s, d in ((pw, gw), (ph, gh)))
        return self._tables[key]

    @torch.no_grad()
    def add_frame(self, gt_trainids, fcn_output):
        """gt_trainids: uint8 CUDA map; fcn_output: uint8 or int64 CUDA map of the same [H,W] (a leading 1 is allowed).
        The reference resizes the prediction to the gt with Image.NEAREST, which is the identity for equal shapes.  Other
        shapes raise unless the evaluator was made with resize_pred=True, which applies that resize."""
        if not (gt_trainids.is_cuda and fcn_output.is_cuda):
            raise RuntimeError("SegEvaluator: label maps must be CUDA tensors (there is no CPU path)")
        if gt_trainids.dtype != torch.uint8 or fcn_output.dtype not in (torch.uint8, torch.int64):
            raise TypeError("SegEvaluator: gt must be uint8 and the prediction uint8 or int64")
        g, p = gt_trainids.squeeze(0), fcn_output.squeeze(0)
        if g.dim() != 2 or p.dim() != 2 or (g.shape != p.shape and not self.resize_pred):
            raise ValueError("SegEvaluator: gt %s and prediction %s must be [H,W] maps of the same shape"
                             % (tuple(gt_trainids.shape), tuple(fcn_output.shape)))
        g, p = g.contiguous(), p.contiguous()
        if self._conf is None:
            self._conf = torch.zeros(self.num_classes, self.num_classes, dtype=torch.int64, device=g.device)
        if g.shape == p.shape:
            ops.check(lib().vps_seg_confusion(ops._ptr(g), ops._ptr(p), p.element_size(), C.c_int64(g.numel()), self.num_classes,
                                              ops._ptr(self._conf), ops.stream()), "seg_confusion")
            return
        (gh, gw), (ph, pw) = g.shape, p.shape
        xtab, ytab = self._nearest_tables(ph, pw, gh, gw, g.device)
        ops.check(lib().vps_seg_confusion_nearest(ops._ptr(g), gh, gw, ops._ptr(p), p.element_size(), ph, pw, ops._ptr(xtab),
                                                  ops._ptr(ytab), self.num_classes, ops._ptr(self._conf), ops.stream()),
                  "seg_confusion_nearest")

    def confusion_matrix(self):
        """the accumulated counts, float64 [C, C] as the reference holds them"""
        if self._conf is None:
            return np.zeros((self.num_classes, self.num_classes))
        return self._conf.cpu().numpy().view(np.uint64).astype(np.float64)

    def result(self):
        """{meanIU, IU_array, confusion_matrix} of evaluate_ssegs (cityscapes.py:142-151), float64"""
        conf = self.confusion_matrix()
        pos, res, tp = conf.sum(1), conf.sum(0), np.diag(conf)
        iu = tp / np.maximum(1.0, pos + res - tp)
        return {"meanIU": iu.mean(), "IU_array": iu, "confusion_matrix": conf}


def image_segment_ids(pan_2ch, num_stuff=11):
    """Image-level unified result (uint8 CUDA [H,W,3], PanUnifier(image=True)) -> int32 CUDA [H,W] segment ids of the
    reference's image converter: 1000 * semantic + instance + 1 for things, 1000 * semantic + 1 for stuff, 0 = VOID.  IPQ is
    invariant to the id values (the reference's are panopticapi colours)."""
    assert pan_2ch.is_cuda and pan_2ch.dtype == torch.uint8 and pan_2ch.shape[-1] == 3
    pan_2ch = pan_2ch.contiguous()
    ids = torch.empty(pan_2ch.shape[:-1], dtype=torch.int32, device=pan_2ch.device)
    ops.check(lib().vps_pan2ch_image_ids(ops._ptr(pan_2ch), C.c_int64(ids.numel()), int(num_stuff), ops._ptr(ids), ops.stream()),
              "pan2ch_image_ids")
    return ids


class IpqEvaluator:
    """Image PQ of `BaseDataset.evaluate_panoptic`: `add_frame` per image in order, then `compute()`."""

    def __init__(self, categories, num_stuff=11):
        self.categories = categories
        self.num_stuff = num_stuff
        self.frames = []            # (gt_segms, pred_segms, pairs, counts)

    def add_frame(self, gt_rgb, gt_segments, pan_2ch):
        """gt_rgb: RGB panoptic ground truth (uint8 CUDA [H,W,3]) with its segments_info list; pan_2ch: the image-level
        unified result (uint8 CUDA [H,W,3]) of the same size.  Other sizes raise, and there is no resizing mode: the
        reference's PQ core compares the PNGs pixel for pixel and fails on maps of different sizes too.  The predicted segments are the converter's: category =
        semantic class, iscrowd 0, area = pixel count (the row sums of the frame's pair table)."""
        if gt_rgb.shape != pan_2ch.shape:
            raise ValueError("IpqEvaluator: gt %s and prediction %s differ in shape" % (tuple(gt_rgb.shape), tuple(pan_2ch.shape)))
        pairs, counts = frame_confusion(rgb_to_id(gt_rgb), image_segment_ids(pan_2ch, self.num_stuff))
        area = defaultdict(int)
        for lab, c in zip((pairs % np.uint64(OFFSET)).tolist(), counts.tolist()):
            area[lab] += c
        pred_segments = [{"id": i, "category_id": (i - 1) // 1000, "iscrowd": 0, "area": a}
                         for i, a in sorted(area.items()) if i != VOID]
        self.add_frame_table(gt_segments, pred_segments, pairs, counts)

    def add_frame_table(self, gt_segments, pred_segments, pairs, counts):
        """host part of add_frame: (pairs, counts) = the image's sorted (gt * 2^24 + pred) codes and their pixel counts.
        Segment lists become plain dicts as in the reference (a duplicate id keeps its last entry); predicted areas are
        recounted from the table with the reference's sanity checks (KeyError)."""
        gt_segms = {el["id"]: dict(el) for el in gt_segments}
        pred_segms = {el["id"]: dict(el) for el in pred_segments}
        recount_pred_areas(pred_segms, pred_segments, pairs, counts, self.categories)
        self.frames.append((gt_segms, pred_segms, pairs, counts))

    def compute(self):
        """_pq_compute_single_core (base_dataset.py:337-431) over the images added so far, in order, into one PQStat:
        dict category -> vps_b200.vpq.CatStat"""
        stat = defaultdict(CatStat)
        for gt_segms, pred_segms, pairs, counts in self.frames:
            gt_pred = {(lab // OFFSET, lab % OFFSET): c for lab, c in zip(pairs.tolist(), counts.tolist())}
            match_segments(stat, gt_segms, pred_segms, gt_pred, check_iou=False)
        return stat

    def write_pq_txt(self, path, stat):
        """The reference's pq.txt (base_dataset.py:196-211) for `stat`; returns its results dict (All / Things / Stuff and
        per_class, as pq_compute returns it)."""
        metrics = [("All", None), ("Things", True), ("Stuff", False)]
        results = {}
        for name, isthing in metrics:
            results[name], per_class = pq_average(stat, self.categories, isthing=isthing)
            if name == "All":
                results["per_class"] = per_class
        with open(path, "w") as f:
            f.write("================================================\n")
            f.write("{:10s}| {:>5s}  {:>5s}  {:>5s} {:>5s}".format("", "PQ", "SQ", "RQ", "N\n"))
            f.write("-" * (10 + 7 * 4) + "\n")
            for name, _ in metrics:
                r = results[name]
                f.write("{:10s}| {:5.1f}  {:5.1f}  {:5.1f} {:5d}\n".format(name, 100 * r["pq"], 100 * r["sq"], 100 * r["rq"], r["n"]))
            f.write("{:4s}| {:>5s} {:>5s} {:>5s} {:>6s} {:>7s} {:>7s} {:>7s}\n".format("IDX", "PQ", "SQ", "RQ", "IoU", "TP", "FP", "FN"))
            for idx, r in results["per_class"].items():
                f.write("{:4d} | {:5.1f} {:5.1f} {:5.1f} {:6.1f} {:7d} {:7d} {:7d}\n".format(
                    idx, 100 * r["pq"], 100 * r["sq"], 100 * r["rq"], r["iou"], r["tp"], r["fp"], r["fn"]))
        return results
