"""VPQ evaluator core (SURVEY 8f rank 2): `vpq_compute_single_core` + `PQStat.pq_average` of the reference's
tools/eval_vpq.py (:73-203, :44-70) with the pixel-level work on the GPU.

The reference stacks the id maps of every `nframes`-long window and runs np.unique on 64-bit (gt, pred) codes -- the same
frame is re-sorted in up to `nframes` windows and for k in {0,5,10,15}.  Here every frame's (gt, pred, count) table is
computed ONCE on the device (`vps_tube_confusion`: pack -> 64-bit radix sort -> run-length encode) and the window tables
are merged from those few hundred rows on the host; the matching logic is the reference's, in the same iteration order
(so the float IoU sums are identical)."""
import copy
import ctypes as C
from collections import defaultdict

import numpy as np
import torch

from . import ops
from ._lib import lib

OFFSET = 256 * 256 * 256          # eval_vpq.py:74
VOID = 0


class CatStat:
    """PQStatCat (eval_vpq.py:20-32)"""
    __slots__ = ("iou", "tp", "fp", "fn")

    def __init__(self):
        self.iou, self.tp, self.fp, self.fn = 0.0, 0, 0, 0

    def __iadd__(self, o):
        self.iou += o.iou; self.tp += o.tp; self.fp += o.fp; self.fn += o.fn
        return self


def frame_confusion(gt_ids, pred_ids):
    """np.unique(gt * 2^24 + pred, return_counts=True) of one frame on the GPU.  gt_ids / pred_ids: CUDA integer tensors of the
    same shape (ids < 2^24).  Returns (pairs uint64 ascending, counts int64) as numpy arrays."""
    if not (gt_ids.is_cuda and pred_ids.is_cuda):
        raise RuntimeError("frame_confusion: id maps must be CUDA tensors (there is no CPU path)")
    g = gt_ids.reshape(-1).to(torch.int32).contiguous()          # bit pattern of uint32 ids < 2^31
    p = pred_ids.reshape(-1).to(torch.int32).contiguous()
    n = g.numel()
    dev = g.device
    pairs = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
    counts = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    nruns = torch.zeros(1, dtype=torch.int32, device=dev)
    ws = torch.empty(int(lib().vps_tube_confusion_ws_bytes(C.c_int64(n))), dtype=torch.uint8, device=dev)
    ops.check(lib().vps_tube_confusion(ops._ptr(g), ops._ptr(p), C.c_int64(n), C.c_uint64(OFFSET), ops._ptr(pairs), ops._ptr(counts),
                                       ops._ptr(nruns), ops._ptr(ws), C.c_int64(ws.numel()), ops.stream()), "tube_confusion")
    k = int(nruns.item())
    return pairs[:k].cpu().numpy().astype(np.uint64), counts[:k].cpu().numpy().astype(np.int64)


def rgb_to_id(rgb):
    """[H,W,3] uint8 CUDA image -> [H,W] int32 ids (r + 256 g + 65536 b, eval_vpq.py:87-89)"""
    assert rgb.is_cuda and rgb.dtype == torch.uint8 and rgb.shape[-1] == 3
    rgb = rgb.contiguous()
    out = torch.empty(rgb.shape[:-1], dtype=torch.int32, device=rgb.device)
    ops.check(lib().vps_rgb_to_id(ops._ptr(rgb), C.c_int64(out.numel()), ops._ptr(out), ops.stream()), "rgb_to_id")
    return out


def segments_from_pan2ch(pan_2ch, num_stuff=11):
    """Unified 3-channel result (uint8 CUDA [H,W,3], vps_b200.postproc.PanUnifier) -> (id map int32 CUDA [H,W], segments list).
    The reference's converter (tools/dataset/cityscapes_vps.py:96-140) makes the colour panopticapi's IdGenerator returns the
    segment id: one fixed colour per stuff category (all its keys merge into one segment per frame), one colour per
    (thing category, track) key kept across frames.  VPQ is invariant to the id values; the deterministic ids here are
    1000 * semantic + 1 for stuff (semantic < num_stuff) and 1000 * semantic + track + 1 for things, 0 = VOID.
    category_id = semantic class, iscrowd = 0, area = pixel count."""
    assert pan_2ch.is_cuda and pan_2ch.dtype == torch.uint8 and pan_2ch.shape[-1] == 3
    pan_2ch = pan_2ch.contiguous()
    ids = torch.empty(pan_2ch.shape[:-1], dtype=torch.int32, device=pan_2ch.device)
    ops.check(lib().vps_pan2ch_ids(ops._ptr(pan_2ch), C.c_int64(ids.numel()), int(num_stuff), ops._ptr(ids), ops.stream()), "pan2ch_ids")
    pairs, counts = frame_confusion(torch.zeros_like(ids), ids)      # gt = 0: the pair code is the id itself
    segs = []
    for i, a in zip(pairs.tolist(), counts.tolist()):
        if i == VOID:
            continue
        segs.append({"id": int(i), "category_id": int((i - 1) // 1000), "iscrowd": 0, "area": int(a)})
    return ids, segs


def _merge_segments(seg_list):
    out = {}
    for el in seg_list:                                          # eval_vpq.py:90-101
        if el["id"] in out:
            out[el["id"]]["area"] += el["area"]
        else:
            out[el["id"]] = copy.deepcopy(el)
    return out


def recount_pred_areas(pred_segms, pred_segments, pairs, counts, categories):
    """Predicted areas recounted from the id map, with the reference's sanity checks (eval_vpq.py:102-116,
    base_dataset.py:352-366): pred_segms (id -> segment, updated in place) from the list pred_segments; (pairs, counts) =
    the frame's sorted (gt * 2^24 + pred) codes and their pixel counts."""
    area = defaultdict(int)
    for lab, c in zip((pairs % np.uint64(OFFSET)).tolist(), counts.tolist()):
        area[lab] += c
    left = set(el["id"] for el in pred_segments)
    for lab in sorted(area):
        if lab not in pred_segms:
            if lab == VOID:
                continue
            raise KeyError("Segment with ID {} is presented in PNG and not presented in JSON.".format(lab))
        pred_segms[lab]["area"] = area[lab]
        left.remove(lab)
        if pred_segms[lab]["category_id"] not in categories:
            raise KeyError("Segment with ID {} has unknown category_id {}.".format(lab, pred_segms[lab]["category_id"]))
    if left:
        raise KeyError("The following segment IDs {} are presented in JSON and not presented in PNG.".format(sorted(left)))


def match_segments(stat, gt_segms, pred_segms, gt_pred, check_iou):
    """The matching of the reference's PQ cores (eval_vpq.py:157-207 for a tube, base_dataset.py:378-431 for an image):
    gt_segms / pred_segms map id -> segment (area, category_id, iscrowd), gt_pred maps (gt id, pred id) -> intersection in
    ascending key order.  A match needs a non-crowd gt of the same category and IoU > 0.5, with the prediction's VOID pixels
    removed from the union; an unmatched gt is a false negative unless it is crowd; an unmatched prediction is a false
    positive unless more than half of it lies on VOID or on the crowd region of its category.  check_iou: the VPQ core's
    `iou <= 1` assertion (the image core has none).  Adds into stat (category -> CatStat) in the reference's order."""
    gt_matched, pred_matched = set(), set()
    for (g, p), inter in gt_pred.items():
        if g not in gt_segms or p not in pred_segms:
            continue
        if gt_segms[g]["iscrowd"] == 1 or gt_segms[g]["category_id"] != pred_segms[p]["category_id"]:
            continue
        union = pred_segms[p]["area"] + gt_segms[g]["area"] - inter - gt_pred.get((VOID, p), 0)
        iou = inter / union
        if check_iou:
            assert iou <= 1.0, "INVALID IOU VALUE : %d" % g
        if iou > 0.5:
            c = stat[gt_segms[g]["category_id"]]
            c.tp += 1
            c.iou += iou
            gt_matched.add(g)
            pred_matched.add(p)
    crowd = {}
    for g, info in gt_segms.items():
        if g in gt_matched:
            continue
        if info["iscrowd"] == 1:
            crowd[info["category_id"]] = g
            continue
        stat[info["category_id"]].fn += 1
    for p, info in pred_segms.items():
        if p in pred_matched:
            continue
        inter = gt_pred.get((VOID, p), 0)
        if info["category_id"] in crowd:
            inter += gt_pred.get((crowd[info["category_id"]], p), 0)
        if inter / info["area"] > 0.5:
            continue
        stat[info["category_id"]].fp += 1


class VpqEvaluator:
    """Feed the sampled frames of one video in order (`add_frame`), then `compute(nframes)` for every window length."""

    def __init__(self, categories):
        self.categories = categories
        self.frames = []            # (gt_segms, pred_segms, pairs, counts)

    def add_frame(self, gt_segments, pred_segments, gt_ids, pred_ids):
        """gt_ids / pred_ids: CUDA id maps of one sampled frame, of one size.  There is no resizing mode: the reference's VPQ
        core compares the PNGs pixel for pixel and fails on maps of different sizes too."""
        pairs, counts = frame_confusion(gt_ids, pred_ids)
        self.add_frame_table(gt_segments, pred_segments, pairs, counts)

    def add_frame_table(self, gt_segments, pred_segments, pairs, counts):
        """host part of add_frame: (pairs, counts) = the frame's sorted (gt * 2^24 + pred) codes and their pixel counts"""
        gt_segms, pred_segms = _merge_segments(gt_segments), _merge_segments(pred_segments)
        recount_pred_areas(pred_segms, pred_segments, pairs, counts, self.categories)
        self.frames.append((gt_segms, pred_segms, pairs, counts))

    @staticmethod
    def _tube_areas(per_frame):
        vid = {}
        for segms in per_frame:                                  # eval_vpq.py:123-136 (the first frame's dict is extended in place there)
            for k, v in segms.items():
                if k not in vid:
                    vid[k] = copy.deepcopy(v)
                else:
                    vid[k]["area"] += v["area"]
        return vid

    def compute(self, nframes):
        """vpq_compute_single_core (eval_vpq.py:73-203) over the frames added so far.  Returns dict category -> CatStat."""
        stat = defaultdict(CatStat)
        for idx in range(0, len(self.frames) - nframes + 1):
            win = self.frames[idx:idx + nframes]
            vid_gt = self._tube_areas([f[0] for f in win])
            vid_pred = self._tube_areas([f[1] for f in win])
            conf = defaultdict(int)
            for _, _, pairs, counts in win:
                for lab, c in zip(pairs.tolist(), counts.tolist()):
                    conf[lab] += c
            gt_pred = {(lab // OFFSET, lab % OFFSET): conf[lab] for lab in sorted(conf)}     # np.unique order
            match_segments(stat, vid_gt, vid_pred, gt_pred, check_iou=True)
        return stat


def pq_average(stat, categories, isthing=None):
    """PQStat.pq_average (eval_vpq.py:44-70)"""
    pq = sq = rq = 0.0
    n = 0
    per_class = {}
    for label, info in categories.items():
        if isthing is not None and isthing != (info["isthing"] == 1):
            continue
        c = stat[label]
        if c.tp + c.fp + c.fn == 0:
            per_class[label] = {"pq": 0.0, "sq": 0.0, "rq": 0.0, "iou": 0.0, "tp": 0, "fp": 0, "fn": 0}
            continue
        n += 1
        pq_c = c.iou / (c.tp + 0.5 * c.fp + 0.5 * c.fn)
        sq_c = c.iou / c.tp if c.tp != 0 else 0
        rq_c = c.tp / (c.tp + 0.5 * c.fp + 0.5 * c.fn)
        per_class[label] = {"pq": pq_c, "sq": sq_c, "rq": rq_c, "iou": c.iou, "tp": c.tp, "fp": c.fp, "fn": c.fn}
        pq += pq_c; sq += sq_c; rq += rq_c
    return {"pq": pq / n, "sq": sq / n, "rq": rq / n, "n": n}, per_class


NFRAMES_PER_VIDEO = 6           # eval_vpq.py:305: the GT frames of one clip
WINDOWS = (1, 2, 3, 4)          # nframes of the tubes, k = 5 * (nframes - 1) = 0, 5, 10, 15


def split_clips(n_frames, n_annotations, nframes_per_video=NFRAMES_PER_VIDEO):
    """frame indices of each clip: np.array_split of the split's frames into len(gt annotations) // 6 clips (eval_vpq.py:306-309;
    the sizes differ by at most one when the count is uneven)"""
    return [c.tolist() for c in np.array_split(np.arange(n_frames), n_annotations // nframes_per_video)]


def _id_map(img):
    """RGB-coded id image (numpy or torch, [H,W,>=3] uint8) -> int32 CUDA id map"""
    t = img if torch.is_tensor(img) else torch.from_numpy(np.ascontiguousarray(img))
    if t.dim() != 3 or t.shape[2] < 3 or t.dtype != torch.uint8:
        raise ValueError("id image must be uint8 [H, W, 3], got %s %s" % (tuple(t.shape), t.dtype))
    return rgb_to_id(t[..., :3].to("cuda", non_blocking=True).contiguous())


def evaluate_split(gt_json, pred_json, gt_maps, pred_maps, nframes_per_video=NFRAMES_PER_VIDEO, windows=WINDOWS):
    """VPQ of a whole split as tools/eval_vpq.py's main computes it (:281-323), without the files: gt_json / pred_json are
    the loaded JSONs, gt_maps / pred_maps iterables of RGB-coded id images (host or CUDA uint8 [H,W,3]) in the order the
    reference pairs them with the annotations -- zip(gt annotations, pred annotations, gt maps, pred maps).  The maps are
    consumed one frame at a time: each frame's (gt, pred) pair table is built once on the device and the images are dropped.
    Returns {k: {"All", "Things", "Stuff": pq_average results, "per_class": per-category results}} for k = 5 * (nframes - 1).
    Each clip's statistics are summed into the split's in clip order, as PQStat.__iadd__ does, so the IoU sums are the
    reference's to the bit."""
    categories = {el["id"]: el for el in gt_json["categories"]}
    gt_anns, pred_anns = gt_json["annotations"], pred_json["annotations"]
    tables = []
    for (g, p), _ in zip(zip(gt_maps, pred_maps), range(min(len(gt_anns), len(pred_anns)))):
        tables.append(frame_confusion(_id_map(g), _id_map(p)))
    stats = {nf: defaultdict(CatStat) for nf in windows}
    for clip in split_clips(len(tables), len(gt_anns), nframes_per_video):
        ev = VpqEvaluator(categories)
        for i in clip:
            ev.add_frame_table(gt_anns[i]["segments_info"], pred_anns[i]["segments_info"], *tables[i])
        for nf in windows:
            for c, v in ev.compute(nf).items():
                stats[nf][c] += v
    out = {}
    for nf in windows:
        res = {}
        for name, isthing in (("All", None), ("Things", True), ("Stuff", False)):
            res[name], per_class = pq_average(stats[nf], categories, isthing=isthing)
            if name == "All":
                res["per_class"] = per_class
        out[5 * (nf - 1)] = res
    return out


def vpq_text(res):
    """the text of vpq-<k>.txt (eval_vpq.py:233-244) for one entry of evaluate_split's result"""
    lines = ["================================================\n",
             "{:10s}| {:>5s}  {:>5s}  {:>5s} {:>5s}".format("", "PQ", "SQ", "RQ", "N\n"),
             "-" * 38 + "\n"]
    for name in ("All", "Things", "Stuff"):
        r = res[name]
        lines.append("{:10s}| {:5.1f}  {:5.1f}  {:5.1f} {:5d}\n".format(name, 100 * r["pq"], 100 * r["sq"], 100 * r["rq"], r["n"]))
    lines.append("{:4s}| {:>5s} {:>5s} {:>5s} {:>6s} {:>7s} {:>7s} {:>7s}\n".format("IDX", "PQ", "SQ", "RQ", "IoU", "TP", "FP", "FN"))
    for idx, r in res["per_class"].items():
        lines.append("{:4d} | {:5.1f} {:5.1f} {:5.1f} {:6.1f} {:7d} {:7d} {:7d}\n".format(
            idx, 100 * r["pq"], 100 * r["sq"], 100 * r["rq"], r["iou"], r["tp"], r["fp"], r["fn"]))
    return "".join(lines)


def vpq_final_text(results):
    """the text of vpq-final.txt (eval_vpq.py:325-330): the mean over k of 100 * PQ for All, Things and Stuff"""
    ks = sorted(results)
    mean = lambda name: sum(100 * results[k][name]["pq"] for k in ks) / len(ks)
    return "vpq_all:%.4f\nvpq_thing:%.4f\nvpq_stuff:%.4f\n" % (mean("All"), mean("Things"), mean("Stuff"))
