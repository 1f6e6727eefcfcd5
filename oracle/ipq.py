"""ORACLE (test infrastructure, not product code) for the evaluation of the image panoptic model (reference
tools/test_eval_ipq.py): CPU restatements in numpy of

* `get_confusion_matrix` (tools/dataset/base_dataset.py:449-467) and the IU / mean IU of `Cityscapes.evaluate_ssegs`
  (tools/dataset/cityscapes.py:112-151);
* the image converter `_converter_2ch_single_core` (base_dataset.py:287-335);
* `_pq_compute_single_core` (:337-431), whose `PQStat.pq_average` (:41-78) is the VPQ one (oracle.vpq.pq_average);
* the `pq.txt` text of `pq_compute` (:196-211).

Pinned against the reference's own `evaluate_panoptic` / `evaluate_ssegs` by tests/golden/ipq_frames.{npz,json} and
ipq_pq.txt (tests/golden/make_ipq_golden.py; tests/test_ipq_cpu.py).  The reference colours segments with panopticapi's
`IdGenerator` (a fixed colour per stuff category, a fresh one per thing key; not reproducible), so the converter here uses
deterministic ids and is compared modulo a bijection of ids, as oracle/writer.py is."""
from collections import defaultdict

import numpy as np

from oracle.vpq import OFFSET, VOID, CatStat, pq_average


def get_confusion_matrix(gt_label, pred_label, class_num):
    """np.bincount of gt * C + pred, bins < C * C copied to [i, j] (a pred >= C aliases into the next row); float64"""
    index = (np.asarray(gt_label).astype(np.int64) * class_num + np.asarray(pred_label).astype(np.int64)).astype(np.int32)
    count = np.bincount(index.reshape(-1), minlength=class_num * class_num)
    return count[:class_num * class_num].reshape(class_num, class_num).astype(np.float64)


def seg_confusion(gt_trainids, pred, class_num=19):
    """one frame of evaluate_ssegs: pixels with gt 255 dropped, the prediction taken as the uint8 the reference saves"""
    gt = np.asarray(gt_trainids)
    pr = np.asarray(pred).astype(np.uint8)
    keep = gt != 255
    return get_confusion_matrix(gt[keep], pr[keep], class_num)


def seg_result(conf):
    """IU / mean IU of evaluate_ssegs from the frame-summed float64 confusion matrix"""
    pos, res, tp = conf.sum(1), conf.sum(0), np.diag(conf)
    iu = tp / np.maximum(1.0, pos + res - tp)
    return {"meanIU": iu.mean(), "IU_array": iu, "confusion_matrix": conf}


def convert_image(pan_2ch, num_stuff=11):
    """_converter_2ch_single_core on one image: keys 1000 * semantic + instance (channel 1) in ascending order, VOID
    (semantic 255) skipped, one segments_info entry per key (bbox [x, y, x_max - x, y_max - y], area = the key's pixels).
    Ids: 1000 * semantic + 1 for a stuff category (its fixed colour: every key of it shares the id), 1000 * semantic +
    instance + 1 for a thing key, 0 = VOID.  Returns (segments_info, ids uint32 [H,W])."""
    p = np.asarray(pan_2ch).astype(np.uint32)
    sem, ins = p[..., 0], p[..., 1]
    key = 1000 * sem + ins
    ids = np.where(sem == 255, 0, 1000 * sem + np.where(sem < num_stuff, 0, ins) + 1).astype(np.uint32)
    info = []
    for k in np.unique(key).tolist():
        if k // 1000 == 255:
            continue
        m = key == k
        ys, xs = np.nonzero(m)
        x, y = int(xs.min()), int(ys.min())
        info.append({"category_id": int(k // 1000), "iscrowd": 0, "id": int(ids[m][0]),
                     "bbox": [x, y, int(xs.max()) - x, int(ys.max()) - y], "area": int(m.sum())})
    return info, ids


def pq_compute_single_core(frames, categories):
    """frames: list of (gt_segments, pred_segments, gt_ids [H,W], pred_ids [H,W]) in order.  Returns category -> CatStat."""
    stat = defaultdict(CatStat)
    for gt_segments, pred_segments, gt_ids, pred_ids in frames:
        gt_segms = {el["id"]: dict(el) for el in gt_segments}
        pred_segms = {el["id"]: dict(el) for el in pred_segments}
        left = set(el["id"] for el in pred_segments)
        labels, cnt = np.unique(np.asarray(pred_ids), return_counts=True)
        for lab, c in zip(labels.tolist(), cnt.tolist()):
            if lab not in pred_segms:
                if lab == VOID:
                    continue
                raise KeyError("segment with ID %d is presented in PNG and not presented in JSON." % lab)
            pred_segms[lab]["area"] = c
            left.remove(lab)
            if pred_segms[lab]["category_id"] not in categories:
                raise KeyError("segment with ID %d has unknown category_id" % lab)
        if left:
            raise KeyError("segment IDs %s are presented in JSON and not presented in PNG." % sorted(left))
        packed = np.asarray(gt_ids).astype(np.uint64) * np.uint64(OFFSET) + np.asarray(pred_ids).astype(np.uint64)
        conf = {}
        for lab, inter in zip(*(a.tolist() for a in np.unique(packed, return_counts=True))):
            conf[(lab // OFFSET, lab % OFFSET)] = inter
        gt_matched, pred_matched = set(), set()
        for (g, p), inter in conf.items():
            if g not in gt_segms or p not in pred_segms:
                continue
            if gt_segms[g]["iscrowd"] == 1 or gt_segms[g]["category_id"] != pred_segms[p]["category_id"]:
                continue
            iou = inter / (pred_segms[p]["area"] + gt_segms[g]["area"] - inter - conf.get((VOID, p), 0))
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
            inter = conf.get((VOID, p), 0)
            if info["category_id"] in crowd:
                inter += conf.get((crowd[info["category_id"]], p), 0)
            if inter / info["area"] > 0.5:
                continue
            stat[info["category_id"]].fp += 1
    return stat


def pq_txt(stat, categories):
    """the text pq_compute writes to pq.txt"""
    metrics = [("All", None), ("Things", True), ("Stuff", False)]
    res = {name: pq_average(stat, categories, isthing=t) for name, t in metrics}
    lines = ["================================================\n",
             "{:10s}| {:>5s}  {:>5s}  {:>5s} {:>5s}".format("", "PQ", "SQ", "RQ", "N\n"),
             "-" * 38 + "\n"]
    for name, _ in metrics:
        r = res[name][0]
        lines.append("{:10s}| {:5.1f}  {:5.1f}  {:5.1f} {:5d}\n".format(name, 100 * r["pq"], 100 * r["sq"], 100 * r["rq"], r["n"]))
    lines.append("{:4s}| {:>5s} {:>5s} {:>5s} {:>6s} {:>7s} {:>7s} {:>7s}\n".format("IDX", "PQ", "SQ", "RQ", "IoU", "TP", "FP", "FN"))
    for idx, r in res["All"][1].items():
        lines.append("{:4d} | {:5.1f} {:5.1f} {:5.1f} {:6.1f} {:7d} {:7d} {:7d}\n".format(
            idx, 100 * r["pq"], 100 * r["sq"], 100 * r["rq"], r["iou"], r["tp"], r["fp"], r["fn"]))
    return "".join(lines)
