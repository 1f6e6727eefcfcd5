"""Golden vectors for the evaluation of the image panoptic model (reference tools/test_eval_ipq.py): runs the REFERENCE's
own `BaseDataset.evaluate_panoptic` (tools/dataset/base_dataset.py:104-229) end to end and `Cityscapes.evaluate_ssegs`
(tools/dataset/cityscapes.py:112-166), imported unmodified through make_unify_golden.import_reference, on seeded synthetic
frames whose predictions come from the reference's own image-level get_unified_pan_result.

* evaluate_panoptic reads GT panoptic PNGs + a GT json written to a temporary directory (through a stub `self` carrying
  panoptic_json_file / panoptic_gt_folder), colours segments with the stand-in panopticapi IdGenerator of
  make_writer_golden.py (ids are compared modulo a bijection), and runs with torch.multiprocessing.cpu_count patched to 1:
  the reference adds per-worker PQStats, so its float IoU sums depend on the worker count; with one worker its order is
  the frame order.
* evaluate_ssegs reads label PNGs through a stub carrying roidb; it prints its results, so they are taken from its frame
  at return, and get_confusion_matrix is recorded per frame for the exact counts.

The frames hold crowd GT segments, VOID GT pixels, a predicted segment mostly on VOID and one mostly on crowd (neither a
false positive), a category mismatch, an IoU of exactly 0.5, a duplicate GT id (the last entry wins), GT trainIds 255 and
20, predicted labels >= 19, a predicted stuff class removed by the stuff area limit, and an odd frame size.
Output: tests/golden/ipq_frames.npz, ipq_frames.json, ipq_pq.txt.
Run where the reference tree is available:  python tests/golden/make_ipq_golden.py"""
import json
import os
import shutil
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_unify_golden import import_reference  # noqa: E402
from make_writer_golden import StandInIdGenerator, rgb2id  # noqa: E402

H, W = 61, 97
NFR = 3
STUFF_AREA_LIMIT = 200
CATEGORIES = [{"id": i, "name": "c%d" % i, "isthing": 1 if i >= 11 else 0} for i in range(19)]


def id2rgb(ids):
    ids = ids.astype(np.uint32)
    return np.stack([ids % 256, (ids // 256) % 256, ids // 65536], -1).astype(np.uint8)


def synth_frame(rng, f):
    """(seg, pan, cls) for the image unify, the GT id map with its segments_info, and the GT trainIds"""
    stuff = rng.choice([0, 1, 2, 3, 5], size=((H + 15) // 16, (W + 15) // 16)).repeat(16, 0).repeat(16, 1)[:H, :W]
    seg = stuff.astype(np.uint8).copy()
    seg[50:58, 5:15] = 9                                      # a stuff class under the area limit -> VOID in the prediction
    pan = seg.copy()
    gkey = 1000 * seg.astype(np.int64)                        # GT keys: 1000 * category + instance
    cls = rng.integers(1, 9, size=6)
    jit = lambda: int(rng.integers(0, 3))                    # noqa: E731
    rects = [(10 + jit(), 25, 2, 20 + jit()),                # 0: crowd in the GT
             (10, 24 + jit(), 25 + jit(), 45),               # 1: category mismatch
             (30 + jit(), 46, 2, 2 + 2 * (6 + jit())),       # 2: GT = left half -> IoU exactly 0.5
             (30, 45 + jit(), 30 + jit(), 50),               # 3: exact match
             (0, 6, 70 + jit(), 82),                         # 4: 4 of 6 rows on VOID, no GT instance
             (48 + jit(), 58, 60, 80 + jit())]               # 5: the semantic head votes stuff -> demoted
    for j, (y0, y1, x0, x1) in enumerate(rects):
        pan[y0:y1, x0:x1] = 11 + j
        seg[y0:y1, x0:x1] = 10 + cls[j] if j != 5 else 2
        if j == 4:
            continue
        if j == 2:
            x1 = (x0 + x1) // 2
        gkey[y0:y1, x0:x1] = 1000 * (10 + cls[j]) + j + 1
    seg[40:43, 85:90] = 21                                    # predicted labels >= 19 alias into the next row
    gkey[:4] = -1                                             # VOID band
    gt_ids = np.where(gkey < 0, 0, gkey + 5).astype(np.uint32)
    segments = []
    for i, a in zip(*np.unique(gt_ids, return_counts=True)):
        if i == 0:
            continue
        k = int(i) - 5
        cat, inst = k // 1000, k % 1000
        if inst == 2:
            cat = 11 + (cat - 10) % 8                         # instance 1: GT category differs from the prediction
        segments.append({"id": int(i), "category_id": int(cat), "iscrowd": int(inst == 1), "area": int(a)})
    if f == 1:                                                # a duplicate id: the plain dict keeps the LAST entry
        segments.insert(0, dict(segments[0], area=segments[0]["area"] + 1000))
    cat_of = {s["id"]: s["category_id"] for s in segments}
    trainid = np.full((H, W), 255, np.uint8)
    for i, c in cat_of.items():
        trainid[gt_ids == i] = c
    trainid[55:58, 88:93] = 20
    return seg, pan, cls.astype(np.int64), gt_ids, segments, trainid


class _Stub:
    pass


def run_evaluate_panoptic(BaseDataset, pans_2ch, gt_ids, gt_segments, tmp):
    import torch.multiprocessing
    torch.multiprocessing.cpu_count = lambda: 1
    gt_folder = os.path.join(tmp, "gt_pan")
    os.makedirs(gt_folder)
    from PIL import Image
    images, anns = [], []
    for i, (ids, segs) in enumerate(zip(gt_ids, gt_segments)):
        name = "f%d_gtFine_panoptic.png" % i
        Image.fromarray(id2rgb(ids)).save(os.path.join(gt_folder, name))
        images.append({"id": i, "file_name": name, "height": H, "width": W})
        anns.append({"image_id": i, "file_name": name, "segments_info": segs})
    json_file = os.path.join(tmp, "gt.json")
    json.dump({"images": images, "annotations": anns, "categories": CATEGORIES}, open(json_file, "w"))
    stub = _Stub()
    stub.panoptic_json_file, stub.panoptic_gt_folder = json_file, gt_folder
    out_dir = os.path.join(tmp, "pans_unified")
    results = BaseDataset.evaluate_panoptic(stub, pans_2ch, out_dir)
    pred_json = json.load(open(os.path.join(out_dir, "pred.json")))
    pq_txt = open(os.path.join(out_dir, "pq.txt")).read()
    return results, pred_json, pq_txt


def run_evaluate_ssegs(Cityscapes, trainids, fcns, tmp):
    from PIL import Image
    os.makedirs(os.path.join(tmp, "images"))
    os.makedirs(os.path.join(tmp, "labels"))
    roidb, names = [], []
    for i, t in enumerate(trainids):
        Image.fromarray(t).save(os.path.join(tmp, "labels", "f%d_gtFine_labelTrainIds.png" % i))
        roidb.append({"image": os.path.join(tmp, "images", "f%d_leftImg8bit.png" % i)})
        names.append("f%d_leftImg8bit.png" % i)
    stub = Cityscapes.__new__(Cityscapes)
    stub.roidb = roidb
    per_frame = []

    def get_confusion_matrix(gt, pred, class_num):
        m = Cityscapes.get_confusion_matrix(stub, gt, pred, class_num)
        per_frame.append(m.copy())
        return m
    stub.get_confusion_matrix = get_confusion_matrix
    captured = {}

    def prof(frame, event, arg):
        if event == "return" and frame.f_code is Cityscapes.evaluate_ssegs.__code__:
            captured.update(frame.f_locals["evaluation_results"])
    sys.setprofile(prof)
    try:
        Cityscapes.evaluate_ssegs(stub, fcns, os.path.join(tmp, "ssegs"), names)
    finally:
        sys.setprofile(None)
    return captured, per_frame


def main():
    utils = types.ModuleType("panopticapi.utils")
    utils.IdGenerator, utils.rgb2id = StandInIdGenerator, rgb2id
    sys.modules["panopticapi"] = types.ModuleType("panopticapi")
    sys.modules["panopticapi.utils"] = utils
    import_reference()
    from tools.dataset.base_dataset import BaseDataset
    from tools.dataset.cityscapes import Cityscapes
    rng = np.random.default_rng(314)
    frames = [synth_frame(rng, f) for f in range(NFR)]
    names = ["f%d" % i for i in range(NFR)]
    uni = BaseDataset.get_unified_pan_result(None, [f[0].copy() for f in frames], [f[1].copy() for f in frames],
                                             [f[2].copy() for f in frames], stuff_area_limit=STUFF_AREA_LIMIT, names=names)
    pans_2ch = [uni[n] for n in names]
    for f, p in zip(frames, pans_2ch):
        assert (p[..., 0][f[1] == 9] == 255).all()           # the small stuff class was removed
    tmp = tempfile.mkdtemp(prefix="ipq_golden_")
    assert "viper" not in tmp and "images" not in tmp and "labels" not in tmp
    try:
        results, pred_json, pq_txt = run_evaluate_panoptic(BaseDataset, pans_2ch, [f[3] for f in frames], [f[4] for f in frames], tmp)
        sseg, per_frame = run_evaluate_ssegs(Cityscapes, [f[5] for f in frames], [f[0] for f in frames], tmp)
    finally:
        shutil.rmtree(tmp)
    assert len(per_frame) == NFR and sseg
    out = {"nframes": np.int64(NFR), "stuff_area_limit": np.int64(STUFF_AREA_LIMIT)}
    for i, f in enumerate(frames):
        out["pan2ch%d" % i], out["gt_ids%d" % i], out["trainid%d" % i], out["fcn%d" % i] = pans_2ch[i], f[3], f[5], f[0]
        out["seg_conf%d" % i] = per_frame[i]
    out["seg_confusion"] = sseg["confusion_matrix"]
    out["IU_array"] = sseg["IU_array"]
    out["meanIU"] = np.float64(sseg["meanIU"])
    pc = results["per_class"]
    out["stat"] = np.array([[pc[c["id"]]["iou"], pc[c["id"]]["tp"], pc[c["id"]]["fp"], pc[c["id"]]["fn"]] for c in CATEGORIES],
                           dtype=np.float64)
    out["avg"] = np.array([[results[n]["pq"], results[n]["sq"], results[n]["rq"], results[n]["n"]] for n in ("All", "Things", "Stuff")],
                          dtype=np.float64)
    np.savez_compressed(os.path.join(HERE, "ipq_frames.npz"), **out)
    json.dump({"categories": CATEGORIES, "gt": [f[4] for f in frames], "pred": [a["segments_info"] for a in pred_json["annotations"]]},
              open(os.path.join(HERE, "ipq_frames.json"), "w"))
    open(os.path.join(HERE, "ipq_pq.txt"), "w").write(pq_txt)
    print(pq_txt)
    print("meanIU", sseg["meanIU"])


if __name__ == "__main__":
    main()
