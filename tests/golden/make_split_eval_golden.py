"""Golden split for the split-level VPQ scorer (vps_b200.eval_vpq): runs the REFERENCE's own tools/eval_vpq.py `main`
(imported unmodified from /root/reference, sys.argv set) on a small synthetic Cityscapes-VPS split written here, and keeps
the split and the texts it writes under tests/golden/split_eval/:

    truth/<name>_final_mask.png | <name>_gtFine_color.png, gt.json       (ground truth, as --truth_dir / --pan_gt_json_file)
    submit/pred.json, submit/pan_pred/<id>.png                             (a prediction, as --submit_dir)
    expected/vpq-{0,5,10,15}.txt, vpq-final.txt                            (the reference's output, byte for byte)
    stats.json                                                             (the split PQStat behind each vpq-k.txt)

20 frames of 48x64 make 20 // 6 = 3 clips of 7, 7 and 6 frames (an uneven np.array_split); the frames come from
make_vpq_golden.synth_clip: VOID bands, a crowd region with a prediction inside it, matched, poorly overlapping (FP + FN),
missed and hallucinated instances.  GT names mix the _newImg8bit and _leftImg8bit suffixes.

The reference's main runs np.array_split on a list of (dict, dict, array, array, dict) tuples.  numpy < 1.24 turned that list
into an (n, 5) object array; numpy >= 1.24 raises on the ragged input.  numpy.array_split is wrapped during the call to build
that object array first, as older numpy did; nothing else of the reference is touched.
Run in the build container only:  python tests/golden/make_split_eval_golden.py"""
import importlib.util
import json
import os
import shutil
import sys

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests.golden.make_vpq_golden import synth_clip, to_rgb  # noqa: E402

REF = "/root/reference/tools/eval_vpq.py"
OUT = os.path.join(HERE, "split_eval")
CLIPS = (7, 7, 6)
H, W = 48, 64


def names():
    out = []
    for i in range(sum(CLIPS)):
        base = "%04d_%04d_frankfurt_000000_%06d" % (i // 6, 5 * i % 30, 1000 + i)
        out.append((base, base + ("_newImg8bit.png" if i % 3 else "_leftImg8bit.png")))
    return out


def gt_png_name(file_name):
    return file_name.replace("_newImg8bit.png", "_final_mask.png").replace("_leftImg8bit.png", "_gtFine_color.png")


def main():
    spec = importlib.util.spec_from_file_location("ref_eval_vpq", REF)
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    rng = np.random.default_rng(11)
    frames = [f for n in CLIPS for f in synth_clip(rng, n, H, W)]
    if os.path.isdir(OUT):
        shutil.rmtree(OUT)
    for d in ("truth", "submit/pan_pred", "expected"):
        os.makedirs(os.path.join(OUT, d))
    categories = [{"id": i, "name": "c%d" % i, "isthing": 1 if i >= 11 else 0} for i in range(19)]
    gt_json = {"images": [], "annotations": [], "categories": categories}
    pred_json = {"annotations": []}
    for (base, fname), (gseg, pseg, gt, pr) in zip(names(), frames):
        gt_json["images"].append({"id": base, "file_name": fname, "width": W, "height": H})
        gt_json["annotations"].append({"image_id": base, "file_name": base + ".png", "segments_info": gseg})
        pred_json["annotations"].append({"segments_info": pseg})
        Image.fromarray(to_rgb(gt)).save(os.path.join(OUT, "truth", gt_png_name(fname)))
        Image.fromarray(to_rgb(pr)).save(os.path.join(OUT, "submit", "pan_pred", base + ".png"))
    json.dump(gt_json, open(os.path.join(OUT, "gt.json"), "w"))
    json.dump(pred_json, open(os.path.join(OUT, "submit", "pred.json"), "w"))

    stats = []
    orig_avg = ref.PQStat.pq_average

    def pq_average(self, cats, isthing):
        if isthing is None:                          # once per k, in k order (vpq_compute)
            stats.append({str(c): [v.iou, v.tp, v.fp, v.fn] for c, v in self.pq_per_cat.items()})
        return orig_avg(self, cats, isthing)
    ref.PQStat.pq_average = pq_average

    orig_split = np.array_split

    def array_split_legacy(ary, n, axis=0):
        if isinstance(ary, list) and ary and isinstance(ary[0], tuple):
            obj = np.empty((len(ary), len(ary[0])), dtype=object)
            for i, row in enumerate(ary):
                for j, v in enumerate(row):
                    obj[i, j] = v
            ary = obj
        return orig_split(ary, n, axis)

    work = os.path.join(OUT, "_run")
    shutil.copytree(os.path.join(OUT, "submit"), work)
    argv = sys.argv
    try:
        np.array_split = array_split_legacy
        sys.argv = ["eval_vpq.py", "--submit_dir", work + "/", "--truth_dir", os.path.join(OUT, "truth"),
                    "--pan_gt_json_file", os.path.join(OUT, "gt.json")]
        ref.main()
    finally:
        np.array_split, sys.argv = orig_split, argv
    for k in (0, 5, 10, 15):
        shutil.copy(os.path.join(work, "vpq-%d.txt" % k), os.path.join(OUT, "expected"))
    shutil.copy(os.path.join(work, "vpq-final.txt"), os.path.join(OUT, "expected"))
    shutil.rmtree(work)
    json.dump({"k": [0, 5, 10, 15], "stats": stats}, open(os.path.join(OUT, "stats.json"), "w"))
    print(open(os.path.join(OUT, "expected", "vpq-final.txt")).read())


if __name__ == "__main__":
    main()
