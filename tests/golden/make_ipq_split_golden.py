"""Golden split for the image panoptic driver (vps_b200.test_eval_ipq): writes a small synthetic Cityscapes layout and the
model outputs of its images, then runs the REFERENCE's own functions on them in the order tools/test_eval_ipq.py's main
runs them after the model -- the image-level `get_unified_pan_result`, `Cityscapes.evaluate_ssegs`,
`BaseDataset.evaluate_panoptic` -- imported unmodified through make_unify_golden.import_reference, with the stand-in
panopticapi IdGenerator of make_writer_golden.py, one PQ worker (see make_ipq_golden.py) and, in place of pycocotools, an
roidb built as JsonDataset.get_roidb builds it (image ids sorted, image = <dataset_path>/images/<file_name>).

tests/golden/ipq_split/:
    annotations/instancesonly_gtFine_val.json   the roidb's images (one prediction is not in it; ids not in file order)
    annotations/cityscapes_fine_val.json        panoptic GT: crowd segments, VOID pixels, a duplicate id
    labels/<name>_gtFine_labelTrainIds.png      trainIds with 255 and 20; one label larger than its prediction
    panoptic/<file_name>                        panoptic GT PNGs (the reference reads data/cityscapes/panoptic/)
    model_outputs.npz                           names, fcn_outputs, panoptic_outputs, panoptic_cls_inds per image
    expected/pq.txt, sseg.txt, pred.json        the reference's pq.txt, evaluate_ssegs' printed block, pred.json
    expected/ssegs.npz                          the decoded palette PNGs (pixels and palette) and IU_array (float64)

Six images of odd sizes come from make_ipq_golden.synth_frame.  evaluate_panoptic runs np.array_split on lists of images of
different shapes; numpy < 1.24 made a 1-d object array of such a list, numpy >= 1.24 raises, so numpy.array_split is
wrapped during the call to build that object array first, as in make_split_eval_golden.py.  Nothing else of the
reference is touched.
Run where the reference tree is available:  python tests/golden/make_ipq_split_golden.py"""
import contextlib
import io
import json
import os
import shutil
import sys
import tempfile
import types

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_ipq_golden as G  # noqa: E402
from make_unify_golden import import_reference  # noqa: E402
from make_writer_golden import StandInIdGenerator, rgb2id  # noqa: E402

OUT = os.path.join(HERE, "ipq_split")
SIZES = [(61, 97), (63, 101), (67, 99), (61, 105), (65, 97), (71, 103)]
NOT_IN_ROIDB = 4                     # a prediction the mIoU does not count
BIG_LABEL = 2                        # its label PNG is larger than the prediction: evaluate_ssegs resizes with NEAREST
STUFF_AREA_LIMIT = 200


def name(i):
    return "city_%06d_%06d" % (i, 19 + i)


def write_split(out, rng):
    """the on-disk layout and the model outputs; returns (names, segs, pans, clss)"""
    for d in ("annotations", "labels", "panoptic", "expected"):
        os.makedirs(os.path.join(out, d))
    inst_images, pan_images, pan_anns = [], [], []
    segs, pans, clss, names = [], [], [], []
    for i, (h, w) in enumerate(SIZES):
        G.H, G.W = h, w
        seg, pan, cls, gt_ids, segments, trainid = G.synth_frame(rng, i % 3)
        fn = name(i) + "_leftImg8bit.png"
        if i != NOT_IN_ROIDB:
            inst_images.append({"id": 500 - 7 * i if i % 2 else 100 + i, "file_name": fn, "height": h, "width": w})
            if i == BIG_LABEL:
                trainid = np.asarray(Image.fromarray(trainid).resize((w + 13, h + 7), Image.NEAREST))
            Image.fromarray(trainid).save(os.path.join(out, "labels", name(i) + "_gtFine_labelTrainIds.png"))
        pan_images.append({"id": name(i), "file_name": fn, "height": h, "width": w})
        pan_anns.append({"image_id": name(i), "file_name": name(i) + "_gtFine_panoptic.png", "segments_info": segments})
        Image.fromarray(G.id2rgb(gt_ids)).save(os.path.join(out, "panoptic", fn))
        segs.append(seg), pans.append(pan), clss.append(cls), names.append(fn)
    json.dump({"images": inst_images, "annotations": [], "categories": []},
              open(os.path.join(out, "annotations", "instancesonly_gtFine_val.json"), "w"))
    json.dump({"images": pan_images, "annotations": pan_anns, "categories": G.CATEGORIES},
              open(os.path.join(out, "annotations", "cityscapes_fine_val.json"), "w"))
    arrays = {"names": np.array(names)}
    for i in range(len(names)):
        arrays["fcn%d" % i], arrays["pano%d" % i], arrays["cls%d" % i] = segs[i][None], pans[i][None], clss[i]
    np.savez_compressed(os.path.join(out, "model_outputs.npz"), **arrays)
    return names, segs, pans, clss


def main():
    utils = types.ModuleType("panopticapi.utils")
    utils.IdGenerator, utils.rgb2id = StandInIdGenerator, rgb2id
    sys.modules["panopticapi"] = types.ModuleType("panopticapi")
    sys.modules["panopticapi.utils"] = utils
    import_reference()
    import torch.multiprocessing
    torch.multiprocessing.cpu_count = lambda: 1
    from tools.dataset.cityscapes import Cityscapes
    if os.path.isdir(OUT):
        shutil.rmtree(OUT)
    names, segs, pans, clss = write_split(OUT, np.random.default_rng(2718))

    tmp = tempfile.mkdtemp(prefix="ipq_split_golden_")
    assert "images" not in tmp and "labels" not in tmp and "viper" not in tmp
    cwd = os.getcwd()
    try:
        root = os.path.join(tmp, "root")
        shutil.copytree(OUT, root)
        os.makedirs(os.path.join(tmp, "data", "cityscapes"))
        shutil.copytree(os.path.join(OUT, "panoptic"), os.path.join(tmp, "data", "cityscapes", "panoptic"))
        os.chdir(tmp)                                               # panoptic_gt_folder is relative
        helper = Cityscapes.__new__(Cityscapes)
        inst = json.load(open(os.path.join(root, "annotations", "instancesonly_gtFine_val.json")))["images"]
        helper.roidb = [dict(im, image=os.path.join(root, "images", im["file_name"])) for im in sorted(inst, key=lambda im: im["id"])]
        helper.panoptic_json_file = os.path.join(root, "annotations", "cityscapes_fine_val.json")
        helper.panoptic_gt_folder = "data/cityscapes/panoptic"
        out = os.path.join(tmp, "val")
        uni = helper.get_unified_pan_result([s.copy() for s in segs], [p.copy() for p in pans], [c.copy() for c in clss],
                                            stuff_area_limit=STUFF_AREA_LIMIT, names=names)
        captured = {}

        def prof(frame, event, arg):
            if event == "return" and frame.f_code is Cityscapes.evaluate_ssegs.__code__:
                captured.update(frame.f_locals["evaluation_results"])
        buf = io.StringIO()
        sys.setprofile(prof)
        try:
            with contextlib.redirect_stdout(buf):
                helper.evaluate_ssegs(segs, out + "_ssegs", names)
        finally:
            sys.setprofile(None)
        keys = sorted(uni.keys())
        orig_split = np.array_split

        def array_split_legacy(ary, n, axis=0):
            if isinstance(ary, list) and ary and isinstance(ary[0], np.ndarray) and len({a.shape for a in ary}) > 1:
                obj = np.empty(len(ary), dtype=object)
                for i, a in enumerate(ary):
                    obj[i] = a
                ary = obj
            return orig_split(ary, n, axis)
        try:
            np.array_split = array_split_legacy
            helper.evaluate_panoptic([uni[k] for k in keys], out + "_pans_unified")
        finally:
            np.array_split = orig_split
        exp = os.path.join(OUT, "expected")
        open(os.path.join(exp, "sseg.txt"), "w").write(buf.getvalue())
        shutil.copy(os.path.join(out + "_pans_unified", "pq.txt"), exp)
        shutil.copy(os.path.join(out + "_pans_unified", "pred.json"), exp)
        ssegs = {"IU_array": np.asarray(captured["IU_array"], np.float64)}
        for f in sorted(os.listdir(out + "_ssegs")):
            im = Image.open(os.path.join(out + "_ssegs", f))
            ssegs["png:" + f] = np.asarray(im)
            ssegs["palette:" + f] = np.asarray(im.getpalette(), np.uint8)
        np.savez_compressed(os.path.join(exp, "ssegs.npz"), **ssegs)
    finally:
        os.chdir(cwd)
        shutil.rmtree(tmp)
    print(open(os.path.join(OUT, "expected", "sseg.txt")).read())
    print(open(os.path.join(OUT, "expected", "pq.txt")).read())


if __name__ == "__main__":
    main()
