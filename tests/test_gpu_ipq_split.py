"""GPU: the image panoptic model tested and scored end to end.
 * vps_pan2ch_image_segments (the image converter's segment table and pan image) equals numpy exactly: golden ipq frames,
   random 1024x2048 frames, odd sizes, an unaligned source, an all-VOID frame, all 256 instance values of one thing class,
   out-of-range semantics;
 * the driver's scoring half on the golden split gives the reference's pq.txt byte for byte and its IU array as float64;
 * vps_b200.test_eval_ipq on an on-disk split writes what ClipRunner + the oracle converter + the host writer write
   in-process, and scores PQ 100 and IU 1 against ground truth made from that output (tc32, fp32; bf16 is reported)."""
import json
import os
import shutil

import numpy as np
import pytest
import torch

from tests.test_ipq_split_cpu import (GOLD, check_ssegs, golden_outputs, ipq_golden_frames, numpy_image_table,
                                      random_image_frame, same_pred_json)

pytestmark = pytest.mark.gpu


def _check_frame(p2_np, src=None):
    from oracle.ipq import convert_image
    from vps_b200.ipq import image_segment_ids
    from vps_b200.writer import id2rgb, image_segments_from_table, pan2ch_segments
    src = torch.from_numpy(p2_np).cuda() if src is None else src
    table, rgb = pan2ch_segments(src, image=True)
    want = numpy_image_table(p2_np)
    area = want[0] > 0                                              # untouched keys: count 0, min 0xFFFFFFFF, max 0
    assert np.array_equal(table[0], want[0])
    for i in range(1, 5):
        assert np.array_equal(table[i][area], want[i][area]), i
    rgb = rgb.cpu().numpy()
    assert np.array_equal(rgb, id2rgb(image_segment_ids(src).cpu().numpy()))
    info, ids = convert_image(p2_np)
    assert np.array_equal(rgb, id2rgb(ids))
    assert image_segments_from_table(table) == info


def test_image_segment_table_golden_frames(cuda):
    for fr in ipq_golden_frames():
        _check_frame(fr)


def test_image_segment_table_random_odd_and_edge_frames(cuda):
    from vps_b200 import ops
    from vps_b200.writer import NKEY, id2rgb, pan2ch_segments
    rng = np.random.default_rng(6)
    _check_frame(random_image_frame(rng, 1024, 2048))
    _check_frame(random_image_frame(rng, 1024, 2048, block=1))      # a run per pixel
    for H, W in ((1, 1), (37, 53), (7, 1000), (333, 17), (64, 48)):
        _check_frame(random_image_frame(rng, H, W, block=5))
    fr = random_image_frame(rng, 96, 160)                           # unaligned source and W % 16 == 0
    buf = torch.zeros(fr.size + 3, dtype=torch.uint8, device="cuda")
    buf[3:] = torch.from_numpy(fr.reshape(-1)).cuda()
    _check_frame(fr, buf[3:].view(96, 160, 3))
    void = np.zeros((128, 256, 3), np.uint8)
    void[..., 0] = 255
    void[..., 1] = 7
    _check_frame(void)
    thing = np.zeros((64, 512, 3), np.uint8)                        # all 256 instance values of thing class 13 (and stuff)
    thing[..., 0] = 13
    thing[..., 1] = np.tile(np.arange(256, dtype=np.uint8).repeat(2), (64, 1))
    thing[40:, 300:, 0] = 3
    _check_frame(thing)
    bad = thing.copy()                                              # out-of-range semantics: counted, coloured 0
    bad[0, :5, 0] = 19
    bad[7, 9, 0] = 200
    p2 = torch.from_numpy(bad).cuda()
    table = torch.empty(5 * NKEY + 1, dtype=torch.int32, device="cuda")
    rgb = torch.empty_like(p2)
    ops.pan2ch_segments(p2, 11, table, rgb, image=True)
    t = table.cpu().numpy().view(np.uint32)
    assert t[-1] == 6
    ok = bad[..., 0] < 19
    want = numpy_image_table(np.where(ok[..., None], bad, np.uint8(255)))
    assert np.array_equal(t[:-1].reshape(5, 19, 256)[0], want[0])
    got = rgb.cpu().numpy()
    assert (got[~ok] == 0).all()
    ids = 1000 * bad[..., 0].astype(np.int64) + np.where(bad[..., 0] < 11, 0, bad[..., 1]) + 1
    assert np.array_equal(got[ok], id2rgb(ids)[ok])
    with pytest.raises(ValueError):
        pan2ch_segments(p2, image=True)


def _golden_scorer(out):
    from vps_b200.test_eval_ipq import EvalHelper, SplitScorer
    names, _ = golden_outputs()
    helper = EvalHelper(GOLD, pan_gt_folder=os.path.join(GOLD, "panoptic"))
    helper.pair(names)
    return SplitScorer(helper, out, workers=3)


def test_golden_split_scored_as_the_reference(cuda, tmp_path, capsys):
    from tests.golden.make_ipq_split_golden import STUFF_AREA_LIMIT
    from vps_b200.postproc import PanUnifier
    from vps_b200.test_eval_ipq import sseg_text
    names, outs = golden_outputs()
    out = str(tmp_path / "val.pkl")
    uni = PanUnifier(image=True, stuff_area_limit=STUFF_AREA_LIMIT)
    with _golden_scorer(out) as scorer:
        for name, (fcn, pano, cls) in zip(names, outs):
            f = torch.from_numpy(fcn).cuda()
            scorer.add(name, f, uni(f, torch.from_numpy(pano).cuda(), cls))
        res = scorer.finish()
    exp = os.path.join(GOLD, "expected")
    pans = out.replace(".pkl", "_pans_unified")
    assert open(os.path.join(pans, "pq.txt"), "rb").read() == open(os.path.join(exp, "pq.txt"), "rb").read()
    assert np.array_equal(res["sseg"]["IU_array"], np.load(os.path.join(exp, "ssegs.npz"))["IU_array"])
    assert sseg_text(res["sseg"]) == open(os.path.join(exp, "sseg.txt")).read()
    assert open(os.path.join(exp, "sseg.txt")).read() in capsys.readouterr().out
    check_ssegs(out.replace(".pkl", "_ssegs"))
    same_pred_json(json.load(open(os.path.join(pans, "pred.json"))), json.load(open(os.path.join(exp, "pred.json"))))


def test_golden_split_shape_mismatch_names_the_image(cuda, tmp_path):
    names, outs = golden_outputs()
    fcn = torch.from_numpy(outs[0][0]).cuda()
    with _golden_scorer(str(tmp_path / "val.pkl")) as scorer:
        p2 = torch.zeros(fcn.shape[1] + 1, fcn.shape[2], 3, dtype=torch.uint8, device="cuda")
        with pytest.raises(ValueError, match=names[0]):
            scorer.add(names[0], fcn, p2)


# ---- the whole chain on an on-disk split ---------------------------------------------------------------------------------
NIMG, H, W = 6, 128, 256

CONFIG = """
from vps_b200.default_cfg import fuse_cfg as _fuse_cfg
_c = _fuse_cfg()
model = _c["model"]
test_cfg = _c["test_cfg"]
img_norm_cfg = dict(mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], to_rgb=True)
test_pipeline = [
    dict(type='LoadRefImageFromFile'),
    dict(type='MultiScaleFlipAug', img_scale=[(%d, %d)], flip=False,
         transforms=[dict(type='Resize', keep_ratio=True), dict(type='RandomFlip'), dict(type='Normalize', **img_norm_cfg),
                     dict(type='Pad', size_divisor=64), dict(type='ImageToTensor', keys=['img', 'ref_img']),
                     dict(type='Collect', keys=['img', 'ref_img'])])]
data = dict(test=dict(type='CityscapesDataset', data_root='{root}', ann_file='annotations/instancesonly_pano_gtFine_val.json',
                      img_prefix='val/', ref_prefix='val_nbr/', pipeline=test_pipeline))
""" % (W, H)


def _name(i):
    return "%s_000000_%06d_leftImg8bit.png" % ("aachen" if i < 3 else "bonn", 19 * i if i % 3 else 0)


def _write_split(root):
    """NIMG images under val/ with their previous frames under val_nbr/ (fid 0 references itself), the dataset json, a
    fuse.py-style config and a checkpoint of the seeded test weights"""
    import cv2

    from oracle.variants import PanopticFuse, from_fusetrack
    from oracle.weights import make_model
    rng = np.random.default_rng(12)
    for d in ("val", "val_nbr", "annotations", "gt/annotations", "gt/labels", "data/cityscapes/panoptic"):
        os.makedirs(os.path.join(root, d))
    images, frames = [], []
    for i in range(NIMG):
        base = rng.integers(0, 256, size=(H // 8, W // 8, 3)).repeat(8, 0).repeat(8, 1).astype(np.int16)
        img, ref = (np.clip(np.roll(base, (s, 2 * s), (0, 1)) + rng.integers(-6, 7, size=(H, W, 3)), 0, 255).astype(np.uint8)
                    for s in (1, 0))
        n = _name(i)
        fid = int(n.split("_")[-2])
        cv2.imwrite(os.path.join(root, "val", n), img)
        cv2.imwrite(os.path.join(root, "val_nbr", n.replace("%06d_" % fid, "%06d_" % (fid - 1)) if fid else n),
                    ref if fid else img)
        images.append({"id": 40 - i, "file_name": n, "width": W, "height": H})
        frames.append((img, ref if fid else img))
    json.dump({"images": images, "categories": []}, open(os.path.join(root, "annotations", "instancesonly_pano_gtFine_val.json"), "w"))
    open(os.path.join(root, "cfg.py"), "w").write(CONFIG.replace("{root}", root))
    open(os.path.join(root, "test.yaml"), "w").write("dataset:\n  dataset_path: %s\n  test_image_set: val\n"
                                                     "test:\n  panoptic_stuff_area_limit: 2048\n" % os.path.join(root, "gt"))
    m = from_fusetrack(PanopticFuse, make_model("C", 0).state_dict())
    torch.save({"state_dict": m.state_dict(), "meta": {}}, os.path.join(root, "w.pth"))
    return images, frames


def _in_process(root, images, frames, precision, out):
    """ClipRunner(unify=True) on the frames in memory + the oracle converter + the host writer"""
    from oracle.ipq import convert_image
    from vps_b200 import test_vpq as TV
    from vps_b200.pipeline import InputStage
    from vps_b200.runner import ClipRunner
    from vps_b200.writer import ImageWriter
    cfg, model = TV.load_model(os.path.join(root, "cfg.py"), os.path.join(root, "w.pth"), "cuda:0", precision)
    pairs = [(torch.from_numpy(a), torch.from_numpy(b)) for a, b in frames]
    metas = [dict(filename=os.path.join(root, "val", im["file_name"]), iid=im["id"], flip=False) for im in images]
    runner = ClipRunner(model, "cuda:0", unify=True, input_stage=InputStage.from_pipeline(cfg.data.test.pipeline))
    runner.unifier.stuff_area_limit = 2048
    w = ImageWriter(out + "_pans_unified", out + "_ssegs")
    fcns = []
    for im, r in zip(images, runner.run(pairs, metas)):
        p2 = r[2]["pan_2ch"].numpy().copy()
        fcns.append(r[2]["fcn_outputs"].numpy()[0].astype(np.uint8))
        w.add_sseg(im["file_name"], fcns[-1])
        w.add_frame_ids(im["file_name"], *convert_image(p2), p2)
    return w.finish(), fcns


def _truth_from(root, images, out, pred, fcns):
    """ground truth = the in-process output: labels = its semantic maps, panoptic PNGs = its pan/ PNGs, segments = pred.json"""
    gt = os.path.join(root, "gt")
    pan_json = {"images": [], "annotations": [], "categories": [{"id": i, "name": "c%d" % i, "isthing": int(i >= 11)}
                                                                for i in range(19)]}
    from PIL import Image
    for i, (im, ann, fcn) in enumerate(zip(images, pred["annotations"], fcns)):
        n = im["file_name"]
        Image.fromarray(fcn).save(os.path.join(gt, "labels", n.replace("leftImg8bit.png", "gtFine_labelTrainIds.png")))
        shutil.copy(os.path.join(out + "_pans_unified", "pan", n.replace("_leftImg8bit", "")),
                    os.path.join(root, "data", "cityscapes", "panoptic", n))
        pan_json["images"].append({"id": i, "file_name": n})
        pan_json["annotations"].append({"image_id": i, "segments_info": ann["segments_info"]})
    json.dump({"images": [dict(im, id=100 - k) for k, im in enumerate(images)], "categories": []},
              open(os.path.join(gt, "annotations", "instancesonly_gtFine_val.json"), "w"))
    json.dump(pan_json, open(os.path.join(gt, "annotations", "cityscapes_fine_val.json"), "w"))
    return pan_json


def _same_tree(a, b):
    from PIL import Image
    assert json.load(open(os.path.join(a + "_pans_unified", "pred.json"))) == json.load(open(os.path.join(b + "_pans_unified", "pred.json")))
    for sub in ("_pans_unified/pan_2ch", "_pans_unified/pan", "_ssegs"):
        fa, fb = sorted(os.listdir(a + sub)), sorted(os.listdir(b + sub))
        assert fa == fb and len(fa) == NIMG
        for f in fa:
            ia, ib = Image.open(os.path.join(a + sub, f)), Image.open(os.path.join(b + sub, f))
            assert ia.mode == ib.mode and ia.getpalette() == ib.getpalette()
            assert np.array_equal(np.asarray(ia), np.asarray(ib))


def _printed_iu(text):
    lines = text.splitlines()
    i = len(lines) - 1 - lines[::-1].index("IU_array:")
    return np.array([float(v) for v in lines[i + 1:i + 20]])


def test_test_eval_ipq_driver_whole_chain(cuda, tmp_path, monkeypatch, capsys):
    from vps_b200 import test_eval_ipq as T
    root = str(tmp_path / "cityscapes")
    images, frames = _write_split(root)
    monkeypatch.chdir(root)                                         # the panoptic GT is read from data/cityscapes/panoptic
    report = {}
    for precision in ("tc32", "fp32", "bf16"):
        out = os.path.join(root, "work", precision)
        if precision != "bf16":                                     # bf16 is scored against the fp32 ground truth
            pred, fcns = _in_process(root, images, frames, precision, os.path.join(root, "inproc", precision))
            pan_json = _truth_from(root, images, os.path.join(root, "inproc", precision), pred, fcns)
        capsys.readouterr()
        assert T.main([os.path.join(root, "cfg.py"), os.path.join(root, "w.pth"), "--out", out + ".pkl", "--precision", precision,
                       "--test_config", os.path.join(root, "test.yaml"), "--workers", "3"]) == 0
        iu = _printed_iu(capsys.readouterr().out)
        pq = open(os.path.join(out + "_pans_unified", "pq.txt")).read().splitlines()
        if precision == "bf16":
            report["bf16_vs_fp32"] = (pq[3:6], iu.tolist())
            continue
        _same_tree(out, os.path.join(root, "inproc", precision))
        assert json.load(open(os.path.join(out + "_pans_unified", "gt.json"))) == pan_json
        for line in pq[3:6]:
            name, vals = line.split("|")
            pq_, sq, rq, n = vals.split()
            assert (pq_, sq, rq) == ("100.0", "100.0", "100.0") or n == "0", (precision, line)
        assert int(pq[3].split()[-1]) > 0
        # mIoU: the labels are the predictions, so every class present has IU 1 and every absent one 0
        present = np.isin(np.arange(19), np.concatenate([f.ravel() for f in fcns]))
        assert present.any() and np.array_equal(iu, present.astype(np.float64)), (precision, iu)
        report[precision] = (int(present.sum()), sum(len(a["segments_info"]) for a in pred["annotations"]))
    with capsys.disabled():
        print("whole chain:", report)
