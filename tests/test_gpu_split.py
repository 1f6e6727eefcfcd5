"""GPU: a Cityscapes-VPS split tested and scored end to end.
 * vps_pan2ch_segments (the writer's segment table and pan_pred image) equals numpy exactly: golden unify / writer frames,
   random 1024x2048 frames, odd sizes, an unaligned source, an all-VOID frame, all 256 track values of one stuff class;
 * vps_pan2ch_segments' table through segments_from_table equals the oracle converter (oracle.writer.convert_frame);
 * PanWriter.add_frame (device table) writes the same pred.json and PNGs as the oracle converter through add_frame_ids on
   a model-produced clip;
 * vps_b200.eval_vpq on the golden split writes the reference's vpq-*.txt byte for byte;
 * vps_b200.test_vpq on an on-disk split writes what ClipRunner + PanUnifier + the oracle converter write in-process, and
   scores VPQ 100 against ground truth made from that output (tc32, fp32; bf16 is reported)."""
import filecmp
import json
import os
import shutil

import numpy as np
import pytest
import torch

from tests.test_split_cpu import GOLD, _numpy_table

pytestmark = pytest.mark.gpu
HERE = os.path.join(os.path.dirname(__file__), "golden")


def _check_frame(p2_np, src=None):
    from oracle.writer import convert_frame
    from vps_b200.writer import id2rgb, pan2ch_segments, segments_from_table
    src = torch.from_numpy(p2_np).cuda() if src is None else src
    table, rgb = pan2ch_segments(src)
    want = _numpy_table(p2_np)
    area = want[0] > 0                                              # untouched keys: count 0, min 0xFFFFFFFF, max 0
    assert np.array_equal(table[0], want[0])
    for i in range(1, 5):
        assert np.array_equal(table[i][area], want[i][area]), i
    segs, ids = convert_frame(p2_np)
    assert np.array_equal(rgb.cpu().numpy(), id2rgb(ids))
    assert segments_from_table(table) == segs


def _random_frame(rng, H, W, block=16):
    hb, wb = (H + block - 1) // block, (W + block - 1) // block
    sem = rng.choice(np.r_[np.arange(19), 255], size=(hb, wb)).repeat(block, 0).repeat(block, 1)[:H, :W]
    trk = rng.integers(0, 256, size=(hb, wb)).repeat(block, 0).repeat(block, 1)[:H, :W]
    out = np.zeros((H, W, 3), np.uint8)
    out[..., 0], out[..., 1], out[..., 2] = sem, rng.integers(0, 256, (H, W)), trk
    return out


def test_segment_table_golden_frames_vs_oracle(cuda):
    d = np.load(os.path.join(HERE, "unify_pan.npz"))
    keys = [k for k in d.keys() if k.startswith("out")]
    assert keys
    for k in keys:
        _check_frame(d[k])
    from tests.test_writer_cpu import _golden
    for fr in _golden()[0]:
        _check_frame(fr)


def test_segment_table_random_odd_and_edge_frames_vs_oracle(cuda):
    rng = np.random.default_rng(5)
    _check_frame(_random_frame(rng, 1024, 2048))
    _check_frame(_random_frame(rng, 1024, 2048, block=1))           # a run per pixel
    for H, W in ((1, 1), (37, 53), (7, 1000), (333, 17), (64, 48)):
        _check_frame(_random_frame(rng, H, W, block=5))
    fr = _random_frame(rng, 96, 160)                                  # unaligned source and W % 16 == 0
    buf = torch.zeros(fr.size + 3, dtype=torch.uint8, device="cuda")
    buf[3:] = torch.from_numpy(fr.reshape(-1)).cuda()
    _check_frame(fr, buf[3:].view(96, 160, 3))
    void = np.zeros((128, 256, 3), np.uint8)
    void[..., 0] = 255
    _check_frame(void)
    from vps_b200.writer import pan2ch_segments, segments_from_table
    assert segments_from_table(pan2ch_segments(torch.from_numpy(void).cuda())[0]) == []
    stuff = np.zeros((64, 512, 3), np.uint8)                          # all 256 track values of stuff class 7 (and a thing)
    stuff[..., 0] = 7
    stuff[..., 2] = np.tile(np.arange(256, dtype=np.uint8).repeat(2), (64, 1))
    stuff[40:, 300:, 0] = 14
    _check_frame(stuff)
    bad = stuff.copy()
    bad[0, 0, 0] = 19
    with pytest.raises(ValueError):
        pan2ch_segments(torch.from_numpy(bad).cuda())


def _model_clip(precision, nfr=6, H=128, W=256):
    from tests.e2e_util import build_models, make_pair, meta
    from vps_b200.runner import ClipRunner
    _, prod = build_models("C", 0, precision, "cuda:0")
    prod.label_dtype = torch.uint8
    frames = [make_pair(H, W, seed=40 + s) for s in range(nfr)]
    metas = [meta(10001 + f, H, W) for f in range(nfr)]
    pinned = [(a.pin_memory(), b.pin_memory()) for a, b in frames]
    return [r[2]["pan_2ch"].clone() for r in ClipRunner(prod, "cuda:0", unify=True).run(pinned, metas)]


def _same_tree(a, b):
    from PIL import Image
    assert json.load(open(os.path.join(a, "pred.json"))) == json.load(open(os.path.join(b, "pred.json")))
    for sub in ("pan_pred", "pan_2ch"):
        fa, fb = sorted(os.listdir(os.path.join(a, sub))), sorted(os.listdir(os.path.join(b, sub)))
        assert fa == fb and fa
        for f in fa:
            assert np.array_equal(np.asarray(Image.open(os.path.join(a, sub, f))), np.asarray(Image.open(os.path.join(b, sub, f))))


def test_writer_device_table_equals_oracle_host_path(cuda, tmp_path):
    from oracle.writer import convert_frame
    from vps_b200.writer import PanWriter
    clip = _model_clip("fp32")
    dev, host = PanWriter(str(tmp_path / "dev"), sample=False, workers=2, max_pending=2), PanWriter(str(tmp_path / "host"), sample=False)
    for i, p2 in enumerate(clip):
        name = "frankfurt_%06d_leftImg8bit.png" % i
        if i % 3 == 0:                                                   # device input
            a = dev.add_frame(name, p2.cuda())
        elif i % 3 == 1:                                                 # host input (uploaded)
            a = dev.add_frame(name, p2)
        else:                                                            # device input with a host copy, as the driver
            a = dev.add_frame(name, p2.cuda(), pan_2ch_host=p2)
        p = p2.numpy()
        assert a == host.add_frame_ids(name, *convert_frame(p), p)
    assert dev.finish() == host.finish()
    _same_tree(str(tmp_path / "dev"), str(tmp_path / "host"))


def test_eval_vpq_golden_split_byte_identical(cuda, tmp_path):
    from vps_b200 import eval_vpq as E
    sub = tmp_path / "submit"
    shutil.copytree(os.path.join(GOLD, "submit"), str(sub))
    os.chmod(str(sub), 0o755)                       # copytree keeps the mode of a read-only checkout; vpq-*.txt go here
    assert E.main(["--submit_dir", str(sub) + "/", "--truth_dir", os.path.join(GOLD, "truth"),
                   "--pan_gt_json_file", os.path.join(GOLD, "gt.json"), "--workers", "3"]) == 0
    for f in ("vpq-0.txt", "vpq-5.txt", "vpq-10.txt", "vpq-15.txt", "vpq-final.txt"):
        assert filecmp.cmp(str(sub / f), os.path.join(GOLD, "expected", f), shallow=False), f


# ---- the whole chain on an on-disk split ---------------------------------------------------------------------------------
NCLIP, NFR, H, W = 2, 30, 128, 256

CONFIG = """
from vps_b200.default_cfg import fusetrack_cfg as _fusetrack_cfg
_c = _fusetrack_cfg()
model = _c["model"]
test_cfg = _c["test_cfg"]
img_norm_cfg = dict(mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], to_rgb=True)
test_pipeline = [
    dict(type='LoadRefImageFromFile'),
    dict(type='MultiScaleFlipAug', img_scale=[(%d, %d)], flip=False,
         transforms=[dict(type='Resize', keep_ratio=True), dict(type='RandomFlip'), dict(type='Normalize', **img_norm_cfg),
                     dict(type='Pad', size_divisor=64), dict(type='ImageToTensor', keys=['img', 'ref_img']),
                     dict(type='Collect', keys=['img', 'ref_img'])])]
data = dict(test=dict(type='CityscapesVPSDataset', data_root=%r, ann_file='im_all_info_test_city_vps.json',
                      img_prefix='test/img_all/', ref_prefix='test/img_all/', nframes_span_test=%d, pipeline=test_pipeline))
""" % (W, H, "{root}", NFR)


def _frame_name(c, f):
    return "%04d_%04d_frankfurt_000000_%06d_leftImg8bit.png" % (c, f, 100 + f)


def _write_split(root):
    """NCLIP clips of NFR frames under root/val/img_all (the config says test/: --mode val rewrites it), im_all_info, the
    pan_im_json of the sampled frames, a config and a checkpoint of the seeded test weights"""
    import cv2
    from oracle.weights import make_model
    rng = np.random.default_rng(9)
    os.makedirs(os.path.join(root, "val", "img_all"))
    images, frames = [], []
    for c in range(NCLIP):
        base = rng.integers(0, 256, size=(H // 8, W // 8, 3)).repeat(8, 0).repeat(8, 1).astype(np.int16)
        for f in range(NFR):
            img = np.clip(np.roll(base, (f, 2 * f), (0, 1)) + rng.integers(-6, 7, size=(H, W, 3)), 0, 255).astype(np.uint8)
            name = _frame_name(c, f)
            cv2.imwrite(os.path.join(root, "val", "img_all", name), img)
            images.append({"id": (c + 1) * 10000 + f + 1, "file_name": name, "width": W, "height": H})
            frames.append(img)
    json.dump({"images": images, "categories": []}, open(os.path.join(root, "im_all_info_val_city_vps.json"), "w"))
    sampled = [im["file_name"] for im in images][4::5]
    json.dump({"images": [{"id": n[:-len("_leftImg8bit.png")], "file_name": n} for n in sampled[::-1]]},
              open(os.path.join(root, "pan_im.json"), "w"))
    open(os.path.join(root, "cfg.py"), "w").write(CONFIG.replace("'{root}'", repr(root)))
    open(os.path.join(root, "test.yaml"), "w").write("test:\n  panoptic_stuff_area_limit: 2048\n")
    torch.save({"state_dict": make_model("C", 0).state_dict(), "meta": {}}, os.path.join(root, "w.pth"))
    return images, frames, sorted(sampled)


def _in_process(root, images, frames, names, precision, out):
    """ClipRunner + PanUnifier + the oracle converter + the host writer, fed directly (frame i references frame i - 1
    inside its clip)"""
    from oracle.writer import convert_frame
    from vps_b200 import test_vpq as T
    from vps_b200.pipeline import InputStage
    from vps_b200.runner import ClipRunner
    from vps_b200.writer import PanWriter
    cfg, model = T.load_model(os.path.join(root, "cfg.py"), os.path.join(root, "w.pth"), "cuda:0", precision)
    pairs, metas = [], []
    for i, (im, fr) in enumerate(zip(images, frames)):
        ref = frames[i - 1] if i % NFR else fr
        pairs.append((torch.from_numpy(fr), torch.from_numpy(ref)))
        metas.append(dict(filename=os.path.join(root, "val/img_all", im["file_name"]), iid=im["id"], flip=False))
    runner = ClipRunner(model, "cuda:0", unify=True, input_stage=InputStage.from_pipeline(cfg.data.test.pipeline))
    runner.unifier.stuff_area_limit = 2048                           # test.yaml, as the reference's test_cityscapes_1gpu.yaml
    w = PanWriter(out)
    it = iter(names)
    for i, r in enumerate(runner.run(pairs, metas)):
        p = r[2]["pan_2ch"].numpy().copy()
        name = next(it) if i >= 4 and (i - 4) % 5 == 0 else None
        w.add_frame_ids(name, *convert_frame(p), p)
    return w.finish()


def _truth_from(out, names, root):
    """ground truth = the in-process output itself: GT PNG = its pan_pred PNG, GT segments = its pred.json"""
    truth = os.path.join(root, "truth")
    os.makedirs(truth, exist_ok=True)
    pred = json.load(open(os.path.join(out, "pred.json")))
    gt = {"images": [], "annotations": [], "categories": [{"id": i, "isthing": int(i >= 11)} for i in range(19)]}
    for n, ann in zip(names, pred["annotations"]):
        base = n[:-len("_leftImg8bit.png")]
        gt["images"].append({"id": base, "file_name": n})
        gt["annotations"].append({"image_id": base, "segments_info": ann["segments_info"]})
        shutil.copy(os.path.join(out, "pan_pred", base + ".png"), os.path.join(truth, base + "_gtFine_color.png"))
    path = os.path.join(root, "gt.json")
    json.dump(gt, open(path, "w"))
    return truth, path, pred


def test_test_vpq_driver_whole_chain_vs_oracle_writer(cuda, tmp_path):
    from vps_b200 import eval_vpq as E
    from vps_b200 import test_vpq as T
    root = str(tmp_path / "cityscapes_vps")         # the tracker reads img_meta filenames under a Cityscapes path
    images, frames, names = _write_split(root)
    report = {}
    for precision in ("tc32", "fp32", "bf16"):
        out = os.path.join(root, precision + ".pkl")
        T.main([os.path.join(root, "cfg.py"), os.path.join(root, "w.pth"), "--out", out, "--pan_im_json_file",
                os.path.join(root, "pan_im.json"), "--n_video", "2", "--mode", "val", "--precision", precision,
                "--test_config", os.path.join(root, "test.yaml")])
        got = out.replace(".pkl", "_pans_unified/")
        if precision == "bf16":                                     # scored against the tc32 chain, reported only
            res = E.evaluate_dirs(got, os.path.join(root, "truth_tc32"), os.path.join(root, "gt_tc32.json"))
            report["bf16"] = {k: 100 * r["All"]["pq"] for k, r in res.items()}
            continue
        ref_out = os.path.join(root, "inproc_" + precision)
        _in_process(root, images, frames, names, precision, ref_out)
        _same_tree(got, ref_out)
        truth, gt_json, pred = _truth_from(ref_out, names, root)
        n_things = sum(s["category_id"] >= 11 for a in pred["annotations"] for s in a["segments_info"])
        report[precision + "_segments"] = (sum(len(a["segments_info"]) for a in pred["annotations"]), n_things)
        res = E.evaluate_dirs(got, truth, gt_json)
        for k, r in res.items():
            assert r["All"]["pq"] == 1.0 and r["Stuff"]["pq"] == 1.0 and r["Things"]["pq"] == 1.0, (precision, k)
        assert open(os.path.join(got, "vpq-final.txt")).read() == "vpq_all:100.0000\nvpq_thing:100.0000\nvpq_stuff:100.0000\n"
        if precision == "tc32":
            shutil.move(truth, os.path.join(root, "truth_tc32"))
            shutil.move(gt_json, os.path.join(root, "gt_tc32.json"))
        else:
            shutil.rmtree(truth)
    print("whole chain:", report)
