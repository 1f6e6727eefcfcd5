"""CPU: the split-level pieces of vps_b200.eval_vpq / test_vpq / datasets / writer that need no device.
 * the vpq-*.txt texts from the statistics the reference's own eval_vpq.py computed on the golden split
   (tests/golden/make_split_eval_golden.py), byte for byte;
 * the GT / prediction file-name mapping and the clip split;
 * the test dataset's order, reference frame and img_meta fields (cityscapes_vps.py:137-148, loading.py:43-67);
 * the command lines, the --mode rewrite and the stuff area limit read from the UPSNet yaml;
 * the writer's host step (key table -> segments_info) against the numpy converter."""
import json
import os

import numpy as np
import pytest

GOLD = os.path.join(os.path.dirname(__file__), "golden", "split_eval")


def _stat(d):
    from collections import defaultdict

    from vps_b200.vpq import CatStat
    stat = defaultdict(CatStat)
    for c, (iou, tp, fp, fn) in d.items():
        s = stat[int(c)]
        s.iou, s.tp, s.fp, s.fn = iou, tp, fp, fn
    return stat


def test_vpq_texts_match_reference_golden():
    from vps_b200.vpq import pq_average, vpq_final_text, vpq_text
    gt = json.load(open(os.path.join(GOLD, "gt.json")))
    cats = {el["id"]: el for el in gt["categories"]}
    st = json.load(open(os.path.join(GOLD, "stats.json")))
    results = {}
    for k, d in zip(st["k"], st["stats"]):
        stat = _stat(d)
        res = {}
        for name, t in (("All", None), ("Things", True), ("Stuff", False)):
            res[name], pc = pq_average(stat, cats, isthing=t)
            if t is None:
                res["per_class"] = pc
        results[k] = res
        assert vpq_text(res) == open(os.path.join(GOLD, "expected", "vpq-%d.txt" % k)).read()
    assert vpq_final_text(results) == open(os.path.join(GOLD, "expected", "vpq-final.txt")).read()


def test_file_names_and_clip_split():
    from vps_b200.eval_vpq import gt_files, pred_files
    from vps_b200.vpq import split_clips
    gt = {"images": [{"id": "b_x", "file_name": "b_x_leftImg8bit.png"}, {"id": "a_y", "file_name": "a_y_newImg8bit.png"}]}
    assert gt_files(gt) == ["a_y_final_mask.png", "b_x_gtFine_color.png"]          # sorted after the mapping
    assert pred_files(gt) == [os.path.join("pan_pred", "b_x.png"), os.path.join("pan_pred", "a_y.png")]   # JSON order
    for n, ann in ((20, 20), (12, 12), (13, 13), (6, 6), (35, 36)):
        want = [list(map(int, c)) for c in np.array_split(np.arange(n), ann // 6)]
        assert split_clips(n, ann) == want
    assert [len(c) for c in split_clips(20, 20)] == [7, 7, 6]
    with pytest.raises(ValueError):
        split_clips(5, 5)                                            # 5 // 6 = 0 clips: np.array_split refuses, as in eval_vpq


def _im_all_info(tmp_path, nvid=2, nfr=4):
    images = []
    for v in range(nvid):
        for f in range(nfr):
            images.append({"id": (v + 1) * 10000 + f + 1, "file_name": "%04d_%04d_city_%d_newImg8bit.png" % (v, f, f),
                           "width": 64, "height": 32})
    images.append(dict(images[1], width=99))                        # a duplicate id: COCO keeps the first place, last entry
    p = tmp_path / "im_all_info_val_city_vps.json"
    p.write_text(json.dumps({"images": images, "categories": []}))
    return str(p), images


def test_dataset_order_reference_frame_and_meta(tmp_path):
    from vps_b200.datasets import CityscapesVPSTestSet
    from vps_b200.pipeline import InputStage
    ann, images = _im_all_info(tmp_path)
    ds = CityscapesVPSTestSet(ann_file=ann, img_prefix="data/val/img_all/", ref_prefix="data/val/ref/", nframes_span_test=4)
    assert len(ds) == 8
    assert [ds.img_info(i)["id"] for i in range(8)] == [im["id"] for im in images[:8]]
    assert ds.img_info(1)["width"] == 99
    for i in range(8):
        info = ds.img_info(i)
        prev = images[i - 1] if i % 4 else images[i]              # prepare_test_img: idx % nframes_span_test
        assert info["ref_filename"] == prev["file_name"] and info["ref_id"] == prev["id"] - 1
        assert info["filename"] == images[i]["file_name"]
        assert ds.paths(i) == ("data/val/img_all/" + images[i]["file_name"], "data/val/ref/" + prev["file_name"])
    stage = InputStage(resize=True, device="cpu")
    m = ds.img_meta(5, stage, (1080, 1920))
    assert m["filename"] == "data/val/img_all/" + images[5]["file_name"] and m["iid"] == 20002 and m["flip"] is False
    assert m["ori_shape"] == (1080, 1920, 3) and m["img_shape"] == (1024, 1820, 3) and m["pad_shape"] == (1024, 1824, 3)
    assert m["scale_factor"] == 1024 / 1080
    assert m["img_norm_cfg"]["to_rgb"] is True and m["img_norm_cfg"]["mean"].dtype == np.float32
    # data_root joins relative paths (custom.py:57-69)
    ds2 = CityscapesVPSTestSet(ann_file=os.path.basename(ann), img_prefix="a/", ref_prefix="/abs/", data_root=str(tmp_path))
    assert ds2.paths(0) == (os.path.join(str(tmp_path), "a/", images[0]["file_name"]), "/abs/" + images[0]["file_name"])


def test_mode_rewrite_and_arguments(tmp_path):
    from vps_b200 import test_vpq as T
    from vps_b200.datasets import rewrite_mode
    cfg = dict(type="CityscapesVPSDataset", ann_file="d/im_all_info_test_city_vps.json", img_prefix="d/test/img_all/",
               ref_prefix="d/test/img_all/", nframes_span_test=30, pipeline=[])
    v = rewrite_mode(cfg, "val")
    assert (v["ann_file"], v["img_prefix"], v["ref_prefix"]) == ("d/im_all_info_val_city_vps.json", "d/val/img_all/", "d/val/img_all/")
    assert rewrite_mode(v, "test") == cfg and cfg["img_prefix"] == "d/test/img_all/"
    with pytest.raises(KeyError):
        rewrite_mode(cfg, "train")
    a = T.parse_args(["c.py", "w.pth", "--out", "x/val.pkl", "--pan_im_json_file", "p.json", "--n_video", "50", "--mode", "test"])
    assert (a.config, a.checkpoint, a.out, a.pan_im_json_file, a.n_video, a.mode, a.precision) == \
        ("c.py", "w.pth", "x/val.pkl", "p.json", 50, "test", "tc32")
    assert a.out.replace(".pkl", "_pans_unified/") == "x/val_pans_unified/"
    with pytest.raises(ValueError):
        T.parse_args(["c.py", "w.pth", "--out", "x/val.json"])
    y = tmp_path / "t.yaml"
    y.write_text("test:\n  scales:\n  - 1024\n  panoptic_stuff_area_limit: 2048\n")
    assert T.stuff_area_limit(str(y)) == 2048
    y.write_text("test:\n  scales:\n  - 1024\n")
    assert T.stuff_area_limit(str(y)) == 4096                      # not set: the default of the UPSNet config
    with pytest.raises(FileNotFoundError):                          # update_config opens the file: no silent default
        T.stuff_area_limit(str(tmp_path / "none.yaml"))
    from vps_b200 import eval_vpq as E
    e = E.parse_args(["--submit_dir", "s/", "--truth_dir", "t/", "--pan_gt_json_file", "g.json"])
    assert (e.submit_dir, e.truth_dir, e.pan_gt_json_file) == ("s/", "t/", "g.json")


def _numpy_table(p2):
    """the key table vps_pan2ch_segments produces, restated with numpy"""
    from vps_b200.writer import NKEY
    p = p2.astype(np.int64)
    sem, trk = p[..., 0], p[..., 2]
    t = np.zeros((5, NKEY), np.uint32)
    t[1:3] = 0xFFFFFFFF
    ys, xs = np.indices(sem.shape)
    ok = sem < 19
    key = (sem * 256 + trk)[ok]
    np.add.at(t[0], key, 1)
    np.minimum.at(t[1], key, xs[ok].astype(np.uint32)); np.minimum.at(t[2], key, ys[ok].astype(np.uint32))
    np.maximum.at(t[3], key, xs[ok].astype(np.uint32)); np.maximum.at(t[4], key, ys[ok].astype(np.uint32))
    return t.reshape(5, 19, 256)


def test_segments_from_table_equals_host_writer():
    from oracle import vpq as V
    from tests.test_writer_cpu import _golden
    from vps_b200.writer import PanWriter, segments_from_table
    frames, _, _ = _golden()
    rng = np.random.default_rng(3)
    extra = np.zeros((20, 30, 3), np.uint8)
    extra[..., 0] = 5
    extra[..., 2] = rng.integers(0, 256, (20, 30))                 # one stuff class, many track values
    for fr in list(frames) + [extra]:
        w = PanWriter(None, sample=False)
        ann = w.add_frame_ids("f", *V.segments_from_pan2ch(fr), fr)
        assert segments_from_table(_numpy_table(fr)) == ann["segments_info"]


def test_driver_refuses_an_unsorted_split(tmp_path):
    """the reference samples the unified results sorted by file name; a dataset listed in another order is refused"""
    from vps_b200 import ConfigDict
    from vps_b200 import test_vpq as T
    from vps_b200.datasets import CityscapesVPSTestSet
    ann, images = _im_all_info(tmp_path)
    data = json.load(open(ann))
    data["images"] = data["images"][:8][::-1]
    open(ann, "w").write(json.dumps(data))
    ds = CityscapesVPSTestSet(ann_file=ann, img_prefix="i/", ref_prefix="i/", nframes_span_test=4)
    pipeline = [dict(type="LoadRefImageFromFile"), dict(type="Resize", img_scale=(2048, 1024), keep_ratio=True),
                dict(type="Normalize", mean=[0, 0, 0], std=[1, 1, 1], to_rgb=True), dict(type="Pad", size_divisor=32)]
    cfg = ConfigDict(data=ConfigDict(test=ConfigDict(pipeline=pipeline)))
    with pytest.raises(ValueError, match="file-name order"):
        T.run_split(cfg, None, ds, ["a"], str(tmp_path / "out"), device="cpu")


def test_writer_pool_errors(tmp_path):
    """a failed PNG write is raised by close(), but does not replace an exception already leaving a `with` block"""
    from vps_b200.writer import PanWriter
    blocker = tmp_path / "file"
    blocker.write_text("")                                          # output_dir is a file: every write fails
    img = np.zeros((4, 4, 3), np.uint8)
    w = PanWriter(str(blocker), sample=False, workers=1)
    w._submit("a_leftImg8bit.png", (("pan_pred", img),))
    with pytest.raises(OSError):
        w.close()
    with pytest.raises(KeyError, match="original"):
        with PanWriter(str(blocker), sample=False, workers=1) as w2:
            w2._submit("a_leftImg8bit.png", (("pan_pred", img),))
            raise KeyError("original")
    assert w2._pool is None and not w2._pending
