"""CPU: the parts of vps_b200.test_eval_ipq / datasets / writer that need no device.
 * the test dataset of the image panoptic model: order, reference frame (mmdet/datasets/cityscapes.py:82-97), img_meta;
 * the eval helper's paths from the yaml, the roidb sort, the file naming of ssegs / pan_2ch / pan, the command line;
 * the pairing of predictions with the panoptic GT json, refused when the reference would mispair;
 * the image converter's segments from a key table, against oracle.ipq.convert_image;
 * the golden split (tests/golden/make_ipq_split_golden.py) driven through the host parts with numpy ids: the reference's
   pq.txt byte for byte, its printed evaluate_ssegs block, pred.json up to the ids, and its palette PNGs."""
import json
import os

import numpy as np
import pytest

HERE = os.path.join(os.path.dirname(__file__), "golden")
GOLD = os.path.join(HERE, "ipq_split")


def _ann(tmp_path, names, ids=None, fname="inst.json"):
    ids = list(range(1, len(names) + 1)) if ids is None else ids
    images = [{"id": i, "file_name": n, "width": 64, "height": 32} for i, n in zip(ids, names)]
    p = tmp_path / fname
    p.write_text(json.dumps({"images": images, "categories": []}))
    return str(p), images


def test_dataset_order_reference_frame_and_meta(tmp_path):
    from vps_b200.datasets import CityscapesTestSet
    from vps_b200.pipeline import InputStage
    names = ["frankfurt_000000_000001_leftImg8bit.png", "frankfurt_000000_000000_leftImg8bit.png",
             "lindau/lindau_000000_000019_leftImg8bit.png", "x_000010_000010_leftImg8bit.png",
             "a_000001_000001_newImg8bit.png"]
    ann, images = _ann(tmp_path, names, ids=[7, 3, 9, 1, 5])
    data = json.loads(open(ann).read())
    data["images"].append(dict(images[0], width=99))                   # a duplicate id: first place, last entry
    open(ann, "w").write(json.dumps(data))
    ds = CityscapesTestSet(ann_file=ann, img_prefix="d/val/", ref_prefix="d/val_nbr/", seg_prefix="d/labels/")
    assert len(ds) == 5 and [ds.img_info(i)["id"] for i in range(5)] == [7, 3, 9, 1, 5]
    assert ds.img_info(0)["width"] == 99
    refs = ["frankfurt_000000_000000_leftImg8bit.png",
            "frankfurt_000000_000000_leftImg8bit.png",                 # fid 0 references itself
            "lindau/lindau_000000_000018_leftImg8bit.png",
            "x_000010_000009_leftImg8bit.png",                         # only '%06d' % fid + suffix is replaced
            "a_000001_000000_newImg8bit.png"]
    for i in range(5):
        assert ds.img_info(i)["ref_filename"] == refs[i], i
        assert ds.paths(i) == ("d/val/" + names[i], "d/val_nbr/" + refs[i])
    stage = InputStage(resize=True, device="cpu")
    m = ds.img_meta(2, stage, (1024, 2048))
    assert m["filename"] == "d/val/" + names[2] and m["iid"] == 9 and m["flip"] is False
    assert m["ori_shape"] == (1024, 2048, 3) and m["img_shape"] == (1024, 2048, 3) and m["pad_shape"] == (1024, 2048, 3)
    assert m["img_norm_cfg"]["to_rgb"] is True
    ds2 = CityscapesTestSet(ann_file=os.path.basename(ann), img_prefix="v/", ref_prefix="/abs/", data_root=str(tmp_path))
    assert ds2.paths(1) == (os.path.join(str(tmp_path), "v/", names[1]), "/abs/" + names[1])
    with pytest.raises(ValueError):
        CityscapesTestSet(ann_file=ann, img_prefix="v/", ref_prefix=None)


def _yaml(tmp_path, text):
    y = tmp_path / "t.yaml"
    y.write_text(text)
    return str(y)


def test_eval_helper_paths_roidb_and_arguments(tmp_path):
    from vps_b200 import test_eval_ipq as T
    y = _yaml(tmp_path, "dataset:\n  dataset_path: %s\n  test_image_set: val\ntest:\n  panoptic_stuff_area_limit: 2048\n"
              % str(tmp_path))
    assert T.eval_helper_config(y) == (str(tmp_path), "val")
    assert T.eval_helper_config(_yaml(tmp_path, "dataset:\n  dataset_path: ./data/cityscapes/\n")) == ("./data/cityscapes/", "val")
    with pytest.raises(ValueError, match="dataset_path"):
        T.eval_helper_config(_yaml(tmp_path, "dataset:\n  test_image_set: val\n"))
    with pytest.raises(FileNotFoundError):
        T.eval_helper_config(str(tmp_path / "none.yaml"))
    os.makedirs(tmp_path / "annotations")
    _ann(tmp_path / "annotations", ["c_1_leftImg8bit.png", "a_2_leftImg8bit.png", "b_3_leftImg8bit.png"], ids=[30, 10, 20],
         fname="instancesonly_gtFine_val.json")
    (tmp_path / "annotations" / "cityscapes_fine_val.json").write_text(json.dumps({"images": [], "annotations": [], "categories": []}))
    h = T.EvalHelper(str(tmp_path))
    assert [e["id"] for e in h.roidb] == [10, 20, 30]                  # sorted by image id (json_dataset.py:64-79)
    assert h.roidb[0]["image"] == os.path.join(str(tmp_path), "images", "a_2_leftImg8bit.png")
    assert T.label_path("/d/images/x/images_leftImg8bit.png") == "/d/labels/x/labels_gtFine_labelTrainIds.png"   # literal
    assert h.panoptic_json_file == os.path.join(str(tmp_path), "annotations", "cityscapes_fine_val.json")
    assert h.panoptic_gt_folder == "data/cityscapes/panoptic"
    a = T.parse_args(["c.py", "w.pth", "--out", "x/val.pkl", "--test_config", y])
    assert (a.config, a.checkpoint, a.out, a.dataset, a.gpus, a.precision, a.workers) == \
        ("c.py", "w.pth", "x/val.pkl", "Cityscapes", "0", "tc32", 4)
    with pytest.raises(ValueError):
        T.parse_args(["c.py", "w.pth", "--out", "x/val.json"])
    with pytest.raises(SystemExit):
        T.parse_args(["c.py", "w.pth", "--out", "x/val.pkl", "--dataset", "Viper"])
    with pytest.raises(FileNotFoundError):                             # main reads the yaml before anything else
        T.main(["c.py", "w.pth", "--out", str(tmp_path / "val.pkl"), "--test_config", str(tmp_path / "none.yaml")])


def test_file_naming():
    from vps_b200.writer import pan_image_name, sseg_path
    assert sseg_path("o/val_ssegs", "frankfurt_000000_000294_leftImg8bit.png") == "o/val_ssegs/frankfurt_000000_000294.png"
    assert sseg_path("o/s", "x_newImg8bit.png") == "o/s/x.png"
    assert sseg_path("o/s", "x_leftImg8bit.jpg") == "o/s/x_leftImg8bit.jpg"
    assert pan_image_name("frankfurt_000000_000294_leftImg8bit.png") == "frankfurt_000000_000294.png"
    assert pan_image_name("a_leftImg8bit.jpeg") == "a.png" and pan_image_name("b.jpg") == "b.png"


def _helper(tmp_path, gt_names, roidb_names):
    from vps_b200 import test_eval_ipq as T
    os.makedirs(tmp_path / "annotations", exist_ok=True)
    _ann(tmp_path / "annotations", roidb_names, fname="instancesonly_gtFine_val.json")
    (tmp_path / "annotations" / "cityscapes_fine_val.json").write_text(json.dumps(
        {"images": [{"id": i, "file_name": n} for i, n in enumerate(gt_names)], "annotations": [], "categories": []}))
    return T.EvalHelper(str(tmp_path))


def test_pairing_checks(tmp_path):
    names = ["a_000001_leftImg8bit.png", "b_000002_leftImg8bit.png", "c_000003_leftImg8bit.png"]
    h = _helper(tmp_path, names, [names[2], names[0]])
    h.pair(names)
    assert h.labels == [[os.path.join(str(tmp_path), "labels", "a_000001_gtFine_labelTrainIds.png")], [],
                        [os.path.join(str(tmp_path), "labels", "c_000003_gtFine_labelTrainIds.png")]]
    with pytest.raises(ValueError, match="file-name order"):
        h.pair([names[1], names[0], names[2]])
    with pytest.raises(ValueError, match="file-name order"):
        h.pair([names[0], names[0], names[2]])
    with pytest.raises(ValueError, match="predictions"):
        h.pair(names[:2])
    with pytest.raises(ValueError, match="does not pair"):
        h.pair([names[0], "b_000009_leftImg8bit.png", names[2]])
    h = _helper(tmp_path, [names[1], names[0], names[2]], names)      # the GT json in another order
    with pytest.raises(ValueError, match="does not pair"):
        h.pair(names)
    h = _helper(tmp_path, names, names + ["d_000004_leftImg8bit.png"])
    with pytest.raises(FileNotFoundError, match="d_000004"):          # a roidb image without a prediction
        h.pair(names)


def numpy_image_table(p2):
    """the key table vps_pan2ch_image_segments produces, restated with numpy"""
    p = p2.astype(np.int64)
    sem, ins = p[..., 0], p[..., 1]
    t = np.zeros((5, 19 * 256), np.uint32)
    t[1:3] = 0xFFFFFFFF
    ys, xs = np.indices(sem.shape)
    ok = sem < 19
    key = (sem * 256 + ins)[ok]
    np.add.at(t[0], key, 1)
    np.minimum.at(t[1], key, xs[ok].astype(np.uint32)); np.minimum.at(t[2], key, ys[ok].astype(np.uint32))
    np.maximum.at(t[3], key, xs[ok].astype(np.uint32)); np.maximum.at(t[4], key, ys[ok].astype(np.uint32))
    return t.reshape(5, 19, 256)


def random_image_frame(rng, H, W, block=16):
    hb, wb = (H + block - 1) // block, (W + block - 1) // block
    sem = rng.choice(np.r_[np.arange(19), 255], size=(hb, wb)).repeat(block, 0).repeat(block, 1)[:H, :W]
    ins = rng.integers(0, 256, size=(hb, wb)).repeat(block, 0).repeat(block, 1)[:H, :W]
    out = np.zeros((H, W, 3), np.uint8)
    out[..., 0], out[..., 1], out[..., 2] = sem, ins, rng.integers(0, 256, (H, W))
    return out


def ipq_golden_frames():
    d = np.load(os.path.join(HERE, "ipq_frames.npz"))
    return [d["pan2ch%d" % i] for i in range(int(d["nframes"]))]


def test_image_segments_from_table_equal_oracle_converter():
    from oracle.ipq import convert_image
    from vps_b200.writer import image_segments_from_table
    rng = np.random.default_rng(8)
    frames = ipq_golden_frames() + [random_image_frame(rng, 40, 70, block=5)]
    stuff = np.zeros((20, 30, 3), np.uint8)                           # one stuff class under several instance values
    stuff[..., 0] = 4
    stuff[..., 1] = rng.integers(0, 4, (20, 30))
    stuff[:5, :, 0] = 255
    frames.append(stuff)
    for fr in frames:
        assert image_segments_from_table(numpy_image_table(fr)) == convert_image(fr)[0]
    assert image_segments_from_table(numpy_image_table(np.full((3, 4, 3), 255, np.uint8))) == []


def same_pred_json(got, want):
    """equal segments_info, with the reference's colour ids mapped one to one onto ours, image by image"""
    assert len(got["annotations"]) == len(want["annotations"])
    for a, b in zip(got["annotations"], want["annotations"]):
        sa, sb = a["segments_info"], b["segments_info"]
        assert len(sa) == len(sb)
        fwd, back = {}, {}
        for x, y in zip(sa, sb):
            assert {k: v for k, v in x.items() if k != "id"} == {k: v for k, v in y.items() if k != "id"}
            assert fwd.setdefault(x["id"], y["id"]) == y["id"] and back.setdefault(y["id"], x["id"]) == x["id"]


def golden_outputs():
    d = np.load(os.path.join(GOLD, "model_outputs.npz"))
    names = [str(n) for n in d["names"]]
    return names, [(d["fcn%d" % i], d["pano%d" % i], d["cls%d" % i]) for i in range(len(names))]


def check_ssegs(folder):
    from PIL import Image
    want = np.load(os.path.join(GOLD, "expected", "ssegs.npz"))
    files = sorted(k[4:] for k in want.files if k.startswith("png:"))
    assert sorted(os.listdir(folder)) == files and files
    for f in files:
        im = Image.open(os.path.join(folder, f))
        assert im.mode == "P"
        assert np.array_equal(np.asarray(im), want["png:" + f])
        assert np.array_equal(np.asarray(im.getpalette(), np.uint8), want["palette:" + f])


def test_golden_split_host_path(tmp_path):
    """the driver's host parts fed with numpy ids (oracle unify and converter, numpy pair tables and confusion counts)"""
    from PIL import Image

    from oracle.ipq import convert_image, seg_confusion, seg_result
    from oracle.variants import unify_image_frame
    from tests.golden.make_ipq_split_golden import STUFF_AREA_LIMIT
    from vps_b200 import test_eval_ipq as T
    from vps_b200.ipq import IpqEvaluator
    from vps_b200.writer import ImageWriter
    names, outs = golden_outputs()
    helper = T.EvalHelper(GOLD, pan_gt_folder=os.path.join(GOLD, "panoptic"))
    helper.pair(names)
    out = str(tmp_path / "val.pkl")
    pans = out.replace(".pkl", "_pans_unified")
    w = ImageWriter(pans, out.replace(".pkl", "_ssegs"), workers=2, max_pending=1)
    ipq = IpqEvaluator(helper.categories)
    conf = np.zeros((19, 19))
    for i, (name, (fcn, pano, cls)) in enumerate(zip(names, outs)):
        labels, gt_rgb = helper.load_gt(i)
        w.add_sseg(name, fcn)
        for lab in labels:
            pred = fcn[0] if lab.shape == fcn[0].shape else \
                np.asarray(Image.fromarray(fcn[0]).resize((lab.shape[1], lab.shape[0]), Image.NEAREST))
            conf += seg_confusion(lab, pred)
        p2 = unify_image_frame(fcn[0], pano[0], cls, stuff_area_limit=STUFF_AREA_LIMIT)
        info, ids = convert_image(p2)
        ann = w.add_frame_ids(helper.pan_gt_json["images"][i]["file_name"], info, ids, p2)
        g = gt_rgb.astype(np.uint64)
        gt_ids = g[..., 0] + 256 * g[..., 1] + 65536 * g[..., 2]
        pairs, counts = np.unique(gt_ids * np.uint64(1 << 24) + ids.astype(np.uint64), return_counts=True)
        ipq.add_frame_table(helper.pan_gt_json["annotations"][i]["segments_info"], ann["segments_info"], pairs, counts)
    assert sum(len(x) for x in helper.labels) == 5 and any(lab.shape != o[0][0].shape
                                                          for x, o in zip(helper.labels, outs) for lab in
                                                          [np.asarray(Image.open(p)) for p in x])
    pred = w.finish(helper.pan_gt_json)
    ipq.write_pq_txt(os.path.join(pans, "pq.txt"), ipq.compute())
    exp = os.path.join(GOLD, "expected")
    assert open(os.path.join(pans, "pq.txt")).read() == open(os.path.join(exp, "pq.txt")).read()
    res = seg_result(conf)
    assert T.sseg_text(res) == open(os.path.join(exp, "sseg.txt")).read()
    assert np.array_equal(res["IU_array"], np.load(os.path.join(exp, "ssegs.npz"))["IU_array"])
    check_ssegs(out.replace(".pkl", "_ssegs"))
    same_pred_json(pred, json.load(open(os.path.join(exp, "pred.json"))))
    assert json.load(open(os.path.join(pans, "pred.json"))) == pred
    assert json.load(open(os.path.join(pans, "gt.json"))) == helper.pan_gt_json
    want = [n.replace("_leftImg8bit", "") for n in names]
    assert sorted(os.listdir(os.path.join(pans, "pan_2ch"))) == want and sorted(os.listdir(os.path.join(pans, "pan"))) == want


def test_image_writer_pool_errors(tmp_path):
    """the image writer shares PanWriter's pool: a failed write is raised by finish(), not over an exception in flight"""
    from vps_b200.writer import ImageWriter
    blocker = tmp_path / "file"
    blocker.write_text("")
    w = ImageWriter(str(blocker), str(blocker), workers=1)
    w.add_sseg("a_leftImg8bit.png", np.zeros((4, 4), np.uint8))
    with pytest.raises(OSError):
        w.finish()
    with pytest.raises(KeyError, match="original"):
        with ImageWriter(str(blocker), str(blocker), workers=1) as w2:
            w2.add_sseg("a_leftImg8bit.png", np.zeros((4, 4), np.uint8))
            raise KeyError("original")
    assert w2._pool is None and not w2._pending
