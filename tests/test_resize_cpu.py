"""CPU: the restatements behind the keep-ratio Resize of the test pipeline and the NEAREST resize of predictions in the
semantic evaluation (oracle/resize.py) -- the cv2 INTER_LINEAR and mmcv.imrescale sizes against OpenCV itself and the golden
digests (tests/golden/make_resize_golden.py), the Pillow index tables against Pillow itself, the resizing
evaluate_ssegs against the reference's own run (tests/golden/make_ipq_resize_golden.py), and the host side of
InputStage(resize=True) (sizes, meta, from_pipeline)."""
import hashlib
import json
import os

import numpy as np
import pytest

from oracle import ipq as OI
from oracle import pipeline as OP
from oracle import resize as OR

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def cases():
    with open(os.path.join(GOLDEN, "resize_cases.json")) as f:
        return json.load(f)


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def frame(seed, h, w):
    return np.random.default_rng(seed).integers(0, 256, size=(h, w, 3), dtype=np.uint8)


def test_oracle_resize_equals_cv2_and_golden_digests():
    cv2 = pytest.importorskip("cv2")
    g = cases()
    norm = g["norm"]
    for c in g["cases"]:
        img = frame(c["seed"], *c["shape"])
        (oh, ow), sf = OR.rescale_size(*c["shape"], tuple(g["img_scale"]))
        assert [oh, ow] == c["resized_shape"] and sf == c["scale_factor"], c
        got = OR.resize_linear_u8(img, oh, ow)
        assert np.array_equal(got, cv2.resize(img, (ow, oh), interpolation=cv2.INTER_LINEAR)), c["shape"]
        assert sha(got) == c["sha256_resized"], c["shape"]
        x = OR.prepare_frame(img, norm["mean"], norm["std"], norm["to_rgb"], 32, img_scale=tuple(g["img_scale"]))
        assert list(x.shape[2:]) == c["pad_shape"] and sha(x) == c["sha256_prepared"], c["shape"]


def test_oracle_resize_small_cases_in_full():
    g = cases()
    d = np.load(os.path.join(GOLDEN, "resize_small.npz"))
    for i, _ in enumerate(g["small"]):
        img = d["img%d" % i]
        got, sf = OR.imrescale(img, tuple(g["small_scale"]))
        np.testing.assert_array_equal(got, d["resized%d" % i])
        assert sf == float(d["scale_factor%d" % i])
        np.testing.assert_array_equal(OR.prepare_frame(img, g["norm"]["mean"], g["norm"]["std"], True, 32,
                                                       img_scale=tuple(g["small_scale"])), d["prepared%d" % i])


def test_prepare_frame_default_keeps_the_frame():
    img = frame(7, 37, 91)
    want = OP.impad_to_multiple(OP.imnormalize(img, [1, 2, 3], [4, 5, 6]), 32).transpose(2, 0, 1)[None]
    np.testing.assert_array_equal(OR.prepare_frame(img, [1, 2, 3], [4, 5, 6]), want)
    np.testing.assert_array_equal(OR.prepare_frame(img, [1, 2, 3], [4, 5, 6]), OP.prepare_frame(img, [1, 2, 3], [4, 5, 6]))
    # a resize to the frame's own size is the identity
    np.testing.assert_array_equal(OR.resize_linear_u8(img, 37, 91), img)


def test_imrescale_sizes_and_factors():
    """mmcv 0.2.14: sf = min(long / max(h, w), short / min(h, w)); size (int(h * sf + 0.5), int(w * sf + 0.5))"""
    want = {(1080, 1920): ((1024, 1820), 1024 / 1080), (720, 1280): ((1024, 1820), 1024 / 720),
            (2160, 3840): ((1024, 1820), 1024 / 2160), (1024, 2048): ((1024, 2048), 1.0),
            (1023, 2047): ((1023, 2048), 2048 / 2047), (3000, 17): ((2048, 12), 2048 / 3000), (1, 1): ((1024, 1024), 1024.0)}
    for (h, w), (size, sf) in want.items():
        got = OR.rescale_size(h, w, (2048, 1024))
        assert got == (size, sf), (h, w, got)
        assert OR.rescale_size(h, w, (1024, 2048)) == got          # the order of img_scale does not matter


def test_pillow_tables_equal_image_resize_nearest():
    pytest.importorskip("PIL")
    from PIL import Image
    g = cases()
    d = np.load(os.path.join(GOLDEN, "resize_small.npz"))

    def pil(p, gh, gw):
        im = Image.fromarray(p)
        im.putpalette(list(range(256)) * 3)
        assert im.mode == "P"
        return np.array(im.resize((gw, gh), Image.NEAREST))
    for i, (_, (gh, gw)) in enumerate(g["nearest_small"]):
        p = d["nn_pred%d" % i]
        np.testing.assert_array_equal(OR.resize_nearest(p, gh, gw), d["nn_out%d" % i])
        np.testing.assert_array_equal(OR.resize_nearest(p, gh, gw), pil(p, gh, gw))
    for c in g["nearest"]:
        p = np.random.default_rng(c["seed"]).integers(0, 19, size=c["pred_shape"], dtype=np.uint8)
        got = OR.resize_nearest(p, *c["gt_shape"])
        assert sha(got) == c["sha256"] and np.array_equal(got, pil(p, *c["gt_shape"])), c
    rng = np.random.default_rng(11)
    for _ in range(20):                                              # random up / down scales per axis
        ph, pw, gh, gw = (int(v) for v in rng.integers(1, 300, size=4))
        p = rng.integers(0, 19, size=(ph, pw), dtype=np.uint8)
        np.testing.assert_array_equal(OR.resize_nearest(p, gh, gw), pil(p, gh, gw), err_msg=str((ph, pw, gh, gw)))


def test_product_tables_equal_oracle_tables():
    from vps_b200.ipq import nearest_table
    for s, d in ((1820, 1920), (1920, 1820), (1, 5), (7, 7), (97, 31), (3000, 2999)):
        np.testing.assert_array_equal(nearest_table(s, d), OR.nearest_table(s, d))
        assert nearest_table(s, d).min() >= 0 and nearest_table(s, d).max() < s


def test_resizing_evaluate_ssegs_equals_reference_golden():
    d = np.load(os.path.join(GOLDEN, "ipq_resize.npz"))
    total = np.zeros((19, 19))
    shapes = set()
    for i in range(int(d["nframes"])):
        gt, pred = d["trainid%d" % i], d["fcn%d" % i]
        shapes.add((pred.shape[0] < gt.shape[0], pred.shape[1] < gt.shape[1], pred.shape == gt.shape))
        conf = OR.seg_confusion_resized(gt, pred.astype(np.int64))
        np.testing.assert_array_equal(conf, d["seg_conf%d" % i])
        total += conf
    assert len(shapes) >= 3                                           # down, up and equal shapes are all in the golden
    r = OI.seg_result(total)
    assert np.array_equal(r["confusion_matrix"], d["seg_confusion"])
    assert np.array_equal(r["IU_array"], d["IU_array"]) and r["meanIU"] == d["meanIU"]


REF_TEST_PIPELINE = [
    dict(type="LoadRefImageFromFile"),
    dict(type="MultiScaleFlipAug", img_scale=[(2048, 1024)], flip=False,
         transforms=[dict(type="Resize", keep_ratio=True), dict(type="RandomFlip"),
                     dict(type="Normalize", mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], to_rgb=True),
                     dict(type="Pad", size_divisor=32), dict(type="ImageToTensor", keys=["img", "ref_img"]),
                     dict(type="Collect", keys=["img", "ref_img"])])]


def test_input_stage_from_pipeline_and_geometry():
    """the stage built from the reference config's test_pipeline, and its meta geometry (no device needed)"""
    import copy

    from vps_b200.pipeline import CITYSCAPES_NORM, InputStage
    st = InputStage.from_pipeline(REF_TEST_PIPELINE)
    assert st.resize and st.img_scale == (2048, 1024) and st.div == 32 and st.to_rgb
    assert list(st.mean) == list(InputStage().mean) and list(st.std) == list(InputStage().std)
    assert CITYSCAPES_NORM["to_rgb"]
    assert st.geometry(1080, 1920) == (1024, 1820, 1024, 1824, 1024 / 1080)
    assert st.geometry(1024, 2048) == (1024, 2048, 1024, 2048, 1.0)
    assert st.geometry(2160, 3840)[:4] == (1024, 1820, 1024, 1824)
    with pytest.raises(NotImplementedError):
        InputStage().geometry(1080, 1920)                                # resize=False keeps the identity-only rule
    for edit in (lambda p: p[1].update(flip=True), lambda p: p[1].update(img_scale=[(2048, 1024), (1024, 512)]),
                 lambda p: p[1]["transforms"][0].update(keep_ratio=False), lambda p: p[1]["transforms"].append(dict(type="Foo")),
                 lambda p: p[1]["transforms"][3].update(size=(1024, 2048), size_divisor=None)):
        bad = copy.deepcopy(REF_TEST_PIPELINE)
        edit(bad)
        with pytest.raises(NotImplementedError):
            InputStage.from_pipeline(bad)
    with pytest.raises(ValueError):
        InputStage.from_pipeline([dict(type="LoadImageFromFile")])

