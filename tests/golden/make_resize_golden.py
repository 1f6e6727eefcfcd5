"""Golden vectors for the keep-ratio Resize of the test pipeline (mmdet/datasets/pipelines/transforms.py:107-121 ->
mmcv.imrescale -> cv2.resize(..., INTER_LINEAR) on the uint8 frame) and for the Image.NEAREST resize evaluate_ssegs applies
to a prediction of another shape (tools/dataset/cityscapes.py:125-126).  Runs OpenCV and Pillow themselves on seeded
`np.random.default_rng` frames:

* every frame shape of CASES is resized to its keep-ratio size under img_scale=(2048, 1024) by cv2.resize, then normalised
  with the Cityscapes cfg, zero-padded to a multiple of 32 and transposed (oracle/pipeline.py restates mmcv 0.2.14's
  imnormalize / impad_to_multiple); the SHA-256 of the resized uint8 frame and of the fp32 [1,3,Hp,Wp] tensor are kept
  (full-size outputs are megabytes each);
* SMALL frames under img_scale=(64, 32) are kept in full (frame, resized frame, tensor), so a failure shows a readable diff;
* NEAREST: uint8 label maps in mode P (as write_segmentation_result saves them) resized with Pillow to another shape, up
  and down; digests for the large pairs, the maps in full for the small ones.

Output: tests/golden/resize_cases.json, resize_small.npz.  Rerunning writes identical files.
Run:  python tests/golden/make_resize_golden.py"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

NORM = dict(mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], to_rgb=True)
IMG_SCALE = (2048, 1024)
CASES = [(1080, 1920), (720, 1280), (600, 800), (480, 640), (1200, 1600), (2160, 3840), (1536, 3072), (1023, 2047),
         (1024, 1024), (37, 91), (5, 7), (3000, 17), (1, 1), (2048, 4096)]
SMALL_SCALE = (64, 32)
SMALL = [(45, 70), (17, 9), (5, 7), (1, 1), (32, 64), (100, 37)]
NEAREST = [((1024, 1820), (1080, 1920)), ((1080, 1920), (1024, 1820)), ((512, 1024), (1024, 2048)), ((333, 777), (1000, 2001))]
NEAREST_SMALL = [((37, 53), (61, 97)), ((61, 97), (37, 53)), ((7, 3), (7, 5)), ((1, 1), (3, 5)), ((17, 30), (16, 31))]


def frame(seed, h, w):
    return np.random.default_rng(seed).integers(0, 256, size=(h, w, 3), dtype=np.uint8)


def label_map(seed, h, w):
    return np.random.default_rng(seed).integers(0, 19, size=(h, w), dtype=np.uint8)


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def cv2_prepare(img, img_scale):
    """the reference's test pipeline on one frame: mmcv.imrescale (restated size, cv2.resize itself), then Normalize / Pad /
    ImageToTensor"""
    import cv2

    from oracle import resize as OR
    (oh, ow), sf = OR.rescale_size(img.shape[0], img.shape[1], img_scale)
    resized = cv2.resize(img, (ow, oh), interpolation=cv2.INTER_LINEAR)
    return resized, OR.prepare_frame(resized, NORM["mean"], NORM["std"], NORM["to_rgb"], 32), sf


def pil_nearest(pred, gh, gw):
    from PIL import Image
    im = Image.fromarray(np.uint8(pred))
    im.putpalette(list(range(256)) * 3)                        # write_segmentation_result saves a palette (mode P) image
    return np.array(im.resize((gw, gh), Image.NEAREST))


def main():
    cases, small = [], {}
    for i, (h, w) in enumerate(CASES):
        seed = 1000 + i
        resized, x, sf = cv2_prepare(frame(seed, h, w), IMG_SCALE)
        cases.append({"seed": seed, "shape": [h, w], "resized_shape": list(resized.shape[:2]), "pad_shape": list(x.shape[2:]),
                      "scale_factor": sf, "sha256_resized": sha(resized), "sha256_prepared": sha(x)})
    for i, (h, w) in enumerate(SMALL):
        img = frame(2000 + i, h, w)
        resized, x, sf = cv2_prepare(img, SMALL_SCALE)
        small["img%d" % i], small["resized%d" % i], small["prepared%d" % i] = img, resized, x
        small["scale_factor%d" % i] = np.float64(sf)
    nearest = []
    for i, ((ph, pw), (gh, gw)) in enumerate(NEAREST):
        seed = 3000 + i
        nearest.append({"seed": seed, "pred_shape": [ph, pw], "gt_shape": [gh, gw],
                        "sha256": sha(pil_nearest(label_map(seed, ph, pw), gh, gw))})
    for i, ((ph, pw), (gh, gw)) in enumerate(NEAREST_SMALL):
        p = label_map(4000 + i, ph, pw)
        small["nn_pred%d" % i], small["nn_out%d" % i] = p, pil_nearest(p, gh, gw)
    import cv2
    import PIL
    with open(os.path.join(HERE, "resize_cases.json"), "w") as f:
        json.dump({"generator": {"opencv": cv2.__version__, "pillow": PIL.__version__}, "img_scale": list(IMG_SCALE),
                   "small_scale": list(SMALL_SCALE), "norm": NORM, "cases": cases, "small": [list(s) for s in SMALL],
                   "nearest": nearest, "nearest_small": [[list(a), list(b)] for a, b in NEAREST_SMALL]}, f, indent=1)
        f.write("\n")
    # np.savez (not _compressed): zip entries carry no time stamp, so rerunning writes the same bytes
    np.savez(os.path.join(HERE, "resize_small.npz"), **small)


if __name__ == "__main__":
    main()
