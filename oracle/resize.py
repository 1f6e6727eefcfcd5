"""ORACLE (test infrastructure, not product code): CPU restatements of the two resizes at the ends of the test path, for
frames that are not 1024x2048 already.

* Before the model: the keep-ratio `Resize` of the test pipeline (mmdet/datasets/pipelines/transforms.py:107-121), i.e.
  mmcv 0.2.14 `imrescale` (not vendored: its size and factor are restated from the published source) and the
  `cv2.resize(..., INTER_LINEAR)` it calls on the uint8 frame, restated from OpenCV's fixed-point path for uint8.  With
  Normalize / Pad / ImageToTensor of oracle/pipeline.py, `prepare_frame(..., img_scale)` is the whole pipeline of one frame.
* After the model: the `Image.NEAREST` resize `Cityscapes.evaluate_ssegs` applies to a prediction of another shape than
  the gt (tools/dataset/cityscapes.py:125-126, after write_segmentation_result saved it as np.uint8, :182-186), restated
  as Pillow's index tables, and the frame's confusion counts through it (oracle/ipq.py's seg_confusion).

Pinned against OpenCV and Pillow themselves and the reference's own evaluate_ssegs by tests/golden/make_resize_golden.py,
make_ipq_resize_golden.py and tests/test_resize_cpu.py."""
import numpy as np

from oracle.ipq import seg_confusion
from oracle.pipeline import impad_to_multiple, imnormalize


def rescale_size(h, w, img_scale):
    """mmcv.imrescale(img, scale=img_scale): the factor min(long / max(h, w), short / min(h, w)) as a Python float and the
    new size (int(h * sf + 0.5), int(w * sf + 0.5))"""
    long_e, short_e = max(img_scale), min(img_scale)
    sf = min(long_e / max(h, w), short_e / min(h, w))
    return (int(h * sf + 0.5), int(w * sf + 0.5)), sf


def _linear_taps(src, dst, clamp_frac):
    """cv2 INTER_LINEAR taps of one axis: (s0, s1, a0, a1) with a0 + a1 ~ 2048.  scale = 1 / (dst / src) in double,
    f = float((d + 0.5) * scale - 0.5) with no fused multiply-add, s = floor(f), f -= s in float.  x (clamp_frac): f is
    zeroed where s leaves [0, src - 1]; y: f is kept and both rows are clamped."""
    scale = 1.0 / (float(dst) / float(src))
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if clamp_frac:
        f = np.where((s < 0) | (s >= src - 1), np.float32(0), f).astype(np.float32)
        s = np.clip(s, 0, src - 1)
    s0, s1 = np.clip(s, 0, src - 1), np.clip(s + 1, 0, src - 1)
    a1 = np.rint(f * np.float32(2048)).astype(np.int64)                           # saturate_cast<short>: half to even
    a0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int64)
    return s0, s1, a0, a1


def resize_linear_u8(img, oh, ow):
    """cv2.resize(img, (ow, oh), interpolation=INTER_LINEAR) of a uint8 [H,W,C] image, bit for bit: horizontal pass
    R = S[s0] * a0 + S[s1] * a1 (int), vertical pass as OpenCV's SIMD VResizeLinearVec_32s8u does it,
    t = ((R0 >> 4) * b0 >> 16) + ((R1 >> 4) * b1 >> 16), out = clamp((t + 2) >> 2, 0, 255)."""
    h, w = img.shape[:2]
    xs0, xs1, a0, a1 = _linear_taps(w, ow, True)
    ys0, ys1, b0, b1 = _linear_taps(h, oh, False)
    src = img.astype(np.int64)
    rows = src[:, xs0] * a0[None, :, None] + src[:, xs1] * a1[None, :, None]      # [H, ow, C]
    r0, r1 = rows[ys0] >> 4, rows[ys1] >> 4
    t = ((r0 * b0[:, None, None]) >> 16) + ((r1 * b1[:, None, None]) >> 16)
    return np.clip((t + 2) >> 2, 0, 255).astype(np.uint8)


def imrescale(img, img_scale):
    """mmcv.imrescale(img, img_scale, return_scale=True) with the default bilinear interpolation"""
    h, w = img.shape[:2]
    (oh, ow), sf = rescale_size(h, w, img_scale)
    return resize_linear_u8(img, oh, ow), sf


def prepare_frame(img_u8_bgr, mean, std, to_rgb=True, divisor=32, img_scale=None):
    """the test pipeline for one frame -> fp32 [1,3,Hp,Wp]: Resize(img_scale, keep_ratio) -> Normalize -> Pad(divisor) ->
    ImageToTensor.  img_scale=None skips the Resize, which gives oracle.pipeline.prepare_frame's output."""
    if img_scale is not None:
        img_u8_bgr, _ = imrescale(img_u8_bgr, img_scale)
    x = impad_to_multiple(imnormalize(img_u8_bgr, mean, std, to_rgb), divisor)
    return np.ascontiguousarray(x.transpose(2, 0, 1))[None]


def nearest_table(src, dst):
    """Pillow's index table of one axis of Image.resize(size, NEAREST) (ImagingScaleAffine, the affine scaler of a pure
    scale): a = src / dst, xo = a / 2, then per output xin = int(xo) and xo += a -- a SEQUENTIAL double sum, reproduced by
    np.cumsum.  An index outside [0, src) would leave the output pixel at the fill value 0; it is marked -1 here.  (The
    running sum overshoots src - a / 2 by far less than a / 2 at any size below 2^25, so it does not happen in practice.)"""
    if src == dst:
        return np.arange(dst, dtype=np.int32)                     # Pillow copies the image when the size is unchanged
    a = float(src) / float(dst)
    xo = np.cumsum(np.concatenate([[a * 0.5], np.full(dst - 1, a)]))
    idx = np.where(xo < 0, -1, xo.astype(np.int64))
    return np.where((idx >= 0) & (idx < src), idx, -1).astype(np.int32)


def resize_nearest(pred, gh, gw):
    """Image.fromarray(np.uint8(pred)).resize((gw, gh), Image.NEAREST) of a [H,W] label map, as evaluate_ssegs reads back
    the prediction it wrote"""
    p = np.asarray(pred).astype(np.uint8)
    ytab, xtab = nearest_table(p.shape[0], gh), nearest_table(p.shape[1], gw)
    out = p[np.clip(ytab, 0, None)][:, np.clip(xtab, 0, None)]
    out[ytab < 0] = 0
    out[:, xtab < 0] = 0
    return out


def seg_confusion_resized(gt_trainids, pred, class_num=19):
    """one frame of evaluate_ssegs for a prediction of any shape: NEAREST-resized to the gt, then seg_confusion"""
    gt = np.asarray(gt_trainids)
    return seg_confusion(gt, resize_nearest(pred, gt.shape[0], gt.shape[1]), class_num)
