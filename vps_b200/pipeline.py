"""GPU input stage (SURVEY 8f rank 4): what the reference's test pipeline does on the host for `img` and `ref_img` between
LoadImageFromFile / LoadRefImageFromFile and the model (configs/cityscapes/fusetrack.py:172-190, mmdet/datasets/pipelines/
{loading,transforms,formating}.py):  Resize(img_scale=(2048,1024), keep_ratio) -> Normalize(mean, std, to_rgb) -> Pad(32) ->
ImageToTensor, plus the `img_meta` fields `simple_test` reads.

`InputStage` takes the decoded uint8 HWC BGR frame (what cv2.imread / mmcv.imread return), uploads it as uint8 (12.6 MB per
1024x2048 pair instead of 50 MB of fp32) and normalises / pads / transposes it on the device in one pass (`vps_preprocess_u8`,
bit-identical to mmcv.imnormalize's float32 arithmetic).  Resize: the rescale factor mmcv.imrescale derives is
min(long_edge / max(h, w), short_edge / min(h, w)); for Cityscapes frames (1024x2048) it is exactly 1 and cv2.resize is the
identity.  By default only that case is accepted (other sizes raise); with `resize=True` any frame is resized on the device
in the same pass (`vps_preprocess_resize_u8`, bit-identical to cv2.resize INTER_LINEAR on the uint8 frame) and the meta
carries the reference's ori_shape / img_shape / pad_shape / scale_factor."""
import ctypes as C

import numpy as np
import torch

from . import ops
from ._lib import lib

CITYSCAPES_NORM = dict(mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], to_rgb=True)    # fusetrack.py:153-154

# the meta fields the stage owns when it resizes: they replace a caller's (ClipRunner)
GEOMETRY_KEYS = ("ori_shape", "img_shape", "pad_shape", "scale_factor")

# transforms of a test pipeline that need nothing from the stage: decoding is the caller's, RandomFlip without flip is the
# identity, and the tensor / collect steps are what the stage's output already is
_PASS_THROUGH = ("LoadImageFromFile", "LoadRefImageFromFile", "RandomFlip", "ImageToTensor", "DefaultFormatBundle", "Collect")


class InputStage:
    def __init__(self, mean=CITYSCAPES_NORM["mean"], std=CITYSCAPES_NORM["std"], to_rgb=True, img_scale=(2048, 1024), size_divisor=32,
                 device="cuda:0", resize=False):
        self.mean = (C.c_float * 3)(*[float(np.float32(v)) for v in mean])
        self.std = (C.c_float * 3)(*[float(np.float32(v)) for v in std])
        self.to_rgb, self.img_scale, self.div = bool(to_rgb), img_scale, int(size_divisor)
        self.resize = bool(resize)
        self.dev = torch.device(device)

    @classmethod
    def from_pipeline(cls, test_pipeline, device="cuda:0"):
        """The stage of a reference config's `test_pipeline` list (fusetrack.py:172-187): img_scale from MultiScaleFlipAug
        (or from Resize), the Normalize cfg, Pad's size_divisor; it always resizes (resize=True).  What the stage does not
        implement is rejected: flip TTA, several scales, keep_ratio=False, Pad to a fixed size, other transforms."""
        steps, img_scale = [], None
        for t in test_pipeline:
            if t["type"] == "MultiScaleFlipAug":
                if t.get("flip", False):
                    raise NotImplementedError("InputStage.from_pipeline: flip test-time augmentation is not implemented")
                img_scale = t["img_scale"]
                steps.extend(t["transforms"])
            else:
                steps.append(t)
        norm = pad = None
        for t in steps:
            kind = t["type"]
            if kind == "Resize":
                if not t.get("keep_ratio", True):
                    raise NotImplementedError("InputStage.from_pipeline: Resize(keep_ratio=False) is not implemented")
                if t.get("ratio_range") is not None:
                    raise NotImplementedError("InputStage.from_pipeline: Resize(ratio_range=...) is not implemented")
                if t.get("img_scale") is not None:
                    img_scale = t["img_scale"]
            elif kind == "Normalize":
                norm = t
            elif kind == "Pad":
                if t.get("size") is not None or t.get("size_divisor") is None:
                    raise NotImplementedError("InputStage.from_pipeline: only Pad(size_divisor=...) is implemented")
                pad = t
            elif kind == "RandomFlip" and t.get("flip_ratio"):
                raise NotImplementedError("InputStage.from_pipeline: RandomFlip with a flip_ratio is not implemented")
            elif kind not in _PASS_THROUGH:
                raise NotImplementedError("InputStage.from_pipeline: transform %r is not implemented" % kind)
        if isinstance(img_scale, list):
            if len(img_scale) != 1:
                raise NotImplementedError("InputStage.from_pipeline: %d scales (multi-scale test-time augmentation) are not "
                                          "implemented" % len(img_scale))
            img_scale = img_scale[0]
        if norm is None or pad is None or img_scale is None or not any(t["type"] == "Resize" for t in steps):
            raise ValueError("InputStage.from_pipeline: the pipeline needs Resize (with an img_scale), Normalize and Pad")
        return cls(mean=norm["mean"], std=norm["std"], to_rgb=norm.get("to_rgb", True), img_scale=tuple(img_scale),
                   size_divisor=pad["size_divisor"], device=device, resize=True)

    def scale_factor(self, h, w):
        """mmcv.imrescale(img, scale=(long, short)): min(long / max(h, w), short / min(h, w))"""
        long_e, short_e = max(self.img_scale), min(self.img_scale)
        return min(long_e / max(h, w), short_e / min(h, w))

    def geometry(self, h, w):
        """(oh, ow, hp, wp, scale_factor) of an h x w frame: the size mmcv.imrescale gives it ((int(h * sf + 0.5),
        int(w * sf + 0.5)) with resize, the frame's own without) and that size padded to the size divisor"""
        sf = self.scale_factor(h, w)
        if self.resize:
            oh, ow = int(h * sf + 0.5), int(w * sf + 0.5)
        elif abs(sf - 1.0) > 1e-12:
            raise NotImplementedError("InputStage: Resize with scale %.4f (frame %dx%d): only the identity case of the Cityscapes "
                                      "pipeline is implemented on the device (InputStage(resize=True) resizes)" % (sf, h, w))
        else:
            oh, ow, sf = h, w, 1.0
        hp, wp = (oh + self.div - 1) // self.div * self.div, (ow + self.div - 1) // self.div * self.div
        return oh, ow, hp, wp, sf

    def __call__(self, img_u8, out=None, stream_tensor=None):
        """img_u8: uint8 [H,W,3] BGR, host (pinned or not) or CUDA tensor.  Returns (fp32 CUDA [1,3,Hp,Wp], meta fields)."""
        assert img_u8.dtype == torch.uint8 and img_u8.dim() == 3 and img_u8.shape[2] == 3
        h, w = int(img_u8.shape[0]), int(img_u8.shape[1])
        oh, ow, hp, wp, sf = self.geometry(h, w)
        d = img_u8 if img_u8.is_cuda else img_u8.to(self.dev, non_blocking=True)
        d = d.contiguous()
        if out is None:
            out = torch.empty(1, 3, hp, wp, dtype=torch.float32, device=d.device)
        elif self.resize and tuple(out.shape) != (1, 3, hp, wp):
            raise ValueError("InputStage: out %s is not [1, 3, %d, %d]" % (tuple(out.shape), hp, wp))
        if (oh, ow) == (h, w):
            ops.check(lib().vps_preprocess_u8(ops._ptr(d), h, w, self.mean, self.std, int(self.to_rgb), ops._ptr(out), hp, wp,
                                              ops.stream()), "preprocess_u8")
        else:
            ops.check(lib().vps_preprocess_resize_u8(ops._ptr(d), h, w, oh, ow, self.mean, self.std, int(self.to_rgb),
                                                     ops._ptr(out), hp, wp, ops.stream()), "preprocess_resize_u8")
        d.record_stream(torch.cuda.current_stream(d.device))
        meta = dict(img_shape=(oh, ow, 3), ori_shape=(h, w, 3), pad_shape=(hp, wp, 3), scale_factor=sf,
                    img_norm_cfg=dict(mean=np.array(list(self.mean), np.float32), std=np.array(list(self.std), np.float32), to_rgb=self.to_rgb))
        return out, meta

    def pair(self, img_u8, ref_u8=None, outs=(None, None)):
        """both frames of a pair (ref_u8 None for a detector that reads the current frame only) -> (img, ref_img, meta).
        The reference resizes img and ref_img with one Resize and keeps one set of meta fields, so with resize both frames
        must share a shape (ValueError otherwise)."""
        if self.resize and ref_u8 is not None and tuple(ref_u8.shape) != tuple(img_u8.shape):
            raise ValueError("InputStage: img %s and ref_img %s differ in shape" % (tuple(img_u8.shape), tuple(ref_u8.shape)))
        x, meta = self(img_u8, out=outs[0])
        r = None if ref_u8 is None else self(ref_u8, out=outs[1])[0]
        return x, r, meta
