"""The step right after the hot path (SURVEY 8f rank 1): `get_unified_pan_result` of the reference's test driver
(tools/dataset/cityscapes_vps.py:162-226) frame by frame on the GPU.

`PanUnifier` mirrors the reference method: call it once per frame, in clip order, with the label maps and the
`panoptic_cls_inds` / `panoptic_det_obj_ids` of `simple_test`; it returns the uint8 [H,W,3] (semantic, instance rank,
track id + 1) image the VPQ writer consumes.  The only host-side state is the reference's duplicate-track-id counter.

`PanUnifier(image=True)` is the image-level function the image panoptic model (PanopticFuse) is evaluated with
(tools/dataset/base_dataset.py:232-274): the same regions and decisions, no track ids, no counter, third channel 0."""
import ctypes as C

import numpy as np
import torch

from . import ops
from ._lib import lib


class PanUnifier:
    def __init__(self, num_seg_classes=19, num_classes=9, stuff_area_limit=4 * 64 * 64, image=False):
        # configs/cityscapes/test_cityscapes_1gpu.yaml:7-8; cityscapes_vps.py:162 (stuff_area_limit), :166 (max_oid)
        self.image = image
        self.id_last_stuff = num_seg_classes - num_classes
        self.stuff_area_limit = stuff_area_limit
        self.max_oid = 100
        self._ws = None

    def dedup_track_ids(self, obj_id):
        """cityscapes_vps.py:171-181: the last occurrence of a repeated id keeps it, earlier ones are re-numbered from a
        counter that runs across frames (the reference patches a reversed copy)."""
        obj_id = np.asarray(obj_id).copy()
        vals, cnt = np.unique(obj_id, return_counts=True)
        out = obj_id.copy()
        for v in vals[cnt > 1]:
            pos = np.nonzero(obj_id == v)[0]
            for p in pos[-2::-1]:
                out[p] = self.max_oid
                self.max_oid += 1
        return out

    def error_word(self):
        """device view (int32[1]) of the flag `check()` reads: copy it on a side stream to test it without synchronising"""
        off = int(lib().vps_unify_pan_error_offset())
        return self._ws[off:off + 4].view(torch.int32)

    def check(self):
        """Raise what the reference raises (IndexError, cityscapes_vps.py:197) if the last frame held a panoptic instance id
        without a `cls_ind` entry.  Synchronises the stream: call it where the results are consumed (ClipRunner does, after
        the download of the frame it yields)."""
        if self._ws is not None and int(lib().vps_unify_pan_error(ops._ptr(self._ws), ops.stream())) != 0:
            raise IndexError("get_unified_pan_result: panoptic instance id beyond len(cls_ind)")

    @torch.no_grad()
    def __call__(self, seg, pan, cls_ind, obj_id=None, out=None):
        """seg, pan: CUDA label maps [H,W] or [1,H,W] (uint8 or int64); cls_ind, obj_id: per-instance arrays (tensor /
        numpy / list); obj_id must be None for the image-level function.  Returns a uint8 CUDA tensor [H,W,3]."""
        if not (seg.is_cuda and pan.is_cuda):
            raise RuntimeError("PanUnifier: label maps must be CUDA tensors (there is no CPU path)")
        seg = seg.reshape(seg.shape[-2:]).contiguous()
        pan = pan.reshape(pan.shape[-2:]).contiguous()
        assert seg.dtype == pan.dtype and seg.dtype in (torch.uint8, torch.int64) and seg.shape == pan.shape
        H, W = pan.shape
        dev = pan.device
        cls_np = np.ascontiguousarray(np.asarray(cls_ind.cpu() if torch.is_tensor(cls_ind) else cls_ind).reshape(-1), dtype=np.int32)
        k = int(cls_np.shape[0])
        obj_np = None
        if self.image and obj_id is not None:
            raise ValueError("PanUnifier(image=True): the image-level result has no track ids")
        if obj_id is not None:
            obj_np = np.asarray(obj_id.cpu() if torch.is_tensor(obj_id) else obj_id).reshape(-1)
            obj_np = np.ascontiguousarray(self.dedup_track_ids(obj_np), dtype=np.int32)
            assert obj_np.shape[0] >= min(k, 1) or k == 0
        cls_p = cls_np.ctypes.data_as(C.c_void_p) if k else None
        obj_p = obj_np.ctypes.data_as(C.c_void_p) if (obj_np is not None and obj_np.shape[0]) else None
        if self._ws is None or self._ws.device != dev:
            self._ws = torch.empty(int(lib().vps_unify_pan_ws_bytes()), dtype=torch.uint8, device=dev)
        if out is None:
            out = torch.empty(H, W, 3, dtype=torch.uint8, device=dev)
        if self.image:
            ops.check(lib().vps_unify_pan_image(ops._ptr(seg), ops._ptr(pan), seg.element_size(), H, W, cls_p, k,
                                                self.id_last_stuff, self.stuff_area_limit, ops._ptr(out), ops._ptr(self._ws),
                                                C.c_int64(self._ws.numel()), ops.stream()), "unify_pan_image")
        else:
            ops.check(lib().vps_unify_pan(ops._ptr(seg), ops._ptr(pan), seg.element_size(), H, W, cls_p, obj_p, k,
                                          self.id_last_stuff, self.stuff_area_limit, ops._ptr(out), ops._ptr(self._ws),
                                          C.c_int64(self._ws.numel()), ops.stream()), "unify_pan")
        return out
