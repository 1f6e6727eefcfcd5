"""ORACLE (test infrastructure): CPU restatements of the reference's two other Cityscapes detectors and of the image-level
unified result, built from the FuseTrack oracle's modules (oracle/model.py) and its unify restatement (oracle/unify.py).

  * PanopticTrack  (mmdet/models/detectors/panoptic_track.py:443-536, configs/cityscapes/track.py): the current frame
    only -- ResNet-50-FPN, no FlowNet2, no BFPTcea -- with the tracker.
  * PanopticFuse   (panoptic_fuse.py:399-473, configs/cityscapes/fuse.py): flow and fuse neck, no tracker; per-class
    bbox results (bbox2result) and pano_results without track ids / labels.
  * unify_image_frame: get_unified_pan_result of tools/dataset/base_dataset.py:232-274 -- the video function of
    cityscapes_vps.py without track ids (no duplicate-id counter) and with the third channel 0.

`from_fusetrack(cls, sd)` builds either detector and loads the FuseTrack state_dict restricted to its own keys, which is
how the golden clips (tests/golden/make_models_golden.py) load the synthetic weight set "C" into the reference models.
Pinned by tests/golden/{track,fuse}_clip_128x256.npz and unify_image.npz (tests/test_models_cpu.py)."""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import unify as U
from .flownet2 import FlowNet2
from .model import (TEST_CFG_RPN, BFPTcea, FCNMaskHead, FPN, PanopticFuseTrack, ResNet50, RPNHead, SharedFCBBoxHead,
                    TrackHead, UPSNetFPN, mask_removal, mask_roi, roi_extract, seg_term)


class _Variant(PanopticFuseTrack):
    with_flow = with_track = True

    def __init__(self):
        nn.Module.__init__(self)
        self.backbone = ResNet50()
        self.neck = FPN()
        if self.with_flow:
            self.extra_neck = BFPTcea()
        self.panopticFPN = UPSNetFPN()
        self.rpn_head = RPNHead()
        self.bbox_head = SharedFCBBoxHead()
        if self.with_track:
            self.track_head = TrackHead()
        self.mask_head = FCNMaskHead()
        if self.with_flow:
            self.flownet2 = FlowNet2()
        self.prev_bboxes = self.prev_roi_feats = self.prev_det_labels = None
        self.eval()

    @torch.no_grad()
    def simple_test(self, img, img_meta, ref_img=None, taps=None):
        """img (and ref_img for Fuse) [1,3,H,W] fp32 normalised; img_meta dict with iid, img_shape."""
        im_info = np.array([[float(img.shape[2]), float(img.shape[3]), 1.0]])
        flow = ref_x = None
        x = self.extract_feat(img)
        xf = x
        if self.with_flow:
            flow = self.compute_flow(img.clone(), ref_img.clone(), 0.25, taps)
            ref_x = self.extract_feat(ref_img)
            xf = self.extra_neck(x, ref_x, flow, taps)
        fcn_output, fcn_score = self.panopticFPN(xf[0:4])
        cls_scores, bbox_preds = self.rpn_head(xf)
        proposals = self.rpn_head.get_bboxes(cls_scores, bbox_preds, img_meta["img_shape"], TEST_CFG_RPN, taps)
        rois = torch.cat([proposals.new_zeros(proposals.size(0), 1), proposals[:, :4]], dim=-1)   # bbox2roi
        roi_feats = roi_extract(xf[:4], rois, 7)
        cls_score, bbox_pred = self.bbox_head(roi_feats)
        cls_prob, det_rois, cls_idx = mask_roi(rois, bbox_pred, F.softmax(cls_score, dim=1), im_info)
        det_labels = cls_idx - 1
        det_bboxes = det_rois[:, 1:]
        det_obj_ids = None
        if self.with_track:
            det_roi_feats = roi_extract(xf[:4], det_rois, 7)
            is_first = (img_meta["iid"] % 10000) == 1
            det_obj_ids = np.asarray(self.track(det_bboxes, det_labels, det_roi_feats, cls_prob, is_first, taps))
        mask_feats = roi_extract(xf[:4], det_rois, 14)
        mask_score = self.mask_head(mask_feats)
        _, _, mh, mw = mask_score.shape
        mask_score = mask_score.gather(1, cls_idx.view(-1, 1, 1, 1).expand(-1, -1, mh, mw))
        keep_inds, mask_logits = mask_removal(det_rois[:, 1:], cls_prob, mask_score, cls_idx, tuple(fcn_output.shape[2:]))
        cls_idx_k = cls_idx[keep_inds]
        stuff, inst = seg_term(cls_idx_k, fcn_output, det_rois[keep_inds] * 4.0)
        panoptic_logits = torch.cat([stuff, inst + mask_logits], dim=1)
        panoptic_output = torch.max(F.softmax(panoptic_logits, dim=1), dim=1)[1]
        sem_output = torch.max(F.softmax(fcn_output, dim=1), dim=1)[1]
        h0, w0 = img_meta["img_shape"][:2]
        pano_results = {
            "fcn_outputs": sem_output[:, 0:h0, 0:w0],
            "panoptic_cls_inds": cls_idx_k,
            "panoptic_cls_prob": cls_prob[keep_inds],
            "panoptic_outputs": panoptic_output[:, 0:h0, 0:w0],
        }
        if taps is not None:
            taps.update(flow=flow, fpn=x, ref_fpn=ref_x, fused=xf, fcn_score=fcn_score, fcn_output=fcn_output,
                        rpn_cls=cls_scores, rpn_reg=bbox_preds, proposals=proposals, roi_feats=roi_feats,
                        cls_score=cls_score, bbox_pred=bbox_pred, det_rois=det_rois, cls_idx=cls_idx, cls_prob=cls_prob,
                        mask_score=mask_score, keep_inds=keep_inds, panoptic_logits=panoptic_logits)
        if self.with_track:
            ids_t = torch.from_numpy(det_obj_ids)
            pano_results["panoptic_det_labels"] = det_labels[keep_inds]
            pano_results["panoptic_det_obj_ids"] = ids_t[keep_inds]
            bbox_results = {}
            for bbox, label, obj_id in zip(det_bboxes.numpy(), det_labels.numpy(), det_obj_ids):
                if obj_id >= 0:
                    bbox_results[int(obj_id)] = {"bbox": bbox, "label": label}
            if taps is not None:
                taps["det_obj_ids_all"] = ids_t
        else:
            # bbox2result (mmdet/core/bbox/transforms.py:138-156); the dummy detection has label -1 and lands nowhere
            b, lab = det_bboxes.numpy(), det_labels.numpy()
            bbox_results = [b[lab == i, :] for i in range(8)]
        return bbox_results, [[] for _ in range(8)], pano_results


class PanopticTrack(_Variant):
    with_flow = False


class PanopticFuse(_Variant):
    with_track = False


def from_fusetrack(cls, state_dict):
    """cls built and loaded (strict) with the entries of a FuseTrack state_dict that it has."""
    m = cls()
    keys = set(m.state_dict())
    m.load_state_dict({k: v for k, v in state_dict.items() if k in keys}, strict=True)
    return m


def unify_image_frame(seg, pan, cls_ind, stuff_area_limit=4 * 64 * 64):
    """base_dataset.py:232-274 for one frame: the video function's channels 0 and 1, channel 2 zero."""
    out = U.unify_frame(seg, pan, cls_ind, None, stuff_area_limit)
    out[:, :, 2] = 0
    return out
