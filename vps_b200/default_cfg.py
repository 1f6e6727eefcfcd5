"""Built-in equivalents of the model / test_cfg sections of the reference's three Cityscapes configs
(configs/cityscapes/fusetrack.py lines 2-148, track.py lines 2-135, fuse.py lines 2-142) for environments where the
reference tree is not mounted.  On a machine that has the reference, load its file instead:
`Config.fromfile('<ref>/configs/cityscapes/fusetrack.py')`."""


def fusetrack_cfg():
    ce = lambda **k: dict(type='CrossEntropyLoss', **k)
    model = dict(
        type='PanopticFuseTrack', pretrained=None,
        backbone=dict(type='ResNet', depth=50, num_stages=4, out_indices=(0, 1, 2, 3), frozen_stages=1, style='pytorch'),
        neck=dict(type='FPN', in_channels=[256, 512, 1024, 2048], out_channels=256, num_outs=5),
        extra_neck=dict(type='BFPTcea', in_channels=256, num_levels=5, refine_level=0, refine_type='conv', center=0, nframes=2),
        panoptic=dict(type='UPSNetFPN', in_channels=256, out_channels=128, num_levels=4, num_things_classes=8,
                      num_classes=19, ignore_label=255, loss_weight=1.0),
        rpn_head=dict(type='RPNHead', in_channels=256, feat_channels=256, anchor_scales=[8], anchor_ratios=[0.5, 1.0, 2.0],
                      anchor_strides=[4, 8, 16, 32, 64], target_means=[.0, .0, .0, .0], target_stds=[1.0, 1.0, 1.0, 1.0],
                      loss_cls=ce(use_sigmoid=True, loss_weight=1.0),
                      loss_bbox=dict(type='SmoothL1Loss', beta=1.0 / 9.0, loss_weight=1.0)),
        bbox_roi_extractor=dict(type='SingleRoIExtractor', roi_layer=dict(type='RoIAlign', out_size=7, sample_num=2),
                                out_channels=256, featmap_strides=[4, 8, 16, 32]),
        bbox_head=dict(type='SharedFCBBoxHead', num_fcs=2, in_channels=256, fc_out_channels=1024, roi_feat_size=7,
                       num_classes=9, target_means=[0., 0., 0., 0.], target_stds=[0.1, 0.1, 0.2, 0.2],
                       reg_class_agnostic=False, loss_cls=ce(use_sigmoid=False, loss_weight=1.0),
                       loss_bbox=dict(type='SmoothL1Loss', beta=1.0, loss_weight=1.0)),
        track_head=dict(type='TrackHead', num_fcs=2, in_channels=256, fc_out_channels=1024, roi_feat_size=7,
                        match_coeff=[1.0, 2.0, 10.0], loss_match=ce(use_sigmoid=False, loss_weight=0.5)),
        mask_roi_extractor=dict(type='SingleRoIExtractor', roi_layer=dict(type='RoIAlign', out_size=14, sample_num=2),
                                out_channels=256, featmap_strides=[4, 8, 16, 32]),
        mask_head=dict(type='FCNMaskHead', num_convs=4, in_channels=256, conv_out_channels=256, num_classes=9,
                       loss_mask=ce(use_mask=True, loss_weight=1.0)))
    cm = {i: 10 + i for i in range(1, 9)}
    test_cfg = dict(
        rpn=dict(nms_across_levels=False, nms_pre=1000, nms_post=1000, max_num=1000, nms_thr=0.7, min_bbox_size=0),
        rcnn=dict(score_thr=0.05, nms=dict(type='nms', iou_thr=0.5), max_per_img=100, mask_thr_binary=0.5),
        loss_pano_weight=None, flownet2=[], class_mapping=cm)
    return dict(model=model, train_cfg=None, test_cfg=test_cfg)


def track_cfg():
    """configs/cityscapes/track.py: FuseTrack's model without the BFPTcea fuse neck, and no `flownet2` in test_cfg (so no
    FlowNet2 either).  Its match_coeff spells the last weight as the integer 10."""
    c = fusetrack_cfg()
    c['model']['type'] = 'PanopticTrack'
    del c['model']['extra_neck']
    c['model']['track_head']['match_coeff'] = [1.0, 2.0, 10]
    del c['test_cfg']['flownet2']
    return c


def fuse_cfg():
    """configs/cityscapes/fuse.py: FuseTrack's model without the track head; the same test_cfg."""
    c = fusetrack_cfg()
    c['model']['type'] = 'PanopticFuse'
    del c['model']['track_head']
    return c
