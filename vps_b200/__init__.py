"""vps_b200: Hopper-native inference for the reference's three Cityscapes models -- PanopticFuseTrack, PanopticTrack and
PanopticFuse (drop-in modules for mcahny/vps's registries).

    from vps_b200 import Config, build_detector
    cfg = Config.fromfile('<reference>/configs/cityscapes/fusetrack.py')      # loads unmodified
    model = build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).cuda()
    model.load_state_dict(torch.load('latest.pth')['state_dict'])
    result = model(return_loss=False, rescale=True, img=[img], img_meta=[[meta]], ref_img=[ref_img])
"""
from .config import Config, ConfigDict  # noqa: F401
from .registry import (BACKBONES, DETECTORS, EXTRA_NECKS, HEADS, LOSSES, NECKS, PANOPTIC, ROI_EXTRACTORS,  # noqa: F401
                       SHARED_HEADS, Registry, build_detector, build_from_cfg)
from . import modules as _modules  # noqa: F401  (registers the classes)
from . import detector as _detector  # noqa: F401
from .detector import PanopticFuse, PanopticFuseTrack, PanopticTrack  # noqa: F401
from .default_cfg import fuse_cfg, fusetrack_cfg, track_cfg  # noqa: F401
