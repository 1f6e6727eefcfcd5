"""Build any of the REFERENCE's three Cityscapes detectors (its own python code, via ref_import stubs) from its
unmodified config: configs/cityscapes/fusetrack.py (PanopticFuseTrack), track.py (PanopticTrack) or fuse.py
(PanopticFuse).  run_reference.py builds FuseTrack from its full state_dict; this builder takes a FuseTrack state_dict
(or any superset of the built model's keys) and loads, strictly, the entries of the model's own keys -- which is how the
synthetic weight set "C" goes into the two models that lack FuseTrack's flow, fuse neck or track head."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def build_reference_model(state_dict, config):
    """config: "fusetrack", "track" or "fuse"."""
    from tests.golden.ref_import import REF, setup
    M = setup()
    from vps_b200.config import Config
    cfg = Config.fromfile(os.path.join(REF, "configs/cityscapes/%s.py" % config))
    cfg.model["pretrained"] = None
    fsd = {k[len("flownet2."):]: v for k, v in state_dict.items() if k.startswith("flownet2.")}
    _load = torch.load
    torch.load = lambda *a, **k: {"state_dict": fsd}      # the flow models' ctor reads work_dirs/flownet/...pth.tar
    _cd = torch.cuda.current_device
    torch.cuda.current_device = lambda: 0                  # ... and prints the device with %d
    try:
        det = M.build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg)
    finally:
        torch.load = _load
        torch.cuda.current_device = _cd
    det.load_state_dict({k: state_dict[k] for k in det.state_dict()}, strict=True)
    det.eval()
    return det
