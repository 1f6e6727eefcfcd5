"""CPU: the drop-in boundary -- registries, config loader, state_dict layout, C-ABI exports, no-fallback rule."""
import ctypes
import json
import os
import re

import pytest
import torch

from tests.golden.ref_import import REF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_CFG = os.path.join(REF, "configs/cityscapes/fusetrack.py")       # REF: where the reference tree is (tests/golden/ref_import.py)
REF_RECORD = os.path.join(ROOT, "tests", "golden", "reference_boundary.json")


def test_registry_semantics_match_reference():
    from vps_b200.registry import Registry, build_from_cfg
    r = Registry("thing")

    @r.register_module
    class A(object):
        def __init__(self, x, y=2):
            self.x, self.y = x, y
    with pytest.raises(KeyError):          # duplicate name (mmdet/utils/registry.py:40-43)
        r.register_module(A)
    with pytest.raises(TypeError):
        r.register_module(3)
    obj = build_from_cfg(dict(type="A", x=1), r, default_args=dict(y=5, x=9))
    assert (obj.x, obj.y) == (1, 5)        # cfg wins over default_args (setdefault)
    with pytest.raises(KeyError):
        build_from_cfg(dict(type="Nope"), r)
    assert r.get("A") is A and r.get("B") is None and "A" in r.module_dict


def test_all_reference_names_are_registered():
    import vps_b200 as V
    assert V.DETECTORS.get("PanopticFuseTrack") is not None
    for reg, names in ((V.BACKBONES, ["ResNet"]), (V.NECKS, ["FPN"]), (V.EXTRA_NECKS, ["BFPTcea"]),
                       (V.PANOPTIC, ["UPSNetFPN"]), (V.ROI_EXTRACTORS, ["SingleRoIExtractor"]),
                       (V.HEADS, ["RPNHead", "SharedFCBBoxHead", "TrackHead", "FCNMaskHead"]),
                       (V.LOSSES, ["CrossEntropyLoss", "SmoothL1Loss"])):
        for n in names:
            assert reg.get(n) is not None, n


def _reference_record():
    """the reference's fusetrack.py as its loader reads it and the contents of its registries, recorded from the reference
    by tests/golden/make_boundary_golden.py"""
    from tests.golden.make_boundary_golden import from_json
    with open(REF_RECORD) as f:
        return from_json(json.load(f))


def test_reference_config_loads_unmodified_and_builds():
    from vps_b200 import Config, build_detector, fusetrack_cfg
    rec = _reference_record()
    if os.path.exists(REF_CFG):                  # where the reference tree is present, the record is still what it loads to
        live = Config.fromfile(REF_CFG)
        assert _plain(dict(live.model.items())) == rec["model"] and _plain(dict(live.test_cfg.items())) == rec["test_cfg"]
    cfg = Config(dict(model=rec["model"], test_cfg=rec["test_cfg"]))
    assert hasattr(cfg.test_cfg, "flownet2") and not hasattr(cfg.test_cfg, "nope")
    assert cfg.test_cfg.rpn.nms_thr == 0.7 and cfg.model.bbox_head.num_classes == 9
    det = build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg)
    mine = fusetrack_cfg()
    ref_model = {k: v for k, v in cfg.model.items()}
    ref_model["pretrained"] = None
    assert _plain(ref_model) == _plain(mine["model"])
    assert _plain(cfg.test_cfg) == _plain(mine["test_cfg"])
    assert det.class_mapping == {i: 10 + i for i in range(1, 9)}


def test_b200_classes_build_through_the_reference_registries():
    """SURVEY 8b, second route: overwrite the reference's registries' module_dict[name] entries with this project's classes
    and build the detector through those registries from the reference's config.  Everywhere: the reference's registries are
    stood in for by registries that hold a placeholder class under every name, and with the defining module, that the
    reference's own registries hold (recorded by tests/golden/make_boundary_golden.py); the detector is built by this
    project's `build` on the stand-in DETECTORS registry.  Where the reference tree is present, additionally the same
    through the reference's OWN registries and its own mmdet build_detector (in a subprocess: importing the reference on an
    mmcv-less machine needs process-wide stubs, tests/golden/ref_import.py)."""
    import types
    from vps_b200.config import Config
    from vps_b200.registry import Registry, build, install_into_reference
    rec = _reference_record()
    RR = types.SimpleNamespace()
    for attr, names in rec["registries"].items():
        reg = Registry(attr.lower())
        for name, module in names.items():
            reg.module_dict[name] = type(name, (object,), {"__module__": module})
        setattr(RR, attr, reg)
    ref_cls = RR.DETECTORS.get('PanopticFuseTrack')
    assert ref_cls is not None and ref_cls.__module__.startswith('mmdet.')
    done = install_into_reference(RR)
    assert ('DETECTORS', 'PanopticFuseTrack') in done and ('BACKBONES', 'ResNet') in done and len(done) >= 12
    for attr, name in done:
        assert getattr(RR, attr).get(name).__module__.startswith('vps_b200.'), (attr, name)
    cfg = Config(dict(model=rec["model"], test_cfg=rec["test_cfg"]))
    cfg.model['pretrained'] = None
    det = build(cfg.model, RR.DETECTORS, dict(train_cfg=None, test_cfg=cfg.test_cfg))
    assert type(det).__module__ == 'vps_b200.detector', type(det)
    for name in ('backbone', 'neck', 'extra_neck', 'panopticFPN', 'rpn_head', 'bbox_head', 'track_head', 'mask_head'):
        assert type(getattr(det, name)).__module__.startswith('vps_b200.'), name
    assert len(det.state_dict()) == 629
    if os.path.exists(REF_CFG):
        _build_through_the_live_reference()


def _build_through_the_live_reference():
    import subprocess
    import sys
    code = r"""
import os, sys
sys.path.insert(0, %r)
from tests.golden.ref_import import REF, setup
M = setup()                                  # the reference's mmdet.models (its registries now hold ITS classes)
import mmdet.models.registry as RR
import mmdet.models.builder as RB
ref_cls = RR.DETECTORS.get('PanopticFuseTrack')
assert ref_cls is not None and ref_cls.__module__.startswith('mmdet.')
import vps_b200
from vps_b200.registry import install_into_reference
done = install_into_reference(RR)
assert ('DETECTORS', 'PanopticFuseTrack') in done and ('BACKBONES', 'ResNet') in done and len(done) >= 12
from vps_b200.config import Config
cfg = Config.fromfile(os.path.join(REF, 'configs/cityscapes/fusetrack.py'))
cfg.model['pretrained'] = None
det = RB.build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg)      # the reference's builder
assert type(det).__module__ == 'vps_b200.detector', type(det)
for name in ('backbone', 'neck', 'extra_neck', 'panopticFPN', 'rpn_head', 'bbox_head', 'track_head', 'mask_head'):
    assert type(getattr(det, name)).__module__.startswith('vps_b200.'), name
assert len(det.state_dict()) == 629
print('OK', len(done))
""" % ROOT
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "OK" in out.stdout, out.stderr[-3000:]


def _plain(x):
    if isinstance(x, dict):
        return {k: _plain(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [_plain(v) for v in x]
    return x


def test_state_dict_layout_matches_oracle_and_reference_names():
    from oracle.model import PanopticFuseTrack as Oracle
    from vps_b200 import ConfigDict, build_detector, fusetrack_cfg
    c = fusetrack_cfg()
    det = build_detector(ConfigDict(c["model"]), train_cfg=None, test_cfg=ConfigDict(c["test_cfg"]))
    o = Oracle()
    a, b = det.state_dict(), o.state_dict()
    assert set(a) == set(b)
    assert all(a[k].shape == b[k].shape for k in a)
    det.load_state_dict(b, strict=True)
    for k in ("backbone.layer1.0.downsample.0.weight", "neck.lateral_convs.3.conv.bias",
              "extra_neck.liteflownet.flow_estimator.convs.2.0.weight", "extra_neck.tcea_fusion.sAtt_add_2.bias",
              "extra_neck.refine.conv.weight", "panopticFPN.deform_convs.0.3.conv_offset.weight",
              "panopticFPN.deform_convs.0.6.conv.weight", "panopticFPN.deform_convs.0.7.bias",
              "panopticFPN.conv_pred.conv.weight", "rpn_head.rpn_reg.bias", "bbox_head.shared_fcs.1.weight",
              "track_head.fcs.0.weight", "mask_head.convs.3.conv.weight", "mask_head.upsample.weight",
              "flownet2.flownetc.conv_redir.0.weight", "flownet2.flownets_2.upsampled_flow6_to_5.weight",
              "flownet2.flownets_d.inter_conv3.0.bias", "flownet2.flownetfusion.predict_flow0.weight"):
        assert k in a, k


def test_cabi_library_exports_every_declared_symbol():
    from vps_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "vps_b200.h")).read()
    declared = set(re.findall(r"^\s*(?:const char\*|int64_t|int|void)\s+(vps_[a-z0-9_]+)\s*\(", hdr, re.M))
    assert len(declared) >= 40
    assert declared == set(_lib.EXPORTS), (declared ^ set(_lib.EXPORTS))
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for s in declared:
        assert hasattr(lib, s), s
    assert lib.vps_version() >= 100


def test_no_cpu_fallback():
    """The product path must fail loudly without CUDA: no oracle / torch fallback."""
    from vps_b200 import ConfigDict, build_detector, fusetrack_cfg
    c = fusetrack_cfg()
    det = build_detector(ConfigDict(c["model"]), train_cfg=None, test_cfg=ConfigDict(c["test_cfg"]))
    img = torch.zeros(1, 3, 64, 64)
    with pytest.raises(Exception):
        det.simple_test(img, [dict(filename="city", iid=1, img_shape=(64, 64, 3))], ref_img=[img])
    src = "".join(open(os.path.join(ROOT, "vps_b200", f)).read() for f in os.listdir(os.path.join(ROOT, "vps_b200"))
                  if f.endswith(".py"))
    assert "import oracle" not in src and "from oracle" not in src


def test_synth_table_matches_oracle_calibration():
    """vps_b200.synth.make_weights (table-driven) reproduces oracle.weights.make_model (measured calibration)."""
    from oracle.weights import make_model
    from vps_b200 import ConfigDict, build_detector, fusetrack_cfg
    from vps_b200.synth import make_weights
    c = fusetrack_cfg()
    det = build_detector(ConfigDict(c["model"]), train_cfg=None, test_cfg=ConfigDict(c["test_cfg"]))
    make_weights(det, "C", 0)
    a, b = det.state_dict(), make_model("C", 0).state_dict()
    for k in a:
        tol = 2e-5 * max(1.0, float(b[k].abs().max()))
        assert float((a[k].float() - b[k].float()).abs().max()) <= tol, k
