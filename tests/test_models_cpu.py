"""CPU: the reference's two other Cityscapes models, PanopticTrack (configs/cityscapes/track.py) and PanopticFuse (fuse.py).

  * the oracle (oracle/variants.py) reproduces the golden clips generated from the REFERENCE's own code
    (tests/golden/make_models_golden.py): integer outputs bit-exact, floats within the bounds of test_golden_cpu.py;
  * the oracle's image-level unified result equals the reference's function (tests/golden/unify_image.npz);
  * the drop-in boundary: both configs load unmodified and build through this project's registries into detectors whose
    state_dict keys are the reference model's, and after install_into_reference() the reference's own build_detector
    builds this project's class for each of the three configs."""
import json
import os

import numpy as np
import pytest

from tests.golden.ref_import import REF
from tests.test_golden_cpu import CROSS_HOST, TIGHT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
RECORD = os.path.join(GOLDEN, "reference_boundary_models.json")
DETECTORS = {"track": "PanopticTrack", "fuse": "PanopticFuse"}


def _record():
    from tests.golden.make_boundary_golden import from_json
    with open(RECORD) as f:
        return from_json(json.load(f))


def _oracle(name):
    from oracle.variants import PanopticFuse, PanopticTrack, from_fusetrack
    from oracle.weights import make_model
    return from_fusetrack(PanopticTrack if name == "track" else PanopticFuse, make_model("C", 0).state_dict())


@pytest.mark.parametrize("name", ["track", "fuse"])
def test_oracle_reproduces_reference_golden_clip(name):
    from tests.golden.make_golden import weights_digest, weights_fingerprint
    from tests.golden.make_models_golden import clip
    g = np.load(os.path.join(GOLDEN, "%s_clip_128x256.npz" % name))
    H, W = int(g["H"]), int(g["W"])
    oracle = _oracle(name)
    sd = oracle.state_dict()
    assert np.allclose(weights_fingerprint(sd), g["weights_fingerprint"], rtol=1e-5, atol=0)
    TOL = TIGHT if weights_digest(sd) == str(g["weights_sha256"]) else CROSS_HOST
    frames = clip(name)
    assert len(frames) == int(g["nframes"])
    for f, (iid, a, b) in enumerate(frames):
        taps = {}
        r = oracle.simple_test(a, dict(iid=iid, img_shape=(H, W, 3)), b, taps)
        p = r[2]
        assert np.array_equal(p["panoptic_outputs"].numpy().astype(np.uint8), g["f%d_pano" % f])
        assert np.array_equal(p["fcn_outputs"].numpy().astype(np.uint8), g["f%d_sem" % f])
        assert np.array_equal(p["panoptic_cls_inds"].numpy(), g["f%d_cls_inds" % f])
        assert np.abs(p["panoptic_cls_prob"].numpy() - g["f%d_cls_prob" % f]).max() <= TOL["cls_prob"]
        assert np.abs(taps["fcn_score"].numpy() - g["f%d_fcn_score" % f]).max() <= TOL["fcn_score"]
        assert np.abs(taps["cls_score"].numpy() - g["f%d_cls_score" % f]).max() <= TOL["cls_score"]
        if name == "track":
            assert np.array_equal(p["panoptic_det_obj_ids"].numpy(), g["f%d_obj_ids" % f])
            assert np.array_equal(p["panoptic_det_labels"].numpy(), g["f%d_det_labels" % f])
            ids = sorted(r[0].keys())
            assert ids == g["f%d_bbox_ids" % f].tolist()
            assert np.abs(np.stack([r[0][i]["bbox"] for i in ids]) - g["f%d_bbox" % f]).max() <= TOL["bbox"]
            assert np.abs(taps["fpn"][0][:, ::32].numpy() - g["f%d_fpn0" % f]).max() <= TOL["fused"]
            assert taps["flow"] is None and not hasattr(oracle, "extra_neck") and not hasattr(oracle, "flownet2")
        else:
            assert "panoptic_det_obj_ids" not in p and "panoptic_det_labels" not in p
            assert isinstance(r[0], list) and len(r[0]) == 8
            rows = np.concatenate(r[0], 0)
            cls = np.concatenate([np.full(len(x), i, np.int32) for i, x in enumerate(r[0])])
            assert np.array_equal(cls, g["f%d_bbox_cls" % f])
            assert np.abs(rows - g["f%d_bbox" % f]).max() <= TOL["bbox"]
            assert np.abs(taps["flow_full"].numpy() - g["f%d_flow_full" % f]).max() <= TOL["flow"]
            assert np.abs(taps["fused"][0][:, ::32].numpy() - g["f%d_fused0" % f]).max() <= TOL["fused"]
            assert not hasattr(oracle, "track_head")
    if name == "track":                  # a later frame both matched earlier tracks and opened new ones
        assert any(np.isin(g["f%d_bbox_ids" % f], np.arange(int(g["f%d_bbox_ids" % (f - 1)].max()) + 1)).any()
                   for f in range(1, len(frames)))


def test_oracle_image_unify_matches_reference():
    from oracle.variants import unify_image_frame
    g = np.load(os.path.join(GOLDEN, "unify_pan.npz"))
    h = np.load(os.path.join(GOLDEN, "unify_image.npz"))
    assert int(h["nframes"]) == int(g["nframes"])
    for i in range(int(g["nframes"])):
        got = unify_image_frame(g["seg%d" % i], g["pan%d" % i], g["cls%d" % i])
        assert np.array_equal(got, h["out%d" % i]), i
        assert not h["out%d" % i][:, :, 2].any()
        # channels 0 and 1 are those of the video function without track ids
        assert np.array_equal(h["out%d" % i][:, :, :2], g["out_noid%d" % i][:, :, :2])


def _plain(x):
    if isinstance(x, dict):
        return {k: _plain(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [_plain(v) for v in x]
    return x


@pytest.mark.parametrize("name", ["track", "fuse"])
def test_reference_config_loads_unmodified_and_builds(name):
    from vps_b200 import Config, ConfigDict, build_detector, fuse_cfg, track_cfg
    rec = _record()[name]
    path = os.path.join(REF, "configs/cityscapes/%s.py" % name)
    if os.path.exists(path):
        live = Config.fromfile(path)
        assert _plain(dict(live.model.items())) == rec["model"] and _plain(dict(live.test_cfg.items())) == rec["test_cfg"]
    cfg = Config(dict(model=rec["model"], test_cfg=rec["test_cfg"]))
    cfg.model["pretrained"] = None
    det = build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg)
    assert type(det).__name__ == DETECTORS[name] == rec["detector"]
    assert type(det).__module__ == "vps_b200.detector"
    assert sorted(det.state_dict()) == rec["state_dict_keys"]
    mine = (track_cfg if name == "track" else fuse_cfg)()
    assert _plain(cfg.model) == _plain(mine["model"]) and _plain(cfg.test_cfg) == _plain(mine["test_cfg"])
    built = build_detector(ConfigDict(mine["model"]), train_cfg=None, test_cfg=ConfigDict(mine["test_cfg"]))
    assert sorted(built.state_dict()) == rec["state_dict_keys"]
    # what each model switches off
    keys = rec["state_dict_keys"]
    if name == "track":
        assert not any(k.startswith(("extra_neck.", "flownet2.")) for k in keys) and det.with_track and not det.with_flow
    else:
        assert not any(k.startswith("track_head.") for k in keys) and det.with_flow and not det.with_track
    # the oracle restatement has the same layout
    from oracle.variants import PanopticFuse, PanopticTrack
    assert sorted((PanopticTrack if name == "track" else PanopticFuse)().state_dict()) == keys


def test_every_config_builds_through_the_reference_registries():
    """install_into_reference() covers all three configs: on stand-ins for the reference's registries (recorded by
    tests/golden/make_boundary_golden.py) everywhere, and through the reference's own registries and its own mmdet
    build_detector where the reference tree is present."""
    import types
    from tests.test_boundary import _reference_record
    from vps_b200.config import Config
    from vps_b200.registry import Registry, build, install_into_reference
    base = _reference_record()
    RR = types.SimpleNamespace()
    for attr, names in base["registries"].items():
        reg = Registry(attr.lower())
        for n, module in names.items():
            reg.module_dict[n] = type(n, (object,), {"__module__": module})
        setattr(RR, attr, reg)
    for n in ("PanopticFuseTrack", "PanopticTrack", "PanopticFuse"):
        assert RR.DETECTORS.get(n).__module__.startswith("mmdet."), n
    done = install_into_reference(RR)
    for n in ("PanopticFuseTrack", "PanopticTrack", "PanopticFuse"):
        assert ("DETECTORS", n) in done
    recs = dict(_record(), fusetrack=dict(model=base["model"], test_cfg=base["test_cfg"], detector="PanopticFuseTrack"))
    for name, rec in recs.items():
        cfg = Config(dict(model=rec["model"], test_cfg=rec["test_cfg"]))
        cfg.model["pretrained"] = None
        det = build(cfg.model, RR.DETECTORS, dict(train_cfg=None, test_cfg=cfg.test_cfg))
        assert type(det).__module__ == "vps_b200.detector" and type(det).__name__ == rec["detector"], name
    if os.path.exists(os.path.join(REF, "configs/cityscapes/track.py")):
        _build_through_the_live_reference()


def _build_through_the_live_reference():
    import subprocess
    import sys
    code = r"""
import os, sys
sys.path.insert(0, %r)
from tests.golden.ref_import import REF, setup
M = setup()
import mmdet.models.registry as RR
import mmdet.models.builder as RB
import vps_b200
from vps_b200.registry import install_into_reference
names = ('PanopticFuseTrack', 'PanopticTrack', 'PanopticFuse')
assert all(RR.DETECTORS.get(n).__module__.startswith('mmdet.') for n in names)
done = install_into_reference(RR)
from vps_b200.config import Config
for cfgname, n in zip(('fusetrack', 'track', 'fuse'), names):
    assert ('DETECTORS', n) in done
    cfg = Config.fromfile(os.path.join(REF, 'configs/cityscapes/%%s.py' %% cfgname))
    cfg.model['pretrained'] = None
    det = RB.build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg)      # the reference's builder
    assert type(det).__module__ == 'vps_b200.detector' and type(det).__name__ == n, type(det)
    for m in det.children():
        assert type(m).__module__.startswith('vps_b200.'), type(m)
print('OK')
""" % ROOT
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "OK" in out.stdout, out.stderr[-3000:]


def test_what_each_detector_builds():
    """PanopticTrack builds neither FlowNet2 nor the fuse neck; PanopticFuse builds both and no track head."""
    from vps_b200 import ConfigDict, build_detector, fuse_cfg, track_cfg
    for f, flow in ((track_cfg, False), (fuse_cfg, True)):
        c = f()
        det = build_detector(ConfigDict(c["model"]), train_cfg=None, test_cfg=ConfigDict(c["test_cfg"]))
        assert det.with_flow == flow and (det.flownet2 is not None) == flow and (det.extra_neck is not None) == flow
        assert det.with_track != flow and (det.track_head is not None) != flow
