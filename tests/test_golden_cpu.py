"""CPU: the oracle restatement reproduces the golden vectors generated from the REFERENCE's own python code
(tests/golden/make_golden.py) on the seeded 2-frame clip: integer outputs bit-exact, floats within TOL."""
import os

import numpy as np
import torch

from tests.e2e_util import make_pair

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fusetrack_clip_128x256.npz")
# Float bounds.  TIGHT: when the synthetic weights are bit-identical to those the golden clip was generated with (the same
# class of host CPU).  CROSS_HOST otherwise: the calibration and the forward pass run CPU convolutions whose last bits
# depend on the host's vector unit; measured between two x86 hosts: class probability 4.4e-6, box corners 3.7e-4 px,
# flow 1.8e-5 px, semantic logits 1.1e-5, class logits 6.0e-5, fused features 4.8e-6 -- the bounds keep ~3x margin.
# Integer outputs (label maps, ids, classes) are bit-exact in both cases.
TIGHT = dict(cls_prob=1e-6, bbox=1e-4, flow=1e-5, fcn_score=1e-5, cls_score=1e-5, fused=1e-5)
CROSS_HOST = dict(cls_prob=1.5e-5, bbox=1e-3, flow=5e-5, fcn_score=4e-5, cls_score=2e-4, fused=1e-5)


def test_oracle_reproduces_reference_golden_clip():
    from oracle.weights import make_model
    from tests.golden.make_golden import weights_digest, weights_fingerprint
    g = np.load(GOLD)
    H, W = int(g["H"]), int(g["W"])
    oracle = make_model("C", 0)
    assert np.allclose(weights_fingerprint(oracle.state_dict()), g["weights_fingerprint"], rtol=1e-5, atol=0), \
        "synthetic weights differ from the ones the golden file was generated with (torch RNG drift?)"
    TOL = TIGHT if weights_digest(oracle.state_dict()) == str(g["weights_sha256"]) else CROSS_HOST
    img, ref = make_pair(H, W)
    for f, (iid, a, b) in enumerate(((10001, img, ref), (10002, ref, img))):
        taps = {}
        r = oracle.simple_test(a, dict(iid=iid, img_shape=(H, W, 3)), b, taps)
        p = r[2]
        assert np.array_equal(p["panoptic_outputs"].numpy().astype(np.uint8), g["f%d_pano" % f])
        assert np.array_equal(p["fcn_outputs"].numpy().astype(np.uint8), g["f%d_sem" % f])
        assert np.array_equal(p["panoptic_cls_inds"].numpy(), g["f%d_cls_inds" % f])
        assert np.array_equal(p["panoptic_det_obj_ids"].numpy(), g["f%d_obj_ids" % f])
        assert np.array_equal(p["panoptic_det_labels"].numpy(), g["f%d_det_labels" % f])
        assert np.abs(p["panoptic_cls_prob"].numpy() - g["f%d_cls_prob" % f]).max() <= TOL["cls_prob"]
        ids = sorted(r[0].keys())
        assert ids == g["f%d_bbox_ids" % f].tolist()
        assert np.abs(np.stack([r[0][i]["bbox"] for i in ids]) - g["f%d_bbox" % f]).max() <= TOL["bbox"]
        assert np.abs(taps["flow_full"].numpy() - g["f%d_flow_full" % f]).max() <= TOL["flow"]
        assert np.abs(taps["fcn_score"].numpy() - g["f%d_fcn_score" % f]).max() <= TOL["fcn_score"]
        assert np.abs(taps["cls_score"].numpy() - g["f%d_cls_score" % f]).max() <= TOL["cls_score"]
        assert np.abs(taps["fused"][0][:, ::32].numpy() - g["f%d_fused0" % f]).max() <= TOL["fused"]
