"""Generate tests/golden/track_clip_128x256.npz and fuse_clip_128x256.npz from the REFERENCE's own python code.

As tests/golden/make_golden.py does for FuseTrack: the reference is imported through tests/golden/ref_import.py, its
PanopticTrack / PanopticFuse is built from the unmodified configs/cityscapes/track.py / fuse.py and loaded with the
synthetic weight set "C" (oracle/weights.py, seed 0) restricted to that model's keys, and run on the seeded 128x256 clip:
  * Track: three frames (10001, 10002, 10003), so that the tracker both matches earlier tracks and opens new ones;
  * Fuse: the two frame pairs of the FuseTrack clip.
The fields follow fusetrack_clip_128x256.npz.  Track has no flow and no fuse neck: "fpn0" (every 32nd channel of the
first FPN level, the features its heads run on) takes the place of "flow_full" / "fused0".  Fuse's bbox results are
per-class arrays: "bbox" holds their rows in class order and "bbox_cls" the class of each row.  The script asserts that
every frame has real detections (not MaskROI's dummy) and that a later Track frame matches at least one earlier track.
Run where the reference tree is available:  python tests/golden/make_models_golden.py"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle.weights import make_model  # noqa: E402
from tests.e2e_util import make_pair, meta  # noqa: E402
from tests.golden.make_golden import weights_digest, weights_fingerprint  # noqa: E402
from tests.golden.run_reference_models import build_reference_model  # noqa: E402

H, W = 128, 256
HERE = os.path.dirname(os.path.abspath(__file__))


def clip(name):
    """[(iid, img, ref_img)] of the golden clip of model `name`"""
    img, ref = make_pair(H, W)
    if name == "fuse":
        return [(10001, img, ref), (10002, ref, img)]
    third = torch.roll(img, shifts=(3, 5), dims=(2, 3))
    return [(10001, img, ref), (10002, ref, img), (10003, third, ref)]


def run(name, sd_full):
    det = build_reference_model(sd_full, name)
    sd = det.state_dict()
    assert set(sd) == _oracle_keys(name)
    cap = {}
    if name == "fuse":
        det.flownet2.register_forward_hook(lambda m, i, o: cap.__setitem__("flow_full", o.detach().clone()))
        det.extra_neck.register_forward_hook(lambda m, i, o: cap.__setitem__("fused0", o[0].detach().clone()))
    else:
        det.neck.register_forward_hook(lambda m, i, o: cap.__setitem__("fpn0", o[0].detach().clone()))
    det.panopticFPN.register_forward_hook(lambda m, i, o: cap.__setitem__("fcn_score", o[1].detach().clone()))

    def _first_cls(m, i, o):
        if "cls_score" not in cap:          # first call of the frame = the 1000-proposal pass
            cap["cls_score"] = o[0].detach().clone()
    det.bbox_head.register_forward_hook(_first_cls)
    out = {"weights_sha256": np.array(weights_digest(sd)), "weights_fingerprint": weights_fingerprint(sd), "H": H, "W": W}
    matched = False
    frames = clip(name)
    out["nframes"] = len(frames)
    with torch.no_grad():
        for f, (iid, a, b) in enumerate(frames):
            cap.clear()
            r = det.simple_test(a, [meta(iid, H, W)], ref_img=[b])
            p = r[2]
            cls = p["panoptic_cls_inds"].numpy()
            assert cls.shape[0] >= 2 and (cls > 0).all(), "%s frame %d: no detections (the dummy)" % (name, f)
            out["f%d_pano" % f] = p["panoptic_outputs"].numpy().astype(np.uint8)
            out["f%d_sem" % f] = p["fcn_outputs"].numpy().astype(np.uint8)
            out["f%d_cls_inds" % f] = cls.astype(np.int32)
            out["f%d_cls_prob" % f] = p["panoptic_cls_prob"].numpy().astype(np.float32)
            out["f%d_fcn_score" % f] = cap["fcn_score"].numpy().astype(np.float32)
            out["f%d_cls_score" % f] = cap["cls_score"].numpy().astype(np.float32)
            if name == "fuse":
                assert "panoptic_det_obj_ids" not in p and isinstance(r[0], list) and len(r[0]) == 8
                out["f%d_bbox" % f] = np.concatenate(r[0], 0).astype(np.float32)
                out["f%d_bbox_cls" % f] = np.concatenate([np.full(len(b_), i, np.int32) for i, b_ in enumerate(r[0])])
                out["f%d_flow_full" % f] = cap["flow_full"].numpy().astype(np.float32)
                out["f%d_fused0" % f] = cap["fused0"][:, ::32].numpy().astype(np.float32)
            else:
                ids = p["panoptic_det_obj_ids"].numpy()
                out["f%d_obj_ids" % f] = ids.astype(np.int32)
                out["f%d_det_labels" % f] = p["panoptic_det_labels"].numpy().astype(np.int32)
                bids = sorted(r[0].keys())
                out["f%d_bbox_ids" % f] = np.array(bids, np.int32)
                out["f%d_bbox" % f] = np.stack([r[0][i]["bbox"] for i in bids]).astype(np.float32)
                out["f%d_fpn0" % f] = cap["fpn0"][:, ::32].numpy().astype(np.float32)
                if f > 0:
                    prev = max(int(out["f%d_bbox_ids" % g].max()) for g in range(f))
                    matched |= bool((np.array(bids) <= prev).any())
                    print("frame %d: %d tracks matched, %d opened" % (f, int((np.array(bids) <= prev).sum()),
                                                                       int((np.array(bids) > prev).sum())))
    if name == "track":
        assert matched, "no later frame matched an earlier track"
    path = os.path.join(HERE, "%s_clip_128x256.npz" % name)
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


def _oracle_keys(name):
    from oracle.variants import PanopticFuse, PanopticTrack
    return set((PanopticTrack if name == "track" else PanopticFuse)().state_dict())


def main():
    sd = make_model("C", 0).state_dict()
    for name in sys.argv[1:] or ("track", "fuse"):
        run(name, sd)


if __name__ == "__main__":
    main()
