"""GPU: PanopticTrack (configs/cityscapes/track.py) and PanopticFuse (fuse.py) on the device, against the oracle
(oracle/variants.py) and the goldens generated from the reference's own code (tests/golden/make_models_golden.py).

  * parity on the golden clip in tc32 and fp32: label maps, class ids and (Track) track ids bit-exact against the oracle
    and the reference golden; bf16 reports its label agreement;
  * one 1024x2048 pair per model in tc32 under the near-tie rule of test_gpu_fullsize.py;
  * CUDA-graph replay equals eager; ClipRunner with prefetch equals direct simple_test calls (Track from (img, None)
    pairs, Fuse also streaming); ClipRunner(unify=True) on Fuse equals the image-level unify oracle;
  * Track's whole VPQ chain (model -> PanUnifier -> segments -> VpqEvaluator) against the oracle chain."""
import os

import numpy as np
import pytest
import torch

from tests.e2e_util import make_pair, meta, near_tie_report

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TIE_TOL = 2e-4


def build(name, precision="tc32"):
    """(oracle, product) of model `name` ("track" / "fuse") with the synthetic weight set "C" restricted to its keys"""
    from oracle.variants import PanopticFuse, PanopticTrack, from_fusetrack
    from oracle.weights import make_model
    from vps_b200 import ConfigDict, build_detector, fuse_cfg, track_cfg
    oracle = from_fusetrack(PanopticTrack if name == "track" else PanopticFuse, make_model("C", 0).state_dict())
    cfg = (track_cfg if name == "track" else fuse_cfg)()
    prod = build_detector(ConfigDict(cfg["model"]), train_cfg=None, test_cfg=ConfigDict(cfg["test_cfg"]))
    prod.load_state_dict(oracle.state_dict(), strict=True)
    prod.precision = precision
    return oracle, prod.to("cuda:0")


@pytest.fixture(scope="module")
def models(cuda):
    return {n: build(n) for n in ("track", "fuse")}


def _run(prod, a, b, iid, H, W, **kw):
    return prod.simple_test(a.cuda(), [meta(iid, H, W)], ref_img=[b.cuda()] if b is not None else None, **kw)


def _labels(r):
    p = r[2]
    out = [p["panoptic_outputs"].cpu().long(), p["fcn_outputs"].cpu().long(), p["panoptic_cls_inds"].cpu().long()]
    if "panoptic_det_obj_ids" in p:
        out.append(p["panoptic_det_obj_ids"].cpu().long())
    return out


@pytest.mark.parametrize("name", ["track", "fuse"])
@pytest.mark.parametrize("precision", ["tc32", "fp32"])
def test_golden_clip_bit_exact(models, name, precision):
    from tests.golden.make_models_golden import clip
    oracle, prod = models[name]
    prod.precision = precision
    prod.reset_tracker()
    oracle.prev_bboxes = None
    g = np.load(os.path.join(GOLDEN, "%s_clip_128x256.npz" % name))
    H, W = int(g["H"]), int(g["W"])
    for f, (iid, a, b) in enumerate(clip(name)):
        o = oracle.simple_test(a, dict(iid=iid, img_shape=(H, W, 3)), b)
        r = _run(prod, a, b if name == "fuse" else None, iid, H, W)
        p, op = r[2], o[2]
        pano, sem = p["panoptic_outputs"].cpu(), p["fcn_outputs"].cpu()
        assert torch.equal(pano, op["panoptic_outputs"]) and torch.equal(sem, op["fcn_outputs"]), (name, f)
        assert np.array_equal(pano.numpy().astype(np.uint8), g["f%d_pano" % f])
        assert np.array_equal(sem.numpy().astype(np.uint8), g["f%d_sem" % f])
        assert p["panoptic_cls_inds"].cpu().tolist() == op["panoptic_cls_inds"].tolist() == g["f%d_cls_inds" % f].tolist()
        if name == "track":
            ids = p["panoptic_det_obj_ids"].cpu().tolist()
            assert ids == op["panoptic_det_obj_ids"].tolist() == g["f%d_obj_ids" % f].tolist(), f
            assert sorted(r[0]) == g["f%d_bbox_ids" % f].tolist()
        else:
            assert "panoptic_det_obj_ids" not in p and "panoptic_det_labels" not in p
            assert [len(x) for x in r[0]] == [len(x) for x in o[0]]
            assert np.array_equal(np.concatenate([np.full(len(x), i) for i, x in enumerate(r[0])]), g["f%d_bbox_cls" % f])
            assert np.abs(np.concatenate(r[0], 0) - g["f%d_bbox" % f]).max() <= 1e-3


@pytest.mark.parametrize("name", ["track", "fuse"])
def test_bf16_clip_close_to_oracle(models, name):
    oracle, prod = models[name]
    prod.precision = "bf16"
    prod.reset_tracker()
    oracle.prev_bboxes = None
    H, W = 128, 256
    img, ref = make_pair(H, W)
    o = oracle.simple_test(img, dict(iid=10001, img_shape=(H, W, 3)), ref)
    r = _run(prod, img, ref if name == "fuse" else None, 10001, H, W)
    prod.precision = "tc32"
    sem = float((r[2]["fcn_outputs"].cpu() == o[2]["fcn_outputs"]).float().mean())
    pan = float((r[2]["panoptic_outputs"].cpu() == o[2]["panoptic_outputs"]).float().mean())
    print("%s bf16 agreement with the oracle: semantic %.4f panoptic %.4f" % (name, sem, pan))
    assert sem >= 0.95, sem


@pytest.mark.parametrize("name", ["track", "fuse"])
def test_full_size_pair_matches_oracle(models, name):
    oracle, prod = models[name]
    prod.precision = "tc32"
    prod.reset_tracker()
    oracle.prev_bboxes = None
    H, W = 1024, 2048
    img, ref = make_pair(H, W, seed=63)
    ot = {}
    o = oracle.simple_test(img, dict(iid=10001, img_shape=(H, W, 3)), ref, ot)
    pt = {}
    r = _run(prod, img, ref if name == "fuse" else None, 10001, H, W, taps=pt)
    torch.cuda.synchronize()
    fcn_abs = float((pt["fcn_score"].float().permute(0, 3, 1, 2).cpu() - ot["fcn_score"]).abs().max())
    assert fcn_abs <= 1e-3, fcn_abs
    # detections as a SET (test_gpu_fullsize.py): boundary ties of noise-like scores may swap the lowest-ranked ones
    pd_, od_ = pt["det_rois"].cpu(), ot["det_rois"]
    dd = torch.cdist(pd_[:, 1:].double(), od_[:, 1:].double(), p=float("inf"))
    ddmin, jj = dd.min(dim=1)
    dm = ddmin <= 5e-3
    dfrac = float(dm.float().mean())
    assert dfrac >= 0.99 and bool((pt["cls_idx"].cpu().long()[dm] == ot["cls_idx"][jj[dm]]).all()), dfrac
    excl = torch.zeros(H, W, dtype=torch.bool)
    matched_o = set(jj[dm].tolist())
    unmatched = [pd_[i, 1:5] for i in (~dm).nonzero().flatten().tolist()] + \
                [od_[k, 1:5] for k in range(od_.shape[0]) if k not in matched_o]
    for b in unmatched:
        x1, y1, x2, y2 = [float(v) for v in b]
        excl[max(0, int(y1) - 2):min(H, int(y2) + 3), max(0, int(x1) - 2):min(W, int(x2) + 3)] = True
    sem_bad, sem_unexpl = near_tie_report(r[2]["fcn_outputs"].cpu(), o[2]["fcn_outputs"], ot["fcn_output"], TIE_TOL)
    pan_bad, pan_unexpl = near_tie_report(r[2]["panoptic_outputs"].cpu(), o[2]["panoptic_outputs"], ot["panoptic_logits"],
                                          TIE_TOL, exclude=excl if unmatched else None)
    print("%s full size tc32: %d detections, matched %.4f; label pixels differing: semantic %d, panoptic %d; not "
          "explained by a near-tie: %d / %d" % (name, pd_.shape[0], dfrac, sem_bad, pan_bad, sem_unexpl, pan_unexpl))
    assert sem_unexpl == 0 and pan_unexpl == 0, (sem_bad, sem_unexpl, pan_bad, pan_unexpl)
    assert sem_bad <= 2e-5 * H * W and pan_bad <= 2e-5 * H * W, (sem_bad, pan_bad)


@pytest.mark.parametrize("name", ["track", "fuse"])
def test_cuda_graph_replay_equals_eager(models, name):
    _, prod = models[name]
    prod.precision = "tc32"
    H, W = 128, 256
    frames = [make_pair(H, W, seed=s) for s in (1, 2, 3, 4)]
    outs = {}
    for use_graph in (False, True):
        prod.use_cuda_graph = use_graph
        prod.reset_tracker()
        outs[use_graph] = [_labels(_run(prod, a, b if name == "fuse" else None, 10001 + f, H, W))
                           for f, (a, b) in enumerate(frames)]
    prod.use_cuda_graph = True
    for e, g in zip(outs[False], outs[True]):
        assert all(torch.equal(x, y) for x, y in zip(e, g))


@pytest.mark.parametrize("name,streaming", [("track", False), ("fuse", False), ("fuse", True)])
def test_clip_runner_equals_direct_calls(models, name, streaming):
    """ClipRunner with prefetch (two ping-pong graph instances) == direct simple_test calls; Track's pairs are
    (img, None) and upload no reference frame; in a streaming Fuse clip the reference frame of t is frame t - 1."""
    from vps_b200.runner import ClipRunner
    _, prod = models[name]
    prod.precision = "tc32"
    H, W = 128, 256
    g = torch.Generator().manual_seed(41)
    imgs = [torch.randn(1, 3, H, W, generator=g) for _ in range(6)]
    metas = [meta(10001 + t, H, W) for t in range(6)]
    if name == "track":
        pairs = [(x, None) for x in imgs]
    else:
        pairs = [(imgs[t], imgs[max(t - 1, 0)]) for t in range(6)]
    prod.reset_tracker()
    direct = [_labels(_run(prod, a, b, m["iid"], H, W)) for (a, b), m in zip(pairs, metas)]
    try:
        prod.label_dtype = torch.uint8
        prod.reset_tracker()
        pinned = [(a.pin_memory(), None if b is None else b.pin_memory()) for a, b in pairs]
        got = [_labels(r) for r in ClipRunner(prod, "cuda:0", streaming=streaming).run(pinned, metas, prefetch=True)]
    finally:
        prod.label_dtype = torch.int64
    assert len(got) == len(direct)
    for d, r in zip(direct, got):
        assert all(torch.equal(x, y) for x, y in zip(d, r))


def test_clip_runner_unify_fuse_is_image_level(models):
    from oracle.variants import unify_image_frame
    from vps_b200.runner import ClipRunner
    _, prod = models["fuse"]
    prod.precision = "fp32"
    H, W = 128, 256
    frames = [make_pair(H, W, seed=s) for s in (21, 22, 23)]
    metas = [meta(10001 + f, H, W) for f in range(len(frames))]
    try:
        prod.label_dtype = torch.uint8
        runner = ClipRunner(prod, "cuda:0", unify=True)
        assert runner.unifier.image
        n = 0
        for r in runner.run([(a.pin_memory(), b.pin_memory()) for a, b in frames], metas):
            seg, pan = r[2]["fcn_outputs"][0].numpy(), r[2]["panoptic_outputs"][0].numpy()
            want = unify_image_frame(seg, pan, r[2]["panoptic_cls_inds"].cpu().numpy())
            assert np.array_equal(r[2]["pan_2ch"].numpy(), want)
            n += int((want[:, :, 1] > 0).any())
        assert n > 0                     # the frames hold instances
    finally:
        prod.label_dtype = torch.int64
        prod.precision = "tc32"


def test_image_unify_kernel_matches_reference_golden(cuda):
    from vps_b200.postproc import PanUnifier
    g = np.load(os.path.join(GOLDEN, "unify_pan.npz"))
    h = np.load(os.path.join(GOLDEN, "unify_image.npz"))
    u = PanUnifier(image=True)
    for i in range(int(g["nframes"])):
        for dt in (torch.uint8, torch.int64):
            seg = torch.from_numpy(g["seg%d" % i]).to(dt).cuda()
            pan = torch.from_numpy(g["pan%d" % i]).to(dt).cuda()
            out = u(seg, pan, g["cls%d" % i]).cpu().numpy()
            assert np.array_equal(out, h["out%d" % i]), (i, dt)
    with pytest.raises(ValueError):
        u(seg, pan, g["cls0"], g["obj0"])


def test_vpq_parity_of_the_track_chain(cuda):
    """Track: model -> PanUnifier -> segments_from_pan2ch -> VpqEvaluator against the oracle chain: PQ = SQ = RQ = 1."""
    from tests.test_gpu_vpq import _oracle_clip, _product_clip
    from tests.test_vpq_cpu import CATEGORIES
    from vps_b200 import vpq as P
    oracle, prod = build("track", "fp32")
    H, W = 128, 256
    frames = [make_pair(H, W, seed=s) for s in (51, 52, 53, 54, 55)]
    gt = _oracle_clip(oracle, frames, H, W)
    for precision in ("tc32", "fp32"):
        pred = _product_clip(prod, frames, H, W, precision)
        ev = P.VpqEvaluator(CATEGORIES)
        for (gi, gs), (pi, ps) in zip(gt, pred):
            ev.add_frame(gs, ps, torch.from_numpy(gi.astype(np.int64)).cuda(), pi)
        for nframes in (1, 2, 3):
            res, _ = P.pq_average(ev.compute(nframes), CATEGORIES, isthing=None)
            print("Track VPQ agreement %s k=%d: PQ %.4f SQ %.4f RQ %.4f (n=%d)" % (precision, nframes, res["pq"], res["sq"],
                                                                               res["rq"], res["n"]))
            assert res["pq"] == 1.0 and res["sq"] == 1.0 and res["rq"] == 1.0, (nframes, res)
