"""GPU: evaluation of the image panoptic model (vps_b200.ipq) -- the seg-confusion and image-id kernels against numpy
restatements, the evaluators against the golden numbers of the reference's own evaluate_ssegs / evaluate_panoptic, and the
whole chain PanopticFuse -> PanUnifier(image=True) -> IpqEvaluator / SegEvaluator against the oracle's chain."""
import numpy as np
import pytest
import torch

from tests.e2e_util import make_pair, meta

pytestmark = pytest.mark.gpu


def _bincount_conf(gt, pred, C):
    """restatement of the reference's counting: gt != 255, index gt * C + (pred & 255) counted iff < C * C"""
    g = gt.reshape(-1).astype(np.int64)
    p = pred.reshape(-1).astype(np.int64) & 255
    keep = g != 255
    idx = g[keep] * C + p[keep]
    return np.bincount(idx[idx < C * C], minlength=C * C).reshape(C, C).astype(np.uint64)


def _blocks(rng, H, W, hi, b):
    return rng.integers(0, hi, size=((H + b - 1) // b, (W + b - 1) // b)).repeat(b, 0).repeat(b, 1)[:H, :W]


def _seg_conf(gt, pred, C, offset=0):
    """vps_seg_confusion through an offset view of a larger buffer (offset > 0: unaligned uint8 pointers)"""
    import ctypes as Ct

    from vps_b200 import ops
    from vps_b200._lib import lib
    n = gt.size
    g = torch.zeros(n + offset, dtype=torch.uint8, device="cuda")
    g[offset:] = torch.from_numpy(gt.reshape(-1))
    p = torch.zeros(n + offset, dtype=torch.from_numpy(pred).dtype, device="cuda")
    p[offset:] = torch.from_numpy(pred.reshape(-1))
    conf = torch.zeros(C * C, dtype=torch.int64, device="cuda")
    ops.check(lib().vps_seg_confusion(ops._ptr(g[offset:]), ops._ptr(p[offset:]), p.element_size(), Ct.c_int64(n), C,
                                      ops._ptr(conf), ops.stream()), "seg_confusion")
    return conf.cpu().numpy().view(np.uint64).reshape(C, C)


@pytest.mark.parametrize("dtype", [np.uint8, np.int64])
def test_seg_confusion_matches_bincount(cuda, dtype):
    """piecewise-constant maps with gt 255, gt in [C, 255), preds >= C (aliasing into the next row); 1024x2048, odd sizes
    and unaligned pointers"""
    rng = np.random.default_rng(3)
    for H, W, off in ((1024, 2048, 0), (37, 53, 0), (61, 97, 3), (1, 1, 1)):
        gt = _blocks(rng, H, W, 24, 8).astype(np.uint8)
        gt[_blocks(rng, H, W, 5, 16) == 0] = 255
        pred = _blocks(rng, H, W, 22, 5)
        if dtype == np.int64:
            pred = pred + 256 * _blocks(rng, H, W, 3, 7)                # only the low byte counts
        pred = pred.astype(dtype)
        got = _seg_conf(gt, pred, 19, off)
        assert np.array_equal(got, _bincount_conf(gt, pred, 19)), (H, W, off)
    import ctypes as Ct

    from vps_b200 import ops
    from vps_b200._lib import VpsError, lib
    with pytest.raises(VpsError):                                      # C > 64 is rejected
        ops.check(lib().vps_seg_confusion(None, None, 1, Ct.c_int64(1), 65, None, ops.stream()), "seg_confusion")


def test_seg_evaluator_accumulates_frames(cuda):
    from oracle import ipq as O
    from vps_b200.ipq import SegEvaluator
    rng = np.random.default_rng(4)
    ev = SegEvaluator()
    total = np.zeros((19, 19))
    for H, W in ((64, 128), (33, 45), (128, 64)):
        gt = _blocks(rng, H, W, 19, 4).astype(np.uint8)
        gt[:2] = 255
        pred = _blocks(rng, H, W, 21, 6).astype(np.int64)
        ev.add_frame(torch.from_numpy(gt).cuda(), torch.from_numpy(pred)[None].cuda())
        total += O.seg_confusion(gt, pred)
    r, want = ev.result(), O.seg_result(total)
    assert np.array_equal(r["confusion_matrix"], want["confusion_matrix"])
    assert np.array_equal(r["IU_array"], want["IU_array"]) and r["meanIU"] == want["meanIU"]
    with pytest.raises(ValueError):
        ev.add_frame(torch.zeros(4, 5, dtype=torch.uint8, device="cuda"), torch.zeros(5, 4, dtype=torch.uint8, device="cuda"))


def test_image_ids_match_oracle(cuda):
    from oracle import ipq as O
    from vps_b200.ipq import image_segment_ids
    rng = np.random.default_rng(6)
    for H, W in ((1024, 2048), (61, 97)):
        p2 = np.zeros((H, W, 3), np.uint8)
        p2[..., 0] = _blocks(rng, H, W, 19, 8)
        p2[..., 0][_blocks(rng, H, W, 6, 16) == 0] = 255
        p2[..., 1] = np.where(p2[..., 0] >= 11, _blocks(rng, H, W, 40, 8), 0)
        p2[..., 2] = _blocks(rng, H, W, 256, 4)                       # channel 2 never matters for the image key
        got = image_segment_ids(torch.from_numpy(p2).cuda()).cpu().numpy().astype(np.uint32)
        _, want = O.convert_image(p2)
        assert np.array_equal(got, want), (H, W)


def test_evaluators_reproduce_reference_golden(cuda, tmp_path):
    import os

    from tests.test_ipq_cpu import load
    from oracle.writer import id2rgb
    from vps_b200.ipq import IpqEvaluator, SegEvaluator
    d, info, categories, txt = load()
    seg, ipq = SegEvaluator(), IpqEvaluator(categories)
    for i in range(int(d["nframes"])):
        seg.add_frame(torch.from_numpy(d["trainid%d" % i]).cuda(), torch.from_numpy(d["fcn%d" % i]).cuda())
        ipq.add_frame(torch.from_numpy(id2rgb(d["gt_ids%d" % i])).cuda(), info["gt"][i], torch.from_numpy(d["pan2ch%d" % i]).cuda())
    r = seg.result()
    assert np.array_equal(r["confusion_matrix"], d["seg_confusion"])
    assert np.array_equal(r["IU_array"], d["IU_array"]) and r["meanIU"] == d["meanIU"]
    stat = ipq.compute()
    for row, c in enumerate(d["stat"]):
        assert [stat[row].tp, stat[row].fp, stat[row].fn] == c[1:].astype(int).tolist(), row
        assert stat[row].iou == c[0], row
    path = os.path.join(str(tmp_path), "pq.txt")
    ipq.write_pq_txt(path, stat)
    assert open(path).read() == txt


def test_ipq_parity_of_the_whole_chain(cuda):
    """PanopticFuse -> PanUnifier(image=True) -> IpqEvaluator / SegEvaluator, all on the GPU, scored against the oracle's
    chain (oracle.variants + oracle.ipq converter) as ground truth, on the golden Fuse clip (whose label maps
    test_gpu_models.py pins bit for bit in tc32 and fp32).  tc32 and fp32: PQ = SQ = RQ = 1 and a diagonal semantic
    confusion equal to the oracle's.  bf16: the agreement is reported (random-init weights give noise-like logits),
    only checked to be a valid score."""
    from oracle import ipq as O
    from oracle.variants import unify_image_frame
    from oracle.writer import id2rgb
    from tests.golden.make_models_golden import clip
    from tests.test_gpu_models import build
    from vps_b200.ipq import IpqEvaluator, SegEvaluator
    from vps_b200.postproc import PanUnifier
    from vps_b200.vpq import pq_average
    oracle, prod = build("fuse", "fp32")
    categories = {i: {"id": i, "isthing": 1 if i >= 11 else 0} for i in range(19)}
    H, W = 128, 256
    frames = list(clip("fuse"))
    gts = []
    for iid, a, b in frames:
        p = oracle.simple_test(a, dict(iid=iid, img_shape=(H, W, 3)), b)[2]
        sem = p["fcn_outputs"][0].numpy().astype(np.uint8)
        p2 = unify_image_frame(sem, p["panoptic_outputs"][0].numpy().astype(np.uint8), np.asarray(p["panoptic_cls_inds"]),
                               stuff_area_limit=256)
        segs, ids = O.convert_image(p2)
        gts.append((sem, id2rgb(ids), segs))
    uni = PanUnifier(image=True, stuff_area_limit=256)
    for precision in ("tc32", "fp32", "bf16"):
        prod.precision = precision
        ipq, seg = IpqEvaluator(categories), SegEvaluator()
        want = np.zeros((19, 19))
        for (iid, a, b), (sem, rgb, segs) in zip(frames, gts):
            r = prod.simple_test(a.cuda(), [meta(iid, H, W)], ref_img=[b.cuda()])
            p2 = uni(r[2]["fcn_outputs"], r[2]["panoptic_outputs"], r[2]["host"]["panoptic_cls_inds"])
            ipq.add_frame(torch.from_numpy(rgb).cuda(), segs, p2)
            seg.add_frame(torch.from_numpy(sem).cuda(), r[2]["fcn_outputs"])
            want += O.seg_confusion(sem, sem)
        res, _ = pq_average(ipq.compute(), categories, isthing=None)
        conf = seg.result()["confusion_matrix"]
        print("IPQ agreement %s: PQ %.4f SQ %.4f RQ %.4f (n=%d); semantic pixel agreement %.4f"
              % (precision, res["pq"], res["sq"], res["rq"], res["n"], np.trace(conf) / conf.sum()))
        if precision in ("tc32", "fp32"):
            assert res["pq"] == 1.0 and res["sq"] == 1.0 and res["rq"] == 1.0, res
            assert np.array_equal(conf, want) and np.array_equal(conf, np.diag(np.diag(conf)))
        else:
            assert 0.0 < res["pq"] <= 1.0 and res["n"] > 0, res
    prod.precision = "tc32"


def test_seg_confusion_on_fusetrack_and_track(cuda):
    """the semantic evaluation applies to every model's fcn_outputs: one fp32 frame of FuseTrack and of Track"""
    from oracle import ipq as O
    from tests.e2e_util import build_models
    from tests.test_gpu_models import build
    from vps_b200.ipq import SegEvaluator
    H, W = 128, 256
    a, b = make_pair(H, W, seed=71)
    for name in ("fusetrack", "track"):
        oracle, prod = build_models("C", 0, "fp32", "cuda:0") if name == "fusetrack" else build(name, "fp32")
        ref = oracle.simple_test(a, dict(iid=10001, img_shape=(H, W, 3)), b if name == "fusetrack" else None, {})[2]
        sem = ref["fcn_outputs"][0].numpy().astype(np.uint8)
        r = prod.simple_test(a.cuda(), [meta(10001, H, W)], ref_img=[b.cuda()] if name == "fusetrack" else None)
        ev = SegEvaluator()
        ev.add_frame(torch.from_numpy(sem).cuda(), r[2]["fcn_outputs"])
        conf = ev.result()["confusion_matrix"]
        assert np.array_equal(conf, O.seg_confusion(sem, sem)), name
