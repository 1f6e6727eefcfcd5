"""GPU: frames of any size through the test pipeline.  The keep-ratio Resize fused into the input stage
(`vps_preprocess_resize_u8`) is bit-identical to cv2.resize INTER_LINEAR + Normalize + Pad (oracle/resize.py, pinned
against OpenCV by tests/test_resize_cpu.py, and the golden digests of OpenCV's own output); the detectors and ClipRunner fed
resized uint8 frames equal the same models fed the host-prepared tensors; the semantic confusion of a prediction of
another shape (`vps_seg_confusion_nearest`) equals a numpy gather through Pillow's NEAREST tables, and SegEvaluator
reproduces the reference's own evaluate_ssegs on such predictions."""
import ctypes as Ct
import hashlib

import numpy as np
import pytest
import torch

from tests.test_resize_cpu import GOLDEN, cases, frame

pytestmark = pytest.mark.gpu

NORM = dict(mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375])


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _resize_prep(img, oh, ow, hp, wp, to_rgb=True, offset=0, fill=float("nan")):
    """vps_preprocess_resize_u8 on a frame copied to `offset` bytes into a device buffer; the output starts as `fill`"""
    from vps_b200 import ops
    from vps_b200._lib import lib
    h, w = img.shape[:2]
    buf = torch.zeros(img.size + offset, dtype=torch.uint8, device="cuda")
    buf[offset:] = torch.from_numpy(img.reshape(-1)).cuda()
    out = torch.full((1, 3, hp, wp), fill, dtype=torch.float32, device="cuda")
    mean = (Ct.c_float * 3)(*[float(np.float32(v)) for v in NORM["mean"]])
    std = (Ct.c_float * 3)(*[float(np.float32(v)) for v in NORM["std"]])
    ops.check(lib().vps_preprocess_resize_u8(ops._ptr(buf[offset:]), h, w, oh, ow, mean, std, int(to_rgb), ops._ptr(out), hp, wp,
                                             ops.stream()), "preprocess_resize_u8")
    return out.cpu().numpy()


def test_preprocess_resize_matches_cv2_goldens(cuda):
    """every golden shape at full size: the digest of cv2's pipeline output, and the oracle bit for bit"""
    from oracle import resize as OR
    g = cases()
    for c in g["cases"]:
        img = frame(c["seed"], *c["shape"])
        (oh, ow), hp_wp = c["resized_shape"], c["pad_shape"]
        got = _resize_prep(img, oh, ow, *hp_wp)
        assert _sha(got) == c["sha256_prepared"], c["shape"]
        if c["shape"][0] * c["shape"][1] <= 1200 * 1600:
            want = OR.prepare_frame(img, NORM["mean"], NORM["std"], True, 32, img_scale=tuple(g["img_scale"]))
            assert np.array_equal(got, want), c["shape"]


@pytest.mark.parametrize("to_rgb", [True, False])
@pytest.mark.parametrize("offset", [0, 1, 3])
def test_preprocess_resize_odd_unaligned_padded(cuda, to_rgb, offset):
    """odd widths, an unaligned source, both channel orders, and zeros over the whole padding of a larger tensor"""
    from oracle import pipeline as OP
    from oracle import resize as OR
    rng = np.random.default_rng(17 + offset)
    for h, w, oh, ow in ((1080, 1920, 1024, 1820), (37, 91, 83, 205), (45, 131, 31, 97), (5, 7, 1, 1), (1, 1, 3, 5), (123, 77, 123, 77)):
        img = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
        hp, wp = oh + 40, ow + 33
        got = _resize_prep(img, oh, ow, hp, wp, to_rgb, offset)
        want = OP.imnormalize(OR.resize_linear_u8(img, oh, ow), NORM["mean"], NORM["std"], to_rgb).transpose(2, 0, 1)
        assert np.array_equal(got[0, :, :oh, :ow], want), (h, w, oh, ow)
        assert not got[0, :, oh:].any() and not got[0, :, :, ow:].any(), (h, w, oh, ow)


def test_preprocess_resize_is_the_identity_at_scale_1(cuda):
    from vps_b200 import ops
    from vps_b200._lib import lib
    from vps_b200.pipeline import InputStage
    st = InputStage()
    for h, w in ((1024, 2048), (61, 97)):
        img = frame(5, h, w)
        hp, wp = (h + 31) // 32 * 32, (w + 31) // 32 * 32
        d = torch.from_numpy(img).cuda()
        want = torch.full((1, 3, hp, wp), float("nan"), device="cuda")
        ops.check(lib().vps_preprocess_u8(ops._ptr(d), h, w, st.mean, st.std, 1, ops._ptr(want), hp, wp, ops.stream()), "preprocess_u8")
        assert np.array_equal(_resize_prep(img, h, w, hp, wp), want.cpu().numpy()), (h, w)


def test_input_stage_resize_meta(cuda):
    """InputStage(resize=True): the tensor of the oracle pipeline and the meta fields mmdet's Resize / Pad give"""
    from oracle import resize as OR
    from vps_b200.pipeline import InputStage
    st = InputStage(resize=True)
    for h, w in ((1080, 1920), (720, 1280), (1024, 2048), (37, 91)):
        img = frame(h * w, h, w)
        x, meta = st(torch.from_numpy(img))
        (oh, ow), sf = OR.rescale_size(h, w, (2048, 1024))
        want = OR.prepare_frame(img, NORM["mean"], NORM["std"], True, 32, img_scale=(2048, 1024))
        assert np.array_equal(x.cpu().numpy(), want), (h, w)
        assert meta["ori_shape"] == (h, w, 3) and meta["img_shape"] == (oh, ow, 3)
        assert meta["pad_shape"] == (want.shape[2], want.shape[3], 3)
        assert type(meta["scale_factor"]) is float and meta["scale_factor"] == sf
    a = torch.from_numpy(frame(1, 1080, 1920))
    xa, xb, meta = st.pair(a, a.clone())
    assert torch.equal(xa, xb) and meta["img_shape"] == (1024, 1820, 3)
    with pytest.raises(ValueError):
        st.pair(a, torch.zeros(720, 1280, 3, dtype=torch.uint8))


def _frames(seed, n, h, w):
    """a short clip: one random frame shifted a little per step (so tracks carry over)"""
    base = np.random.default_rng(seed).integers(0, 256, size=(h, w, 3), dtype=np.uint8)
    return [np.ascontiguousarray(np.roll(base, (2 * t, 3 * t), axis=(0, 1))) for t in range(n)]


@pytest.mark.parametrize("name", ["fusetrack", "track"])
def test_detectors_from_resized_frames(cuda, name):
    """a detector fed uint8 frames resized on the device == the same detector fed the oracle-prepared fp32 tensors"""
    from oracle import resize as OR
    from tests.e2e_util import build_models
    from tests.test_gpu_models import build
    from vps_b200.pipeline import InputStage
    _, prod = build_models("C", 0, "tc32", "cuda:0") if name == "fusetrack" else build(name, "tc32")
    a, b = _frames(23, 2, 150, 303)
    st = InputStage(img_scale=(256, 128), resize=True)
    xa, xb, m = st.pair(torch.from_numpy(a), torch.from_numpy(b))
    assert m["img_shape"] == (127, 256, 3) and tuple(xa.shape) == (1, 3, 128, 256)      # img_shape inside the padding
    meta = dict(m, filename="synthetic_city_%06d.png" % 10001, iid=10001)
    outs = []
    for x, r in ((xa, xb), tuple(torch.from_numpy(OR.prepare_frame(f, NORM["mean"], NORM["std"], True, 32, img_scale=(256, 128))).cuda()
                                 for f in (a, b))):
        prod.reset_tracker()
        res = prod.simple_test(x, [meta], ref_img=[r] if name == "fusetrack" else None)[2]
        ids = res.get("panoptic_det_obj_ids")
        outs.append((res["panoptic_outputs"].clone(), res["fcn_outputs"].clone(), None if ids is None else ids.cpu().clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert (outs[0][2] is None) == (outs[1][2] is None) and (outs[0][2] is None or torch.equal(outs[0][2], outs[1][2]))


@pytest.mark.parametrize("name,divisor,streaming", [("track", 32, False), ("fusetrack", 64, False), ("fusetrack", 64, True)])
def test_clip_runner_resizes_1080p(cuda, name, divisor, streaming):
    """ClipRunner(input_stage=InputStage(resize=True)) on a 1080x1920 clip == ClipRunner fed the host-prepared tensors with the
    reference's meta: label maps and track ids.  The clip resizes to 1024x1820; Pad(32) gives 1024x1824, which PanopticTrack
    takes.  FuseTrack's FlowNet2 needs sides divisible by 64 (panoptic_fusetrack.py:129-130 asserts it, as the product
    does), so FuseTrack runs the same clip under Pad(64): 1024x1856."""
    from oracle import resize as OR
    from tests.e2e_util import build_models
    from tests.test_gpu_models import build
    from vps_b200.pipeline import InputStage
    from vps_b200.runner import ClipRunner
    _, prod = build_models("C", 0, "tc32", "cuda:0") if name == "fusetrack" else build(name, "tc32")
    n = 4
    frames = _frames(31, n, 1080, 1920)
    ref = (lambda t: None) if name == "track" else (lambda t: max(t - 1, 0))
    pairs_u8 = [(torch.from_numpy(frames[t]).pin_memory(), None if ref(t) is None else torch.from_numpy(frames[ref(t)]).pin_memory())
                for t in range(n)]
    f32 = [torch.from_numpy(OR.prepare_frame(f, NORM["mean"], NORM["std"], True, divisor, img_scale=(2048, 1024))) for f in frames]
    hp = (1820 + divisor - 1) // divisor * divisor
    assert tuple(f32[0].shape) == (1, 3, 1024, hp)
    pairs_f32 = [(f32[t].pin_memory(), None if ref(t) is None else f32[ref(t)].pin_memory()) for t in range(n)]
    geo = dict(ori_shape=(1080, 1920, 3), img_shape=(1024, 1820, 3), pad_shape=(1024, hp, 3), scale_factor=1024 / 1080)
    ids = [dict(filename="synthetic_city_%06d.png" % (10001 + t), iid=10001 + t) for t in range(n)]
    outs = []
    try:
        prod.label_dtype = torch.uint8
        for pairs, stage, metas in ((pairs_f32, None, [dict(m, **geo) for m in ids]),
                                    (pairs_u8, InputStage(size_divisor=divisor, resize=True), ids)):
            prod.reset_tracker()
            runner = ClipRunner(prod, "cuda:0", input_stage=stage, streaming=streaming)
            outs.append([(r[2]["panoptic_outputs"].clone(), r[2]["fcn_outputs"].clone(), r[2]["panoptic_det_obj_ids"].cpu().clone())
                         for r in runner.run(pairs, metas)])
    finally:
        prod.label_dtype = torch.int64
    assert len(outs[0]) == len(outs[1]) == n
    for t, (a, b) in enumerate(zip(*outs)):
        assert tuple(a[0].shape[-2:]) == (1024, 1820)
        assert all(torch.equal(x, y) for x, y in zip(a, b)), t


def _nearest_conf(gt, pred, C, xtab, ytab):
    """numpy: gather through the tables (index < 0 reads 0), then the counting rule of vps_seg_confusion"""
    p = pred.astype(np.int64)[np.clip(ytab, 0, None)][:, np.clip(xtab, 0, None)] & 255
    p[ytab < 0] = 0
    p[:, xtab < 0] = 0
    g = gt.reshape(-1).astype(np.int64)
    keep = g != 255
    idx = g[keep] * C + p.reshape(-1)[keep]
    return np.bincount(idx[idx < C * C], minlength=C * C).reshape(C, C).astype(np.uint64)


def _run_nearest(gt, pred, C, xtab, ytab, offset=0):
    from vps_b200 import ops
    from vps_b200._lib import lib
    gh, gw = gt.shape
    ph, pw = pred.shape
    g = torch.zeros(gt.size + offset, dtype=torch.uint8, device="cuda")
    g[offset:] = torch.from_numpy(gt.reshape(-1))
    p = torch.from_numpy(pred).cuda()
    xt, yt = torch.from_numpy(xtab).cuda(), torch.from_numpy(ytab).cuda()
    conf = torch.zeros(C * C, dtype=torch.int64, device="cuda")
    ops.check(lib().vps_seg_confusion_nearest(ops._ptr(g[offset:]), gh, gw, ops._ptr(p), p.element_size(), ph, pw, ops._ptr(xt),
                                              ops._ptr(yt), C, ops._ptr(conf), ops.stream()), "seg_confusion_nearest")
    return conf.cpu().numpy().view(np.uint64).reshape(C, C)


@pytest.mark.parametrize("dtype", [np.uint8, np.int64])
def test_seg_confusion_nearest_matches_numpy(cuda, dtype):
    from tests.test_gpu_ipq import _blocks, _seg_conf
    from vps_b200.ipq import nearest_table
    rng = np.random.default_rng(8)
    C = 19
    for (gh, gw), (ph, pw), off in (((1080, 1920), (1024, 1820), 0), ((1024, 1820), (1080, 1920), 0), ((61, 97), (37, 53), 3),
                                    ((37, 53), (61, 97), 1), ((45, 131), (61, 97), 0), ((1, 1), (3, 5), 1), ((17, 16), (1, 1), 0)):
        gt = _blocks(rng, gh, gw, 24, 8).astype(np.uint8)
        gt[_blocks(rng, gh, gw, 5, 16) == 0] = 255
        pred = _blocks(rng, ph, pw, 22, 5)
        if dtype == np.int64:
            pred = pred + 256 * _blocks(rng, ph, pw, 3, 7)                     # only the low byte counts
        pred = pred.astype(dtype)
        xtab, ytab = nearest_table(pw, gw), nearest_table(ph, gh)
        got = _run_nearest(gt, pred, C, xtab, ytab, off)
        assert np.array_equal(got, _nearest_conf(gt, pred, C, xtab, ytab)), (gh, gw, ph, pw)
    # tables with out-of-source entries read 0
    gt = _blocks(rng, 20, 30, 19, 4).astype(np.uint8)
    pred = _blocks(rng, 10, 15, 19, 3).astype(dtype)
    xtab, ytab = nearest_table(15, 30), nearest_table(10, 20)
    xtab[[0, 7, 29]] = -1
    ytab[[5, 19]] = -1
    assert np.array_equal(_run_nearest(gt, pred, C, xtab, ytab), _nearest_conf(gt, pred, C, xtab, ytab))
    # equal shapes through identity tables == vps_seg_confusion
    gt = _blocks(rng, 1024, 2048, 24, 8).astype(np.uint8)
    pred = _blocks(rng, 1024, 2048, 22, 5).astype(dtype)
    got = _run_nearest(gt, pred, C, nearest_table(2048, 2048), nearest_table(1024, 1024))
    assert np.array_equal(got, _seg_conf(gt, pred, C))


def test_seg_evaluator_resize_pred_reproduces_reference_golden(cuda):
    import os

    from vps_b200.ipq import SegEvaluator
    d = np.load(os.path.join(GOLDEN, "ipq_resize.npz"))
    for dtype in (torch.uint8, torch.int64):
        ev = SegEvaluator(resize_pred=True)
        for i in range(int(d["nframes"])):
            gt, pred = d["trainid%d" % i], d["fcn%d" % i]
            ev.add_frame(torch.from_numpy(gt).cuda(), torch.from_numpy(pred).to(dtype)[None].cuda())
        r = ev.result()
        assert np.array_equal(r["confusion_matrix"], d["seg_confusion"]), dtype
        assert np.array_equal(r["IU_array"], d["IU_array"]) and r["meanIU"] == d["meanIU"]
    with pytest.raises(ValueError):
        SegEvaluator().add_frame(torch.zeros(4, 5, dtype=torch.uint8, device="cuda"), torch.zeros(5, 4, dtype=torch.uint8, device="cuda"))
