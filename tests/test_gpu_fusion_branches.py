"""MaskRemoval (vps_mask_removal) and the panoptic fusion (vps_panoptic_fuse) on each of their branches, against the
oracle written as the reference writes it: mask_removal, then seg_term on rois[keep] * 4, then
max(softmax(cat[stuff, inst + energy])) with fcn_output = bilinear x4 of fcn_score.  Keep lists, nkeep and the
panoptic and semantic label maps must be identical.

Branches: the thread-block-cluster MaskRemoval (k <= 128 and num_things <= 8) and the per-position one (otherwise),
a device detection count below k, uint8 and int64 label maps, fp32 and bf16 fcn_score, frames that are not a
multiple of the 32 x 8 fusion tile, 128 kept instances, the dummy result, and the keep_inds = [0] fallback when
MaskRemoval keeps nothing.

Inputs come from fixed seeds and are continuous.  None of them places two logits a few ulps apart on purpose: there
the reference's softmax can make two probabilities equal where the kernel's first-max argmax over the logits still
tells them apart."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

NS, MS, CAP = 11, 28, 128      # stuff classes, mask logit size, fusion instance capacity (MAX_DET_CAP)
FILL = 200                     # label-map sentinel: a pixel the kernel never writes keeps it


def to_nhwc(t, dtype=torch.float32):
    """[n,c,h,w] -> device NHWC view with channels padded to a multiple of 8 (the library's activation layout)"""
    n, c, h, w = t.shape
    buf = torch.zeros(n, h, w, (c + 7) // 8 * 8, dtype=dtype)
    buf[..., :c] = t.permute(0, 2, 3, 1).to(dtype)
    return buf.cuda()[..., :c]


def stable_order(prob):
    return np.argsort(-prob.numpy(), kind="stable").astype(np.int32)


# ---------------------------------------------------------------------------------------------------- oracle
def oracle(boxes, prob, mlog, cls_idx, fcn_score, H, W):
    """(keep_inds, pano, sem) of panoptic_fusetrack.py:572-593; boxes [k,4], mlog [k,28,28], cls_idx 1-based."""
    from oracle.model import mask_removal, seg_term
    keep, energy = mask_removal(boxes, prob, mlog[:, None], cls_idx, (H, W))
    fcn_output = F.interpolate(fcn_score, scale_factor=4, mode="bilinear", align_corners=False)
    rois = torch.cat([torch.zeros(boxes.shape[0], 1), boxes], 1)
    stuff, inst = seg_term(cls_idx[keep], fcn_output, rois[keep] * 4.0)
    pano = torch.max(F.softmax(torch.cat([stuff, inst + energy], 1), 1), 1)[1][0]
    sem = torch.max(F.softmax(fcn_output, 1), 1)[1][0]
    return keep.numpy(), pano, sem


# ---------------------------------------------------------------------------------------------------- kernels
def gpu_mask_removal(boxes, order, mlog, cls_idx, H, W, num_things=8, k_dev=None):
    """vps_mask_removal; returns (keep_sorted, nkeep) on the device"""
    from vps_b200 import ops
    dev, k = "cuda", boxes.shape[0]
    keep_sorted = torch.zeros(max(k, CAP), dtype=torch.int32, device=dev)
    nkeep = torch.zeros(1, dtype=torch.int32, device=dev)
    kd = None if k_dev is None else torch.tensor([k_dev], dtype=torch.int32, device=dev)
    ops.mask_removal(boxes.cuda(), torch.as_tensor(order, dtype=torch.int32).cuda(), k, mlog.contiguous().cuda(), MS,
                     cls_idx.int().cuda(), H, W, 0.3, torch.empty(num_things, H, W, dtype=torch.uint8, device=dev),
                     num_things, torch.empty(2 * k, dtype=torch.int32, device=dev),
                     torch.empty(k, dtype=torch.int32, device=dev), keep_sorted, nkeep, k_dev=kd)
    return keep_sorted, nkeep


def kept(keep_sorted, nkeep):
    return keep_sorted[:int(nkeep.item())].cpu().numpy().astype(np.int64)


def gpu_fuse(fcn_score, boxes, cls_idx, mlog, keep_sorted, nkeep, H, W, dummy=False, score_dtype=torch.float32):
    """vps_panoptic_fuse into int64 and into uint8 label maps; the two must hold the same values.  Returns (pano, sem)."""
    from vps_b200 import ops
    maps = []
    for ldt in (torch.int64, torch.uint8):
        pano = torch.full((H, W), FILL, dtype=ldt, device="cuda")
        sem = torch.full((H, W), FILL, dtype=ldt, device="cuda")
        ops.panoptic_fuse(to_nhwc(fcn_score, score_dtype), boxes.cuda(), cls_idx.int().cuda(), mlog.contiguous().cuda(),
                          MS, keep_sorted, nkeep, CAP, NS, dummy, H, W, pano, sem)
        maps.append((pano.cpu().long(), sem.cpu().long()))
    (p64, s64), (p8, s8) = maps
    assert torch.equal(p8, p64) and torch.equal(s8, s64), "uint8 and int64 label maps differ"
    return p64, s64


def check_frame(fcn_score, boxes, prob, mlog, cls_idx, num_things=8, score_dtype=torch.float32):
    """MaskRemoval and fusion of one frame against the oracle; returns the oracle's keep list and pano map"""
    H, W = fcn_score.shape[2] * 4, fcn_score.shape[3] * 4
    keep_ref, pano_ref, sem_ref = oracle(boxes, prob, mlog, cls_idx, fcn_score, H, W)
    keep_sorted, nkeep = gpu_mask_removal(boxes, stable_order(prob), mlog, cls_idx, H, W, num_things)
    got = kept(keep_sorted, nkeep)
    # the host maps an empty keep list to [0] (mask_removal.py:89-91); the device count stays 0
    assert np.array_equal(got if got.size else np.zeros(1, np.int64), keep_ref)
    pano, sem = gpu_fuse(fcn_score, boxes, cls_idx, mlog, keep_sorted, nkeep, H, W, score_dtype=score_dtype)
    assert torch.equal(sem, sem_ref)
    assert torch.equal(pano, pano_ref)
    return keep_ref, pano_ref


def random_frame(seed, H, W, k):
    """fcn_score [1,19,H/4,W/4], boxes clipped to the frame (as MaskROI clips them), scores, mask logits, classes"""
    g = torch.Generator().manual_seed(seed)
    fcn_score = torch.randn(1, 19, H // 4, W // 4, generator=g) * 2
    xy = torch.rand(k, 2, generator=g) * torch.tensor([W * 1.0, H * 1.0])
    wh = torch.exp(torch.rand(k, 2, generator=g) * 3.5) + 1
    boxes = torch.cat([xy - wh / 2, xy + wh / 2], 1)
    boxes[:, 0::2].clamp_(0, W - 1)
    boxes[:, 1::2].clamp_(0, H - 1)
    prob = torch.rand(k, generator=g) * 0.39 + 0.6
    mlog = torch.randn(k, MS, MS, generator=g) * 2 + 0.3
    cls_idx = torch.randint(1, 9, (k,), generator=g)
    cls_idx[:k // 4] = 3                                       # same-class overlaps
    return fcn_score, boxes, prob, mlog, cls_idx


PATHS = pytest.mark.parametrize("num_things", [8, 9], ids=["cluster", "per_position"])


# ---------------------------------------------------------------------------------------------------- MaskRemoval
@PATHS
def test_empty_keep_fuses_detection_zero(cuda, num_things):
    """Every resized mask is empty, so MaskRemoval keeps nothing and the reference falls back to keep_inds = [0]:
    detection 0 in the original order (not the best-scoring one) with its SegTerm channel and zero mask energy."""
    H, W, k = 96, 160, 6
    fcn_score, boxes, prob, mlog, cls_idx = random_frame(21, H, W, k)
    boxes[0] = torch.tensor([30.6, 20.2, 101.3, 77.9])
    mlog = -(mlog.abs() + 0.1)                                  # strictly negative: cv2.resize keeps it so
    prob[0] = 0.61                                              # detection 0 is last in score order
    prob[1:] = torch.linspace(0.95, 0.7, k - 1)
    fcn_score[0, :NS, :, :(W // 4) // 2] -= 4.0                 # stuff logits below 0 on the left half
    keep_ref, pano_ref = check_frame(fcn_score, boxes, prob, mlog, cls_idx, num_things)
    assert list(keep_ref) == [0] and stable_order(prob)[0] != 0
    assert int((pano_ref == NS).sum()) > 0                      # the fallback channel wins somewhere


def fraction_chain(seed):
    """Boxes of exactly 28 x 28 pixels (x2 - x1 + 1 == 28): cv2.resize is the identity there, so each mask is the
    pixel set written here.  Returns the frame and the detections MaskRemoval must keep, in score order."""
    rng = np.random.RandomState(seed)
    H, W = 64, 96
    pool = list(rng.permutation(MS * MS))          # mask pixels no detection of the chain has used yet
    occupied = []                                  # pixels of the kept class-3 masks
    # (positive pixels already occupied, fresh positive pixels, zero-valued pixels on occupied ones, kept)
    chain = [(0, 100, 0, True),
             (3, 7, 0, True),                      # 3/10 == 0.3: not above the threshold
             (10, 23, 0, False),                   # 10/33 > 0.3
             (6, 14, 0, True),                     # 6/20
             (3, 7, 5, True),                      # logits == 0 are no mask pixels: 3/10, not 8/15
             (31, 69, 0, False),                   # 0.31
             (0, 0, 12, False),                    # only zero logits: mask_sum == 0
             (30, 70, 0, True)]                    # 30/100 == 0.3
    masks, classes, boxes, expect = [], [], [], []
    for n_occ, n_new, n_zero, keep in chain:
        m = -rng.uniform(0.5, 3.0, MS * MS)
        on = list(rng.choice(occupied, n_occ, replace=False)) if n_occ else []
        on += [pool.pop() for _ in range(n_new)]
        m[on] = rng.uniform(0.5, 3.0, len(on))
        if n_zero:
            m[rng.choice(sorted(set(occupied) - set(on)), n_zero, replace=False)] = 0.0
        if keep:
            occupied = sorted(set(occupied) | set(on))
        masks.append(m); classes.append(3); boxes.append([8.0, 8.0, 35.0, 35.0]); expect.append(keep)
    # class 5 on the same pixels: the occupancy is per class, so its first mask is kept whatever class 3 holds
    first = masks[0].copy()
    for keep in (True, False):                     # the second one is fully covered by the first
        masks.append(first.copy()); classes.append(5); boxes.append([8.7, 8.2, 35.2, 35.9]); expect.append(keep)
    n = len(masks)
    # scores in chain order, detection indices shuffled so that index order and score order differ
    det = rng.permutation(n)
    prob = torch.zeros(n)
    prob[det] = torch.linspace(0.99, 0.7, n)
    mlog = torch.zeros(n, MS, MS)
    mlog[det] = torch.from_numpy(np.stack(masks).reshape(n, MS, MS)).float()
    bx = torch.zeros(n, 4)
    bx[det] = torch.tensor(boxes)
    cls_idx = torch.zeros(n, dtype=torch.long)
    cls_idx[det] = torch.tensor(classes)
    fcn_score = torch.randn(1, 19, H // 4, W // 4, generator=torch.Generator().manual_seed(seed)) * 2
    return fcn_score, bx, prob, mlog, cls_idx, det[np.array(expect)]


@PATHS
def test_fraction_rule_on_exact_masks(cuda, num_things):
    fcn_score, boxes, prob, mlog, cls_idx, expect = fraction_chain(22)
    keep_ref, _ = check_frame(fcn_score, boxes, prob, mlog, cls_idx, num_things)
    assert np.array_equal(keep_ref, expect)                     # the chain is what it claims to be


def geometry_frame(seed):
    H, W, k = 96, 160, 40
    fcn_score, boxes, prob, mlog, cls_idx = random_frame(seed, H, W, k)
    special = [
        [30.2, 10.5, 30.9, 40.3],                  # 1 px wide
        [50.0, 60.1, 90.2, 60.7],                  # 1 px high
        [5.3, 7.2, 5.9, 7.8],                      # 1 x 1
        [100.5, 20.25, 117.75, 33.5],              # 18 x 14: cv2 shrinks the mask
        [60.0, 70.0, 73.0, 83.0],                  # 14 x 14: an exact 2x shrink
        [2.6, 3.4, 150.8, 90.9],                   # 149 x 88: cv2 enlarges it
        [10.999, 40.001, 47.999, 79.5],            # corners astype(int32) truncates
        [120.3, 70.6, W - 1.0, H - 1.0],           # reaches x2 = W-1 and y2 = H-1
        [140.5, 80.25, W + 12.7, H + 5.5],         # runs past the frame
        [20.0, 30.0, 40.5, 22.5 + 30.0],           # SegTerm x2, y2 at .5: np.round to even (40, 52)
        [44.0, 5.0, 61.5, 23.5],                   # ... and to the odd side (62, 24)
        [70.25, 40.75, 89.5, 41.5],                # .5 ends on a 1-2 px tall box
    ]
    n = len(special)
    boxes[:n] = torch.tensor(special)
    # the special boxes come first in score order, and boxes of one class among them do not overlap, so all of them
    # are kept and their edges decide labels; raised thing logits let instances win inside their boxes
    cls_idx[:n] = torch.tensor([1, 2, 1, 1, 2, 8, 3, 4, 5, 6, 7, 7])
    prob[:n] = torch.linspace(0.999, 0.99, n)
    prob[n:] *= 0.98
    mlog[:3] += 2.5                                            # the 1-px boxes get a positive mask pixel
    fcn_score[0, NS:NS + 8] += 1.5
    return fcn_score, boxes, prob, mlog, cls_idx


@PATHS
def test_resize_geometry(cuda, num_things):
    check_frame(*geometry_frame(23), num_things=num_things)


def test_mask_removal_paths_agree(cuda):
    """The cluster path (num_things 8) and the per-position path (num_things 9) on the same dense frame"""
    H, W, k = 96, 160, 120
    fcn_score, boxes, prob, mlog, cls_idx = random_frame(24, H, W, k)
    keep_ref, _, _ = oracle(boxes, prob, mlog, cls_idx, fcn_score, H, W)
    got = [kept(*gpu_mask_removal(boxes, stable_order(prob), mlog, cls_idx, H, W, nt)) for nt in (8, 9)]
    assert np.array_equal(got[0], got[1])
    assert np.array_equal(got[0], keep_ref)
    assert 0 < len(keep_ref) < k                                 # both decisions occur


def test_per_position_path_beyond_128(cuda):
    """k = 160 > 128 takes the per-position path.  The fusion holds at most 128 instances, so only the keep list
    is compared."""
    from oracle.model import mask_removal
    H, W, k = 96, 160, 160
    _, boxes, prob, mlog, cls_idx = random_frame(25, H, W, k)
    keep_ref, _ = mask_removal(boxes, prob, mlog[:, None], cls_idx, (H, W))
    keep_sorted, nkeep = gpu_mask_removal(boxes, stable_order(prob), mlog, cls_idx, H, W, 8)
    assert np.array_equal(kept(keep_sorted, nkeep), keep_ref.numpy())
    assert 0 < len(keep_ref) < k


@PATHS
def test_device_count_below_k(cuda, num_things):
    """k_dev < k: only the first k_dev detections exist.  The order array still lists the other ones after them, so
    a kernel that read past k_dev would keep some of them."""
    H, W, k, kd = 96, 160, 40, 23
    fcn_score, boxes, prob, mlog, cls_idx = random_frame(26, H, W, k)
    keep_ref, pano_ref, sem_ref = oracle(boxes[:kd], prob[:kd], mlog[:kd], cls_idx[:kd], fcn_score, H, W)
    order = np.concatenate([stable_order(prob[:kd]), kd + stable_order(prob[kd:])])
    keep_sorted, nkeep = gpu_mask_removal(boxes, order, mlog, cls_idx, H, W, num_things, k_dev=kd)
    assert np.array_equal(kept(keep_sorted, nkeep), keep_ref)
    pano, sem = gpu_fuse(fcn_score, boxes, cls_idx, mlog, keep_sorted, nkeep, H, W)
    assert torch.equal(sem, sem_ref) and torch.equal(pano, pano_ref)


# ---------------------------------------------------------------------------------------------------- fusion
def test_fusion_bf16_score(cuda):
    H, W = 96, 160
    fcn_score, boxes, prob, mlog, cls_idx = random_frame(27, H, W, 40)
    fcn_score = fcn_score.bfloat16().float()                    # scores a bf16 tensor holds exactly
    check_frame(fcn_score, boxes, prob, mlog, cls_idx, score_dtype=torch.bfloat16)


def test_fusion_partial_tiles(cuda):
    """100 x 172: neither side is a multiple of the 32 x 8 tile"""
    check_frame(*random_frame(28, 100, 172, 40))


def test_fusion_128_instances(cuda):
    """128 kept instances.  Sorted position j spans x >= 4j, so the first instance that misses the 32-px tile column t
    is 8t + 8: the tiles' candidate lists end in all four warps of the instance scan, and the last column lists
    every instance."""
    H, W, k = 40, 512, 128
    rng = np.random.RandomState(29)
    j = np.arange(k)
    boxes = torch.tensor(np.stack([4.0 * j + 0.5, np.full(k, 0.3), np.full(k, W - 1.0), np.full(k, H - 1.0)], 1)).float()
    # position j has class j % 8 + 1 and a mask that is positive over its ~20 leftmost pixels: the masks of one
    # class start 32 px apart and never overlap, so MaskRemoval keeps all 128
    mlog = -rng.uniform(0.5, 2.0, (k, MS, MS))
    for i in range(k):
        n_on = int(np.clip(round(20 * MS / (W - 4 * i)), 1, MS))
        mlog[i, :, :n_on] = rng.uniform(0.5, 2.0, (MS, n_on))
    det = rng.permutation(k)                                     # detection index of sorted position j
    inv = np.argsort(det)
    boxes, mlog = boxes[inv], torch.from_numpy(mlog[inv]).float()
    cls_idx = torch.from_numpy(j % 8 + 1)[inv]
    prob = torch.linspace(0.99, 0.7, k)[inv]
    fcn_score = torch.randn(1, 19, H // 4, W // 4, generator=torch.Generator().manual_seed(29)) * 2
    first_miss = [next((i for i in range(k) if 4 * i >= 32 * t + 32), None) for t in range(W // 32)]
    assert {m // 32 for m in first_miss if m is not None} == {0, 1, 2, 3} and first_miss[-1] is None
    keep_ref, _ = check_frame(fcn_score, boxes, prob, mlog, cls_idx)
    assert np.array_equal(keep_ref, det)


def test_fusion_dummy(cuda):
    """dummy = 1 (MaskROI found nothing): one all-zero instance channel; keep_sorted and nkeep are not read"""
    H, W = 96, 160
    fcn_score = random_frame(30, H, W, 1)[0]
    fcn_score[0, :NS, :H // 8] -= 4.0                            # stuff logits below 0 on the top half
    keep_ref, pano_ref, sem_ref = oracle(torch.zeros(1, 4), torch.ones(1), torch.zeros(1, MS, MS),
                                         torch.zeros(1, dtype=torch.long), fcn_score, H, W)
    assert list(keep_ref) == [0] and int((pano_ref == NS).sum()) > 0
    keep_sorted = torch.arange(CAP, dtype=torch.int32, device="cuda")
    nkeep = torch.full((1,), 5, dtype=torch.int32, device="cuda")
    pano, sem = gpu_fuse(fcn_score, torch.rand(CAP, 4) * 50, torch.ones(CAP, dtype=torch.long), torch.randn(CAP, MS, MS),
                         keep_sorted, nkeep, H, W, dummy=True)
    assert torch.equal(sem, sem_ref) and torch.equal(pano, pano_ref)


# ---------------------------------------------------------------------------------------------------- MaskROI tail
def maskroi_case(case):
    """120 RoIs, 40-px boxes on a 32-px grid (neighbours overlap with IoU < 0.5, so NMS keeps every survivor) and
    zero box deltas, so that the decoded boxes are the RoIs on both sides bit for bit.
    none: every foreground probability is below the 0.6 score threshold.
    ties: 95 distinct scores, then 10 RoIs with identical rows (equal probabilities) holding the 96th to 105th
    places, then 15 lower ones: the 100th best score is tied, and numpy's >= keeps k = 105 > max_det = 100."""
    rng = np.random.RandomState({"none": 31, "ties": 32}[case])
    H, W, n, nc = 320, 384, 120, 9
    gy, gx = np.divmod(np.arange(n), 12)
    x1 = gx * 32.0 + rng.choice([0.0, 0.25, 0.5, 0.75], n)
    y1 = gy * 32.0 + rng.choice([0.0, 0.25, 0.5, 0.75], n)
    rois = np.stack([np.zeros(n), x1, y1, np.minimum(x1 + 39.5, W - 1), np.minimum(y1 + 39.5, H - 1)], 1)
    cls_score = np.zeros((n, nc))
    if case == "none":
        cls_score[:, 0] = 3.0
        cls_score[:, 1:] = rng.uniform(-1.0, 1.0, (n, nc - 1))
    else:
        slots = rng.permutation(n)
        logit = np.empty(n)
        logit[slots[:95]] = rng.permutation(np.linspace(7.0, 3.6, 95))
        logit[slots[95:105]] = 3.4
        logit[slots[105:]] = rng.permutation(np.linspace(3.2, 2.8, 15))
        cls = rng.randint(1, nc, n)
        cls[slots[95:105]] = 2                                  # identical rows: equal probabilities on both sides
        cls_score[np.arange(n), cls] = logit
    g = torch.Generator().manual_seed(33)
    mask_pred = torch.randn(CAP, nc, MS, MS, generator=g) * 2 + 0.3
    fcn_score = torch.randn(1, 19, H // 4, W // 4, generator=g) * 2
    return (torch.from_numpy(rois).float(), torch.from_numpy(cls_score).float(), torch.zeros(n, 4 * nc), mask_pred,
            fcn_score, H, W)


@pytest.mark.parametrize("mask_dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("case", ["none", "ties"])
def test_maskroi_tail_to_fusion(cuda, case, mask_dtype):
    """vps_maskroi_finalize -> vps_det_split -> vps_select_class -> sort -> MaskRemoval -> fusion, as the detector
    chains them, against the oracle's tail (mask_roi, gather, mask_removal, seg_term, softmax-max)."""
    from oracle.model import mask_roi
    from vps_b200 import ops
    rois, cls_score, bbox_pred, mask_pred, fcn_score, H, W = maskroi_case(case)
    mask_pred = mask_pred.to(mask_dtype).float()                # values the chosen dtype holds exactly
    n, nc = cls_score.shape
    # ---- oracle
    o_prob, o_rois, o_cls = mask_roi(rois, bbox_pred, F.softmax(cls_score, 1), np.array([[H * 1.0, W * 1.0, 1.0]]))
    ko = o_rois.shape[0]
    o_mask = mask_pred[:ko].gather(1, o_cls.view(-1, 1, 1, 1).expand(-1, -1, MS, MS))[:, 0]
    keep_ref, pano_ref, sem_ref = oracle(o_rois[:, 1:], o_prob, o_mask, o_cls, fcn_score, H, W)
    # ---- device chain (detector._mask_roi + the tail of simple_test)
    dev, m = "cuda", n * (nc - 1)
    y = torch.cat([cls_score, bbox_pred], 1).cuda()
    cand, ccls = torch.empty(m, 5, device=dev), torch.empty(m, dtype=torch.int32, device=dev)
    cprob, ncand = torch.empty(m, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
    ops.maskroi_candidates(rois.cuda(), y[:, :nc], y[:, nc:], n, nc, 0.6, H, W, cand, ccls, cprob, ncand)
    psort, slot = torch.empty(m, device=dev), torch.empty(m, dtype=torch.int32, device=dev)
    ops.sort_desc(cprob, psort, slot, m, torch.empty(ops.sort_ws_bytes(m), dtype=torch.uint8, device=dev))
    csort = torch.empty(m, 5, device=dev)
    ops.gather_rows(cand, slot, m, 5, csort)
    keep, nk = torch.empty(m, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
    ops.nms(csort, m, 0.5, keep, nk, torch.empty(ops.nms_ws_bytes(m), dtype=torch.uint8, device=dev), n_dev=ncand)
    det_rois = torch.empty(CAP, 5, device=dev)
    cidx, cp = torch.empty(CAP, dtype=torch.int32, device=dev), torch.empty(CAP, device=dev)
    kout = torch.zeros(2, dtype=torch.int32, device=dev)
    ops.maskroi_finalize(csort, slot, ccls, keep, nk, 100, CAP, det_rois, cidx, cp, kout)
    k, dummy = kout.tolist()
    if case == "none":
        assert (k, dummy) == (1, 1)
    else:
        assert (k, dummy) == (105, 0)
    assert k == ko
    boxes_c, labels = torch.empty(CAP, 4, device=dev), torch.empty(CAP, dtype=torch.int32, device=dev)
    ops.det_split(det_rois, cidx, CAP, boxes_c, labels)
    assert torch.equal(cidx[:k].cpu().long(), o_cls) and torch.equal(labels[:k].cpu().long(), o_cls - 1)
    assert torch.equal(boxes_c[:k].cpu(), o_rois[:, 1:])
    assert float((cp[:k].cpu() - o_prob).abs().max()) <= 1e-5
    mask_logit = torch.empty(k, MS, MS, device=dev)
    ops.select_class(to_nhwc(mask_pred, mask_dtype), cidx, k, mask_logit)
    assert torch.equal(mask_logit.cpu(), o_mask)
    order = torch.empty(k, dtype=torch.int32, device=dev)
    ops.sort_desc(cp, torch.empty(k, device=dev), order, k, torch.empty(ops.sort_ws_bytes(k), dtype=torch.uint8, device=dev))
    keep_sorted = torch.zeros(CAP, dtype=torch.int32, device=dev)
    nkeep = torch.zeros(1, dtype=torch.int32, device=dev)
    if not dummy:
        ops.mask_removal(boxes_c, order, k, mask_logit, MS, cidx, H, W, 0.3, torch.empty(8, H, W, dtype=torch.uint8, device=dev),
                         8, torch.empty(2 * k, dtype=torch.int32, device=dev), torch.empty(k, dtype=torch.int32, device=dev),
                         keep_sorted, nkeep)
    got = kept(keep_sorted, nkeep)
    assert np.array_equal(got if got.size else np.zeros(1, np.int64), keep_ref)
    pano, sem = gpu_fuse(fcn_score, boxes_c.cpu(), cidx.cpu(), mask_logit.cpu(), keep_sorted, nkeep, H, W, dummy=bool(dummy))
    assert torch.equal(sem, sem_ref) and torch.equal(pano, pano_ref)
