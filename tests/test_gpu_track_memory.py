"""GPU: the tracker memory past the size of one allocation -- growable buffers, cached track embeddings and the tiled
match kernels.

1. A long stream (memory past 4096 tracks) through PanopticFuseTrack._track against the oracle's torch.cat-grown memory.
2. Cached embeddings and memory growth change no bits: the same stream against a loop that re-embeds the whole memory
   every frame into fixed buffers, also across a weight change mid-stream.
3. Embedding a row gives the same bits in any batch, for every precision (what makes the cache exact).
4. The dots keep the one-warp-per-pair fmaf order bit for bit, and the match / update kernels take memories whose size
   no longer fits a grid dimension."""
import ctypes
import ctypes.util

import numpy as np
import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu

COEFF = [1.0, 2.0, 10.0]


@pytest.fixture
def tc32_flag():
    from vps_b200 import ops
    saved = ops.F32_TC[0]
    yield ops.F32_TC
    ops.F32_TC[0] = saved


class _NoWeights(nn.Module):
    def prepare(self, force=False):
        return self


def _tracker(track_head, precision):
    """A PanopticFuseTrack that holds only a track head: _track, prepare and reset_tracker are the product's."""
    from vps_b200.detector import PanopticFuseTrack
    det = PanopticFuseTrack.__new__(PanopticFuseTrack)
    nn.Module.__init__(det)
    for name in ("backbone", "neck", "extra_neck", "panopticFPN", "rpn_head", "bbox_head", "mask_head", "flownet2"):
        setattr(det, name, _NoWeights())
    det.track_head = track_head
    det.precision = precision
    det._graphs, det._pf_queue, det._tail_done = {}, [], [None, None]
    det.reset_tracker()
    return det


def _track_head(in_channels, roi_feat_size, fc_out, seed):
    from vps_b200.modules import TrackHead
    torch.manual_seed(seed)
    return TrackHead(in_channels=in_channels, roi_feat_size=roi_feat_size, fc_out_channels=fc_out,
                     match_coeff=COEFF).cuda()


class Stream:
    """Frames of up to 100 detections against a memory (features, boxes, labels) the caller passes in: re-detections of
    remembered tracks (stored features + small noise, jittered box, same label), duplicates of some of them that score
    lower and come first (the "undo" branch of the id loop), and new objects with labels no track has (so a new object
    never matches a remembered one, and a re-detection only matches its own track)."""

    def __init__(self, feat_shape, seed, k=100, n_redet=10, n_dup=3, scale=0.5):
        self.g = torch.Generator().manual_seed(seed)
        self.feat_shape, self.k, self.n_redet, self.n_dup, self.scale = feat_shape, k, n_redet, n_dup, scale
        self.next_label = 0

    def _boxes(self, n):
        xy = torch.rand(n, 2, generator=self.g) * 1000
        wh = torch.rand(n, 2, generator=self.g) * 60 + 20
        return torch.cat([xy, xy + wh], 1)

    def _new_labels(self, n):
        lab = torch.arange(self.next_label, self.next_label + n, dtype=torch.int32)
        self.next_label += n
        return lab

    def frame(self, mem_feats, mem_boxes, mem_labels):
        g, m = self.g, mem_boxes.shape[0]
        feats, boxes, labels, probs = [], [], [], []
        if m > 0:
            rows = torch.randperm(m, generator=g)[:self.n_redet]
            at = rows.to(mem_feats.device)
            base = mem_feats[at].float().cpu()
            rboxes, rlabels = mem_boxes[at].cpu(), mem_labels[at].cpu()
            jit = lambda b, s: b + (torch.rand(b.shape, generator=g) - 0.5) * s
            for d in range(min(self.n_dup, rows.numel())):             # weaker duplicates first
                feats.append(base[d:d + 1] + 0.2 * self.scale * torch.randn(base[d:d + 1].shape, generator=g))
                boxes.append(jit(rboxes[d:d + 1], 16.0))
                labels.append(rlabels[d:d + 1])
                probs.append(torch.full((1,), 0.65))
            feats.append(base + 0.02 * self.scale * torch.randn(base.shape, generator=g))
            boxes.append(jit(rboxes, 2.0))
            labels.append(rlabels)
            probs.append(torch.rand(rows.numel(), generator=g) * 0.05 + 0.9)
        n_new = self.k - sum(b.shape[0] for b in boxes)
        feats.append(torch.randn((n_new,) + self.feat_shape, generator=g) * self.scale)
        boxes.append(self._boxes(n_new))
        labels.append(self._new_labels(n_new))
        probs.append(torch.rand(n_new, generator=g) * 0.3 + 0.65)
        perm = torch.randperm(self.k, generator=g)
        keep_first = torch.arange(min(self.n_dup, m))                   # duplicates stay ahead of their originals
        order = torch.cat([keep_first, perm[perm >= keep_first.numel()]])
        return tuple(torch.cat(x)[order] for x in (feats, boxes, labels, probs))


def _product_frame(det, feats, boxes, labels, probs, is_first, dtype):
    k = boxes.shape[0]
    taps = {}
    ids = det._track(feats.to("cuda", dtype), boxes.cuda(), labels.cuda(), probs.cuda(), k, is_first, taps)
    return ids.cpu().numpy(), taps.get("comp_scores")


@pytest.mark.parametrize("precision", ["tc32", "fp32"])
def test_long_stream_vs_oracle(cuda, tc32_flag, precision):
    """60 frames of 100 detections: the memory passes 4096 tracks and its buffers grow past 4096 slots; ids, comp scores
    and the memory itself follow the oracle's torch.cat-grown tensors every frame."""
    from oracle.model import PanopticFuseTrack as Oracle, TrackHead as OTrackHead
    tc32_flag[0] = precision == "tc32"
    th = _track_head(16, 1, 64, seed=3)
    det = _tracker(th, precision)
    oth = OTrackHead(cin=16, fc=64, match_coeff=tuple(COEFF))
    oth.fcs = nn.ModuleList([nn.Linear(16, 64), nn.Linear(64, 64)])
    oth.fcs.load_state_dict({k_: v.detach().cpu() for k_, v in th.fcs.state_dict().items()})
    o = Oracle.__new__(Oracle)
    nn.Module.__init__(o)
    o.track_head = oth
    o.prev_bboxes = o.prev_roi_feats = o.prev_det_labels = None
    st = Stream((16, 1, 1), seed=5)
    caps = set()
    for f in range(60):
        if o.prev_bboxes is None:
            mem = (torch.zeros(0, 16, 1, 1), torch.zeros(0, 4), torch.zeros(0, dtype=torch.int32))
        else:
            mem = (o.prev_roi_feats, o.prev_bboxes, o.prev_det_labels.int())
        feats, boxes, labels, probs = st.frame(*mem)
        taps = {}
        with torch.no_grad():
            ids_ref = o.track(boxes, labels.long(), feats, probs, f == 0, taps)
        # the product keeps RoI features NHWC: [k, 1, 1, 16]
        ids, comp = _product_frame(det, feats.permute(0, 2, 3, 1), boxes, labels, probs, f == 0, torch.float32)
        assert np.array_equal(ids, np.asarray(ids_ref)), f
        if f > 0:
            assert float((comp.cpu() - taps["comp_scores"]).abs().max()) <= 1e-4, f
        m = det.prev_n
        assert m == o.prev_roi_feats.shape[0], f
        assert torch.equal(det.prev_roi_feats[:m].cpu().permute(0, 3, 1, 2), o.prev_roi_feats), f
        assert torch.equal(det.prev_bboxes[:m].cpu(), o.prev_bboxes), f
        assert torch.equal(det.prev_det_labels[:m].cpu().long(), o.prev_det_labels), f
        caps.add(det.prev_bboxes.shape[0])
    assert det.prev_n > 4096 and max(caps) >= 8192, (det.prev_n, sorted(caps))


def _uncached_loop_frame(ref, th, feats, boxes, labels, probs, is_first, cap):
    """One frame of the tracker without the embedding cache and without growth: every memory row is re-embedded, the
    buffers have `cap` slots from the start."""
    from vps_b200 import ops
    k = boxes.shape[0]
    if ref.get("feats") is None or is_first:
        ref.update(feats=torch.zeros((cap,) + tuple(feats.shape[1:]), dtype=feats.dtype, device="cuda"),
                   boxes=torch.zeros(cap, 4, device="cuda"), labels=torch.zeros(cap, dtype=torch.int32, device="cuda"), m=0)
    m = ref["m"]
    feat_len = feats[0].numel()
    ids = torch.empty(k, dtype=torch.int32, device="cuda")
    new_m = torch.zeros(1, dtype=torch.int32, device="cuda")
    if m == 0:
        mem_src = torch.arange(k, dtype=torch.int32, device="cuda")
        ids.copy_(mem_src)
        new_m.fill_(k)
        comp = None
    else:
        emb = th.embed(feats)
        ref_emb = th.embed(ref["feats"][:m])
        mids = torch.empty(k, dtype=torch.int32, device="cuda")
        comp = torch.empty(k, m + 1, device="cuda")
        mem_src = torch.empty(cap, dtype=torch.int32, device="cuda")
        ws = torch.empty((k * m + k + 2 * cap) * 4, dtype=torch.uint8, device="cuda")
        ops.track_assign(emb, ref_emb, k, m, emb.shape[1], boxes, ref["boxes"], labels, ref["labels"], probs, COEFF, cap,
                         ids, mids, comp, mem_src, new_m, ws)
    ops.track_update(ref["feats"], feats, feat_len, ref["boxes"], boxes, ref["labels"], labels, mem_src, m, cap, new_m)
    ref["m"] = int(new_m.item())
    return ids.cpu().numpy(), comp


@pytest.mark.parametrize("precision", ["tc32", "bf16", "fp32"])
def test_cache_and_growth_change_no_bits(cuda, tc32_flag, precision):
    """The full-size track head, 50 frames of k = 100 (memory past 4096): comp, ids, memory size and contents identical
    bit for bit to the uncached fixed-capacity loop; mid-stream new weights + prepare(force=True) re-embed the cache."""
    tc32_flag[0] = precision == "tc32"
    dtype = torch.bfloat16 if precision == "bf16" else torch.float32
    th = _track_head(256, 7, 1024, seed=7)
    det = _tracker(th, precision)
    # small features: the embeddings of unrelated objects stay far below the label term, so new objects open tracks
    st = Stream((7, 7, 256), seed=9, n_redet=4, n_dup=1, scale=0.1)
    ref = {}
    for f in range(50):
        m = det.prev_n
        mem = (det.prev_roi_feats[:m], det.prev_bboxes[:m], det.prev_det_labels[:m]) if m else \
            (torch.zeros((0, 7, 7, 256)), torch.zeros(0, 4), torch.zeros(0, dtype=torch.int32))
        feats, boxes, labels, probs = st.frame(*mem)
        if f == 30:                                         # new weights mid-clip
            with torch.no_grad():
                for p in th.parameters():
                    p.mul_(1.25)
            det.prepare(force=True)
        fd = feats.to("cuda", dtype)
        ids, comp = _product_frame(det, fd, boxes, labels, probs, f == 0, dtype)
        ids_ref, comp_ref = _uncached_loop_frame(ref, th, fd, boxes.cuda(), labels.cuda(), probs.cuda(), f == 0, 8192)
        assert np.array_equal(ids, ids_ref), f
        if comp_ref is not None:
            assert torch.equal(comp, comp_ref), f
        m = det.prev_n
        assert m == ref["m"], f
        assert torch.equal(det.prev_roi_feats[:m], ref["feats"][:m]), f
        assert torch.equal(det.prev_bboxes[:m], ref["boxes"][:m]) and torch.equal(det.prev_det_labels[:m], ref["labels"][:m])
        if f == 30:
            assert torch.equal(det.prev_emb[:m], th.embed(det.prev_roi_feats[:m])), "cache did not follow the new weights"
    assert det.prev_n > 4096, det.prev_n


@pytest.mark.parametrize("precision", ["tc32", "bf16", "fp32"])
def test_embedding_rows_are_batch_invariant(cuda, tc32_flag, precision):
    tc32_flag[0] = precision == "tc32"
    dtype = torch.bfloat16 if precision == "bf16" else torch.float32
    th = _track_head(256, 7, 1024, seed=13)
    g = torch.Generator().manual_seed(17)
    x = (torch.randn(5000, 7, 7, 256, generator=g) * 0.5).to("cuda", dtype)
    for M in (1, 7, 100, 128, 129, 1000, 5000):
        full = th.embed(x[:M])
        rows = sorted({0, M // 3, M // 2, M - 1})
        for r in rows:
            assert torch.equal(full[r:r + 1], th.embed(x[r:r + 1])), (M, r)
        idx = torch.tensor(rows, device="cuda")
        assert torch.equal(full[idx], th.embed(x[idx])), M


def _fmaf():
    libm = ctypes.CDLL(ctypes.util.find_library("m"))
    f = libm.fmaf
    f.argtypes, f.restype = [ctypes.c_float] * 3, ctypes.c_float
    return f


def _warp_dot(fmaf, a, b):
    """one warp per pair: lane l chains fmaf over c = l (mod 32) in increasing c, then lane 0 of the xor butterfly"""
    s = [0.0] * 32
    for c in range(a.shape[0]):
        s[c % 32] = fmaf(float(a[c]), float(b[c]), s[c % 32])
    s = np.array(s, dtype=np.float32)
    o = 16
    while o:
        s = (s[:o] + s[o:2 * o]).astype(np.float32)
        o //= 2
    return s[0]


def _assign(emb, ref_emb, boxes, ref_boxes, labels, ref_labels, probs, cap):
    from vps_b200 import ops
    k, m, dim = emb.shape[0], ref_emb.shape[0], emb.shape[1]
    ids = torch.empty(k, dtype=torch.int32, device="cuda")
    mids = torch.empty(k, dtype=torch.int32, device="cuda")
    comp = torch.empty(k, m + 1, device="cuda")
    mem_src = torch.empty(cap, dtype=torch.int32, device="cuda")
    new_m = torch.zeros(1, dtype=torch.int32, device="cuda")
    ws = torch.empty((k * m + k + 2 * cap) * 4, dtype=torch.uint8, device="cuda")
    ops.track_assign(emb, ref_emb, k, m, dim, boxes, ref_boxes, labels, ref_labels, probs, COEFF, cap, ids, mids, comp,
                     mem_src, new_m, ws)
    torch.cuda.synchronize()
    return ws[:k * m * 4].view(torch.float32).view(k, m), ids, mem_src, new_m


@pytest.mark.parametrize("k,m,dim", [(5, 37, 1024), (19, 33, 200)])
def test_dot_order_bitwise(cuda, k, m, dim):
    """dots in ws equal a CPU restatement of the one-warp-per-pair order with a correctly rounded fmaf (libm)"""
    g = torch.Generator().manual_seed(k * 1000 + m)
    emb, ref_emb = torch.randn(k, dim, generator=g), torch.randn(m, dim, generator=g)
    boxes, ref_boxes = torch.rand(k, 4, generator=g) * 100, torch.rand(m, 4, generator=g) * 100
    boxes[:, 2:] += 100
    ref_boxes[:, 2:] += 100
    dots, _, _, _ = _assign(emb.cuda(), ref_emb.cuda(), boxes.cuda(), ref_boxes.cuda(),
                            torch.zeros(k, dtype=torch.int32, device="cuda"), torch.ones(m, dtype=torch.int32, device="cuda"),
                            torch.full((k,), 0.9, device="cuda"), 64)
    fmaf = _fmaf()
    want = np.array([[_warp_dot(fmaf, emb[i].numpy(), ref_emb[j].numpy()) for j in range(m)] for i in range(k)],
                    dtype=np.float32)
    got = dots.cpu().numpy()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.abs(got - want).max()


def test_match_and_update_past_grid_dimension(cuda):
    """m = 70000 tracks, cap = 2^17: integer-valued embeddings make every dot exact (== the int64 product), and the
    update writes every touched slot, including those past 65535 (the most blocks one grid dimension y can hold)."""
    from vps_b200 import ops
    k, m, dim, feat_len, cap = 6, 70000, 8, 4, 1 << 17
    g = torch.Generator().manual_seed(23)
    # dots of a re-detection with its own track are 64, with any other track |dot| <= 8; the new detection's are <= 8,
    # below the label term (10) a match to a track of another label would need
    ref_emb = torch.randint(-1, 2, (m, dim), generator=g)
    emb = torch.zeros(k, dim, dtype=torch.int64)
    emb[torch.arange(5), torch.arange(5)] = 8
    emb[5] = torch.randint(0, 2, (dim,), generator=g) * 2 - 1
    targets = torch.tensor([65535, 65536, 69999, 1000, 42])         # detection i < 5 re-detects track targets[i]
    ref_emb[targets] = emb[:5]
    ref_boxes = torch.rand(m, 4, generator=g) * 500
    ref_boxes[:, 2:] += 500
    ref_labels = torch.arange(m, dtype=torch.int32)
    boxes = torch.cat([ref_boxes[targets], torch.tensor([[1.0, 1.0, 30.0, 30.0]])])
    labels = torch.cat([ref_labels[targets], torch.tensor([-5], dtype=torch.int32)])   # the last one is a new track
    probs = torch.full((k,), 0.9)
    dots, ids, mem_src, new_m = _assign(emb.float().cuda(), ref_emb.float().cuda(), boxes.cuda(), ref_boxes.cuda(),
                                        labels.cuda(), ref_labels.cuda(), probs.cuda(), cap)
    assert torch.equal(dots.cpu().double(), (emb[:, None, :] * ref_emb[None]).sum(-1).double())
    assert ids.cpu().tolist() == targets.tolist() + [m]
    assert int(new_m.item()) == m + 1
    feats = torch.zeros(cap, feat_len, device="cuda")
    mem_boxes = torch.zeros(cap, 4, device="cuda")
    mem_boxes[:m] = ref_boxes.cuda()
    mem_labels = torch.full((cap,), -1, dtype=torch.int32, device="cuda")
    mem_labels[:m] = ref_labels.cuda()
    det_feats = (torch.arange(k * feat_len, dtype=torch.float32).view(k, feat_len) + 1).cuda()
    det_boxes = boxes.cuda() + 0.5
    ops.track_update(feats, det_feats, feat_len, mem_boxes, det_boxes, mem_labels, labels.cuda(), mem_src, m, cap, new_m)
    slots = targets.tolist() + [m]
    want = torch.zeros(cap, feat_len)
    want[slots] = det_feats.cpu()
    assert torch.equal(feats.cpu(), want)
    assert torch.equal(mem_boxes[slots].cpu(), det_boxes.cpu())
    untouched = torch.ones(m, dtype=torch.bool)
    untouched[targets] = False
    assert torch.equal(mem_boxes[:m][untouched.cuda()].cpu(), ref_boxes[untouched])
    assert int(mem_labels[m]) == -5 and torch.equal(mem_labels[:m].cpu(), ref_labels)     # labels only for new slots
    # the same scatter on a table without boxes / labels (the cached embeddings)
    table = torch.zeros(cap, feat_len, device="cuda")
    ops.track_update(table, det_feats, feat_len, None, None, None, None, mem_src, m, cap, new_m)
    assert torch.equal(table.cpu(), want)
