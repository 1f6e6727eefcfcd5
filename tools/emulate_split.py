"""Design experiment (CPU, test infrastructure): how many bf16 planes does the tensor-core parity mode need?

Every dense contraction of the oracle (conv / conv_transpose / linear / DCN matmul / correlation / tracker dot) is
replaced by the arithmetic a split-bf16 tensor-core path performs: operands split into P bf16 planes
(x = x0 + x1 (+ x2), x_k = bf16(residual)), products x_i * w_j for i + j < P accumulated in fp32.  The clip of the
e2e parity test is then compared with the unmodified fp32 oracle.

    python tools/emulate_split.py [P ...]
"""
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, ".")
from oracle import ops as oops            # noqa: E402
from oracle.weights import make_model     # noqa: E402
from tests.e2e_util import make_pair      # noqa: E402

P = 2
MAXABS = 0.0
_conv2d, _convT, _linear, _matmul = F.conv2d, F.conv_transpose2d, F.linear, torch.matmul


def tf32(x):
    b = x.float().contiguous().view(torch.int32)
    b = (b + 0xFFF + ((b >> 13) & 1)) & ~0x1FFF
    return b.view(torch.float32)


def split(x, p):
    """p = 2, 3: bf16 planes.  p = 10: hybrid planes [tf32(x), bf16(x - tf32(x)), bf16(x)].
    p = 11: [bf16(x), fp16(x - bf16(x))]"""
    x = x.float()
    if p == 10:
        t = tf32(x)
        return [t, (x - t).bfloat16().float(), x.bfloat16().float()]
    if p == 11:
        h = x.bfloat16().float()
        return [h, (x - h).half().float()]
    if p == 13:      # the scheme of vps_conv2d_tc32: A = fp16(x), A2 = fp16(2^11 (x - A)); products A*B + 2^-11 (A2*B + A*B2)
        t = x.half().float()
        assert torch.isfinite(t).all(), "fp16 overflow"
        return [t, ((x - t) * 2048.0).half().float() / 2048.0]
    if p == 12:      # fp16 main (11 bits, limited range) + bf16 corrections
        global MAXABS, MINNZ
        MAXABS = max(MAXABS, float(x.abs().max()))
        t = x.half().float()
        assert torch.isfinite(t).all(), "fp16 overflow"
        return [t, (x - t).bfloat16().float(), x.bfloat16().float()]
    out, r = [], x
    for _ in range(p):
        h = r.bfloat16().float()
        out.append(h)
        r = r - h
    return out


def pairs(p):
    if p == 10:      # tf32 x tf32  +  bf16(a_lo) x bf16(b)  +  bf16(a) x bf16(b_lo)
        return [(0, 0), (1, 2), (2, 1)]
    if p == 11:
        return [(0, 0), (0, 1), (1, 0), (1, 1)]
    if p == 12:
        return [(0, 0), (1, 2), (2, 1)]
    if p == 13:
        return [(0, 0), (1, 0), (0, 1)]
    return [(i, j) for i in range(p) for j in range(p) if i + j < p]


def emu(fn, x, w, bias, *a, **k):
    xs, ws = split(x, P), split(w, P)
    acc = None
    for i, j in pairs(P)[::-1]:       # small terms first (any order on the GPU)
        t = fn(xs[i], ws[j], None, *a, **k)
        acc = t if acc is None else acc + t
    if bias is not None:
        acc = acc + (bias.view(1, -1, 1, 1) if acc.dim() == 4 else bias)
    return acc


def conv2d(x, w, bias=None, *a, **k):
    return emu(_conv2d, x, w, bias, *a, **k)


def convT(x, w, bias=None, *a, **k):
    return emu(_convT, x, w, bias, *a, **k)


def linear(x, w, bias=None):
    return emu(_linear, x, w, bias)


def matmul(a, b):
    As, Bs = split(a, P), split(b, P)
    acc = None
    for i, j in pairs(P)[::-1]:
        t = _matmul(As[i], Bs[j])
        acc = t if acc is None else acc + t
    return acc


def correlation(f1, f2, *a, **k):
    f1s, f2s = split(f1, P), split(f2, P)
    acc = None
    for i, j in pairs(P)[::-1]:
        t = _corr(f1s[i], f2s[j], *a, **k)
        acc = t if acc is None else acc + t
    return acc


_corr = oops.correlation


def run(model, frames, H, W):
    model.prev_bboxes = None
    if hasattr(model, "reset_tracker"):
        model.reset_tracker()
    outs = []
    for iid, a, b in frames:
        taps = {}
        r = model.simple_test(a, dict(iid=iid, img_shape=(H, W, 3)), b, taps)
        outs.append((r, taps))
    return outs


def main():
    global P
    Ps = [int(a) for a in sys.argv[1:]] or [2, 3]
    H, W = 128, 256
    img, ref = make_pair(H, W)
    frames = [(10001, img, ref), (10002, ref, img), (10003, img, ref)]
    import oracle.model as om
    model = make_model("C", 0)
    base = run(model, frames, H, W)
    for p in Ps:
        P = p
        F.conv2d, F.conv_transpose2d, F.linear = conv2d, convT, linear
        torch.matmul = matmul
        oops.correlation = correlation
        try:
            model = make_model("C", 0)
            F.conv2d, F.conv_transpose2d, F.linear = conv2d, convT, linear
            res = run(model, frames, H, W)
        finally:
            F.conv2d, F.conv_transpose2d, F.linear = _conv2d, _convT, _linear
            torch.matmul = _matmul
            oops.correlation = _corr
        for f, ((r0, t0), (r1, t1)) in enumerate(zip(base, res)):
            def rel(k, i=None):
                a, b = (t1[k], t0[k]) if i is None else (t1[k][i], t0[k][i])
                return float((a - b).abs().max() / max(1e-6, float(b.abs().max())))
            rep = dict(flow_full=rel("flow_full"), flow_fine=rel("flow_fine"),
                       fused=max(rel("fused", i) for i in range(5)), fpn=max(rel("fpn", i) for i in range(5)),
                       refined=rel("refined"),
                       fcn_score_abs=float((t1["fcn_score"] - t0["fcn_score"]).abs().max()),
                       fcn_score_max=float(t0["fcn_score"].abs().max()),
                       rpn_cls=max(float((t1["rpn_cls"][l] - t0["rpn_cls"][l]).abs().max()) for l in range(5)),
                       nprop=(t1["proposals"].shape[0], t0["proposals"].shape[0]),
                       ndet=(t1["det_rois"].shape[0], t0["det_rois"].shape[0]))
            if rep["nprop"][0] == rep["nprop"][1]:
                rep["cls_score_abs"] = float((t1["cls_score"] - t0["cls_score"]).abs().max())
            if rep["ndet"][0] == rep["ndet"][1]:
                rep["mask_logit_abs"] = float((t1["mask_score"] - t0["mask_score"]).abs().max())
            rep["pano_diff_px"] = int((r1[2]["panoptic_outputs"] != r0[2]["panoptic_outputs"]).sum())
            rep["sem_diff_px"] = int((r1[2]["fcn_outputs"] != r0[2]["fcn_outputs"]).sum())
            rep["ids_equal"] = bool(np.array_equal(r1[2]["panoptic_det_obj_ids"].numpy(), r0[2]["panoptic_det_obj_ids"].numpy()))
            print("P=%d frame %d: %s" % (p, f, rep), flush=True)
        print("max |operand| seen:", MAXABS)


if __name__ == "__main__":
    main()
