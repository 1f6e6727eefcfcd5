"""Golden vectors for the semantic evaluation of predictions whose shape differs from the ground truth: runs the
REFERENCE's own `Cityscapes.evaluate_ssegs` (tools/dataset/cityscapes.py:112-166, imported unmodified through
make_unify_golden.import_reference) on seeded synthetic frames.  evaluate_ssegs writes each prediction as np.uint8 into a
palette PNG, reads it back and resizes it to the gt with Image.NEAREST (:125-126) before counting.

The frames hold a downscaled prediction, an upscaled one, one of an odd size in both axes, one of the gt's own shape, gt
trainIds 255 and 20 and predicted labels >= 19.  Per-frame confusion counts come from the reference's get_confusion_matrix,
the totals, IU and mean IU from evaluate_ssegs at return (the harness of make_ipq_golden.py).
Output: tests/golden/ipq_resize.npz.  Rerunning writes identical files.
Run where the reference tree is available:  python tests/golden/make_ipq_resize_golden.py"""
import os
import shutil
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_ipq_golden import run_evaluate_ssegs  # noqa: E402
from make_unify_golden import import_reference  # noqa: E402

GT_SHAPE = (61, 97)
PRED_SHAPES = [(31, 49), (128, 200), (45, 131), (61, 97)]     # down, up, odd (down in y, up in x), equal


def blocks(rng, h, w, hi, b):
    return rng.integers(0, hi, size=((h + b - 1) // b, (w + b - 1) // b)).repeat(b, 0).repeat(b, 1)[:h, :w]


def synth(rng, ph, pw):
    gh, gw = GT_SHAPE
    gt = blocks(rng, gh, gw, 19, 6).astype(np.uint8)
    gt[blocks(rng, gh, gw, 5, 12) == 0] = 255
    gt[50:55, 80:90] = 20
    pred = blocks(rng, ph, pw, 19, 5).astype(np.int64)
    pred[:3, :5] = 21                                           # >= 19: aliases into the next row
    return gt, pred


def main():
    import_reference()
    from tools.dataset.cityscapes import Cityscapes
    rng = np.random.default_rng(2718)
    frames = [synth(rng, ph, pw) for ph, pw in PRED_SHAPES]
    tmp = tempfile.mkdtemp(prefix="ipq_resize_golden_")
    assert "images" not in tmp and "labels" not in tmp
    try:
        sseg, per_frame = run_evaluate_ssegs(Cityscapes, [f[0] for f in frames], [f[1] for f in frames], tmp)
    finally:
        shutil.rmtree(tmp)
    assert len(per_frame) == len(frames) and sseg
    out = {"nframes": np.int64(len(frames))}
    for i, (gt, pred) in enumerate(frames):
        # the int64 prediction holds labels < 256, so its uint8 copy is what the reference wrote and read back
        out["trainid%d" % i], out["fcn%d" % i], out["seg_conf%d" % i] = gt, pred.astype(np.uint8), per_frame[i]
    out["seg_confusion"] = sseg["confusion_matrix"]
    out["IU_array"] = sseg["IU_array"]
    out["meanIU"] = np.float64(sseg["meanIU"])
    np.savez(os.path.join(HERE, "ipq_resize.npz"), **out)
    print("meanIU", sseg["meanIU"])


if __name__ == "__main__":
    main()
