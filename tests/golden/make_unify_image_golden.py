"""Golden vectors for the image-level get_unified_pan_result (reference tools/dataset/base_dataset.py:232-274, what
tools/test_eval_ipq.py evaluates the image panoptic model PanopticFuse with): runs the REFERENCE's own function, imported
unmodified as make_unify_golden.py imports the video one, on the seeded synthetic frames of unify_pan.npz and stores the
outputs in tests/golden/unify_image.npz (inputs are read from unify_pan.npz, not copied).
Run where the reference tree is available:  python tests/golden/make_unify_image_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_unify_golden import import_reference  # noqa: E402


def main():
    import_reference()
    from tools.dataset.base_dataset import BaseDataset
    g = np.load(os.path.join(HERE, "unify_pan.npz"))
    n = int(g["nframes"])
    names = ["f%d" % i for i in range(n)]
    out = BaseDataset.get_unified_pan_result(None, [g["seg%d" % i].copy() for i in range(n)],
                                             [g["pan%d" % i].copy() for i in range(n)],
                                             [g["cls%d" % i].copy() for i in range(n)], names=names)
    d = {"out%d" % i: out[nm] for i, nm in enumerate(names)}
    d["nframes"] = np.int64(n)
    path = os.path.join(HERE, "unify_image.npz")
    np.savez_compressed(path, **d)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
