"""CPU: the oracle of the image panoptic model's evaluation (oracle/ipq.py) reproduces the reference's own evaluate_ssegs
and evaluate_panoptic on the golden frames (tests/golden/make_ipq_golden.py), and so does the product's host matching
(vps_b200.ipq.IpqEvaluator fed numpy-made pair tables)."""
import json
import os

import numpy as np
import pytest

HERE = os.path.join(os.path.dirname(__file__), "golden")


def load():
    d = np.load(os.path.join(HERE, "ipq_frames.npz"))
    meta = json.load(open(os.path.join(HERE, "ipq_frames.json")))
    categories = {c["id"]: c for c in meta["categories"]}
    with open(os.path.join(HERE, "ipq_pq.txt")) as f:
        txt = f.read()
    return d, meta, categories, txt


def oracle_frames(d, meta):
    from oracle import ipq as O
    frames = []
    for i in range(int(d["nframes"])):
        segs, ids = O.convert_image(d["pan2ch%d" % i])
        frames.append((meta["gt"][i], segs, d["gt_ids%d" % i], ids))
    return frames


def check_stat(stat, d):
    for row, c in enumerate(d["stat"]):
        s = stat[row]
        assert [s.tp, s.fp, s.fn] == c[1:].astype(int).tolist(), row
        assert s.iou == c[0], row                                   # same summation order -> identical float64


def test_seg_confusion_and_iu_match_reference():
    from oracle import ipq as O
    d, _, _, _ = load()
    total = np.zeros((19, 19))
    for i in range(int(d["nframes"])):
        m = O.seg_confusion(d["trainid%d" % i], d["fcn%d" % i])
        assert np.array_equal(m, d["seg_conf%d" % i]), i
        total += m
    r = O.seg_result(total)
    assert np.array_equal(r["confusion_matrix"], d["seg_confusion"])
    assert np.array_equal(r["IU_array"], d["IU_array"]) and r["meanIU"] == d["meanIU"]
    # the golden exercises the reference's quirks: a pred >= 19 aliases into the next row, gt 20 / 255 are dropped
    assert any((d["fcn%d" % i] >= 19).any() and (d["trainid%d" % i] == 20).any() for i in range(int(d["nframes"])))


def test_converter_matches_reference_pred_json_modulo_ids():
    from oracle import ipq as O
    d, meta, _, _ = load()
    for i in range(int(d["nframes"])):
        segs, _ = O.convert_image(d["pan2ch%d" % i])
        ref = meta["pred"][i]
        assert len(segs) == len(ref), i
        fwd, bwd = {}, {}
        for a, b in zip(segs, ref):                                 # both walk the keys in ascending order
            assert fwd.setdefault(a["id"], b["id"]) == b["id"] and bwd.setdefault(b["id"], a["id"]) == a["id"], i
            assert {k: v for k, v in a.items() if k != "id"} == {k: v for k, v in b.items() if k != "id"}, i


def test_pq_core_and_pq_txt_match_reference():
    from oracle import ipq as O
    from oracle import vpq as V
    d, meta, categories, txt = load()
    stat = O.pq_compute_single_core(oracle_frames(d, meta), categories)
    check_stat(stat, d)
    for row, t in enumerate((None, True, False)):
        r, _ = V.pq_average(stat, categories, isthing=t)
        assert [r["pq"], r["sq"], r["rq"], float(r["n"])] == d["avg"][row].tolist()
    assert O.pq_txt(stat, categories) == txt
    assert d["stat"][:, 1].sum() > 0 and d["stat"][:, 2].sum() > 0 and d["stat"][:, 3].sum() > 0


def test_product_host_matching_matches_reference(tmp_path):
    """IpqEvaluator's host side (the shared matching loop, dict semantics, pq.txt) on numpy-made pair tables"""
    from vps_b200 import ipq as P
    from vps_b200 import vpq as V
    d, meta, categories, txt = load()
    ev = P.IpqEvaluator(categories)
    for gseg, pseg, gt, pr in oracle_frames(d, meta):
        pairs, counts = np.unique(gt.astype(np.uint64) * np.uint64(V.OFFSET) + pr.astype(np.uint64), return_counts=True)
        ev.add_frame_table(gseg, pseg, pairs, counts)
    stat = ev.compute()
    check_stat(stat, d)
    ev.write_pq_txt(str(tmp_path / "pq.txt"), stat)
    assert (tmp_path / "pq.txt").read_text() == txt


def test_product_sanity_checks_raise():
    from vps_b200 import ipq as P
    from vps_b200 import vpq as V
    categories = {i: {"id": i, "isthing": int(i >= 11)} for i in range(19)}
    pairs = np.array([5 * V.OFFSET + 3001, 5 * V.OFFSET + 30001], dtype=np.uint64)
    counts = np.array([4, 6])
    with pytest.raises(KeyError):                    # 30001 is in the PNG, not in the JSON
        P.IpqEvaluator(categories).add_frame_table([], [{"id": 3001, "category_id": 3, "iscrowd": 0, "area": 4}], pairs, counts)
    with pytest.raises(KeyError):                    # category 30 is unknown
        P.IpqEvaluator(categories).add_frame_table([], [{"id": 3001, "category_id": 3, "iscrowd": 0, "area": 4},
                                                        {"id": 30001, "category_id": 30, "iscrowd": 0, "area": 6}], pairs, counts)


def test_iou_of_one_half_is_not_a_match():
    """the golden's half-covered instance: intersection = half the prediction, union = the prediction -> IoU 0.5, no match"""
    d, meta, _, _ = load()
    found = 0
    for gseg, pseg, gt, pr in oracle_frames(d, meta):
        area_p = {s["id"]: int((pr == s["id"]).sum()) for s in pseg}
        gmap = {s["id"]: s for s in gseg}
        for g in np.unique(gt):
            for p in np.unique(pr[gt == g]):
                inter = int(((gt == g) & (pr == p)).sum())
                if g in gmap and p in area_p and p != 0 and 2 * inter == area_p[p] and gmap[int(g)]["area"] == inter:
                    found += 1
    assert found >= 1
