"""CPU: the 2-channel -> PNG/JSON converter row (SURVEY 8f rank 1b).
 * oracle/writer.py vs the reference's own converter_2ch_track_core (golden made by tests/golden/make_writer_golden.py with a
   stand-in colour generator): same segments (category, bbox, area) and the same pixel partition, ids modulo a bijection that
   keeps a thing's id across frames;
 * vps_b200.writer.PanWriter's host part fed by the oracle: PNG round trip, pred.json and frame sampling."""
import json
import os

import numpy as np

HERE = os.path.join(os.path.dirname(__file__), "golden")


def _golden():
    d = np.load(os.path.join(HERE, "writer_frames.npz"))
    ann = json.load(open(os.path.join(HERE, "writer_frames.json")))
    n = int(d["nframes"])
    return [d["in%d" % i] for i in range(n)], [d["png%d" % i] for i in range(n)], ann


def test_oracle_matches_reference_modulo_ids():
    from oracle import writer as Wo
    frames, pngs, ann = _golden()
    thing_map = {}
    seen_multi = False
    for fr, png, a in zip(frames, pngs, ann):
        segs, ids = Wo.convert_frame(fr)
        ref_ids = Wo.rgb2id(png)
        key = lambda s: (s["category_id"], s["iscrowd"], tuple(s["bbox"]), s["area"])
        assert sorted(key(s) for s in segs) == sorted(key(s) for s in a["segments_info"])
        # same partition of the pixels: id pairs form a bijection (VOID <-> 0)
        pairs = np.unique(np.stack([ids.ravel(), ref_ids.ravel()], 1), axis=0)
        assert len(set(pairs[:, 0].tolist())) == len(pairs) == len(set(pairs[:, 1].tolist()))
        assert all((m == 0) == (t == 0) for m, t in pairs.tolist())          # VOID <-> VOID
        for mine, theirs in pairs.tolist():
            if mine and (mine - 1) // 1000 >= 11:                    # a thing keeps its id across the frames of the clip
                assert thing_map.setdefault(mine, theirs) == theirs
        # the case the first golden missed (ADVICE r1): a stuff category whose pixels carry several track-channel values
        # (native stuff: its pan value; demoted thing region: 0) is ONE segment
        p = fr.astype(np.uint32)
        stuff_keys = {}
        for k in np.unique(1000 * p[..., 0] + p[..., 2]).tolist():
            if k // 1000 <= 10:
                stuff_keys.setdefault(k // 1000, []).append(k)
        multi = [c for c, ks in stuff_keys.items() if len(ks) > 1]
        seen_multi = seen_multi or bool(multi)
        for c in multi:
            assert sum(1 for s_ in segs if s_["category_id"] == c) == 1
    assert seen_multi, "golden clip must contain a stuff category with more than one key"


def test_product_writer_host_part_fed_by_oracle(tmp_path):
    from oracle import vpq as V
    from oracle import writer as Wo
    from PIL import Image
    from vps_b200.writer import PanWriter
    frames, _, _ = _golden()
    names = ["frankfurt_%06d_leftImg8bit.png" % i for i in range(len(frames))]
    w = PanWriter(str(tmp_path), sample=False)
    converted = [Wo.convert_frame(fr) for fr in frames]
    for name, fr, (segs, ids) in zip(names, frames, converted):
        v_ids, v_segs = V.segments_from_pan2ch(fr)                  # the numpy VPQ chain segments frames as the converter
        assert np.array_equal(v_ids, ids)
        assert v_segs == [{k: s[k] for k in ("id", "category_id", "iscrowd", "area")} for s in segs]
        assert w.add_frame_ids(name, segs, ids, fr) == {"segments_info": segs}
    pred = w.finish()
    assert json.load(open(os.path.join(str(tmp_path), "pred.json"))) == pred
    assert pred["annotations"] == [{"segments_info": segs} for segs, _ in converted]
    for name, fr, (_, ids) in zip(names, frames, converted):
        png = np.asarray(Image.open(os.path.join(str(tmp_path), "pan_pred", name.replace("_leftImg8bit", ""))))
        assert np.array_equal(Wo.rgb2id(png), ids)
        p2 = np.asarray(Image.open(os.path.join(str(tmp_path), "pan_2ch", name.replace("_leftImg8bit", ""))))
        assert np.array_equal(p2, fr)
    # frame sampling of inference_panoptic_video: [(20 // 5)::5]
    w2 = PanWriter(None)
    kept = [i for i in range(30) if w2.add_frame_ids("f%d" % i, *converted[0], frames[0]) is not None]
    assert kept == list(range(30))[4::5]
