"""Record configs/cityscapes/track.py and fuse.py the way make_boundary_golden.py records fusetrack.py, into
tests/golden/reference_boundary_models.json: for each config, "model" and "test_cfg" as the config loader reads them, and
"state_dict_keys", the sorted state_dict keys of the reference's own PanopticTrack / PanopticFuse built from it
(imported through tests/golden/ref_import.py).
Run where the reference tree is available:  python tests/golden/make_models_boundary_golden.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_boundary_models.json")


def main():
    from oracle.weights import make_model
    from tests.golden.make_boundary_golden import from_json, plain, to_json
    from tests.golden.ref_import import REF
    from tests.golden.run_reference_models import build_reference_model
    from vps_b200.config import Config
    sd = make_model("C", 0).state_dict()
    rec = {}
    for name in ("track", "fuse"):
        cfg = Config.fromfile(os.path.join(REF, "configs/cityscapes/%s.py" % name))
        det = build_reference_model(sd, name)
        rec[name] = {"model": plain(dict(cfg.model.items())), "test_cfg": plain(dict(cfg.test_cfg.items())),
                     "detector": type(det).__name__, "state_dict_keys": sorted(det.state_dict())}
    enc = to_json(rec)
    assert from_json(json.loads(json.dumps(enc))) == rec, "config does not survive a JSON round trip"
    with open(OUT, "w") as f:
        json.dump(enc, f, indent=1)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
