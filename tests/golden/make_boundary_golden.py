"""Record what the drop-in boundary tests (tests/test_boundary.py) compare against, from the REFERENCE itself, into
tests/golden/reference_boundary.json:
  * "model", "test_cfg": configs/cityscapes/fusetrack.py as loaded by the config loader (plain dicts / lists);
  * "registries": for each of the reference's mmdet.models.registry registries, the class names it holds and the module
    each class is defined in (imported through tests/golden/ref_import.py).
Run where the reference tree is available:  python tests/golden/make_boundary_golden.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_boundary.json")


def plain(x):
    if isinstance(x, dict):
        return {k: plain(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [plain(v) for v in x]
    return x


def to_json(x):
    """plain() value -> JSON value; a dict with integer keys (test_cfg.class_mapping) becomes {"__int_keys__": [[k, v], ..]}"""
    if isinstance(x, dict):
        if x and all(isinstance(k, int) for k in x):
            return {"__int_keys__": [[k, to_json(v)] for k, v in x.items()]}
        return {k: to_json(v) for k, v in x.items()}
    if isinstance(x, list):
        return [to_json(v) for v in x]
    return x


def from_json(x):
    if isinstance(x, dict):
        if set(x) == {"__int_keys__"}:
            return {int(k): from_json(v) for k, v in x["__int_keys__"]}
        return {k: from_json(v) for k, v in x.items()}
    if isinstance(x, list):
        return [from_json(v) for v in x]
    return x


def main():
    from tests.golden.ref_import import REF, setup
    from vps_b200.config import Config
    from vps_b200.registry import REGISTRIES
    cfg = Config.fromfile(os.path.join(REF, "configs/cityscapes/fusetrack.py"))
    setup()                                          # the reference's mmdet.models (its registries hold ITS classes)
    import mmdet.models.registry as RR
    regs = {}
    for attr in REGISTRIES:
        theirs = getattr(RR, attr, None)
        if theirs is not None:
            regs[attr] = {name: cls.__module__ for name, cls in sorted(theirs.module_dict.items())}
    rec = {"model": plain(dict(cfg.model.items())), "test_cfg": plain(dict(cfg.test_cfg.items())), "registries": regs}
    enc = to_json(rec)
    assert from_json(json.loads(json.dumps(enc))) == rec, "config does not survive a JSON round trip"
    with open(OUT, "w") as f:
        json.dump(enc, f, indent=1)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
