"""Run a video panoptic model over a Cityscapes-VPS split and write what the reference's tools/test_vpq.py writes for
eval_vpq: <out>_pans_unified/pan_2ch/*.png, pan_pred/*.png and pred.json.

    python -m vps_b200.test_vpq configs/cityscapes/fusetrack.py latest.pth --out work_dirs/fusetrack/val.pkl \\
        --pan_im_json_file data/cityscapes_vps/panoptic_im_val_city_vps.json --n_video 50 --mode val

The chain: frames decoded on the host (cv2.imread, a few threads ahead of the loop) -> the config's test pipeline on the
device (`InputStage.from_pipeline`) -> the model (`ClipRunner`, the unified result computed per frame on the GPU) ->
`PanWriter` (every 5th frame from the 5th, [(20//5)::5] over the whole frame list, named by the sorted pan_im_json names).
The .pkl side files of the reference (_mask.pkl, _pred_pans_2ch.pkl) and --load are not implemented: --out only names the
output directory."""
import argparse
import itertools
import json
import os
import sys
import time

_DESC = ("VPSNet test on the GPU: writes <out>_pans_unified/ (pan_2ch/, pan_pred/, pred.json) for vps_b200.eval_vpq.  "
         "The reference's .pkl side files and --load are not implemented; --out only names the output directory.")


def parse_args(argv=None):
    p = argparse.ArgumentParser(description=_DESC)
    p.add_argument("config", help="test config file path (configs/cityscapes/{fusetrack,track,fuse}.py)")
    p.add_argument("checkpoint", help="checkpoint file (a dict with 'state_dict', or a state dict)")
    p.add_argument("--out", required=True, help="X.pkl: the results go to X_pans_unified/ (no .pkl is written)")
    p.add_argument("--gpus", type=str, default="0", help="the first id is the device used")
    p.add_argument("--dataset", type=str, default="CityscapesVps", choices=["CityscapesVps"])
    p.add_argument("--test_config", type=str, default="configs/cityscapes/test_cityscapes_1gpu.yaml",
                   help="UPSNet test yaml (must exist): test.panoptic_stuff_area_limit is read from it (4096 when it "
                        "does not set it, the default of tools/config/config.py)")
    p.add_argument("--n_video", type=int, default=50, help="accepted for compatibility; the output does not depend on it")
    p.add_argument("--pan_im_json_file", type=str, default="data/cityscapes_vps/panoptic_im_val_city_vps.json")
    p.add_argument("--mode", type=str, default="val", help="val or test: rewrites the paths of cfg.data.test")
    p.add_argument("--precision", type=str, default="tc32", choices=["tc32", "fp32", "bf16"])
    p.add_argument("--workers", type=int, default=4, help="host decode / PNG encode threads")
    args = p.parse_args(argv)
    if not args.out.endswith((".pkl", "pickle")):
        raise ValueError("The output file must be a .pkl file.")
    return args


def stuff_area_limit(test_config):
    """test.panoptic_stuff_area_limit of the UPSNet yaml (update_config, test_vpq.py:88; 4096, the default of
    tools/config/config.py, when the yaml does not set it).  The file must exist, as update_config opens it: the
    reference's test_cityscapes_1gpu.yaml sets 2048, and silently using another limit would change the results."""
    import yaml
    if not os.path.isfile(test_config):
        raise FileNotFoundError("--test_config %r not found (the reference's configs/cityscapes/test_cityscapes_1gpu.yaml "
                                "sets panoptic_stuff_area_limit: 2048)" % test_config)
    with open(test_config) as f:
        y = yaml.safe_load(f) or {}
    v = (y.get("test") or {}).get("panoptic_stuff_area_limit")
    return 4096 if v is None else int(v)


def load_model(config, checkpoint, device, precision):
    import torch

    from . import Config, build_detector
    cfg = Config.fromfile(config)
    cfg.model.pretrained = None
    model = build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg)
    ck = torch.load(checkpoint, map_location="cpu")
    model.load_state_dict(ck.get("state_dict", ck) if isinstance(ck, dict) else ck, strict=True)
    model = model.to(device)
    model.precision = precision
    model.label_dtype = torch.uint8
    model.prepare(force=True)
    return cfg, model


def run_split(cfg, model, dataset, names, output_dir, area_limit=4096, workers=4, device="cuda:0"):
    """the loop of single_gpu_test + get_unified_pan_result + inference_panoptic_video over a whole split; returns pred.json"""
    import cv2
    import torch

    from .pipeline import InputStage
    from .runner import ClipRunner
    from .writer import PanWriter
    stage = InputStage.from_pipeline(cfg.data.test.pipeline, device=device)
    # the reference keys the unified results by file basename and sorts them before sampling (test_vpq.py:170-176); the
    # frames run in dataset order, so the two orders must agree (they do for Cityscapes-VPS names)
    base = [dataset.img_info(i)["filename"].split("/")[-1] for i in range(len(dataset))]
    if base != sorted(set(base)):
        raise ValueError("the dataset's images are not in ascending, unique file-name order: the reference samples the "
                         "sorted results, which this driver does not reorder")
    writer = PanWriter(output_dir, workers=workers)
    sampled = list(range(len(dataset)))[writer.start::writer.step]
    if len(sampled) != len(names):
        raise ValueError("%d frames are sampled from %d images but the pan_im_json lists %d names"
                         % (len(sampled), len(dataset), len(names)))
    name_of = dict(zip(sampled, names))
    with_ref = model.with_flow

    def read(idx):
        img_path, ref_path = dataset.paths(idx)
        img = cv2.imread(img_path, cv2.IMREAD_COLOR)
        if img is None:
            raise FileNotFoundError(img_path)
        ref = None
        if with_ref:
            ref = cv2.imread(ref_path, cv2.IMREAD_COLOR)
            if ref is None:
                raise FileNotFoundError(ref_path)
        pair = (torch.from_numpy(img), None if ref is None else torch.from_numpy(ref))
        return pair, dataset.img_meta(idx)

    from .datasets import prefetch_map
    a, b = itertools.tee(prefetch_map(read, range(len(dataset)), workers=workers, depth=8))   # zip below keeps them in step
    pairs, metas = (pair for pair, _ in a), (meta for _, meta in b)
    runner = ClipRunner(model, device, unify=True, input_stage=stage)
    runner.unifier.stuff_area_limit = int(area_limit)
    model.reset_tracker()
    with writer:
        for idx, r in enumerate(runner.run(pairs, metas)):
            writer.add_frame(name_of.get(idx), r[2]["pan_2ch_device"], pan_2ch_host=r[2]["pan_2ch"])
        return writer.finish()


def main(argv=None):
    args = parse_args(argv)
    import torch

    from .datasets import CityscapesVPSTestSet, rewrite_mode
    device = "cuda:%d" % int(args.gpus.split(",")[0])
    torch.cuda.set_device(device)
    cfg, model = load_model(args.config, args.checkpoint, device, args.precision)
    test = rewrite_mode(cfg.data.test, args.mode)
    cfg.data.test.update(test)
    dataset = CityscapesVPSTestSet.from_cfg(test)
    output_dir = args.out.replace(".pkl", "_pans_unified/")
    print("==> Video Panoptic Segmentation results will be saved at:")
    print("---", output_dir)
    with open(args.pan_im_json_file) as f:
        names = sorted(x["file_name"] for x in json.load(f)["images"])
    t0 = time.time()
    run_split(cfg, model, dataset, names, output_dir, stuff_area_limit(args.test_config), args.workers, device)
    print("==> Done: %d frames in %.1f s" % (len(dataset), time.time() - t0))
    return 0


if __name__ == "__main__":
    sys.exit(main())
