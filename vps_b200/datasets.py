"""The Cityscapes-VPS test split as the reference's loader walks it (mmdet/datasets/cityscapes_vps.py, custom.py, coco.py,
pipelines/loading.py), the Cityscapes test split of the image panoptic model (mmdet/datasets/cityscapes.py,
`CityscapesTestSet`), and a small ordered prefetcher for host decoding.

Order: the images of the annotation file (`im_all_info_{val,test}_city_vps.json`) in file order, as pycocotools' COCO keeps
them (one entry per image id).  Reference frame (`prepare_test_img`, cityscapes_vps.py:137-148): the previous image of the
list, unless the index is a multiple of `nframes_span_test` (30 in the configs: one clip), where the frame references itself;
`ref_id` is the previous image's id minus one, as the reference sets it.  `LoadRefImageFromFile` (loading.py:43-67) reads
img_prefix/filename and ref_prefix/ref_filename.  The img_meta `Collect` hands the model (formating.py:172-175): filename,
ori_shape, img_shape, pad_shape, scale_factor, flip, img_norm_cfg and iid; the geometry fields come from the input stage."""
import json
import os.path as osp
from collections import deque
from concurrent.futures import ThreadPoolExecutor


def prefetch_map(fn, items, workers=4, depth=8):
    """fn(item) for every item, in order, computed on `workers` threads at most `depth` items ahead of the consumer.  The
    threads are joined when the generator finishes, is closed or is dropped."""
    pool = ThreadPoolExecutor(max_workers=max(1, int(workers)), thread_name_prefix="prefetch")
    pending = deque()
    try:
        for x in items:
            pending.append(pool.submit(fn, x))
            if len(pending) >= max(1, int(depth)):
                yield pending.popleft().result()
        while pending:
            yield pending.popleft().result()
    finally:
        for f in pending:
            f.cancel()
        pool.shutdown(wait=True)


def rewrite_mode(test_cfg, mode):
    """the --mode rewrite of tools/test_vpq.py:108-117 on a copy of cfg.data.test: 'val' replaces every "test" in ann_file,
    img_prefix and ref_prefix by "val", 'test' the reverse; any other mode is a KeyError"""
    if mode == "val":
        a, b = "test", "val"
    elif mode == "test":
        a, b = "val", "test"
    else:
        raise KeyError("Argument 'mode' must be either 'val' or 'test'.")
    out = dict(test_cfg)
    for k in ("ann_file", "img_prefix", "ref_prefix"):
        out[k] = out[k].replace(a, b)
    return out


def coco_images(ann_file):
    """the images of a COCO-style annotation file as mmdet's CocoDataset lists them in test mode (coco.py): file order, one
    entry per image id (pycocotools' COCO(ann_file).imgs keeps an id's first position and its last entry), with
    filename = file_name"""
    with open(ann_file) as f:
        images = json.load(f)["images"]
    by_id = {}
    for im in images:
        by_id[im["id"]] = im
    return [dict(im, filename=im["file_name"]) for im in by_id.values()]


class _TestSet:
    """`len(ds)`, `ds.img_info(i)` (with ref_filename), `ds.paths(i)` (image and reference-image paths) and
    `ds.img_meta(i, stage, shape)` of a test-mode dataset; subclasses set the reference-frame rule in img_info"""

    def __init__(self, ann_file, img_prefix, ref_prefix, data_root=None, **_):
        if data_root is not None:                                   # custom.py:57-69
            join = lambda p: p if p is None or osp.isabs(p) else osp.join(data_root, p)
            ann_file, img_prefix, ref_prefix = join(ann_file), join(img_prefix), join(ref_prefix)
        if ref_prefix is None:
            raise ValueError("ref_prefix must be specified.")
        self.ann_file, self.img_prefix, self.ref_prefix = ann_file, img_prefix, ref_prefix
        self.img_infos = coco_images(ann_file)

    @classmethod
    def from_cfg(cls, test_cfg):
        """from cfg.data.test"""
        return cls(**{k: v for k, v in test_cfg.items() if k not in ("type", "pipeline", "test_mode")})

    def __len__(self):
        return len(self.img_infos)

    def paths(self, idx):
        info = self.img_info(idx)
        return osp.join(self.img_prefix, info["filename"]), osp.join(self.ref_prefix, info["ref_filename"])

    def img_meta(self, idx, stage=None, shape=None):
        """filename, iid and flip; with an InputStage and the decoded frame's (h, w) also the geometry fields and
        img_norm_cfg that stage produces"""
        info = self.img_info(idx)
        meta = dict(filename=osp.join(self.img_prefix, info["filename"]), iid=info["id"], flip=False)
        if stage is not None and shape is not None:
            import numpy as np
            h, w = int(shape[0]), int(shape[1])
            oh, ow, hp, wp, sf = stage.geometry(h, w)
            meta.update(ori_shape=(h, w, 3), img_shape=(oh, ow, 3), pad_shape=(hp, wp, 3), scale_factor=sf,
                        img_norm_cfg=dict(mean=np.array(list(stage.mean), np.float32), std=np.array(list(stage.std), np.float32),
                                          to_rgb=stage.to_rgb))
        return meta


class CityscapesVPSTestSet(_TestSet):
    """Test-mode CityscapesVPSDataset (cfg.data.test after rewrite_mode)."""

    def __init__(self, ann_file, img_prefix, ref_prefix, nframes_span_test=6, data_root=None, **_):
        super().__init__(ann_file, img_prefix, ref_prefix, data_root)
        self.nframes_span_test = int(nframes_span_test)

    def img_info(self, idx):
        info = dict(self.img_infos[idx])
        prev = self.img_infos[idx - 1] if idx % self.nframes_span_test > 0 else self.img_infos[idx]
        info["ref_id"] = prev["id"] - 1
        info["ref_filename"] = prev["file_name"]
        return info


class CityscapesTestSet(_TestSet):
    """Test-mode CityscapesDataset of the image panoptic model (configs/cityscapes/fuse.py; mmdet/datasets/cityscapes.py:
    82-97): the reference frame is the file of the previous frame id, read from ref_prefix (the val_nbr directory of
    Cityscapes' neighbouring frames).  With fid = int(filename.split('_')[-2]) and suffix = '_' + filename.split('_')[-1],
    ref_filename = filename.replace('%06d' % fid + suffix, '%06d' % (fid - 1) + suffix) when fid >= 1, else the image
    itself; the replace is applied to the whole filename, as the reference does."""

    def img_info(self, idx):
        info = dict(self.img_infos[idx])
        filename = info["filename"]
        fid = int(filename.split('_')[-2])
        suffix = '_' + filename.split('_')[-1]
        info["ref_filename"] = filename.replace('%06d' % fid + suffix, '%06d' % (fid - 1) + suffix) if fid >= 1 else filename
        return info
