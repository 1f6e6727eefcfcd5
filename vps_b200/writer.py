"""2-channel -> PNG / JSON writer (SURVEY 8f rank 1b): `converter_2ch_track_core` + the file layout of
`inference_panoptic_video` (reference tools/dataset/cityscapes_vps.py:26-160), frame by frame.

`PanWriter.add_frame` makes one device pass per sampled frame (`vps_pan2ch_segments`): the pixel count and bounding box of
every (semantic, track) key and the pan_pred image, id2rgb of the segment id.  The host turns the 19 x 256 key table into
segments_info (`segments_from_table`) and hands the two PNGs to a small pool of writer threads, so their encoding overlaps
the next frames; `finish()` waits for them.  `add_frame_ids` is the same host part fed from numpy (scipy find_objects).  Segment ids: the reference uses the colours of panopticapi's `IdGenerator` (one fixed
colour per stuff category, random per thing key; everything downstream is invariant to the values); here id =
1000 * semantic + 1 for stuff, 1000 * semantic + track + 1 for things, colour = id2rgb(id).  One reference quirk is kept:
the bbox of a stuff segment that merges several keys is the bbox of its LAST key (segm_info[colour] is overwritten per key,
cityscapes_vps.py:131-138) -- `add_frame_ids` takes it from `bbox_ids` when given.

`ImageWriter` is the same for the image panoptic model (tools/test_eval_ipq.py): the image converter's table keyed on the
instance channel (`vps_pan2ch_image_segments`, `image_segments_from_table`), the pan_2ch / pan PNGs, pred.json and gt.json
of evaluate_panoptic, and the palette PNGs of write_segmentation_result, on the same pool of writer threads (`_PngPool`)."""
import ctypes as C
import json
import os
from collections import deque
from concurrent.futures import ThreadPoolExecutor

import numpy as np

NSEM, NTRK = 19, 256            # key space of vps_pan2ch_segments (include/vps_b200.h: VPS_SEG_*)
NKEY = NSEM * NTRK


def id2rgb(ids):
    ids = np.asarray(ids).astype(np.uint32)
    return np.stack([ids % 256, (ids // 256) % 256, ids // 65536], axis=-1).astype(np.uint8)


def _clean_name(name):
    # inference_panoptic_video.save_image (:69)
    return name.replace('_leftImg8bit', '').replace('_newImg8bit', '').replace('jpg', 'png').replace('jpeg', 'png')


def last_key_ids(pan_2ch, num_stuff=11):
    """id map in which a stuff segment keeps only the pixels of its LARGEST key 1000 * semantic + track channel: the reference
    overwrites segm_info[colour] for every key of a category in ascending key order (cityscapes_vps.py:112-138), so the bbox
    that survives is the last key's, while the area is re-counted from the merged PNG."""
    p = np.asarray(pan_2ch).astype(np.uint32)
    sem, trk = p[..., 0], p[..., 2]
    ids = np.where(sem == 255, 0, 1000 * sem + np.where(sem < num_stuff, 0, trk) + 1).astype(np.uint32)
    out = ids.copy()
    for c in np.unique(sem[sem < num_stuff]).tolist():
        m = sem == c
        out[m & (trk != trk[m].max())] = 0
    return out


def pan2ch_segments(pan_2ch, num_stuff=11, rgb=True, image=False):
    """The device pass of add_frame: pan_2ch uint8 CUDA [H,W,3] -> (table uint32 numpy [5, 19, 256] of per-key pixel count,
    min x, min y, max x, max y; pan_pred uint8 CUDA [H,W,3] or None).  Semantics other than 0..18 and 255 raise ValueError.
    image=True keys the image converter's (semantic, instance rank = channel 1) pairs instead of (semantic, track) and
    colours the image converter's ids (`ImageWriter`)."""
    import torch

    from . import ops
    assert pan_2ch.is_cuda and pan_2ch.dtype == torch.uint8 and pan_2ch.dim() == 3 and pan_2ch.shape[2] == 3
    p2 = pan_2ch.contiguous()
    table = torch.empty(5 * NKEY + 1, dtype=torch.int32, device=p2.device)
    out = torch.empty_like(p2) if rgb else None
    ops.pan2ch_segments(p2, num_stuff, table, out, image=image)
    t = table.cpu().numpy().view(np.uint32)
    if t[-1]:
        raise ValueError("pan2ch_segments: %d pixels have a semantic class outside 0..%d and 255" % (int(t[-1]), NSEM - 1))
    return t[:-1].reshape(5, NSEM, NTRK), out


def segments_from_table(table, num_stuff=11):
    """segments_info of one frame from the key table of `pan2ch_segments`, in ascending id order (add_frame_ids' order).
    A stuff category is one segment: its area is the sum over its keys and its bbox is the bbox of its LARGEST track key
    (the converter overwrites segm_info[colour] per key in ascending order, `last_key_ids`); a thing key is its own segment."""
    area, x0, y0, x1, y1 = (table[i] for i in range(5))
    info = []
    for sem in range(NSEM):
        trks = np.flatnonzero(area[sem])
        if len(trks) == 0:
            continue
        if sem < num_stuff:
            segs = [(1000 * sem + 1, int(area[sem].sum(dtype=np.int64)), int(trks[-1]))]
        else:
            segs = [(1000 * sem + int(t) + 1, int(area[sem, t]), int(t)) for t in trks.tolist()]
        for i, a, t in segs:
            x, y = int(x0[sem, t]), int(y0[sem, t])
            info.append({"category_id": sem, "iscrowd": 0, "id": i, "bbox": [x, y, int(x1[sem, t]) - x, int(y1[sem, t]) - y],
                         "area": a})
    return info


def image_segments_from_table(table, num_stuff=11):
    """segments_info of one image from the key table of `pan2ch_segments(..., image=True)`, as the image converter
    (_converter_2ch_single_core, base_dataset.py:287-335) makes it: one entry per key in ascending 1000 * semantic +
    instance order, each with the area and bbox of its own key.  The reference appends one entry per key rather than one
    per colour, so two keys of one stuff category (a fixed colour) give two entries with the same id 1000 * semantic + 1;
    a thing key's id is 1000 * semantic + instance + 1."""
    area, x0, y0, x1, y1 = (table[i] for i in range(5))
    info = []
    for sem, ins in zip(*(a.tolist() for a in np.nonzero(area))):
        x, y = int(x0[sem, ins]), int(y0[sem, ins])
        info.append({"category_id": sem, "iscrowd": 0, "id": 1000 * sem + (0 if sem < num_stuff else ins) + 1,
                     "bbox": [x, y, int(x1[sem, ins]) - x, int(y1[sem, ins]) - y], "area": int(area[sem, ins])})
    return info


def _save_png(path, img, palette=None):
    from PIL import Image
    os.makedirs(os.path.dirname(path), exist_ok=True)
    im = Image.fromarray(img)
    if palette is not None:
        im.putpalette(palette)
    im.save(path)


class _PngPool:
    """PNG encoding on `workers` threads with at most `max_queued` images queued, so host memory stays bounded; close()
    (also on leaving a `with` block) joins them, and a failed write is raised there or by a later submission."""

    def __init__(self, workers=4, max_queued=16):
        self.workers, self.max_queued = max(1, int(workers)), max(1, int(max_queued))
        self._pool, self._pending = None, deque()

    def __enter__(self):
        return self

    def __exit__(self, exc_type, exc, tb):
        # an exception already on its way out is not replaced by a failed PNG write
        self.close(raise_errors=exc_type is None)
        return False

    def _queue(self, jobs):
        """jobs: [(path, image) or (path, image, palette)]"""
        if self._pool is None:
            self._pool = ThreadPoolExecutor(max_workers=self.workers, thread_name_prefix="pan_writer")
        while self._pending and len(self._pending) + len(jobs) > self.max_queued:
            self._pending.popleft().result()
        for job in jobs:
            self._pending.append(self._pool.submit(_save_png, *job))

    def _drain(self, raise_errors=True):
        while self._pending:
            f = self._pending.popleft()
            if raise_errors:
                f.result()
            else:
                f.exception()                                      # wait for it, keep its error out of the way

    def close(self, raise_errors=True):
        """wait for the queued PNGs and stop the writer threads (the first failed write is raised unless raise_errors is
        False)"""
        try:
            self._drain(raise_errors)
        finally:
            self._pending.clear()
            if self._pool is not None:
                self._pool.shutdown(wait=True)
                self._pool = None


class PanWriter(_PngPool):
    """Feed the unified 3-channel results of a clip in order; sampled frames ([(labeled_fid // lambda_)::lambda_], :35) are
    converted and written to <output_dir>/pan_2ch/ and <output_dir>/pan_pred/; `finish()` writes pred.json.

    add_frame encodes its PNGs on `workers` threads with at most `max_pending` frames queued (each holds two host images),
    so host memory stays bounded; finish() or close() (also on leaving a `with` block) joins them, and a failed write is
    raised there or by a later add_frame."""

    def __init__(self, output_dir=None, labeled_fid=20, lambda_=5, sample=True, workers=4, max_pending=8):
        super().__init__(workers, 2 * max(1, int(max_pending)))
        self.output_dir = output_dir
        self.start, self.step = (labeled_fid // lambda_, lambda_) if sample else (0, 1)
        self.index = 0
        self.annotations, self.names = [], []

    def _submit(self, name, images):
        fn = _clean_name(name)
        self._queue([(os.path.join(self.output_dir, sub, fn), img) for sub, img in images])

    def _sampled(self):
        i = self.index
        self.index += 1
        return i >= self.start and (i - self.start) % self.step == 0

    def add_frame(self, name, pan_2ch, num_stuff=11, pan_2ch_host=None):
        """pan_2ch: uint8 tensor [H,W,3] (vps_b200.postproc.PanUnifier), on the device (ClipRunner's
        pano_results['pan_2ch_device']) or on the host (pano_results['pan_2ch']; it is then uploaded).  pan_2ch_host: a host
        copy of the same image, if the caller has one (pano_results['pan_2ch']): the pan_2ch PNG is encoded from it instead
        of downloading the device tensor.  Returns the frame's annotation or None if the frame is not a sampled one."""
        if not self._sampled():
            return None
        import torch
        if pan_2ch_host is None and not pan_2ch.is_cuda:
            pan_2ch_host = pan_2ch
        dev = pan_2ch if pan_2ch.is_cuda else pan_2ch.to(torch.device("cuda", torch.cuda.current_device()))
        table, rgb = pan2ch_segments(dev, num_stuff, rgb=self.output_dir is not None)
        ann = {"segments_info": segments_from_table(table, num_stuff)}
        self.annotations.append(ann)
        self.names.append(name)
        if self.output_dir is not None:
            p2 = pan_2ch.cpu().numpy() if pan_2ch_host is None else pan_2ch_host.numpy().copy()   # host buffers may be reused
            self._submit(name, (("pan_pred", rgb.cpu().numpy()), ("pan_2ch", p2)))
        return ann

    def add_frame_ids(self, name, ids, segs, pan_2ch=None, _counted=False, bbox_ids=None):
        """host part: ids [H,W] uint32 (0 = VOID), segs = [{id, category_id, iscrowd, area}] (any order); bbox_ids: id map
        restricted to the pixels the reference takes a segment's bbox from (`last_key_ids`), default = ids"""
        if not _counted and not self._sampled():
            return None
        from scipy import ndimage
        ids = np.asarray(ids)
        if bbox_ids is None and pan_2ch is not None:
            bbox_ids = last_key_ids(pan_2ch)
        box_src = ids if bbox_ids is None else np.asarray(bbox_ids)
        uniq = sorted(s["id"] for s in segs)
        # dense relabelling so that find_objects does not scan 19000 empty labels
        lut = np.zeros(int(ids.max()) + 1, dtype=np.int32)
        lut[np.asarray(uniq, dtype=np.int64)] = np.arange(1, len(uniq) + 1, dtype=np.int32)
        boxes = ndimage.find_objects(lut[box_src])
        by_id = {s["id"]: s for s in segs}
        info = []
        for rank, i in enumerate(uniq):
            sl = boxes[rank]
            y, x = sl[0].start, sl[1].start
            s = by_id[i]
            info.append({"category_id": int(s["category_id"]), "iscrowd": 0, "id": int(i),
                         "bbox": [int(x), int(y), int(sl[1].stop - 1 - x), int(sl[0].stop - 1 - y)], "area": int(s["area"])})
        ann = {"segments_info": info}
        self.annotations.append(ann)
        self.names.append(name)
        if self.output_dir is not None:
            from PIL import Image
            fn = _clean_name(name)
            for sub, img in (("pan_pred", id2rgb(ids)), ("pan_2ch", pan_2ch)):
                if img is None:
                    continue
                path = os.path.join(self.output_dir, sub, fn)
                os.makedirs(os.path.dirname(path), exist_ok=True)
                Image.fromarray(np.ascontiguousarray(img)).save(path)
        return ann

    def finish(self):
        self.close()
        pred_json = {"annotations": self.annotations}
        if self.output_dir is not None:
            os.makedirs(self.output_dir, exist_ok=True)
            with open(os.path.join(self.output_dir, "pred.json"), "w") as f:
                json.dump(pred_json, f)
        return pred_json


# get_pallete (tools/dataset/cityscapes.py:66-110): the Cityscapes colours of trainIds 0..18, every other entry black
CITYSCAPES_PALETTE = np.zeros((256, 3), np.uint8)
CITYSCAPES_PALETTE[:19] = [(128, 64, 128), (244, 35, 232), (70, 70, 70), (102, 102, 156), (190, 153, 153), (153, 153, 153),
                           (250, 170, 30), (220, 220, 0), (107, 142, 35), (152, 251, 152), (70, 130, 180), (220, 20, 60),
                           (255, 0, 0), (0, 0, 142), (0, 0, 70), (0, 60, 100), (0, 80, 100), (0, 0, 230), (119, 11, 32)]
CITYSCAPES_PALETTE = CITYSCAPES_PALETTE.reshape(-1)


def sseg_path(folder, name):
    """the palette PNG write_segmentation_result writes for the image `name` (cityscapes.py:180), replaces as written there"""
    return os.path.join(folder, name.replace('_leftImg8bit.png', '.png')).replace('_newImg8bit.png', '.png')


def pan_image_name(file_name):
    """the name evaluate_panoptic's save_image gives the PNGs of the GT json image `file_name` (base_dataset.py:158)"""
    return file_name.replace('_leftImg8bit', '').replace('jpg', 'png').replace('jpeg', 'png')


class ImageWriter(_PngPool):
    """The files tools/test_eval_ipq.py writes for the image panoptic model, image by image:
    * `add_sseg`: <sseg_dir>/<name>.png, the semantic map as a palette PNG (Cityscapes.write_segmentation_result);
    * `add_frame`: <output_dir>/pan_2ch/<name>.png and pan/<name>.png (evaluate_panoptic's save_image), and the image's
      segments_info (the image converter `_converter_2ch_single_core`, keyed on the instance channel).  The pan image is
      id2rgb of the converter's ids (`image_segments_from_table`), where the reference draws random panopticapi colours;
    * `finish(gt_json)`: <output_dir>/gt.json (a copy of the GT json) and pred.json.
    PNGs are encoded on `workers` threads with at most `max_pending` images queued (three PNGs each), as in PanWriter."""

    def __init__(self, output_dir=None, sseg_dir=None, workers=4, max_pending=8):
        super().__init__(workers, 3 * max(1, int(max_pending)))
        self.output_dir, self.sseg_dir = output_dir, sseg_dir
        self.annotations = []

    def add_sseg(self, name, fcn_output):
        """fcn_output: host label map [H,W] (a leading 1 is allowed), written as uint8 trainIds with the Cityscapes palette"""
        if self.sseg_dir is not None:
            img = np.asarray(fcn_output).squeeze().astype(np.uint8)
            self._queue([(sseg_path(self.sseg_dir, name), img, CITYSCAPES_PALETTE)])

    def add_frame(self, file_name, pan_2ch, num_stuff=11, pan_2ch_host=None):
        """file_name: the paired GT json image's file_name; pan_2ch: the image-level unified result (uint8 [H,W,3],
        PanUnifier(image=True)) on the device (ClipRunner's pano_results['pan_2ch_device']) or on the host (then uploaded);
        pan_2ch_host: a host copy of it, which the pan_2ch PNG is encoded from.  Returns the image's annotation."""
        import torch
        if pan_2ch_host is None and not pan_2ch.is_cuda:
            pan_2ch_host = pan_2ch
        dev = pan_2ch if pan_2ch.is_cuda else pan_2ch.to(torch.device("cuda", torch.cuda.current_device()))
        table, rgb = pan2ch_segments(dev, num_stuff, rgb=self.output_dir is not None, image=True)
        info = image_segments_from_table(table, num_stuff)
        if self.output_dir is not None:
            p2 = pan_2ch.cpu().numpy() if pan_2ch_host is None else pan_2ch_host.numpy().copy()   # host buffers may be reused
            return self._add(file_name, info, rgb.cpu().numpy(), p2)
        return self._add(file_name, info, None, None)

    def add_frame_ids(self, file_name, segments_info, ids, pan_2ch):
        """host part of add_frame: segments_info and ids [H,W] of the image converter (oracle.ipq.convert_image)"""
        return self._add(file_name, segments_info, None if self.output_dir is None else id2rgb(ids), pan_2ch)

    def _add(self, file_name, info, rgb, p2):
        ann = {"segments_info": info}
        self.annotations.append(ann)
        if self.output_dir is not None:
            fn = pan_image_name(file_name)
            self._queue([(os.path.join(self.output_dir, "pan_2ch", fn), np.ascontiguousarray(p2)),
                         (os.path.join(self.output_dir, "pan", fn), rgb)])
        return ann

    def finish(self, gt_json=None):
        """wait for the PNGs, write gt.json (when given) and pred.json; returns pred.json"""
        self.close()
        pred_json = {"annotations": self.annotations}
        if self.output_dir is not None:
            os.makedirs(self.output_dir, exist_ok=True)
            if gt_json is not None:
                with open(os.path.join(self.output_dir, "gt.json"), "w") as f:
                    json.dump(gt_json, f)
            with open(os.path.join(self.output_dir, "pred.json"), "w") as f:
                json.dump(pred_json, f)
        return pred_json
