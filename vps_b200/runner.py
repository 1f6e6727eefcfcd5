"""Clip inference loop: the host side of `single_gpu_test` (reference tools/test_vpq.py:27-63 -- iterate the loader,
`model(return_loss=False, rescale=True, **data)`, collect the results) with the two copies a loader + collector do
around the model call made asynchronous:

  * the NEXT pair's frames are uploaded from pinned host memory on a copy stream while the current pair computes
    (what `DataLoader(pin_memory=True)` + `non_blocking` gives a user of the reference), and
  * the label maps of the finished pair are downloaded into pinned buffers on the same copy stream, so the next
    pair's kernels do not wait for the D2H.

  * the tracker-independent static part of the NEXT pair (`det.prefetch`: one CUDA-graph replay on a side stream, two
    graph instances ping-pong) is enqueued before the current pair's data-dependent tail, so the tail and its host
    round-trips overlap the next pair's graph.

Nothing about the model call changes: `det.simple_test` is the same entry the parity tests use.

The loop serves all three detectors.  PanopticTrack reads the current frame only: its pairs are `(img, None)`, and no
reference frame is uploaded or normalised.  PanopticFuse has no tracker: with `unify` it gets the image-level unified
result (`PanUnifier(image=True)`)."""
import torch

from .pipeline import GEOMETRY_KEYS


class ClipRunner:
    def __init__(self, det, device=None, depth=2, unify=False, streaming=False, input_stage=None):
        self.det = det
        # input_stage: a vps_b200.pipeline.InputStage -- the pairs are then decoded uint8 HWC BGR frames (what the reference's
        # loader produces before Normalize / Pad / ImageToTensor); they are uploaded as uint8 (4x fewer bytes) and normalised,
        # padded and transposed on the device; a stage with resize=True also resizes them, and its geometry fields replace the
        # caller's in the meta handed to the detector
        self.input_stage = input_stage
        self._f32, self._nf32 = [], 0
        # streaming: every pair's reference frame is the previous pair's current frame (the clip chain of
        # tools/dataset/cityscapes_vps.py:137-142; the first frame of a clip, iid % 10000 == 1, references itself): the
        # previous pair's FPN features are reused as the reference features -- half the backbone work, identical results
        self.streaming = streaming
        self._prev_feats = None
        # unify: also run get_unified_pan_result (tools/dataset/cityscapes_vps.py:162-226) on the GPU for every pair
        # (vps_b200.postproc.PanUnifier) and return the uint8 [H,W,3] image as pano_results['pan_2ch'] (host); a detector
        # without a tracker gets the image-level function (tools/dataset/base_dataset.py:232-274)
        self.unifier = None
        if unify:
            from .postproc import PanUnifier
            self.unifier = PanUnifier(image=not det.with_track)
        self._out2 = []
        self._err = None
        self.dev = torch.device(device) if device is not None else next(det.parameters()).device
        self.copy = torch.cuda.Stream(self.dev)
        self.depth = depth
        self._out = []          # ring of pinned (pano, sem) host buffers
        self._in, self._nup = [], 0   # ring of device input buffers

    def _upload(self, pair):
        """H2D into a fixed ring of device buffers (no allocation in steady state).  Slot reuse is safe with 3 slots: the
        upload of pair i+3 is issued after simple_test(i) returned, i.e. after everything that read slot i finished."""
        main = torch.cuda.current_stream(self.dev)
        slot = self._nup % 3
        self._nup += 1
        while len(self._in) <= slot:
            self._in.append(None)
        bufs = self._in[slot]
        if bufs is None or any((b is None) != (p is None) or (p is not None and (b.shape != p.shape or b.dtype != p.dtype))
                               for b, p in zip(bufs, pair)):
            bufs = self._in[slot] = tuple(None if p is None else torch.empty(p.shape, dtype=p.dtype, device=self.dev)
                                          for p in pair[:2])
        with torch.cuda.stream(self.copy):
            for b, p in zip(bufs, pair):
                if p is not None:                           # (img, None): a detector that reads the current frame only
                    b.copy_(p, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.copy)
        return bufs[0], bufs[1], ev

    def _host_buf(self, i, like):
        k = i % (self.depth + 1)
        while len(self._out) <= k:
            self._out.append(None)
        buf = self._out[k]
        if buf is None or buf[0].shape != like.shape or buf[0].dtype != like.dtype:
            buf = (torch.empty(like.shape, dtype=like.dtype).pin_memory(), torch.empty(like.shape, dtype=like.dtype).pin_memory(),
                   torch.cuda.Event())
            self._out[k] = buf
        return buf

    def _prefetch(self, staged, meta):
        """enqueue the static part of a pair; in streaming mode the previous ENQUEUED pair's features are its reference
        features (they are produced on the same side stream, in order)"""
        feats = None
        ref = [staged[1]] if staged[1] is not None else None
        if self.streaming and (meta['iid'] % 10000) != 1 and self.det._pf_queue:
            feats = self.det._pf_queue[-1][2]['x']
        elif self.streaming and (meta['iid'] % 10000) != 1:
            feats = self._prev_feats
        self.det.prefetch(staged[0], [meta], ref_img=ref, ref_feats=feats)
        if self.streaming:
            self._prev_feats = self.det._pf_queue[-1][2]['x'] if self.det._pf_queue else None

    def _normalise(self, staged, meta):
        """uint8 HWC device frames -> fp32 NCHW padded tensors (ring of 3 like the upload ring) and the pair's meta: when the
        stage resizes, its ori_shape / img_shape / pad_shape / scale_factor replace the caller's (filename / iid stay)"""
        slot = self._nf32 % 3
        self._nf32 += 1
        while len(self._f32) <= slot:
            self._f32.append([None, None])
        ring = self._f32[slot]
        for k in (0, 1):                            # a buffer is reused only for the output shape it was made for
            if ring[k] is not None and (staged[k] is None or tuple(ring[k].shape[2:]) !=
                                        self.input_stage.geometry(int(staged[k].shape[0]), int(staged[k].shape[1]))[2:4]):
                ring[k] = None
        a, b, m = self.input_stage.pair(staged[0], staged[1], outs=ring)
        ring[0], ring[1] = a, b
        if self.input_stage.resize:
            meta = dict(meta, **{k: m[k] for k in GEOMETRY_KEYS})
        return (a, b, None), meta

    def _stage(self, pair, resident):
        """make the pair available on the device: (img, ref, event or None)"""
        if resident:
            return pair[0], pair[1], None
        return self._upload(pair)

    def run(self, pairs, metas, resident=False, prefetch=True):
        """pairs: iterable of (img, ref_img) pinned host tensors [1,3,H,W] fp32 (device tensors if `resident`; ref_img is
        None for a detector that reads the current frame only, PanopticTrack); metas:
        matching img_meta dicts.  Yields (bbox_results, segm_results, pano_results) per pair, in order;
        pano_results['panoptic_outputs'] and ['fcn_outputs'] are HOST tensors in a ring of depth + 1 pinned buffers: the
        download of pair i + depth + 1 reuses the slot of pair i and is issued right before result i + depth is yielded, so a
        result stays valid while the next `depth - 1` results are consumed (depth = 2: the previous result may still be
        read while the current one is processed); clone to keep results longer.  With `prefetch` the tracker-independent static part of pair i+1
        (`det.prefetch`) is enqueued before pair i's data-dependent tail runs, so the two overlap."""
        main = torch.cuda.current_stream(self.dev)
        it = iter(zip(pairs, metas))
        cur = next(it, None)
        if cur is None:
            return
        staged = self._stage(cur[0], resident)
        if staged[2] is not None:
            main.wait_event(staged[2])
        if self.input_stage is not None:
            staged, m = self._normalise(staged, cur[1])
            cur = (cur[0], m)
        self._prev_feats = None
        self._chain = []        # streaming: static-part outputs of enqueued pairs, in order (their 'x' feeds the next pair)
        if prefetch:
            self._prefetch(staged, cur[1])
        pending = None
        i = 0
        while cur is not None:
            a, b, _ = staged
            meta = cur[1]
            cur = next(it, None)
            if cur is not None:
                staged = self._stage(cur[0], resident)          # upload overlaps the compute already in flight
                if staged[2] is not None:
                    main.wait_event(staged[2])
                if self.input_stage is not None:
                    staged, m = self._normalise(staged, cur[1])
                    cur = (cur[0], m)
                if prefetch:
                    self._prefetch(staged, cur[1])
            rb = [b] if b is not None else None
            if prefetch or not self.streaming:
                r = self.det.simple_test(a, [meta], ref_img=rb)
            else:
                first = (meta['iid'] % 10000) == 1
                r = self.det.simple_test(a, [meta], ref_img=rb, ref_feats=None if first else self._prev_feats)
                self._prev_feats = r[2]['fpn_feats']
            pano, sem = r[2]["panoptic_outputs"], r[2]["fcn_outputs"]
            p2 = None
            if self.unifier is not None:
                hk = r[2].get("host", {})
                p2 = self.unifier(sem, pano, hk.get("panoptic_cls_inds", r[2]["panoptic_cls_inds"]),
                                  hk.get("panoptic_det_obj_ids", r[2].get("panoptic_det_obj_ids")))
            done = torch.cuda.Event()
            done.record(main)
            hp, hs, hev = self._host_buf(i, pano)
            h2 = None
            if p2 is not None:
                k2 = i % (self.depth + 1)
                while len(self._out2) <= k2:
                    self._out2.append(None)
                h2 = self._out2[k2]
                if h2 is None or h2.shape != p2.shape:
                    h2 = self._out2[k2] = torch.empty(p2.shape, dtype=torch.uint8).pin_memory()
            herr = None
            if p2 is not None:
                if self._err is None:
                    self._err = [torch.zeros(1, dtype=torch.int32).pin_memory() for _ in range(self.depth + 1)]
                herr = self._err[i % (self.depth + 1)]
            with torch.cuda.stream(self.copy):
                self.copy.wait_event(done)
                hp.copy_(pano, non_blocking=True)
                hs.copy_(sem, non_blocking=True)
                if p2 is not None:
                    h2.copy_(p2, non_blocking=True)
                    herr.copy_(self.unifier.error_word(), non_blocking=True)     # flag of this frame, read without a sync
                hev.record(self.copy)
            pano.record_stream(self.copy)
            sem.record_stream(self.copy)
            if p2 is not None:
                p2.record_stream(self.copy)
                r[2]["pan_2ch"] = h2
            if pending is not None:
                pending[1].synchronize()               # the previous pair's maps are on the host now
                self._raise_if_flagged(pending[2])
                yield pending[0]

            r[2]["panoptic_outputs"], r[2]["fcn_outputs"] = hp, hs
            pending = (r, hev, herr)
            i += 1
        pending[1].synchronize()
        self._raise_if_flagged(pending[2])
        yield pending[0]

    @staticmethod
    def _raise_if_flagged(herr):
        if herr is not None and int(herr[0]) != 0:      # what the reference raises (cityscapes_vps.py:197)
            raise IndexError("get_unified_pan_result: panoptic instance id beyond len(cls_ind)")
