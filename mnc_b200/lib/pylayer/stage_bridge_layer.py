"""pylayer.stage_bridge_layer.StageBridgeLayer -- reference lib/pylayer/stage_bridge_layer.py:
setup :26-63, forward_train :131-235 and backward :82-129 (TRAIN), forward_test :237-255 (TEST);
the bodies run on the device (ops.stage_bridge_train / stage_bridge_train_backward / stage_bridge)."""
import numpy as np
import torch
import yaml

import caffe
from mnc_config import cfg
from mnc_b200 import ops

_TRAIN_TOPS = ("rois", "labels", "mask_targets", "mask_weight", "gt_mask_info", "bbox_targets",
               "bbox_inside_weights", "bbox_outside_weights")


class StageBridgeLayer(caffe.Layer):
    def setup(self, bottom, top):
        self._phase = str(self.phase)
        if self._phase == "TRAIN":
            p = yaml.safe_load(self.param_str_) if self.param_str_ else {}
            self._use_clip = p["use_clip"]
            self._clip_denominator = float(p.get("clip_base", 64))
            self._clip_thresh = 1.0 / self._clip_denominator
            self._num_classes = p["num_classes"]
            self._top_name_map = {k: i for i, k in enumerate(_TRAIN_TOPS)}
            shapes = ((1, 5), (1, 1), (1, 1, cfg.MASK_SIZE, cfg.MASK_SIZE),
                      (1, 1, cfg.MASK_SIZE, cfg.MASK_SIZE), (1, 4), (1, self._num_classes * 4),
                      (1, self._num_classes * 4), (1, self._num_classes * 4))
            for t, s in zip(top, shapes):
                t.reshape(*s)
        else:
            top[0].reshape(1, 5)

    def forward(self, bottom, top):
        if str(self.phase) == "TRAIN":
            return self._forward_train(bottom, top)
        dev = torch.device("cuda", cfg.GPU_ID)
        t = lambda b: torch.from_numpy(np.ascontiguousarray(b.data, dtype=np.float32)).to(dev)
        rois, deltas, scores, im_info = t(bottom[0]), t(bottom[1]), t(bottom[2]), t(bottom[3])
        with torch.cuda.device(dev):
            out = ops.stage_bridge(rois.view(-1, 5), deltas, scores, im_info.view(-1, 3),
                                   rois.shape[0])
            blob = out.cpu().numpy()
        blob[:, 0] = 0
        top[0].reshape(*blob.shape)
        top[0].data[...] = blob

    def _forward_train(self, bottom, top):
        dev = torch.device("cuda", cfg.GPU_ID)
        t = lambda b: torch.from_numpy(np.ascontiguousarray(b.data, dtype=np.float32)).to(dev)
        norm = cfg.TRAIN.BBOX_NORMALIZE_TARGETS_PRECOMPUTED
        with torch.cuda.device(dev):
            self._rois = t(bottom[0]).view(-1, 5)
            self._deltas = t(bottom[1])
            out = ops.stage_bridge_train(
                self._rois, self._deltas, t(bottom[2]), t(bottom[3]), t(bottom[4]),
                t(bottom[5]).view(-1)[:3], t(bottom[6]).view(-1, 2),
                means=cfg.TRAIN.BBOX_NORMALIZE_MEANS if norm else None,
                stds=cfg.TRAIN.BBOX_NORMALIZE_STDS if norm else None,
                inside_weights=cfg.TRAIN.BBOX_INSIDE_WEIGHTS, bbox_thresh=cfg.TRAIN.BBOX_THRESH,
                mask_size=cfg.MASK_SIZE, binarize_thresh=cfg.BINARIZE_THRESH)
            self._state, self._G = out["state"], bottom[3].data.shape[0]
            for name in _TRAIN_TOPS:
                blob = out[name].cpu().numpy()
                top[self._top_name_map[name]].reshape(*blob.shape)
                top[self._top_name_map[name]].data[...] = blob

    def backward(self, top, propagate_down, bottom):
        """:82-129: a bottom diff is zeroed and written only when it is propagated."""
        if str(self.phase) != "TRAIN":
            return super(StageBridgeLayer, self).backward(top, propagate_down, bottom)
        want_r, want_b = bool(propagate_down[0]), bool(propagate_down[1])
        if not (want_r or want_b):
            return
        dev = torch.device("cuda", cfg.GPU_ID)
        with torch.cuda.device(dev):
            td = torch.from_numpy(np.ascontiguousarray(top[0].diff, dtype=np.float32)).to(dev)
            rd, bd = ops.stage_bridge_train_backward(
                td.view(-1, 5), self._state, self._rois, self._deltas, self._G,
                self._clip_thresh if self._use_clip else 0.0, want_rois=want_r, want_bbox=want_b)
            for i, g in ((0, rd), (1, bd)):
                if g is not None:
                    b = bottom[i]
                    if b.diff is None or b.diff.shape != b.data.shape:
                        b.diff = np.zeros(b.data.shape, dtype=np.float32)
                    b.diff[...] = g.cpu().numpy().reshape(b.data.shape)
