"""pylayer.mask_layer.MaskLayer -- reference lib/pylayer/mask_layer.py: setup :22-29,
forward_train :56-93 and backward :50-54 (TRAIN, on the device: ops.mask_layer_train /
mask_layer_train_backward), forward_test :95-102 (a pure reshape (N,441) -> (N,1,21,21); the fused
engine never leaves the device for it)."""
import numpy as np
import torch

import caffe
from mnc_config import cfg
from mnc_b200 import ops


class MaskLayer(caffe.Layer):
    def setup(self, bottom, top):
        top[0].reshape(1, 1, cfg.MASK_SIZE, cfg.MASK_SIZE)
        if str(self.phase) == "TRAIN":
            top[1].reshape(1, 1)

    def forward(self, bottom, top):
        mask_pred = bottom[0].data
        n = mask_pred.shape[0]
        out = mask_pred.reshape((n, 1, cfg.MASK_SIZE, cfg.MASK_SIZE))
        top[0].reshape(*out.shape)
        top[0].data[...] = out
        if str(self.phase) != "TRAIN":
            return
        dev = torch.device("cuda", cfg.GPU_ID)
        t = lambda b: torch.from_numpy(np.ascontiguousarray(b.data, dtype=np.float32)).to(dev)
        with torch.cuda.device(dev):
            self._labels = ops.mask_layer_train(
                t(bottom[0]), t(bottom[1]), t(bottom[2]).view(-1, 12),
                binarize_thresh=cfg.BINARIZE_THRESH, fg_seg_thresh=cfg.TRAIN.FG_SEG_THRESH)
            labels = self._labels.cpu().numpy().reshape(-1, 1)
        top[1].reshape(*labels.shape)
        top[1].data[...] = labels

    def backward(self, top, propagate_down, bottom):
        """:50-54: the bottom diff is zeroed and written only when it is propagated."""
        if str(self.phase) != "TRAIN":
            return super(MaskLayer, self).backward(top, propagate_down, bottom)
        if not propagate_down[0]:
            return
        dev = torch.device("cuda", cfg.GPU_ID)
        with torch.cuda.device(dev):
            td = torch.from_numpy(np.ascontiguousarray(top[0].diff, dtype=np.float32)).to(dev)
            g = ops.mask_layer_train_backward(td.view(td.shape[0], 1, cfg.MASK_SIZE, cfg.MASK_SIZE),
                                              self._labels).cpu().numpy()
        b = bottom[0]
        if b.diff is None or b.diff.shape != b.data.shape:
            b.diff = np.zeros(b.data.shape, dtype=np.float32)
        b.diff[...] = g.reshape(b.data.shape)
