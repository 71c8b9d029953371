"""pylayer.anchor_target_layer.AnchorTargetLayer -- reference lib/pylayer/anchor_target_layer.py:
19-213 (setup, forward; param_str_ keys feat_stride and allowed_border; the backward does
nothing).  The body runs on the device (ops.anchor_target); its sampling keys are drawn with
torch's generator on the device, or taken from `self.keys` when set (a recorded draw)."""
import numpy as np
import torch
import yaml

import caffe
from mnc_config import cfg
from mnc_b200 import ops


class AnchorTargetLayer(caffe.Layer):
    keys = None

    def setup(self, bottom, top):
        layer_params = yaml.safe_load(self.param_str_) if self.param_str_ else {}
        self._feat_stride = layer_params["feat_stride"]
        self._allowed_border = layer_params.get("allowed_border", 0)
        self._num_anchors = 9
        H, W = bottom[0].data.shape[-2:]
        A = self._num_anchors
        top[0].reshape(1, 1, A * H, W)
        for t in top[1:4]:
            t.reshape(1, A * 4, H, W)

    def reshape(self, bottom, top):
        """Reshaping happens during the call to forward"""
        pass

    def forward(self, bottom, top):
        assert bottom[0].data.shape[0] == 1, 'Only single item batches are supported'
        H, W = bottom[0].data.shape[-2:]
        dev = torch.device("cuda", cfg.GPU_ID)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)
        tr = cfg.TRAIN
        with torch.cuda.device(dev):
            fg = bg = counts = None
            if tr.MIX_INDEX:
                fg, bg = t(bottom[3].data).view(-1), t(bottom[4].data).view(-1)
                cap = max(fg.numel(), bg.numel(), 1)
                fg = torch.cat([fg, fg.new_full((cap - fg.numel(),), -1.0)])
                bg = torch.cat([bg, bg.new_full((cap - bg.numel(),), -1.0)])
                counts = torch.tensor([0, bottom[3].data.size, bottom[4].data.size, 0],
                                      dtype=torch.int32, device=dev)
            keys = self.keys if self.keys is not None else ops.sample_keys(
                H * W * self._num_anchors, device=dev)
            tops = ops.anchor_target(
                H, W, t(bottom[1].data), t(bottom[2].data).view(-1)[:3], keys, fg, bg, counts,
                feat_stride=self._feat_stride, allowed_border=self._allowed_border,
                negative_overlap=tr.RPN_NEGATIVE_OVERLAP, positive_overlap=tr.RPN_POSITIVE_OVERLAP,
                clobber_positives=tr.RPN_CLOBBER_POSITIVES, fg_fraction=tr.RPN_FG_FRACTION,
                batch_size=tr.RPN_BATCHSIZE, positive_weight=tr.RPN_POSITIVE_WEIGHT,
                inside_weights=tr.RPN_BBOX_INSIDE_WEIGHTS)
            for i, x in enumerate(tops):
                blob = x.cpu().numpy()
                top[i].reshape(*blob.shape)
                top[i].data[...] = blob

    def backward(self, top, propagate_down, bottom):
        """This layer does not propagate gradients."""
        pass
