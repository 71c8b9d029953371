"""pylayer.proposal_layer.ProposalLayer -- reference lib/pylayer/proposal_layer.py:21-230.

Same caffe.Layer protocol (param_str_ YAML with feat_stride, use_clip, clip_base; setup / reshape /
forward / backward, tops reshaped inside forward), but the body runs on the device: decode + clip +
min-size filter, rank sort, top-N, bitmask NMS with device-side scan, top-N (TEST and TRAIN), plus,
in TRAIN, the proposal_index top (cfg.TRAIN.MIX_INDEX) and the backward into rpn_bbox_pred
(ops.proposal_train / proposal_backward)."""
import numpy as np
import torch
import yaml

import caffe
from mnc_config import cfg
from mnc_b200 import ops


class ProposalLayer(caffe.Layer):
    def setup(self, bottom, top):
        layer_params = yaml.safe_load(self.param_str_) if self.param_str_ else {}
        self._feat_stride = layer_params.get("feat_stride", 16)
        self._num_anchors = 9
        self._use_clip = layer_params.get("use_clip", 0)
        self._clip_thresh = 1.0 / float(layer_params.get("clip_base", 256))
        self._top_name_map = {"rois": 0}
        top[0].reshape(1, 5)
        if str(self.phase) == "TRAIN" and cfg.TRAIN.MIX_INDEX:
            top[1].reshape(1, 1)
            self._top_name_map["proposal_index"] = 1

    def reshape(self, bottom, top):
        """Reshaping happens during the call to forward."""
        pass

    def forward(self, bottom, top):
        assert bottom[0].data.shape[0] == 1, 'Only single item batches are supported'
        cfg_key = str(self.phase)
        c = cfg[cfg_key]
        dev = torch.device("cuda", cfg.GPU_ID)
        cls = torch.from_numpy(np.ascontiguousarray(bottom[0].data, dtype=np.float32)).to(dev)
        bbox = torch.from_numpy(np.ascontiguousarray(bottom[1].data, dtype=np.float32)).to(dev)
        im_info = torch.from_numpy(np.ascontiguousarray(bottom[2].data, dtype=np.float32)).to(dev)
        H, W = cls.shape[-2:]
        with torch.cuda.device(dev):
            if cfg_key == "TRAIN":
                rois, index, counts, self._state = ops.proposal_train(
                    cls, bbox, im_info.view(-1)[:3], H, W, pre_nms_top_n=c.RPN_PRE_NMS_TOP_N,
                    post_nms_top_n=c.RPN_POST_NMS_TOP_N, nms_thresh=c.RPN_NMS_THRESH,
                    min_size=float(c.RPN_MIN_SIZE), feat_stride=self._feat_stride)
                self._bbox = bbox
                rois = rois[None]
            else:
                rois, counts = ops.proposals_from_rpn(
                    cls, bbox, im_info.view(-1, 3), 1, H, W, "nchw", apply_softmax=False,
                    pre_nms_top_n=c.RPN_PRE_NMS_TOP_N, post_nms_top_n=c.RPN_POST_NMS_TOP_N,
                    nms_thresh=c.RPN_NMS_THRESH, min_size=float(c.RPN_MIN_SIZE),
                    batch_index_mode=False)
            n = int(counts[0].item())
            blobs = {"rois": rois[0, :n].cpu().numpy()}
            if cfg_key == "TRAIN" and cfg.TRAIN.MIX_INDEX:
                blobs["proposal_index"] = index[:n].cpu().numpy().reshape(1, n)
        for name, blob in blobs.items():
            top[self._top_name_map[name]].reshape(*blob.shape)
            top[self._top_name_map[name]].data[...] = blob

    def backward(self, top, propagate_down, bottom):
        if str(self.phase) != "TRAIN":
            raise NotImplementedError("ProposalLayer has no backward in TEST")
        if not propagate_down[1]:
            return
        dev = torch.device("cuda", cfg.GPU_ID)
        R = self._state.shape[0]
        d = np.zeros((R, 5), np.float32)
        d[:top[0].diff.shape[0]] = top[0].diff
        with torch.cuda.device(dev):
            out = ops.proposal_backward(torch.from_numpy(d).to(dev), self._state, self._bbox,
                                        self._clip_thresh if self._use_clip else 0.0)
        b = bottom[1]
        if b.diff is None or b.diff.shape != b.data.shape:
            b.diff = np.zeros(b.data.shape, dtype=np.float32)
        b.diff[...] = out.cpu().numpy().reshape(b.data.shape)   # in place: pycaffe's diff is read-only
