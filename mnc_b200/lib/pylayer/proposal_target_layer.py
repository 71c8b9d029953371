"""pylayer.proposal_target_layer.ProposalTargetLayer -- reference
lib/pylayer/proposal_target_layer.py:21-216 (setup, forward, backward; param_str_ keys num_classes
and bp_all, the reference's top map).  The body runs on the device (ops.proposal_target /
proposal_target_backward); its sampling keys are drawn with torch's generator on the device
(torch.manual_seed reproduces a run), or taken from `self.keys` when set (a recorded draw).  The
device writes the tops at a padded capacity; forward trims them to K with one synchronisation, so
the blob shapes are the reference's."""
import numpy as np
import torch
import yaml

import caffe
from mnc_config import cfg
from mnc_b200 import ops

_TOPS = ("rois", "labels", "bbox_targets", "bbox_inside_weights", "bbox_outside_weights",
         "mask_targets", "mask_weight", "gt_masks_info", "fg_inds", "bg_inds")


class ProposalTargetLayer(caffe.Layer):
    keys = None

    def setup(self, bottom, top):
        layer_params = yaml.safe_load(self.param_str_) if self.param_str_ else {}
        self._num_classes = layer_params["num_classes"]
        self._bp_all = layer_params.get("bp_all", True)
        M, C4 = cfg.MASK_SIZE, self._num_classes * 4
        shapes = [(1, 5), (1, 1), (1, C4), (1, C4), (1, C4)]
        if cfg.MNC_MODE:
            shapes += [(1, 1, M, M), (1, 1, M, M), (1, 4)]
            if cfg.TRAIN.MIX_INDEX:
                shapes += [(1, 4), (1, 4)]
        self._top_name_map = {k: i for i, k in enumerate(_TOPS[:len(shapes)])}
        for t, s in zip(top, shapes):
            t.reshape(*s)

    def reshape(self, bottom, top):
        """Reshaping happens during the call to forward."""
        pass

    def forward(self, bottom, top):
        dev = torch.device("cuda", cfg.GPU_ID)
        t = lambda b: torch.from_numpy(np.ascontiguousarray(b.data, dtype=np.float32)).to(dev)
        tr = cfg.TRAIN
        norm = tr.BBOX_NORMALIZE_TARGETS_PRECOMPUTED
        n = bottom[0].data.shape[0]
        G = bottom[1].data.shape[0]
        with torch.cuda.device(dev):
            index = t(bottom[5]).view(-1) if tr.MIX_INDEX else torch.zeros(n, device=dev)
            keys = self.keys if self.keys is not None else ops.sample_keys(
                len(tr.FG_FRACTION) + len(tr.BG_FRACTION), n + G, device=dev)
            out = ops.proposal_target(
                t(bottom[0]).view(-1, 5), index, t(bottom[1]), t(bottom[3]), t(bottom[4]).view(-1, 2),
                t(bottom[2]).view(-1)[:3], keys, batch_size=tr.BATCH_SIZE,
                fg_fraction=tr.FG_FRACTION, fg_thresh_lo=tr.FG_THRESH_LO,
                fg_thresh_hi=tr.FG_THRESH_HI, bg_fraction=tr.BG_FRACTION,
                bg_thresh_lo=tr.BG_THRESH_LO, bg_thresh_hi=tr.BG_THRESH_HI,
                means=tr.BBOX_NORMALIZE_MEANS if norm else None,
                stds=tr.BBOX_NORMALIZE_STDS if norm else None,
                inside_weights=tr.BBOX_INSIDE_WEIGHTS, mask_size=cfg.MASK_SIZE,
                binarize_thresh=cfg.BINARIZE_THRESH, num_classes=self._num_classes)
            self._state, self._n, self._G = out["state"], n, G
            K, nfg, nbg, _ = (int(v) for v in out["counts"].cpu())    # the one synchronisation
            blobs = {k: out[k][:K].cpu().numpy() for k in _TOPS[:8]}
            blobs["fg_inds"] = out["fg_inds"][:nfg].cpu().numpy()
            blobs["bg_inds"] = out["bg_inds"][:nbg].cpu().numpy()
        for name, i in self._top_name_map.items():
            top[i].reshape(*blobs[name].shape)
            top[i].data[...] = blobs[name]

    def backward(self, top, propagate_down, bottom):
        if not propagate_down[0]:
            return
        dev = torch.device("cuda", cfg.GPU_ID)
        Kmax = ops.proposal_target_capacity(cfg.TRAIN.BATCH_SIZE, cfg.TRAIN.FG_FRACTION,
                                            cfg.TRAIN.BG_FRACTION)
        d = np.zeros((Kmax, 5), np.float32)
        d[:top[0].diff.shape[0]] = top[0].diff.reshape(-1, 5)
        with torch.cuda.device(dev):
            rd = ops.proposal_target_backward(torch.from_numpy(d).to(dev), self._state, self._n,
                                              self._G, self._bp_all)
        b = bottom[0]
        if b.diff is None or b.diff.shape != b.data.shape:
            b.diff = np.zeros(b.data.shape, dtype=np.float32)
        b.diff[...] = rd.cpu().numpy().reshape(b.data.shape)   # in place: pycaffe's diff is read-only
