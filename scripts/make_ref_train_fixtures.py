#!/usr/bin/env python
"""Run the REFERENCE's own TRAIN-phase bridge layers and freeze what they produce as golden
fixtures: tests/golden/ref_train_bridge.npz (+ .partN.npz).

TEST INFRASTRUCTURE, like scripts/make_ref_fixtures.py, whose reference environment and import
hook it reuses (same shims, same reference files unmodified on disk):
  lib/pylayer/stage_bridge_layer.py   StageBridgeLayer.setup / forward (TRAIN) / backward  :26-235
  lib/pylayer/mask_layer.py           MaskLayer.setup / forward (TRAIN) / backward         :22-93
  lib/transform/bbox_transform.py     bbox_transform_inv / clip_boxes / bbox_compute_targets /
                                      get_bbox_regression_label
  lib/transform/mask_transform.py     intersect_mask / mask_overlap
  lib/utils/bbox.pyx                  bbox_overlaps (oracle/_ref/cython_bbox.so)

Two more numpy-version shims, both float-index semantics numpy 1.x accepted and numpy 2 rejects:
  * bbox_transform.py:199 `start = 4 * cls` with cls a float32 slices bbox_targets; numpy 2 raises
    TypeError.  The import hook rewrites that line to `start = int(4 * cls)` (the truncation
    numpy 1.x applied).
  * stage_bridge_layer.py:224 `gt_mask[0:gt_mask_info[0], ...]` and mask_layer.py:75
    `gt_masks[info[0]]` index with blob values.  The stub blobs for mask_info and gt_masks_info
    hold integers (the values are integral, so nothing else changes).

Cases (seeded, oracle_train.make_case): the training shape (600x1000 at im_scale 1.6, 64 RoIs,
3 gt, BBOX_NORMALIZE_TARGETS_PRECOMPUTED on, use_clip on with clip_base 512), a second scale
(500x800 at 1.0, 48 RoIs, 5 gt, PRECOMPUTED off, use_clip off) and n = 0.  Seeds are chosen so
that every decision keeps a margin: max overlap vs BBOX_THRESH, resized mask values vs
BINARIZE_THRESH, region IoU vs FG_SEG_THRESH, bbox_pred diffs vs the clip threshold.  The MaskLayer
input of each case gets one foreground row whose ex box is moved off its gt box (empty box
intersection).  Top diffs are ~1e-5 so that some bbox_pred diffs clamp and some do not.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True

from scripts import make_ref_fixtures as MR   # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ref_train_bridge.npz")
MARGIN = 1e-6
CASES = {   # name: (make_case kwargs, PRECOMPUTED, use_clip)
    "A": (dict(H=600, W=1000, im_scale=1.6, n=64, G=3), True, 1),
    "B": (dict(H=500, W=800, im_scale=1.0, n=48, G=5), False, 0),
    "C": (dict(H=600, W=1000, im_scale=1.6, n=0, G=2), True, 1),
}


def _patch_hook():
    orig = MR._RefLoader.source_to_code

    def source_to_code(self, data, path, *, _optimize=-1):
        if path.endswith(os.path.join("transform", "bbox_transform.py")):
            src = data.decode()
            assert src.count("start = 4 * cls") == 1
            data = src.replace("start = 4 * cls", "start = int(4 * cls)").encode()
        return orig(self, data, path, _optimize=_optimize)
    MR._RefLoader.source_to_code = source_to_code


class Blob(MR.Blob):
    """A blob with .diff, holding `dtype` (float32 unless an integer blob is asked for)."""

    def __init__(self, data=None, dtype=np.float32):
        self.data = np.zeros((1,), dtype) if data is None else np.ascontiguousarray(data, dtype)
        self.diff = np.zeros(self.data.shape, np.float32)

    def reshape(self, *dims):
        if tuple(dims) != self.data.shape:
            self.data = np.zeros(dims, np.float32)
            self.diff = np.zeros(dims, np.float32)


def margins_ok(case, out, pred, tops, top_diff, clip_thresh):
    from oracle import oracle_train as T
    if out["max_overlaps"].size and np.abs(out["max_overlaps"] - 0.5).min() < MARGIN:
        return False
    tv = T.target_values(case, out)
    if tv.size and np.abs(tv - 0.4).min() < MARGIN:
        return False
    rv = T.resize_values(pred, tops)
    if rv.size and np.abs(rv - 0.4).min() < MARGIN:
        return False
    _, bd = T.stage_bridge_backward(top_diff, out, case["rois"], case["bbox_pred"], 0.0,
                                    want_rois=False)
    if clip_thresh and np.any(np.abs(np.abs(bd[bd != 0]) - clip_thresh) < 1e-5 * clip_thresh):
        return False
    return True


def main():
    _patch_hook()
    caffe = MR.install_reference_environment({"nms": [], "mv": []})
    from mnc_config import cfg                      # reference lib/mnc_config.py
    from pylayer.stage_bridge_layer import StageBridgeLayer
    from pylayer.mask_layer import MaskLayer
    from oracle import oracle_train as T
    assert caffe is sys.modules["caffe"]
    fx = {}
    for name, (kw, precomputed, use_clip) in CASES.items():
        cfg.TRAIN.BBOX_NORMALIZE_TARGETS_PRECOMPUTED = precomputed
        for seed in range(100):
            case = T.make_case(seed, **kw)
            sb = StageBridgeLayer()
            sb.phase = "TRAIN"
            sb.param_str_ = "{ 'feat_stride': 16, 'use_clip': %d, 'clip_base': 512, 'num_classes': 21}" % use_clip
            bottom = [Blob(case["rois"]), Blob(case["bbox_pred"]), Blob(case["seg_cls_prob"]),
                      Blob(case["gt_boxes"]), Blob(case["gt_masks"]), Blob(case["im_info"][None]),
                      Blob(case["mask_info"], np.int64)]
            top = [Blob() for _ in range(8)]
            sb.setup(bottom, top)
            sb.forward(bottom, top)
            out = T.stage_bridge_forward(**case, num_classes=21, normalize=precomputed)
            K = top[0].data.shape[0]
            rng = np.random.default_rng(1000 + seed)
            top[0].diff = (rng.normal(0, 1e-5, (K, 5))).astype(np.float32)
            sb.backward(top, [True, True], bottom)

            info = top[4].data.copy()
            pred = T.mask_predictions(seed, top[2].data, info)
            if out["nfg"] > 1:                       # empty box intersection in MaskLayer
                info[1, 4:8] = info[1, 8:12] + np.float32(1000)
            ml = MaskLayer()
            ml.phase = "TRAIN"
            mb = [Blob(pred), Blob(case["gt_masks"]), Blob(info, np.int64)]
            mt = [Blob(), Blob()]
            ml.setup(mb, mt)
            ml.forward(mb, mt)
            mt[0].diff = rng.normal(0, 1, mt[0].data.shape).astype(np.float32)
            ml.backward(mt, [True], mb)
            clip = 1.0 / 512 if use_clip else 0.0
            if margins_ok(case, out, pred, info, top[0].diff, clip):
                break
        else:
            raise RuntimeError("no seed with margins for case %s" % name)
        print("case %s: seed %d, K %d, nfg %d" % (name, seed, K, out["nfg"]))
        p = name + "_"
        for k in ("rois", "bbox_pred", "seg_cls_prob", "gt_boxes", "im_info", "mask_info"):
            fx[p + k] = case[k]
        fx[p + "gt_masks"] = case["gt_masks"].astype(bool)
        fx[p + "cfg"] = np.array([precomputed, use_clip, 512, 21], np.int64)
        for i, k in enumerate(T_TOPS):
            fx[p + "top_" + k] = top[i].data
        fx[p + "keep_inds"] = np.asarray(sb._keep_inds, np.int64)
        fx[p + "reg_labels"] = np.asarray(sb._bbox_reg_labels, np.int64)
        fx[p + "clip_keep"] = np.asarray(sb._clip_keep, np.int64)
        fx[p + "top_diff"] = top[0].diff
        fx[p + "rois_diff"] = bottom[0].diff
        fx[p + "bbox_pred_diff"] = bottom[1].diff
        fx[p + "ml_pred"] = pred
        fx[p + "ml_info"] = info
        fx[p + "ml_labels"] = mt[1].data
        fx[p + "ml_top_diff"] = mt[0].diff
        fx[p + "ml_bottom_diff"] = mb[0].diff
    MR.save_parts(OUT, fx)
    print("wrote", OUT)


T_TOPS = ("rois", "labels", "mask_targets", "mask_weight", "gt_mask_info", "bbox_targets",
          "bbox_inside_weights", "bbox_outside_weights")

if __name__ == "__main__":
    main()
