#!/usr/bin/env python
"""Run the REFERENCE's own TRAIN-phase RPN-stage layers and freeze what they produce as golden
fixtures: tests/golden/ref_rpn_train.npz (+ .partN.npz).

TEST INFRASTRUCTURE, like scripts/make_ref_train_fixtures.py, whose Blob and (through it)
scripts/make_ref_fixtures.py's reference environment and import hook it reuses:
  lib/pylayer/proposal_layer.py          ProposalLayer.setup / forward (TRAIN) / backward  :27-230
  lib/pylayer/proposal_target_layer.py   ProposalTargetLayer.setup / forward / backward    :26-216
  lib/pylayer/anchor_target_layer.py     AnchorTargetLayer.setup / forward                 :25-209
  lib/transform/bbox_transform.py, mask_transform.py, lib/utils/bbox.pyx, lib/utils/unmap.py
NMS inside ProposalLayer is answered by make_ref_fixtures' recording stand-in (py_cpu_nms).

Shims, each touching one line of the reference:
  (a) sampling.  npr.choice(cands, size, replace=False) (proposal_target_layer.py:139, :152) and
      np.random.choice (anchor_target_layer.py:126, :134) become oracle_rpn_train.choice: the
      `size` candidates with the smallest (key, index) pairs for the case's keys.  The import hook
      adds `key_row=i` (fg loop) / `key_row=len(cfg.TRAIN.FG_FRACTION) + i` (bg loop) to the two
      proposal_target_layer.py calls, so each category reads its own key row; AnchorTargetLayer's
      calls read the anchor keys of the candidates (positions in inds_inside, which is sorted, so
      position order is anchor order).
  (b) proposal_layer.py:196-197 `unmap_val / self._num_anchors` and `/ self._width`: Python 2
      integer division, written `//`.
  (c) proposal_target_layer.py:190,193,194,201 `gt_assignment[val]` with the float64 values
      np.hstack(([], ...)) gives fg_inds: numpy >= 1.12 rejects float indices; `int(val)`.
  (d) bbox_transform.py:199 `start = 4 * cls` (float32 slice bound), `int(4 * cls)`, and the
      mask_info blob holding integers -- the two numpy-2 shims make_ref_train_fixtures documents.

Cases (seeded): A the training shape (600x1000 at im_scale 1.6, 38x63 map, 300 proposals, 3 gt,
use_clip, bp_all 1, targets normalised); B a second scale (480x800 at 1.0, 30x50 map, 12 gt,
bp_all 0, no clip, not normalised) with an RoI at IoU exactly 50/100 to a gt box whose bg key is 0
(it is sampled as fg and bg: a duplicate keep index); C n = 0 (gt rows only); D a gt box overlapping
no inside anchor (every zero-overlap anchor ties its column maximum).  Seeds keep a margin at every
threshold that is not deliberate: NMS IoU and min-size, the clip tests of the unclipped proposals,
max overlaps vs FG/BG thresholds and RPN_NEGATIVE/POSITIVE_OVERLAP, mask values vs BINARIZE_THRESH.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True

from scripts import make_ref_fixtures as MR          # noqa: E402
from scripts import make_ref_train_fixtures as MT    # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ref_rpn_train.npz")
MARGIN = 1e-6
CASES = {   # name: (H, W, im_info, G, n proposals or 0, normalise, use_clip, bp_all)
    "A": (38, 63, (600, 1000, 1.6), 3, 300, True, 1, 1),
    "B": (30, 50, (480, 800, 1.0), 12, 300, False, 0, 0),
    "C": (38, 63, (600, 1000, 1.6), 2, 0, True, 1, 1),
    "D": (30, 50, (480, 800, 1.0), 4, 300, True, 1, 1),
}
_KEYS = {}


def _patch_hook():
    MT._patch_hook()
    orig = MR._RefLoader.source_to_code

    def source_to_code(self, data, path, *, _optimize=-1):
        src = data.decode() if isinstance(data, bytes) else data
        if path.endswith(os.path.join("pylayer", "proposal_target_layer.py")):
            call = "npr.choice(cur_inds, size=cur_rois_this_image, replace=False)"
            assert src.count(call) == 2
            i = src.index(call)
            src = src[:i] + call[:-1] + ", key_row=i)" + src[i + len(call):]
            src = src.replace(call, call[:-1] + ", key_row=len(cfg.TRAIN.FG_FRACTION) + i)")
            assert src.count("gt_assignment[val]") == 4
            src = src.replace("gt_assignment[val]", "gt_assignment[int(val)]")
            data = src.encode()
        elif path.endswith(os.path.join("pylayer", "proposal_layer.py")):
            for a in ("(unmap_val / self._num_anchors)", "/ self._width)"):
                assert a in src
            src = src.replace("(unmap_val / self._num_anchors)", "(unmap_val // self._num_anchors)")
            src = src.replace("(unmap_val / self._num_anchors / self._width)",
                              "(unmap_val // self._num_anchors // self._width)")
            data = src.encode()
        return orig(self, data, path, _optimize=_optimize)
    MR._RefLoader.source_to_code = source_to_code


def _choice(a, size=None, replace=True, key_row=None):
    from oracle import oracle_rpn_train as R
    assert not replace
    keys = _KEYS["pt"][key_row] if key_row is not None else _KEYS["anchor_pos"]
    return R.choice(a, size, keys)


def margins_ok(native_dets, deltas, H, W, im_info, pt, at_ov, case_gm, mask_info, deliberate,
               index):
    from oracle import oracle as O
    from oracle import oracle_train as T
    if native_dets is not None:
        m_iou, m_side = _proposal_margins(*native_dets, deltas, H, W, im_info)
        if m_iou < 2e-6 or m_side < 1e-3:
            return _fail("nms/min-size", m_iou, m_side)
        # the clip tests of the kept proposals' unclipped boxes (the backward's weights)
        t = index.ravel().astype(np.int64)
        unclipped = O.bbox_transform_inv(O.shifted_anchors(H, W)[t],
                                         deltas.transpose(0, 2, 3, 1).reshape(-1, 4)[t])
        lim = np.array([0, 0, im_info[1] - 1, im_info[0] - 1], np.float32)
        if np.abs(unclipped - lim).min() < 1e-3:
            return _fail("clip", np.abs(unclipped - lim).min())
    mo = np.delete(pt["max_overlaps"], deliberate)
    for t in (0.5, 0.1):
        if mo.size and np.abs(mo - t).min() < MARGIN:
            return _fail("max overlap", t)
    if at_ov.size and min(np.abs(at_ov - 0.3).min(), np.abs(at_ov - 0.7).min()) < MARGIN:
        return _fail("anchor overlap")
    out = {"nfg": int(pt["mask_weight"][:, 0, 0, 0].sum()), "gt_mask_info": pt["gt_masks_info"]}
    tv = T.target_values({"gt_masks": case_gm, "mask_info": mask_info}, out)
    return not (tv.size and np.abs(tv - 0.4).min() < MARGIN) or _fail("mask")


def _fail(*why):
    print("  margin:", *why)
    return False


def _proposal_margins(dets, keep, deltas, H, W, im_info):
    """Smallest |IoU - RPN_NMS_THRESH| between one of the first 300 boxes NMS kept and a box after
    it, up to the 300th kept (the only comparisons that decide the RoIs), and smallest
    |side - min_size| of every decoded proposal."""
    from oracle import oracle as O
    keep = np.asarray(keep)[:300]
    b64 = dets[:int(keep[-1]) + 1, :4].astype(np.float64) if len(keep) else dets[:0, :4]
    area = (b64[:, 2] - b64[:, 0] + 1) * (b64[:, 3] - b64[:, 1] + 1)
    worst = 1.0
    for s0 in range(0, len(keep), 256):
        k = keep[s0:s0 + 256]
        c = b64[k]
        iw = np.minimum(c[:, None, 2], b64[None, :, 2]) - np.maximum(c[:, None, 0], b64[None, :, 0]) + 1
        ih = np.minimum(c[:, None, 3], b64[None, :, 3]) - np.maximum(c[:, None, 1], b64[None, :, 1]) + 1
        inter = np.clip(iw, 0, None) * np.clip(ih, 0, None)
        iou = inter / (area[k, None] + area[None, :] - inter)
        iou[np.arange(len(b64))[None, :] <= k[:, None]] = 0.0
        worst = min(worst, np.abs(iou - 0.7).min())
    pr, _ = O.clip_boxes(O.bbox_transform_inv(O.shifted_anchors(H, W), deltas.transpose(0, 2, 3, 1).reshape(-1, 4)),
                         np.array(im_info[:2], np.float32))
    sides = np.concatenate([pr[:, 2] - pr[:, 0] + 1, pr[:, 3] - pr[:, 1] + 1])
    return float(worst), float(np.abs(sides - 16 * np.float32(im_info[2])).min())


def anchor_max_overlaps(H, W, gt, im_info):
    from oracle import oracle as O
    a = O.shifted_anchors(H, W)
    ins = np.where((a[:, 0] >= 0) & (a[:, 1] >= 0) & (a[:, 2] < im_info[1]) & (a[:, 3] < im_info[0]))[0]
    return O.bbox_overlaps(a[ins], gt[:, :4]).max(axis=1), ins


def main():
    _patch_hook()
    native = {"nms": [], "mv": []}
    MR.install_reference_environment(native)
    np.random.choice = _choice
    from mnc_config import cfg                      # reference lib/mnc_config.py
    from pylayer.proposal_layer import ProposalLayer
    from pylayer.proposal_target_layer import ProposalTargetLayer
    from pylayer.anchor_target_layer import AnchorTargetLayer
    from oracle import oracle_rpn_train as R
    Blob = MT.Blob
    cfg.TRAIN.RPN_POST_NMS_TOP_N = 300              # experiments/cfgs/VGG16/mnc_5stage.yml:4
    fx = {}
    for name, (H, W, im_info, G, n, normalise, use_clip, bp_all) in CASES.items():
        cfg.TRAIN.BBOX_NORMALIZE_TARGETS_PRECOMPUTED = normalise
        for seed in range(40):
            rng = np.random.default_rng(8000 + 100 * ord(name) + seed)
            cs = R.make_case(7000 + 100 * ord(name) + seed, H, W, im_info, G)
            prob, deltas, gt, gm, mask_info = (cs[k] for k in ("prob", "deltas", "gt_boxes", "gt_masks", "mask_info"))
            deliberate = []
            if name == "D":
                gt[0, :4] = (0, 0, 5, 5)                  # no inside anchor reaches x, y < 8
                mask_info[0] = (6, 6)
            info = np.array([im_info], np.float32)
            # ---- ProposalLayer (TRAIN)
            pl = ProposalLayer()
            pl.phase = "TRAIN"
            pl.param_str_ = "{'feat_stride': 16, 'use_clip': %d, 'clip_base': 512}" % use_clip
            pb = [Blob(prob), Blob(deltas), Blob(info)]
            ptop = [Blob(), Blob()]
            pl.setup(pb, ptop)
            n_nms = len(native["nms"])
            pl.forward(pb, ptop)
            dets = (native["nms"][-1][0], native["nms"][-1][2]) if len(native["nms"]) > n_nms else None
            rpn_rois, rois_index = ptop[0].data.copy(), ptop[1].data.copy()
            if n == 0:
                rpn_rois, rois_index = np.zeros((0, 5), np.float32), np.zeros((1, 0), np.float32)
            if name == "B":                               # IoU 5000 / 10000 with gt 0, exactly
                x, y = gt[0, 0], gt[0, 1]
                gt[0, 2:4] = (x + 99, y + 99)
                rpn_rois[7, 1:] = (x, y, x + 99, y + 49)
                deliberate = [7]
            N = rpn_rois.shape[0] + G
            ncat = len(cfg.TRAIN.FG_FRACTION) + len(cfg.TRAIN.BG_FRACTION)
            keys = rng.integers(0, 2 ** 32, (ncat, N), dtype=np.uint64).astype(np.uint32)
            if name == "B":
                keys[1, 7] = 0                            # sampled as bg too
            akeys = rng.integers(0, 2 ** 32, H * W * 9, dtype=np.uint64).astype(np.uint32)
            # ---- ProposalTargetLayer
            _KEYS["pt"] = keys
            tl = ProposalTargetLayer()
            tl.phase = "TRAIN"
            tl.param_str_ = "{'num_classes': 21, 'bp_all': %d}" % bp_all
            tb = [Blob(rpn_rois), Blob(gt), Blob(info), Blob(gm.astype(np.float32)),
                  Blob(mask_info, np.int64), Blob(rois_index)]
            ttop = [Blob() for _ in range(10)]
            tl.setup(tb, ttop)
            tl.forward(tb, ttop)
            pt = R.proposal_target_forward(rpn_rois, rois_index, gt, gm, mask_info, info, keys,
                                           normalize=normalise, bp_all=bool(bp_all))
            # ---- AnchorTargetLayer
            at_ov, ins = anchor_max_overlaps(H, W, gt, im_info)
            _KEYS["anchor_pos"] = akeys[ins]
            al = AnchorTargetLayer()
            al.phase = "TRAIN"
            al.param_str_ = "{'feat_stride': 16}"
            ab = [Blob(np.zeros((1, 18, H, W), np.float32)), Blob(gt), Blob(info),
                  Blob(ttop[8].data.copy()), Blob(ttop[9].data.copy())]
            atop = [Blob() for _ in range(4)]
            al.setup(ab, atop)
            al.forward(ab, atop)
            if not margins_ok(dets if n else None, deltas, H, W, im_info, pt, at_ov, gm, mask_info,
                              deliberate, rois_index):
                continue
            break
        else:
            raise RuntimeError("no seed with margins for case %s" % name)
        # ---- backward passes, in the prototxt's reverse order
        K = ttop[0].data.shape[0]
        drng = np.random.default_rng(9000 + ord(name))
        ttop[0].diff = drng.normal(0, 1e-3, (K, 5)).astype(np.float32)
        ttop[0].diff[::5] = 0                              # rows the Proposal backward skips
        tl.backward(ttop, [True, False, False, False, False, False], tb)
        R_ = ptop[0].data.shape[0]
        if n:
            ptop[0].diff = tb[0].diff.copy()
            pb[1].diff = np.full(deltas.shape, 7, np.float32)
            pl.backward(ptop, [False, True, False], pb)
        print("case %s: seed %d, R %d, K %d, fg %d, bg %d, mix fg %d bg %d" % (
            name, seed, R_, K, int(ttop[6].data[:, 0, 0, 0].sum()), K - int(ttop[6].data[:, 0, 0, 0].sum()),
            ttop[8].data.size, ttop[9].data.size))
        p = name + "_"
        fx[p + "cfg"] = np.array([H, W, G, n, normalise, use_clip, 512, bp_all], np.int64)
        fx[p + "im_info"] = info
        fx[p + "gt_boxes"] = gt
        fx[p + "gt_masks"] = gm
        fx[p + "mask_info"] = mask_info
        fx[p + "keys"] = keys
        fx[p + "anchor_keys"] = akeys
        if n:
            fx[p + "prob"] = prob
            fx[p + "deltas"] = deltas
            fx[p + "pl_rois"] = ptop[0].data
            fx[p + "pl_index"] = ptop[1].data
            fx[p + "pl_top_diff"] = ptop[0].diff
            fx[p + "pl_bbox_diff"] = pb[1].diff
        fx[p + "rpn_rois"] = rpn_rois
        fx[p + "rois_index"] = rois_index
        for i, k in enumerate(PT_TOPS):
            fx[p + "pt_" + k] = ttop[i].data
        fx[p + "pt_keep_ind"] = np.asarray(tl._keep_ind).astype(np.int64)
        fx[p + "pt_top_diff"] = ttop[0].diff
        fx[p + "pt_rois_diff"] = tb[0].diff
        for i, k in enumerate(AT_TOPS):
            fx[p + "at_" + k] = atop[i].data
    MR.save_parts(OUT, fx)
    print("wrote", OUT)


PT_TOPS = ("rois", "labels", "bbox_targets", "bbox_inside_weights", "bbox_outside_weights",
           "mask_targets", "mask_weight", "gt_masks_info", "fg_inds", "bg_inds")
AT_TOPS = ("labels", "bbox_targets", "bbox_inside_weights", "bbox_outside_weights")

if __name__ == "__main__":
    main()
