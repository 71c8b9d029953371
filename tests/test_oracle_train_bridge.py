"""oracle/oracle_train.py (numpy restatement of the TRAIN phase of StageBridgeLayer and MaskLayer)
against the reference's own layers run unmodified (tests/golden/ref_train_bridge*.npz,
scripts/make_ref_train_fixtures.py): every array bit for bit, and the fixtures cover each branch."""
import numpy as np
import pytest

from oracle import oracle_train as T
from tests.test_ref_fixtures import load

CASES = ("A", "B", "C")
TOPS = ("rois", "labels", "mask_targets", "mask_weight", "gt_mask_info", "bbox_targets",
        "bbox_inside_weights", "bbox_outside_weights")


def fixture(name):
    f = load("ref_train_bridge.npz")
    return {k[2:]: v for k, v in f.items() if k.startswith(name + "_")}


def run_oracle(f):
    precomputed, use_clip, clip_base, C = (int(v) for v in f["cfg"])
    out = T.stage_bridge_forward(f["rois"], f["bbox_pred"], f["seg_cls_prob"], f["gt_boxes"],
                                 f["gt_masks"].astype(np.float32), f["im_info"], f["mask_info"],
                                 C, normalize=bool(precomputed))
    clip = 1.0 / clip_base if use_clip else 0.0
    rd, bd = T.stage_bridge_backward(f["top_diff"], out, f["rois"], f["bbox_pred"], clip)
    labels = T.mask_layer_forward(f["ml_pred"], f["gt_masks"].astype(np.float32), f["ml_info"])
    mbd = T.mask_layer_backward(f["ml_top_diff"], labels)
    return out, rd, bd, labels, mbd


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_bit_for_bit(name):
    f = fixture(name)
    out, rd, bd, labels, mbd = run_oracle(f)
    for k in TOPS:
        assert out[k].dtype == np.float32 and out[k].shape == f["top_" + k].shape, k
        assert np.array_equal(out[k], f["top_" + k]), k
    for k in ("keep_inds", "reg_labels", "clip_keep"):
        assert np.array_equal(out[k], f[k]), k
    assert np.array_equal(rd, f["rois_diff"]) and np.array_equal(bd, f["bbox_pred_diff"])
    assert np.array_equal(labels, f["ml_labels"])
    assert np.array_equal(mbd, f["ml_bottom_diff"].reshape(mbd.shape))


def test_fixtures_cover_every_branch():
    seen = dict(fg=0, bg=0, off_image=0, clamped=0, unclamped=0, ml_pos=0, ml_zeroed=0,
                empty_box=0, ties=0, scales=set(), precomputed=set(), use_clip=set())
    for name in CASES:
        f = fixture(name)
        precomputed, use_clip, clip_base, C = (int(v) for v in f["cfg"])
        n, K = f["rois"].shape[0], f["top_labels"].shape[0]
        nfg = int(f["top_mask_weight"][:, 0, 0, 0].sum())
        seen["fg"] += nfg
        seen["bg"] += K - nfg
        seen["off_image"] += n - int(np.sum(f["clip_keep"] < n))
        bd = f["bbox_pred_diff"]
        if use_clip:
            seen["clamped"] += int(np.sum(np.abs(bd) == np.float32(1.0 / clip_base)))
            seen["unclamped"] += int(np.sum((bd != 0) & (np.abs(bd) < np.float32(1.0 / clip_base))))
        pos = f["ml_info"][:, 0] != -1
        seen["ml_pos"] += int(np.sum(f["ml_labels"][pos] > 0))
        seen["ml_zeroed"] += int(np.sum(f["ml_labels"][pos] == 0))
        info = f["ml_info"][pos]
        seen["empty_box"] += int(np.sum((np.maximum(info[:, 4], info[:, 8]) > np.minimum(info[:, 6], info[:, 10])) |
                                        (np.maximum(info[:, 5], info[:, 9]) > np.minimum(info[:, 7], info[:, 11]))))
        s = f["seg_cls_prob"][:, 1:]
        tie = (s == s.max(1, keepdims=True)).sum(1) > 1
        seen["ties"] += int(tie.sum())
        if tie.any():   # the first maximum wins
            assert np.array_equal(f["reg_labels"][tie], s[tie].argmax(1) + 1)
        seen["scales"].add(float(f["im_info"][2]))
        seen["precomputed"].add(precomputed)
        seen["use_clip"].add(use_clip)
    for k in ("fg", "bg", "off_image", "clamped", "unclamped", "ml_pos", "ml_zeroed", "empty_box",
              "ties"):
        assert seen[k] > 0, (k, seen)
    assert len(seen["scales"]) == 2 and seen["precomputed"] == {0, 1} and seen["use_clip"] == {0, 1}
    # n = 0 with G > 0 is valid: every row is a gt row
    assert fixture("C")["rois"].shape[0] == 0 and fixture("C")["top_labels"].shape[0] > 0
