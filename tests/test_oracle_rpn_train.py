"""oracle/oracle_rpn_train.py (numpy restatement of the TRAIN phase of ProposalLayer,
ProposalTargetLayer and AnchorTargetLayer) against the reference's own layers run unmodified but
for the documented shims (tests/golden/ref_rpn_train*.npz, scripts/make_ref_rpn_train_fixtures.py):
every array bit for bit, and the fixtures cover each branch."""
import numpy as np
import pytest

from oracle import oracle_rpn_train as R
from tests.test_ref_fixtures import load

CASES = ("A", "B", "C", "D")
PT_TOPS = ("rois", "labels", "bbox_targets", "bbox_inside_weights", "bbox_outside_weights",
           "mask_targets", "mask_weight", "gt_masks_info", "fg_inds", "bg_inds")
AT_TOPS = ("labels", "bbox_targets", "bbox_inside_weights", "bbox_outside_weights")


def fixture(name):
    f = load("ref_rpn_train.npz")
    return {k[2:]: v for k, v in f.items() if k.startswith(name + "_")}


def config(f):
    H, W, G, n, normalise, use_clip, clip_base, bp_all = (int(v) for v in f["cfg"])
    return dict(H=H, W=W, G=G, n=n, normalize=bool(normalise),
                clip=1.0 / clip_base if use_clip else 0.0, bp_all=bool(bp_all))


def run_oracle(f):
    c = config(f)
    out = {}
    if c["n"]:
        rois, index, st = R.proposal_train_forward(f["prob"], f["deltas"], f["im_info"])
        out.update(pl_rois=rois, pl_index=index,
                   pl_bbox_diff=R.proposal_backward(f["pl_top_diff"], st, f["deltas"], c["clip"]))
    pt = R.proposal_target_forward(f["rpn_rois"], f["rois_index"], f["gt_boxes"], f["gt_masks"],
                                   f["mask_info"], f["im_info"], f["keys"], normalize=c["normalize"],
                                   bp_all=c["bp_all"])
    pt["rois_diff"] = R.proposal_target_backward(f["pt_top_diff"], pt["keep_ind"], c["n"])
    at = R.anchor_target_forward(c["H"], c["W"], f["gt_boxes"], f["im_info"], f["anchor_keys"],
                                 f["pt_fg_inds"], f["pt_bg_inds"])
    return out, pt, at


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_bit_for_bit(name):
    f = fixture(name)
    out, pt, at = run_oracle(f)
    for k, v in out.items():
        assert v.dtype == f[k].dtype and np.array_equal(v, f[k]), k
    for k in PT_TOPS:
        assert pt[k].dtype == np.float32 and pt[k].shape == f["pt_" + k].shape, k
        assert np.array_equal(pt[k], f["pt_" + k]), k
    assert np.array_equal(pt["keep_ind"], f["pt_keep_ind"])
    assert np.array_equal(pt["rois_diff"], f["pt_rois_diff"])
    for k, v in zip(AT_TOPS, at):
        assert v.dtype == np.float32 and v.shape == f["at_" + k].shape, k
        assert np.array_equal(v, f["at_" + k]), k


def test_choice_is_the_smallest_keys_with_index_ties():
    keys = np.array([5, 1, 5, 0, 9, 1], np.uint32)
    assert list(R.choice([0, 1, 2, 3, 4, 5], 3, keys)) == [1, 3, 5]
    assert list(R.choice([0, 2, 4], 2, keys)) == [0, 2]        # tie 5 / 5: the lower index
    assert R.choice([0, 2], 0, keys).size == 0
    # with uniform keys every subset is equally likely (here: 3 of 5, 10 subsets)
    rng = np.random.default_rng(0)
    seen = {}
    for _ in range(4000):
        k = rng.integers(0, 2 ** 32, 5, dtype=np.uint64).astype(np.uint32)
        s = tuple(R.choice(np.arange(5), 3, k))
        seen[s] = seen.get(s, 0) + 1
    assert len(seen) == 10 and max(seen.values()) < 1.25 * 400 and min(seen.values()) > 0.75 * 400


def test_fixtures_cover_every_branch():
    seen = dict(dup_keep=0, short_category=0, mix_inside=0, mix_outside=0, no_inside_gt=0,
                skipped_rows=0, clamped=0, pl_weight0=0, n0=0, bp_all=set(),
                normalize=set(), fg=0, bg_labels=0, pos_anchor=0, neg_anchor=0, off_anchor=0)
    for name in CASES:
        f = fixture(name)
        c = config(f)
        seen["bp_all"].add(c["bp_all"])
        seen["normalize"].add(c["normalize"])
        seen["n0"] += c["n"] == 0
        _, pt, at = run_oracle(f)
        keep = pt["keep_inds"]
        seen["dup_keep"] += len(keep) - len(np.unique(keep))
        K = len(keep)
        nfg = int(pt["mask_weight"][:, 0, 0, 0].sum())
        seen["fg"] += nfg
        seen["bg_labels"] += K - nfg
        # a category with fewer candidates than it asks for (every fg candidate is taken)
        mo = pt["max_overlaps"]
        seen["short_category"] += int(np.sum(mo >= 0.5) < 19)
        lab = at[0].reshape(9, c["H"], c["W"]).transpose(1, 2, 0).ravel()
        seen["pos_anchor"] += int(np.sum(lab == 1))
        seen["neg_anchor"] += int(np.sum(lab == 0))
        from oracle import oracle as O
        a = O.shifted_anchors(c["H"], c["W"])
        im = f["im_info"].ravel()
        inside = (a[:, 0] >= 0) & (a[:, 1] >= 0) & (a[:, 2] < im[1]) & (a[:, 3] < im[0])
        seen["off_anchor"] += int(np.sum(~inside))
        for v in np.concatenate([f["pt_fg_inds"].ravel(), f["pt_bg_inds"].ravel()]):
            seen["mix_inside" if inside[int(v)] else "mix_outside"] += 1
        ov = O.bbox_overlaps(a[inside], f["gt_boxes"][:, :4])
        seen["no_inside_gt"] += int(np.sum(ov.max(axis=0) == 0))
        if c["n"]:
            td = f["pl_top_diff"]
            seen["skipped_rows"] += int(np.sum(~np.any(np.abs(td) > 0, axis=1)))
            d = f["pl_bbox_diff"]
            seen["clamped"] += int(np.sum(np.abs(d) == np.float32(c["clip"]))) if c["clip"] else 0
            rows = np.unique(np.where(np.abs(td) > 0)[0])
            _, _, st = R.proposal_train_forward(f["prob"], f["deltas"], f["im_info"])
            idx = f["pl_index"].ravel()[rows].astype(np.int64)
            seen["pl_weight0"] += int(np.sum(~(np.isin(idx, st["proposal_keep"]) &
                                               np.isin(idx, st["anchor_keep"]))))
    assert seen["dup_keep"] >= 1 and seen["short_category"] >= 1 and seen["n0"] == 1
    assert seen["mix_inside"] > 0 and seen["mix_outside"] > 0 and seen["no_inside_gt"] >= 1
    assert seen["skipped_rows"] > 0 and seen["clamped"] > 0 and seen["pl_weight0"] > 0
    assert seen["bp_all"] == {True, False} and seen["normalize"] == {True, False}
    assert seen["fg"] > 0 and seen["bg_labels"] > 0
    assert seen["pos_anchor"] > 0 and seen["neg_anchor"] > 0 and seen["off_anchor"] > 0
