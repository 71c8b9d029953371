"""CPU checks of the bounds mask voting's device kernels rely on (mnc_b200/csrc/mask_voting.cu),
against the oracle's full aggregate: they must hold for every result, or the pruned search would
miss pixels."""
import numpy as np

from tests.mv_ties import rel_margin
from tests.test_ref_pin import _voting_inputs


def _lists(boxes, scores):
    from oracle import oracle as O
    inds, start, weights, _, _ = O.mask_voting_candidates(boxes, scores, 21, 100)
    beg = np.concatenate([[0], start[:-1]])
    return inds, start, weights, beg


def test_covering_weight_region_contains_every_on_pixel():
    """mv_aggregate_kernel cuts the search region to the columns / rows whose covering weight
    sum_i w_i [x in box_i] exceeds 0.4 (with the kernel's rounding margin, 1 + (n + 4) 2^-21):
    valid because render <= 1 + 6 ulp for masks in [0, 1] and weights >= 0.  Every pixel of {agg > 0.4} must lie inside."""
    from oracle import oracle as O
    nb, H, W = 120, 150, 200
    rng = np.random.default_rng(5)
    boxes, masks, scores = _voting_inputs(nb, H, W, 21)
    # clustered copies so that several lists have many candidates
    src = rng.integers(0, 10, nb)
    boxes = boxes[src] + rng.normal(0, 3, (nb, 4)).astype(np.float32)
    boxes[:, 0::2] = np.clip(np.sort(boxes[:, 0::2], axis=1), 0, W - 1)
    boxes[:, 1::2] = np.clip(np.sort(boxes[:, 1::2], axis=1), 0, H - 1)
    inds, start, weights, beg = _lists(boxes, scores)
    _, rb, agg = O.mv(boxes, masks, inds, start, weights, H, W, return_agg=True)
    xs, ys = np.arange(W, dtype=np.float32), np.arange(H, dtype=np.float32)
    checked = long_lists = 0
    for t, (b, e) in enumerate(zip(beg, start)):
        ii, ww = inds[b:e], weights[b:e]
        on = agg[t] > 0.4
        if not on.any():
            continue
        ux, uy = np.zeros(W, np.float32), np.zeros(H, np.float32)
        for i, w in zip(ii, ww):                       # the kernel's box test: !(p < lo || p > hi)
            bx = boxes[i]
            ux += np.where(~((xs < bx[0]) | (xs > bx[2])), w, 0).astype(np.float32)
            uy += np.where(~((ys < bx[1]) | (ys > bx[3])), w, 0).astype(np.float32)
        rel = rel_margin(len(ii))
        col_ok = ux * rel > np.float32(0.4)
        row_ok = uy * rel > np.float32(0.4)
        yy, xx = np.where(on)
        assert col_ok[xx].all() and row_ok[yy].all(), "result %d: an on pixel lies outside the pruned region" % t
        # and the tight box the oracle reports is the bounding box of the on pixels
        assert list(rb[t]) == [xx.min(), yy.min(), xx.max(), yy.max()]
        checked += 1
        long_lists += len(ii) > 3
    assert checked > 10 and long_lists > 3


def test_coarse_pass_box_is_inside_the_tight_box():
    """The two-pass search skips pixels inside the box spanned by the coarse pass's on pixels: that
    box is always contained in the tight box, so no skipped pixel can move a side."""
    from oracle import oracle as O
    nb, H, W = 120, 150, 200
    boxes, masks, scores = _voting_inputs(nb, H, W, 23)
    inds, start, weights, beg = _lists(boxes, scores)
    _, rb, agg = O.mv(boxes, masks, inds, start, weights, H, W, return_agg=True)
    n = 0
    for t in range(len(start)):
        on = agg[t] > 0.4
        for stride in (4, 6):
            sub = on[::stride, ::stride]
            if not sub.any():
                continue
            yy, xx = np.where(sub)
            x0, y0, x1, y1 = xx.min() * stride, yy.min() * stride, xx.max() * stride, yy.max() * stride
            assert rb[t][0] <= x0 and rb[t][1] <= y0 and x1 <= rb[t][2] and y1 <= rb[t][3]
            n += 1
    assert n > 10
