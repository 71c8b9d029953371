"""CPU model of the capped NMS the device runs for the ProposalLayer (mnc_b200/csrc/nms.cu,
nms_lazy_*): candidates walked in blocks, each block first tested against the boxes kept so far,
then resolved serially from its own upper-triangular suppression words.  The model must give the
oracle's keep list truncated at max_keep for every block size -- the claim the kernels rest on."""
import numpy as np
import pytest

from tests import util


def _iou_gt(a, b, thresh):
    """IoU(a, b) > thresh with the +1 convention, fp32 like devIoU (nms_kernel.cu:24-32)."""
    f = np.float32
    w = max(f(min(a[2], b[2]) - max(a[0], b[0]) + f(1)), f(0))
    h = max(f(min(a[3], b[3]) - max(a[1], b[1]) + f(1)), f(0))
    inter = f(w * h)
    sa = f((a[2] - a[0] + f(1)) * (a[3] - a[1] + f(1)))
    sb = f((b[2] - b[0] + f(1)) * (b[3] - b[1] + f(1)))
    return bool(inter / f(sa + sb - inter) > f(thresh))


def capped_nms_blocks(n, suppresses, max_keep, block):
    """suppresses(i, j): box i, earlier in score order, suppresses box j."""
    kept = []
    for r0 in range(0, n, block):
        cand = range(r0, min(r0 + block, n))
        # phase A: suppression by earlier kept boxes + the block's own strictly upper triangle
        sup = {c: any(suppresses(k, c) for k in kept) for c in cand}
        diag = {i: {c for c in cand if c > i and suppresses(i, c)} for i in cand}
        # phase B: serial resolve
        dead = {c for c in cand if sup[c]}
        for i in cand:
            if i in dead:
                continue
            kept.append(i)
            if len(kept) == max_keep:
                return kept
            dead |= diag[i]
    return kept


@pytest.mark.parametrize("block", [64, 256])
@pytest.mark.parametrize("kind", ["clustered", "sparse"])
def test_block_walk_equals_greedy_nms(block, kind):
    from oracle import oracle as O
    n, max_keep, thresh = 700, 60, 0.7
    if kind == "clustered":
        rng = np.random.default_rng(3)
        c = rng.integers(0, 12, n)
        cx, cy = rng.uniform(50, 950, 12)[c], rng.uniform(50, 550, 12)[c]
        s = np.exp(rng.uniform(np.log(40), np.log(250), 12))[c]
        w, h = s * np.exp(rng.normal(0, 0.15, n)), s * np.exp(rng.normal(0, 0.15, n))
        x, y = cx + rng.normal(0, 6, n), cy + rng.normal(0, 6, n)
        boxes = np.stack([x - w / 2, y - h / 2, x + w / 2, y + h / 2], 1).astype(np.float32)
    else:
        boxes = util.random_boxes(n, seed=4)
    boxes = util.nudge_off_threshold(boxes, thresh)
    want = [int(i) for i in O.nms_sorted(boxes, thresh)[:max_keep]]
    got = capped_nms_blocks(len(boxes), lambda i, j: _iou_gt(boxes[i], boxes[j], thresh), max_keep, block)
    assert got == want
    if kind == "clustered":
        assert len(want) == max_keep and want[-1] > 1.5 * max_keep    # suppression did happen
