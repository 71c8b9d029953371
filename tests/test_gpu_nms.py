"""gpu_nms / `_nms` drop-in vs the oracle: keep lists must be bit-exact (BASELINE.json north_star)."""
import ctypes

import numpy as np
import pytest

from tests import util

pytestmark = pytest.mark.gpu


def _install():
    import mnc_b200.lib as L
    L.install()


@pytest.mark.parametrize("n,thresh", [(1, 0.7), (63, 0.7), (64, 0.5), (65, 0.3), (600, 0.3),
                                      (6000, 0.7), (10000, 0.7)])
def test_nms_host_matches_oracle(n, thresh):
    from oracle import oracle as O
    from mnc_b200._lib import lib, check
    boxes = util.random_boxes(n, seed=10 + n)
    if n <= 6000:
        boxes = util.nudge_off_threshold(boxes, thresh)
    scores = util.tie_free_scores(n, seed=11)
    dets = np.hstack([boxes, scores[:, None]]).astype(np.float32)
    order = O.order_desc(scores)
    sorted_dets = np.ascontiguousarray(dets[order])
    want = O.nms_sorted(sorted_dets, thresh)
    keep = np.zeros(n, dtype=np.int32)
    num = ctypes.c_int(0)
    check(lib.mnc_nms_host(keep.ctypes.data_as(ctypes.c_void_p), ctypes.byref(num),
                           sorted_dets.ctypes.data_as(ctypes.c_void_p), n, 5, thresh, 0),
          "mnc_nms_host")
    got = keep[:num.value]
    assert num.value == len(want)
    assert np.array_equal(got, want)


def test_gpu_nms_wrapper_matches_oracle_and_handles_empty():
    _install()
    from nms.nms_wrapper import nms
    from oracle import oracle as O
    assert nms(np.zeros((0, 5), dtype=np.float32), 0.7) == []
    boxes = util.nudge_off_threshold(util.random_boxes(2000, seed=3), 0.7)
    dets = np.hstack([boxes, util.tie_free_scores(2000, seed=4)[:, None]]).astype(np.float32)
    got = nms(dets, 0.7)
    want = O.gpu_nms(dets, 0.7)
    assert [int(x) for x in got] == [int(x) for x in want]
    with pytest.raises(ValueError):
        nms(dets.astype(np.float64), 0.7)


def test_nms_score_ties_follow_documented_rule():
    """equal scores: (score desc, index asc)."""
    _install()
    from nms.gpu_nms import gpu_nms
    from oracle import oracle as O
    boxes = util.random_boxes(500, seed=5, integer=True)
    scores = np.repeat(np.linspace(0.9, 0.1, 50), 10).astype(np.float32)
    dets = np.hstack([boxes, scores[:, None]]).astype(np.float32)
    assert [int(x) for x in gpu_nms(dets, 0.3)] == [int(x) for x in O.gpu_nms(dets, 0.3)]


def test_batched_device_nms_with_counts_and_max_keep():
    import torch
    from mnc_b200 import ops
    from oracle import oracle as O
    P, n_max = 5, 700
    counts = [700, 1, 0, 333, 64]
    boxes = np.zeros((P, n_max, 4), dtype=np.float32)
    for p in range(P):
        boxes[p] = util.random_boxes(n_max, seed=100 + p, integer=True)
    tb = torch.from_numpy(boxes).cuda()
    tc = torch.tensor(counts, dtype=torch.int32).cuda()
    keep, num = ops.nms_sorted(tb, tc, 0.3, 100)
    keep, num = keep.cpu().numpy(), num.cpu().numpy()
    for p in range(P):
        want = O.nms_sorted(boxes[p, :counts[p]], 0.3)[:100]
        assert num[p] == len(want)
        assert np.array_equal(keep[p, :num[p]], want)


def test_rank_sort_matches_tie_rule():
    import torch
    from mnc_b200 import ops
    from oracle import oracle as O
    rng = np.random.default_rng(0)
    n = 5000
    s = rng.integers(0, 300, size=(3, n)).astype(np.float32) / 300.0  # many ties
    valid = (rng.uniform(size=(3, n)) > 0.2).astype(np.uint8)
    order, nv = ops.rank_sort_desc(torch.from_numpy(s).cuda(), n, 3, outer_stride=n,
                                   valid=torch.from_numpy(valid).cuda())
    order, nv = order.cpu().numpy(), nv.cpu().numpy()
    for p in range(3):
        idx = np.where(valid[p])[0]
        want = idx[O.order_desc(s[p, idx])]
        assert nv[p] == len(idx)
        assert np.array_equal(order[p, :nv[p]], want)


@pytest.mark.parametrize("n,k,tie_levels", [(21546, 6000, 0), (21546, 6000, 300), (5000, 6000, 50),
                                            (9000, 100, 7), (3000, 1, 0), (12000, 8192, 2)])
def test_topk_sort_is_prefix_of_full_order(n, k, tie_levels):
    """mnc_topk_sort_desc == first k entries of the (score desc, index asc) order, including when
    the k-th score is shared by more entries than there are slots (lowest indices win)."""
    import torch
    from mnc_b200 import ops
    from oracle import oracle as O
    rng = np.random.default_rng(n + k)
    P = 3
    if tie_levels:
        s = rng.integers(0, tie_levels, size=(P, n)).astype(np.float32) / tie_levels
    else:
        s = rng.uniform(-1, 1, size=(P, n)).astype(np.float32)
    valid = (rng.uniform(size=(P, n)) > 0.15).astype(np.uint8)
    valid[2, :] = 0
    valid[2, 17:40] = 1                       # fewer valid entries than k
    order, cnt = ops.topk_sort_desc(torch.from_numpy(s).cuda(), n, P, k, outer_stride=n,
                                    valid=torch.from_numpy(valid).cuda())
    order, cnt = order.cpu().numpy(), cnt.cpu().numpy()
    for p in range(P):
        idx = np.where(valid[p])[0]
        want = idx[O.order_desc(s[p, idx])][:k]
        assert cnt[p] == len(want)
        assert np.array_equal(order[p, :cnt[p]], want)
    # no `valid` array: everything takes part
    order, cnt = ops.topk_sort_desc(torch.from_numpy(s).cuda(), n, P, k, outer_stride=n)
    assert np.array_equal(order[0].cpu().numpy()[:min(k, n)], O.order_desc(s[0])[:k])


def _clustered_boxes(n, seed, clusters=40):
    """RPN-like candidates: many near-duplicates around a few centres (heavy suppression, so the
    capped NMS has to walk most of the list before it has max_keep survivors)."""
    rng = np.random.default_rng(seed)
    cx = rng.uniform(50, 950, clusters)
    cy = rng.uniform(50, 550, clusters)
    sz = np.exp(rng.uniform(np.log(40), np.log(300), clusters))
    k = rng.integers(0, clusters, n)
    w = sz[k] * np.exp(rng.normal(0, 0.15, n))
    h = sz[k] * np.exp(rng.normal(0, 0.15, n))
    x = cx[k] + rng.normal(0, 6, n)
    y = cy[k] + rng.normal(0, 6, n)
    b = np.stack([x - w / 2, y - h / 2, x + w / 2, y + h / 2], axis=1)
    b[:, 0::2] = np.clip(b[:, 0::2], 0, 999)
    b[:, 1::2] = np.clip(b[:, 1::2], 0, 599)
    return b.astype(np.float32)


@pytest.mark.parametrize("n_max,max_keep,kind", [(6000, 300, "clustered"), (6000, 300, "sparse"),
                                                 (10000, 300, "sparse"), (1024 + 17, 100, "clustered"),
                                                 (4096, 1, "clustered"), (2500, 600, "clustered"),
                                                 (5000, 1024, "clustered"), (8000, 1500, "clustered")])
def test_capped_nms_equals_mask_scan_and_oracle(n_max, max_keep, kind):
    """mnc_nms_sorted's capped forms (no suppression matrix, kept boxes in shared memory: a cluster
    of 8 CTAs per problem, or one CTA) == the mask + scan pair == the oracle, with per-problem counts (full, ragged last block,
    one box, empty)."""
    import torch
    from mnc_b200 import ops
    from mnc_b200._lib import lib
    from oracle import oracle as O
    counts = [n_max, n_max - 37, 1, 0, 65]
    P = len(counts)
    boxes = np.zeros((P, n_max, 4), dtype=np.float32)
    for p in range(P):
        boxes[p] = (_clustered_boxes(n_max, 7 + p) if kind == "clustered"
                    else util.random_boxes(n_max, seed=7 + p))
    oracle_check = kind == "clustered" and n_max <= 6000
    if oracle_check:    # problem 0 is also held to the (FMA-free) oracle: keep IoUs off the threshold
        boxes[0] = util.nudge_off_threshold(boxes[0], 0.7)
    tb = torch.from_numpy(boxes).cuda()
    tc = torch.tensor(counts, dtype=torch.int32).cuda()
    assert lib.mnc_nms_sorted_launches(n_max, max_keep) == 1     # these sizes take the capped form
    prev = ops.nms_set_lazy(3)                                   # cluster, 256-candidate rounds
    try:
        k3, n3 = ops.nms_sorted(tb, tc, 0.7, max_keep)
        ops.nms_set_lazy(2)                                      # cluster of 8 CTAs, 64-candidate rounds
        k2, n2 = ops.nms_sorted(tb, tc, 0.7, max_keep)
        ops.nms_set_lazy(1)                                      # one CTA per problem
        k1, n1 = ops.nms_sorted(tb, tc, 0.7, max_keep)
        ops.nms_set_lazy(0)
        assert lib.mnc_nms_sorted_launches(n_max, max_keep) == 2
        k0, n0 = ops.nms_sorted(tb, tc, 0.7, max_keep)
    finally:
        ops.nms_set_lazy(prev)
    k1, n1, k0, n0 = k1.cpu().numpy(), n1.cpu().numpy(), k0.cpu().numpy(), n0.cpu().numpy()
    k2, n2, k3, n3 = k2.cpu().numpy(), n2.cpu().numpy(), k3.cpu().numpy(), n3.cpu().numpy()
    assert np.array_equal(n1, n0) and np.array_equal(n2, n0) and np.array_equal(n3, n0)
    for p in range(P):
        assert np.array_equal(k1[p, :n1[p]], k0[p, :n0[p]])
        assert np.array_equal(k2[p, :n2[p]], k0[p, :n0[p]])
        assert np.array_equal(k3[p, :n3[p]], k0[p, :n0[p]])
        if p == 0 and oracle_check:
            want = O.nms_sorted(boxes[p, :counts[p]], 0.7)[:max_keep]
            assert n1[p] == len(want) and np.array_equal(k1[p, :n1[p]], want)
    if kind == "clustered" and max_keep > 1:
        assert n1[0] < counts[0]                                 # suppression did happen
