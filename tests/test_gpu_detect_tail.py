"""The detection tail's selection and box kernels one by one, each against a plain numpy restatement
of the reference's Python at the shapes and values where they can go wrong:

  mnc_vote_select         global score threshold of mask voting (mask_transform.py:240-270)
  mnc_gather_boxes        score-order gather of boxes per problem
  mnc_write_rois          keep list -> [bi, x1, y1, x2, y2] rows (proposal_layer.py:169-175)
  mnc_unscale_clip        rois[:, 1:5] / im_scale, clip_boxes (demo.py:92-95)
  mnc_detect_tail         the same boxes, plus the copies into the per-step output record
  mnc_decode_class_boxes  TesterWrapper._detection_forward: unscale, bbox_transform_inv, clip_boxes

Copies are compared bit for bit.  Every output buffer starts filled with a sentinel, and the rows a
kernel must not write (past a count, past the end of the buffer) must still hold it afterwards."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SENT_I = -7777
SENT_F = np.float32(-1234.5)
SENT_BITS = np.float32(SENT_F).view(np.uint32)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _same_bits(got, want, what):
    """Bitwise equality; a NaN matches a NaN whatever its payload (numpy keeps the input's, the
    device writes its canonical one)."""
    got = np.asarray(got, dtype=np.float32)
    want = np.asarray(want, dtype=np.float32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    gn, wn = np.isnan(got), np.isnan(want)
    assert np.array_equal(gn, wn), "%s: NaN at %s, expected at %s" % (
        what, np.argwhere(gn)[:5].tolist(), np.argwhere(wn)[:5].tolist())
    bad = (_bits(got) != _bits(want)) & ~wn
    assert not bad.any(), "%s: %d elements differ, first at %s: %r != %r" % (
        what, int(bad.sum()), np.argwhere(bad)[0].tolist(), got[bad][0], want[bad][0])


def _lib():
    from mnc_b200._lib import lib
    return lib


def _stream():
    from mnc_b200._lib import cur_stream
    return cur_stream()


# ============================================================================ vote_select
def vote_select_ref(scores, order, keep, num_keep, max_per_image):
    """mask_transform.py:240-270 from given keep lists, one image at a time.
    -> per image: (box_idx, cls, score) of every result in order, and class_bar."""
    B, nb, ncls = scores.shape
    nprob = ncls - 1
    out = []
    for img in range(B):
        sup_idx, sup_scores, tobesort = [], [], []
        for p in range(nprob):
            prob = img * nprob + p
            k = keep[prob, :min(int(num_keep[prob]), max_per_image)]      # ind_scores[0:num_keep]
            idx = order[prob, k]
            sup_idx.append(idx)
            sup_scores.append(scores[img, idx, p + 1])
            tobesort.extend(sup_scores[-1])
        box_idx, cls, res_score, class_bar = [], [], [], []
        if tobesort:
            sorted_scores = np.sort(np.asarray(tobesort, dtype=np.float32))[::-1]
            thresh = sorted_scores[min(len(sorted_scores), max_per_image) - 1]
            for p in range(nprob):
                sel = np.where(sup_scores[p] >= thresh)[0]
                box_idx.extend(sup_idx[p][sel])
                cls.extend([p + 1] * len(sel))
                res_score.extend(sup_scores[p][sel])
                class_bar.append(len(res_score))
        else:       # the reference indexes an empty list here; the device reports no results
            class_bar = [0] * nprob
        out.append((np.asarray(box_idx, np.int64), np.asarray(cls, np.int64),
                    np.asarray(res_score, np.float32), np.asarray(class_bar, np.int64)))
    return out


def build_vote_case(classes, nb, keep_stride, seed):
    """classes[img][p]: scores of class p+1's keep list, in keep order (its length is num_keep).
    Keep positions and the per-class score order are random, so box index = order[keep[k]] is a
    real two-step lookup; every score the kernel must not read is NaN, and keep slots past
    num_keep point at such boxes."""
    rng = np.random.default_rng(seed)
    B, nprob = len(classes), len(classes[0])
    scores = np.full((B, nb, nprob + 1), np.nan, dtype=np.float32)
    order = np.zeros((B * nprob, nb), dtype=np.int32)
    keep = np.zeros((B * nprob, keep_stride), dtype=np.int32)
    num_keep = np.zeros(B * nprob, dtype=np.int32)
    for img in range(B):
        for p in range(nprob):
            s = np.asarray(classes[img][p], dtype=np.float32)
            n = len(s)
            assert n < nb and n <= keep_stride
            prob = img * nprob + p
            order[prob] = rng.permutation(nb)
            pos = np.sort(rng.choice(nb, size=n, replace=False))
            rest = np.setdiff1d(np.arange(nb), pos)
            keep[prob, :n] = pos
            keep[prob, n:] = rest[np.arange(keep_stride - n) % len(rest)]
            num_keep[prob] = n
            scores[img, order[prob, pos], p + 1] = s
    return scores, order, keep, num_keep


def run_vote_select(scores, order, keep, num_keep, max_per_image, max_results, pad=64):
    """mnc_vote_select through the library, with sentinel-filled outputs and `pad` spare entries
    after the last image's result slots.  -> (status, dict of numpy outputs)."""
    B, nb, ncls = scores.shape
    nprob = ncls - 1
    n = B * max_results + pad
    res_idx = torch.full((n,), SENT_I, dtype=torch.int32, device="cuda")
    res_cls = torch.full((n,), SENT_I, dtype=torch.int32, device="cuda")
    res_score = torch.full((n,), float(SENT_F), dtype=torch.float32, device="cuda")
    n_res = torch.full((B + 1,), SENT_I, dtype=torch.int32, device="cuda")
    class_bar = torch.full((B * nprob + 1,), SENT_I, dtype=torch.int32, device="cuda")
    overflow = torch.zeros(1, dtype=torch.int32, device="cuda")
    d_scores, d_order, d_keep, d_num = _dev(scores), _dev(order), _dev(keep), _dev(num_keep)
    rc = _lib().mnc_vote_select(d_scores.data_ptr(), nb, ncls, d_order.data_ptr(), d_keep.data_ptr(),
                                keep.shape[1], d_num.data_ptr(), max_per_image, max_results, B,
                                res_idx.data_ptr(), res_cls.data_ptr(), res_score.data_ptr(),
                                n_res.data_ptr(), class_bar.data_ptr(), overflow.data_ptr(),
                                _stream())
    torch.cuda.synchronize()
    return rc, dict(res_box_idx=res_idx.cpu().numpy(), res_class=res_cls.cpu().numpy(),
                    res_score=res_score.cpu().numpy(), n_res=n_res.cpu().numpy(),
                    class_bar=class_bar.cpu().numpy(), overflow=int(overflow.item()))


def check_vote_select(classes, nb, keep_stride, max_per_image, max_results, seed=0):
    """All six outputs against vote_select_ref; returns the reference results."""
    from mnc_b200._lib import MNC_OK
    scores, order, keep, num_keep = build_vote_case(classes, nb, keep_stride, seed)
    B, nprob = scores.shape[0], scores.shape[2] - 1
    want = vote_select_ref(scores, order, keep, num_keep, max_per_image)
    rc, got = run_vote_select(scores, order, keep, num_keep, max_per_image, max_results)
    assert rc == MNC_OK
    mr = max_results
    for img, (w_idx, w_cls, w_score, w_bar) in enumerate(want):
        k = min(len(w_idx), mr)
        assert got["n_res"][img] == k, (img, got["n_res"][img], len(w_idx))
        sl = slice(img * mr, img * mr + k)
        assert np.array_equal(got["res_box_idx"][sl], w_idx[:k]), img
        assert np.array_equal(got["res_class"][sl], w_cls[:k]), img
        _same_bits(got["res_score"][sl], w_score[:k], "res_score image %d" % img)
        rest = slice(img * mr + k, (img + 1) * mr)
        assert np.all(got["res_box_idx"][rest] == SENT_I) and np.all(got["res_class"][rest] == SENT_I)
        assert np.all(_bits(got["res_score"][rest]) == SENT_BITS), "image %d: slot past n_res written" % img
        assert np.array_equal(got["class_bar"][img * nprob:(img + 1) * nprob], np.minimum(w_bar, mr)), img
    # nothing past the last image's slots, n_res[B] or class_bar[B * nprob]
    assert np.all(got["res_box_idx"][B * mr:] == SENT_I) and np.all(got["res_class"][B * mr:] == SENT_I)
    assert np.all(_bits(got["res_score"][B * mr:]) == SENT_BITS)
    assert got["n_res"][B] == SENT_I and got["class_bar"][B * nprob] == SENT_I
    assert got["overflow"] == int(any(len(w[0]) > mr for w in want))
    return want


def _f32_bits(u):
    return np.array([u], dtype=np.uint32).view(np.float32)[0]


def test_vote_select_counts_around_max_per_image():
    """Total kept entries one below, equal to and one above max_per_image, a batch of 3 with
    keep_stride > max_per_image and nb not a multiple of 32."""
    mpi = 5
    classes = [
        [[0.9, 0.3], [], [0.5, 0.2]],                          # 4 < 5: everything
        [[0.9, 0.3], [0.8], [0.5, 0.2]],                       # 5 == 5: everything
        [[0.9, 0.3], [0.8, 0.25], [0.5, 0.2]],                 # 6 > 5: 0.2 drops
    ]
    want = check_vote_select(classes, nb=45, keep_stride=9, max_per_image=mpi, max_results=16)
    assert [len(w[0]) for w in want] == [4, 5, 5]


def test_vote_select_threshold_ties_across_classes():
    """Ties at the threshold in four classes: every tied entry is kept, so the result count exceeds
    max_per_image; the empty class 4 sits in the middle."""
    classes = [[[0.9, 0.5, 0.5], [0.5, 0.5], [0.8, 0.5], [], [0.5, 0.25]]]
    want = check_vote_select(classes, nb=33, keep_stride=4, max_per_image=4, max_results=32)
    assert len(want[0][0]) == 8


def test_vote_select_last_radix_pass_decides():
    """Scores that agree in their top 24 bits (and some in the top 16 only): the threshold is
    fixed by the last byte of the 4-pass radix select."""
    base = 0x3F333300
    lo = [_f32_bits(base | b) for b in (0x10, 0x80, 0x7F, 0xFF, 0x01, 0x80, 0x81)]
    mid = [_f32_bits((base & 0xFFFF0000) | 0x3400 | b) for b in (0x00, 0x7F)]
    classes = [[[lo[0], lo[1]], [lo[2], mid[0], lo[3]], [lo[4], lo[5], mid[1], lo[6]]]]
    for mpi in (2, 3, 4, 5, 6, 8):
        check_vote_select(classes, nb=40, keep_stride=6, max_per_image=mpi, max_results=16)


def test_vote_select_one_ulp_at_threshold():
    t = np.float32(0.6)
    up, dn = np.nextafter(t, np.float32(2)), np.nextafter(t, np.float32(0))
    classes = [[[up, dn], [t], [dn, t, up]],
               [[dn], [dn, dn], [up]]]
    want = check_vote_select(classes, nb=37, keep_stride=5, max_per_image=4, max_results=8)
    assert sorted(want[0][2].tolist()) == sorted([up, up, t, t])
    assert sorted(want[1][2].tolist()) == sorted([up, dn, dn, dn])


def test_vote_select_signed_zero_subnormal_one():
    """0.0 and -0.0 compare equal (both pass a threshold of either); a subnormal lies above both."""
    sub = np.float32(1e-40)
    z, nz = np.float32(0.0), np.float32(-0.0)
    classes = [
        [[1.0, z], [nz, 1.0], [sub], []],                     # thresh = the subnormal: 3 results
        [[1.0], [z, nz], [nz], [z]],                          # thresh = +-0: all 5
        [[sub, -sub], [z], [nz, 1.0], [-sub]],                # thresh = +-0: both -sub drop
    ]
    want = check_vote_select(classes, nb=35, keep_stride=4, max_per_image=3, max_results=8)
    assert [len(w[0]) for w in want] == [3, 5, 4]
    check_vote_select(classes, nb=35, keep_stride=4, max_per_image=4, max_results=8)


def test_vote_select_empty_classes():
    """Empty classes first, in the middle and last; an image with no kept entry at all gives no
    result and a zero class_bar."""
    classes = [
        [[], [0.4, 0.3], [], [0.9], []],
        [[], [], [], [], []],
        [[0.2], [], [], [], [0.7, 0.1]],
    ]
    want = check_vote_select(classes, nb=50, keep_stride=3, max_per_image=3, max_results=8)
    assert [len(w[0]) for w in want] == [3, 0, 3]


def test_vote_select_truncates_keep_lists_by_position():
    """num_keep > max_per_image: the first max_per_image entries in keep order count (the scores are
    not monotone, and the two best sit past the cut).  The totals stay within the kernel's
    (ncls - 1) * max_per_image entries even without the cut."""
    classes = [
        [[0.6], [0.1, 0.7], [0.3, 0.8, 0.2, 0.5, 0.95, 0.99]],
        [[0.3, 0.8, 0.2, 0.5, 0.95, 0.99], [0.6], [0.1, 0.7]],
    ]
    want = check_vote_select(classes, nb=41, keep_stride=7, max_per_image=4, max_results=8)
    for w in want:
        assert len(w[0]) == 4 and not np.isin(np.float32([0.95, 0.99]), w[2]).any()


def _random_classes(rng, nprob, counts, levels):
    """Scores from a coarse grid, so that many entries tie at any threshold."""
    return [(rng.integers(1, levels, size=n) / np.float32(levels)).astype(np.float32).tolist()
            for n in counts[:nprob]]


def test_vote_select_two_compaction_rounds():
    """21 classes, max_per_image 100, 1200 entries: results come from both 1024-entry compaction
    rounds, so the running count carried between rounds places the second round's results."""
    rng = np.random.default_rng(7)
    classes = [_random_classes(rng, 20, [60] * 20, 40) for _ in range(3)]
    classes[1][19] = []                                       # an empty last class
    classes[2][0] = []                                        # an empty first class
    want = check_vote_select(classes, nb=300, keep_stride=100, max_per_image=100, max_results=512)
    for img, w in enumerate(want):
        # entry index (position in the concatenated keep lists) of every result
        s = [np.asarray(c, np.float32) for c in classes[img]]
        start = np.cumsum([0] + [len(c) for c in s])
        entries = np.concatenate([start[p] + np.where(c >= w[2].min())[0] for p, c in enumerate(s)])
        assert len(entries) == len(w[0]) > 100, img           # ties past max_per_image
        assert (entries < 1024).any() and (entries >= 1024).any(), img


def test_vote_select_largest_shared_memory_case_and_limit():
    """max_per_image 199 with 21 classes: 3980 entries, four compaction rounds, 47.8 KB of dynamic
    shared memory.  One more (48.1 KB, plus the kernel's static histogram and warp counts) does not
    fit the 48 KB a launch gets without an opt-in: MNC_ERR_ARG, and nothing is written."""
    MNC_ERR_ARG = 1
    rng = np.random.default_rng(11)
    classes = [_random_classes(rng, 20, [199] * 20, 200)]
    want = check_vote_select(classes, nb=230, keep_stride=199, max_per_image=199, max_results=4096)
    assert len(want[0][0]) >= 199
    scores, order, keep, num_keep = build_vote_case(classes, 230, 199, 0)
    for mpi in (200, 205):
        rc, got = run_vote_select(scores, order, keep, num_keep, mpi, 4096)
        assert rc == MNC_ERR_ARG, (mpi, rc)
        assert np.all(got["res_box_idx"] == SENT_I) and np.all(got["n_res"] == SENT_I)
        assert np.all(got["class_bar"] == SENT_I) and got["overflow"] == 0


def test_vote_select_overflow():
    """More results than max_results: overflow is set, each image holds exactly its first
    max_results results in order with class_bar clamped, and nothing is written past an image's
    slots (the overflowing images are the first and the last; the middle one has no result)."""
    ties = [[0.5, 0.5], [0.9, 0.5], [], [0.5, 0.5, 0.5], [0.5]]
    classes = [ties, [[], [], [], [], []], [[0.5], [0.5, 0.5], [0.5, 0.5], [0.7, 0.5], [0.5, 0.5]]]
    want = check_vote_select(classes, nb=39, keep_stride=5, max_per_image=3, max_results=4)
    assert [len(w[0]) for w in want] == [8, 0, 9]
    want = check_vote_select(classes, nb=39, keep_stride=5, max_per_image=3, max_results=9)
    assert [len(w[0]) for w in want] == [8, 0, 9]


# ============================================================================ mask_voting_checked
def _tied_voting_inputs(nb=24, H=120, W=160, seed=3):
    """nb disjoint 10x10 boxes, one score shared by every class: each class keeps every box, so
    all 20 * nb kept rows tie at the threshold."""
    rng = np.random.default_rng(seed)
    cols = W // 20
    boxes = np.array([[20 * (i % cols) + 2, 20 * (i // cols) + 2, 20 * (i % cols) + 11,
                       20 * (i // cols) + 11] for i in range(nb)], dtype=np.float32)
    assert boxes[:, 3].max() < H
    scores = np.full((nb, 21), 0.5, dtype=np.float32)
    scores[:, 0] = 0.1
    masks = rng.uniform(0, 1, size=(nb, 1, 21, 21)).astype(np.float32)
    return boxes, masks, scores


def test_mask_voting_checked_retries_on_overflow():
    from mnc_b200 import ops
    from oracle import oracle as O
    from tests import util
    H, W = 120, 160
    boxes, masks, scores = _tied_voting_inputs(H=H, W=W)
    nb = boxes.shape[0]
    args = (_dev(boxes)[None], _dev(masks)[None], _dev(scores)[None],
            torch.tensor([[H, W]], dtype=torch.int32, device="cuda"))
    first = ops.mask_voting(*args, max_per_image=100, max_results=128)
    assert int(first["overflow"].item()) == 1 and int(first["n_res"][0].item()) == 128
    r = ops.mask_voting_checked(*args, max_per_image=100)
    k = int(r["n_res"][0].item())
    inds, start, weights, cscores, class_bar = O.mask_voting_candidates(boxes, scores, 21, 100)
    assert int(r["overflow"].item()) == 0 and k == len(start) == 20 * nb
    assert np.array_equal(r["class_bar"][0].cpu().numpy(), np.asarray(class_bar))
    # disjoint boxes: each result's candidate list is its own box, in the reference's result order
    assert np.array_equal(r["res_box_idx"][0, :k].cpu().numpy(), inds)
    assert np.array_equal(r["res_class"][0, :k].cpu().numpy(), np.repeat(np.arange(1, 21), nb))
    assert np.array_equal(r["res_score"][0, :k].cpu().numpy(), cscores)
    lm_o, lb_o = O.gpu_mask_voting(masks, boxes, scores, 21, 100, W, H)
    got_box = r["result_box"][0, :k].cpu().numpy()
    got_mask = r["result_mask"][0, :k].cpu().numpy()
    assert np.array_equal(got_box, np.concatenate([b[:, :4] for b in lb_o]).astype(np.int32))
    assert util.rel_err(got_mask, np.concatenate(lm_o)) < 1e-3


def test_mask_voting_checked_raises_at_full_capacity(monkeypatch):
    """Real inputs cannot overflow the last capacity, nb * (ncls - 1): at most min(nb,
    max_per_image) rows per class are kept.  With every call reporting overflow the retries
    double the capacity up to that bound and then raise VotingOverflow."""
    from mnc_b200 import ops
    boxes, masks, scores = _tied_voting_inputs()
    real, caps = ops.mask_voting, []

    def always_overflows(*a, **kw):
        caps.append(kw["max_results"])
        r = real(*a, **kw)
        r["overflow"].fill_(1)
        return r

    monkeypatch.setattr(ops, "mask_voting", always_overflows)
    with pytest.raises(ops.VotingOverflow):
        ops.mask_voting_checked(_dev(boxes)[None], _dev(masks)[None], _dev(scores)[None],
                                torch.tensor([[120, 160]], dtype=torch.int32, device="cuda"))
    assert caps == [128, 256, 480]


# ============================================================================ gather_boxes
def _special_floats(rng, shape):
    """Random coordinates with a few values a copy must keep bit for bit."""
    a = (rng.standard_normal(shape) * 500).astype(np.float32)
    flat = a.reshape(-1)
    flat[:5] = [np.float32(-0.0), np.float32(1e-40), np.inf,
                np.array([0x7FC01234], np.uint32).view(np.float32)[0], np.float32(3.4e38)]
    return np.ascontiguousarray(rng.permutation(flat).reshape(shape))


def _run_gather(src, src_stride, outer_stride, inner, order, counts, n_out, problems, want_counts):
    from mnc_b200._lib import MNC_OK
    pad = 16
    dst = torch.full((problems * n_out * 4 + pad,), float(SENT_F), dtype=torch.float32, device="cuda")
    oc = torch.full((problems + 1,), SENT_I, dtype=torch.int32, device="cuda") if want_counts else None
    d_src, d_order = _dev(src), _dev(order)
    d_counts = None if counts is None else _dev(counts)
    rc = _lib().mnc_gather_boxes(d_src.data_ptr(), src_stride, outer_stride, inner, d_order.data_ptr(),
                                 order.shape[1], None if d_counts is None else d_counts.data_ptr(),
                                 n_out, problems, dst.data_ptr(), None if oc is None else oc.data_ptr(),
                                 _stream())
    assert rc == MNC_OK
    torch.cuda.synchronize()
    return dst.cpu().numpy(), (None if oc is None else oc.cpu().numpy())


def _check_gather(src, src_stride, outer_stride, inner, order, counts, n_out, problems, want_counts=True):
    dst, oc = _run_gather(src, src_stride, outer_stride, inner, order, counts, n_out, problems, want_counts)
    flat = src.reshape(-1)
    body = dst[:problems * n_out * 4].reshape(problems, n_out, 4)
    for p in range(problems):
        c = min(n_out if counts is None else int(counts[p]), n_out)
        base = (p // inner) * outer_stride + order[p, :c].astype(np.int64) * src_stride
        want = flat[base[:, None] + np.arange(4)[None, :]]
        _same_bits(body[p, :c], want, "problem %d" % p)
        assert np.all(_bits(body[p, c:]) == SENT_BITS), "problem %d: row past the count written" % p
        if oc is not None:
            assert oc[p] == c
    assert np.all(_bits(dst[problems * n_out * 4:]) == SENT_BITS)
    if oc is not None:
        assert oc[problems] == SENT_I


def test_gather_boxes_one_problem_per_image():
    """inner = 1, 5-float rows (dets), padding between images, order_stride > n_out, counts above,
    equal to and at 0 against n_out."""
    rng = np.random.default_rng(1)
    n_src, n_out, problems, order_stride = 50, 40, 3, 64
    outer = n_src * 5 + 7
    src = _special_floats(rng, (problems * outer,))
    order = np.stack([np.concatenate([rng.permutation(n_src), np.full(order_stride - n_src, -1)])
                      for _ in range(problems)]).astype(np.int32)
    _check_gather(src, 5, outer, 1, order, np.array([45, 40, 0], np.int32), n_out, problems)


def test_gather_boxes_per_class_problems():
    """inner = 20 (the per-class voting problems of 2 images share their image's boxes), n_out
    not a multiple of the 256-thread block, ragged counts; counts = NULL (all n_out rows) with and
    without out_counts."""
    rng = np.random.default_rng(2)
    nb, inner, B = 300, 20, 2
    problems = B * inner
    src = _special_floats(rng, (B * nb * 4,))
    order = np.stack([rng.permutation(nb) for _ in range(problems)]).astype(np.int32)
    counts = rng.integers(0, nb + 5, size=problems).astype(np.int32)
    counts[:3] = [0, nb, nb + 4]
    _check_gather(src, 4, nb * 4, inner, order, counts, nb, problems)
    _check_gather(src, 4, nb * 4, inner, order, counts, 257, problems)
    _check_gather(src, 4, nb * 4, inner, order, None, 257, problems)
    _check_gather(src, 4, nb * 4, inner, order, None, 257, problems, want_counts=False)


# ============================================================================ write_rois
def test_write_rois():
    """num_keep 0, above max_rois and in between; max_rois not a multiple of the 128-thread block;
    keep_stride != max_rois; both batch-index modes.  Rows past the count are [bi, 0, 0, 0, 0]
    (bi = the image in batch-index mode, else 0), exactly +0.0."""
    from mnc_b200._lib import MNC_OK
    rng = np.random.default_rng(4)
    B, n_sorted, max_rois, keep_stride = 3, 260, 200, 230
    boxes = _special_floats(rng, (B, n_sorted, 4))
    keep = np.stack([rng.permutation(n_sorted)[:keep_stride] for _ in range(B)]).astype(np.int32)
    num_keep = np.array([0, max_rois + 10, 57], np.int32)
    d_boxes, d_keep, d_num = _dev(boxes), _dev(keep), _dev(num_keep)
    pad = 16
    for mode in (1, 0):
        rois = torch.full((B * max_rois * 5 + pad,), float(SENT_F), dtype=torch.float32, device="cuda")
        counts = torch.full((B + 1,), SENT_I, dtype=torch.int32, device="cuda")
        rc = _lib().mnc_write_rois(d_boxes.data_ptr(), n_sorted, d_keep.data_ptr(), keep_stride,
                                   d_num.data_ptr(), max_rois, B, mode, rois.data_ptr(),
                                   counts.data_ptr(), _stream())
        assert rc == MNC_OK
        got = rois.cpu().numpy()
        cnt = counts.cpu().numpy()
        want = np.zeros((B, max_rois, 5), np.float32)
        for img in range(B):
            nk = min(int(num_keep[img]), max_rois)
            want[img, :, 0] = img if mode else 0
            want[img, :nk, 1:] = boxes[img, keep[img, :nk]]
            assert cnt[img] == nk
        assert cnt[B] == SENT_I
        _same_bits(got[:B * max_rois * 5].reshape(B, max_rois, 5), want, "rois mode %d" % mode)
        assert np.all(_bits(got[B * max_rois * 5:]) == SENT_BITS)


# ============================================================================ unscale_clip / detect_tail
def clip_ref(boxes, H, W):
    """clip_boxes (bbox_transform.py:102-120) with im.shape's ints."""
    out = np.zeros(boxes.shape, dtype=boxes.dtype)
    out[:, 0::4] = np.maximum(np.minimum(boxes[:, 0::4], W - 1), 0)
    out[:, 1::4] = np.maximum(np.minimum(boxes[:, 1::4], H - 1), 0)
    out[:, 2::4] = np.maximum(np.minimum(boxes[:, 2::4], W - 1), 0)
    out[:, 3::4] = np.maximum(np.minimum(boxes[:, 3::4], H - 1), 0)
    return out


def unscale_clip_ref(rois, rois_per_img, im_scale, im_hw):
    """demo.py:92-95 per image: rois[:, 1:5] / im_scale (float32, as numpy 1.x divides a float32
    array by a Python float), then clip_boxes."""
    out = np.zeros((rois.shape[0], 4), np.float32)
    for img in range(len(im_scale)):
        sl = slice(img * rois_per_img, (img + 1) * rois_per_img)
        out[sl] = clip_ref(rois[sl, 1:5] / np.float32(im_scale[img]), int(im_hw[img][0]),
                           int(im_hw[img][1]))
    return out


def _coord_dividing_to(q, s):
    """An fp32 coordinate r with fl(r / s) == q, searched around q * s."""
    r = np.float32(np.float64(q) * np.float64(s))
    for _ in range(64):
        d = np.float32(r / s)
        if d == q:
            return r
        r = np.nextafter(r, np.float32(np.inf) if d < q else np.float32(-np.inf))
    return None


IM_SCALE = np.array([1.6, 0.75, 2.0], np.float32)
IM_HW = np.array([[600, 1000], [333, 517], [480, 640]], np.float32)


def _tail_rois(rng, n, seed_scale=IM_SCALE, im_hw=IM_HW):
    """n RoIs per image in the resized image, plus edge rows: coordinates that divide back to
    exactly W-1 / H-1, to one ulp either side of them, past the image, and negative."""
    B = len(seed_scale)
    rois = np.zeros((B * n, 5), np.float32)
    for img in range(B):
        s, (H, W) = seed_scale[img], im_hw[img]
        sl = slice(img * n, (img + 1) * n)
        rois[sl, 0] = img
        rois[sl, 1:5] = rng.uniform(-30, 1.1 * max(H, W), size=(n, 4)) * s
        edge = []
        for lim in (W - 1, H - 1):
            lim = np.float32(lim)
            for q in (lim, np.nextafter(lim, np.float32(0)), np.nextafter(lim, np.float32(1e9))):
                r = _coord_dividing_to(q, s)
                assert r is not None, (img, q)
                edge.append(r)
        x_lim, x_dn, x_up, y_lim, y_dn, y_up = edge
        rows = [[x_lim, y_lim, x_dn, y_dn], [x_up, y_up, x_lim, y_lim], [x_dn, y_up, x_up, y_dn],
                [-s, -0.25 * s, -1e-3, -1e-30], [np.float32(1e-40), 0.0, 2 * W * s, 2 * H * s]]
        rois[img * n:img * n + len(rows), 1:5] = np.asarray(rows, np.float32)
    return rois


def test_unscale_clip_batch():
    from mnc_b200._lib import MNC_OK
    rng = np.random.default_rng(5)
    n = 70                                     # 210 RoIs: two blocks, the second partial
    rois = _tail_rois(rng, n)
    total = rois.shape[0]
    out = torch.full((total * 4 + 8,), float(SENT_F), dtype=torch.float32, device="cuda")
    d_rois, d_s, d_hw = _dev(rois), _dev(IM_SCALE), _dev(IM_HW)
    rc = _lib().mnc_unscale_clip(d_rois.data_ptr(), total, n, d_s.data_ptr(), d_hw.data_ptr(),
                                 out.data_ptr(), _stream())
    assert rc == MNC_OK
    got = out.cpu().numpy()
    want = unscale_clip_ref(rois, n, IM_SCALE, IM_HW)
    _same_bits(got[:total * 4].reshape(total, 4), want, "unscale_clip")
    assert np.all(_bits(got[total * 4:]) == SENT_BITS)
    # the edge rows reach both sides of the limits
    for img in range(3):
        H, W = IM_HW[img]
        w = want[img * n:img * n + 5]
        assert (w[:, 0::2] == W - 1).sum() >= 3 and (w[:, 1::2] == H - 1).sum() >= 3
        assert ((w[:, 0::2] < W - 1) & (w[:, 0::2] > W - 2)).any()
        assert (w[3] == 0).all()
    # ops wrapper: same result
    assert np.array_equal(_bits(ops_unscale_clip(d_rois, n, d_s, d_hw)), _bits(want))


def ops_unscale_clip(d_rois, n, d_s, d_hw):
    from mnc_b200 import ops
    return ops.unscale_clip(d_rois, n, d_s, d_hw).cpu().numpy()


def test_detect_tail_record():
    """The per-step output record: counts = 2 * roi_counts, boxes of stage 1 then stage 2 (every
    row, valid or not), scores and masks copied bit for bit, valid = row < roi_counts in each
    stage; the padding after counts and the space past the record stay untouched."""
    from mnc_b200 import ops
    rng = np.random.default_rng(6)
    B, n, msz, ncls = 3, 37, 441, 21
    rois, rois_ext = _tail_rois(rng, n), _tail_rois(rng, n)[::-1].copy()
    o = {"rois": _dev(rois), "rois_ext": _dev(rois_ext),
         "mask_proposal": _dev(_special_floats(rng, (B * n, 1, 21, 21))),
         "mask_proposal_ext": _dev(_special_floats(rng, (B * n, 1, 21, 21))),
         "seg_cls_prob": _dev(_special_floats(rng, (B * n, ncls))),
         "seg_cls_prob_ext": _dev(_special_floats(rng, (B * n, ncls))),
         "roi_counts": _dev(np.array([n, 0, 20], np.int32))}
    ob, os_, om, end = ops.record_layout(B, n, msz, ncls)
    rec = torch.full((end + 32,), float(SENT_F), dtype=torch.float32, device="cuda")
    valid = torch.full((B * 2 * n + 8,), 0xAB, dtype=torch.uint8, device="cuda")
    d_s, d_hw = _dev(IM_SCALE), _dev(IM_HW)
    ops.detect_tail(o, B, n, d_s, d_hw, rec[:end], valid[:B * 2 * n])
    got, v = rec.cpu().numpy(), valid.cpu().numpy()
    cnt = np.array([n, 0, 20])
    _same_bits(got[:B], 2 * cnt, "counts")
    assert np.all(_bits(got[B:ob]) == SENT_BITS) and np.all(_bits(got[end:]) == SENT_BITS)
    b1 = unscale_clip_ref(rois, n, IM_SCALE, IM_HW).reshape(B, n, 4)
    b2 = unscale_clip_ref(rois_ext, n, IM_SCALE, IM_HW).reshape(B, n, 4)
    _same_bits(got[ob:os_].reshape(B, 2 * n, 4), np.concatenate([b1, b2], axis=1), "boxes")
    host = {k: t.cpu().numpy() for k, t in o.items()}
    sc = np.concatenate([host["seg_cls_prob"].reshape(B, n, ncls),
                         host["seg_cls_prob_ext"].reshape(B, n, ncls)], axis=1)
    _same_bits(got[os_:om].reshape(B, 2 * n, ncls), sc, "scores")
    mk = np.concatenate([host["mask_proposal"].reshape(B, n, msz),
                         host["mask_proposal_ext"].reshape(B, n, msz)], axis=1)
    _same_bits(got[om:end].reshape(B, 2 * n, msz), mk, "masks")
    row = np.arange(2 * n) % n
    assert np.array_equal(v[:B * 2 * n].reshape(B, 2 * n), (row[None, :] < cnt[:, None]).astype(np.uint8))
    assert np.all(v[B * 2 * n:] == 0xAB)


# ============================================================================ decode_class_boxes
def bbox_transform_inv_ref(boxes, deltas):
    """bbox_transform.py:64-99, every operation in float32 as numpy evaluates it."""
    widths = boxes[:, 2] - boxes[:, 0] + 1.0
    heights = boxes[:, 3] - boxes[:, 1] + 1.0
    ctr_x = boxes[:, 0] + 0.5 * widths
    ctr_y = boxes[:, 1] + 0.5 * heights
    dx, dy, dw, dh = deltas[:, 0::4], deltas[:, 1::4], deltas[:, 2::4], deltas[:, 3::4]
    pred_ctr_x = dx * widths[:, None] + ctr_x[:, None]
    pred_ctr_y = dy * heights[:, None] + ctr_y[:, None]
    with np.errstate(over="ignore", invalid="ignore"):
        pred_w = np.exp(dw) * widths[:, None]
        pred_h = np.exp(dh) * heights[:, None]
        pred = np.zeros(deltas.shape, dtype=deltas.dtype)
        pred[:, 0::4] = pred_ctr_x - 0.5 * pred_w
        pred[:, 1::4] = pred_ctr_y - 0.5 * pred_h
        pred[:, 2::4] = pred_ctr_x + 0.5 * pred_w
        pred[:, 3::4] = pred_ctr_y + 0.5 * pred_h
    return pred


def decode_class_boxes_ref(rois, deltas, rois_per_img, im_scale, im_hw):
    """TesterWrapper._detection_forward tail per image: boxes = rois[:, 1:5] / im_scale,
    bbox_transform_inv, clip_boxes to the original image."""
    out = np.zeros(deltas.shape, np.float32)
    for img in range(len(im_scale)):
        sl = slice(img * rois_per_img, (img + 1) * rois_per_img)
        boxes = rois[sl, 1:5] / np.float32(im_scale[img])
        with np.errstate(invalid="ignore"):
            out[sl] = clip_ref(bbox_transform_inv_ref(boxes, deltas[sl]), int(im_hw[img][0]),
                               int(im_hw[img][1]))
    return out


def _run_decode(rois, bbox_full, ncls, rois_per_img, im_scale, im_hw):
    """mnc_decode_class_boxes with bbox_stride = bbox_full's row length (> 4 * ncls allowed)."""
    from mnc_b200._lib import MNC_OK
    R = rois.shape[0]
    out = torch.full((R * ncls * 4 + 16,), float(SENT_F), dtype=torch.float32, device="cuda")
    d_rois, d_bbox, d_s, d_hw = _dev(rois), _dev(bbox_full), _dev(im_scale), _dev(im_hw)
    rc = _lib().mnc_decode_class_boxes(d_rois.data_ptr(), R, rois_per_img, d_bbox.data_ptr(),
                                       bbox_full.shape[1], ncls, d_s.data_ptr(), d_hw.data_ptr(),
                                       out.data_ptr(), _stream())
    assert rc == MNC_OK
    got = out.cpu().numpy()
    assert np.all(_bits(got[R * ncls * 4:]) == SENT_BITS)
    return got[:R * ncls * 4].reshape(R, ncls * 4)


def _decode_inputs(rng, n, ncls, extra):
    """Per (RoI, class) a kind: 0 = dw = dh = 0 (exp is exactly 1 on both sides), 1 = dw, dh =
    +-100 (exp is inf or underflows on both sides), 2 = random dw, dh."""
    rois = _tail_rois(rng, n)
    R = rois.shape[0]
    rois[:, 3:5] = np.maximum(rois[:, 3:5], rois[:, 1:3])      # x2 >= x1: positive widths
    kind = rng.integers(0, 3, size=(R, ncls))
    d = np.zeros((R, ncls, 4), np.float32)
    d[:, :, :2] = rng.normal(0, 0.3, size=(R, ncls, 2))
    big = np.where(rng.integers(0, 2, size=(R, ncls, 2)) == 1, 100.0, -100.0)
    d[:, :, 2:] = np.where((kind == 1)[:, :, None], big,
                           np.where((kind == 2)[:, :, None], rng.normal(0, 0.5, size=(R, ncls, 2)), 0))
    full = np.full((R, 4 * ncls + extra), np.nan, np.float32)     # columns past 4*ncls never read
    full[:, :4 * ncls] = d.reshape(R, 4 * ncls)
    return rois, full, kind


@pytest.mark.parametrize("ncls,extra", [(21, 12), (3, 0), (5, 3)])
def test_decode_class_boxes(ncls, extra):
    """Bit-exact where exp cannot differ (kinds 0 and 1), 1e-5 relative elsewhere; bbox_stride >
    4 * ncls, 3 images split by rois_per_img with their own scale and size, R * ncls not a multiple
    of 128."""
    rng = np.random.default_rng(8 + ncls)
    n = 45
    rois, full, kind = _decode_inputs(rng, n, ncls, extra)
    R = rois.shape[0]
    assert (R * ncls) % 128
    got = _run_decode(rois, full, ncls, n, IM_SCALE, IM_HW).reshape(R, ncls, 4)
    want = decode_class_boxes_ref(rois, full[:, :4 * ncls], n, IM_SCALE, IM_HW).reshape(R, ncls, 4)
    exact = kind != 2
    _same_bits(got[exact], want[exact], "decode (exp exact)")
    assert np.allclose(got[~exact], want[~exact], rtol=1e-5, atol=2e-3)
    # exp(+100) = inf: the box spans the image; exp(-100) ~ 0: x1 == x2
    W = np.repeat(IM_HW[:, 1], n)[:, None]
    dw = full[:, 2:4 * ncls:4]
    assert np.all(got[:, :, 0][dw == 100] == 0) and np.all(got[:, :, 2][dw == 100] == np.broadcast_to(W - 1, dw.shape)[dw == 100])
    assert np.array_equal(got[:, :, 0][dw == -100], got[:, :, 2][dw == -100])
    assert (dw == 100).any() and (dw == -100).any()
    # ops wrapper: bbox_stride from the view's row stride
    from mnc_b200 import ops
    d_full = _dev(full)
    via_ops = ops.decode_class_boxes(_dev(rois), d_full[:, :4 * ncls], n, _dev(IM_SCALE), _dev(IM_HW),
                                     ncls=ncls).cpu().numpy()
    _same_bits(via_ops.reshape(R, ncls, 4), got, "ops.decode_class_boxes")


def test_decode_class_boxes_rejects_short_stride():
    rng = np.random.default_rng(9)
    rois, full, _ = _decode_inputs(rng, 8, 21, 0)
    d_rois, d_bbox, d_s, d_hw = _dev(rois), _dev(full), _dev(IM_SCALE), _dev(IM_HW)
    out = torch.empty((rois.shape[0], 21 * 4), dtype=torch.float32, device="cuda")
    rc = _lib().mnc_decode_class_boxes(d_rois.data_ptr(), rois.shape[0], 8, d_bbox.data_ptr(), 4 * 21 - 1,
                                       21, d_s.data_ptr(), d_hw.data_ptr(), out.data_ptr(), _stream())
    assert rc == 1                                            # MNC_ERR_ARG


# ============================================================================ NaN deltas
def test_decode_class_boxes_nan_delta_propagates():
    """A NaN delta gives a NaN coordinate, as clip_boxes' np.maximum(np.minimum(...)) does: dx / dw
    poison x1 and x2, dy / dh poison y1 and y2, and the other class columns are unaffected."""
    rng = np.random.default_rng(10)
    n, ncls = 8, 21
    rois, full, kind = _decode_inputs(rng, n, ncls, 4)
    R = rois.shape[0]
    full[:, 2:4 * ncls:4][kind == 2] = 0.0                    # exact everywhere ...
    full[:, 3:4 * ncls:4][kind == 2] = 0.0
    for r, c, j in [(0, 1, 0), (1, 5, 1), (2, 20, 2), (n + 3, 0, 3), (2 * n + 4, 7, 2), (2 * n + 4, 8, 1)]:
        full[r, 4 * c + j] = np.nan                           # ... but for the NaN deltas
    got = _run_decode(rois, full, ncls, n, IM_SCALE, IM_HW)
    want = decode_class_boxes_ref(rois, full[:, :4 * ncls], n, IM_SCALE, IM_HW)
    assert np.isnan(want).sum() == 12
    _same_bits(got, want, "decode with NaN deltas")


def test_rpn_nan_delta_is_filtered():
    """In the proposal path a NaN coordinate fails the min-size test (as in filter_small_boxes), so
    the RoIs are those of the reference on the same inputs and hold no NaN."""
    from mnc_b200 import ops
    from oracle import oracle as O
    from tests.test_gpu_proposal import _rpn_inputs, _oracle_from_device_decode
    H, W = 14, 20
    _, prob, deltas = _rpn_inputs(H, W, seed=H)
    im_info = np.array([[224, 320, 1.0]], dtype=np.float32)
    # anchor t = (y * W + x) * 9 + a reads deltas[0, 4a + j, y, x]
    poisoned = []
    for (y, x, a, j) in [(3, 4, 0, 0), (7, 11, 4, 1), (10, 2, 8, 2), (0, 19, 5, 3)]:
        deltas[0, 4 * a + j, y, x] = np.nan
        prob[0, 9 + a, y, x] = 0.999                          # would be among the first RoIs
        poisoned.append((y * W + x) * 9 + a)
    r, cnt, mid = ops.proposals_from_rpn(_dev(prob), _dev(deltas), _dev(im_info), 1, H, W, "nchw", False,
                                         batch_index_mode=False, return_intermediate=True)
    props = mid["proposals"][0].cpu().numpy()
    valid = mid["valid"][0].cpu().numpy()
    scores = mid["scores"][0].cpu().numpy()
    assert np.all(valid[poisoned] == 0)
    assert np.all(np.isnan(props[poisoned]).any(axis=1))
    want_rois, inter = O.proposal_layer_forward(prob, deltas, im_info, return_intermediate=True)
    assert np.array_equal(np.isnan(props), np.isnan(inter["all_proposals"]))
    k = int(cnt[0].item())
    rois = r[0, :k].cpu().numpy()
    assert k > 0 and np.isfinite(rois).all()
    forced_boxes, forced_idx = _oracle_from_device_decode(props, scores, valid)
    assert np.array_equal(rois[:, 1:], forced_boxes)
    assert np.array_equal(forced_idx, inter["roi_anchor_index"])
    assert not np.isin(poisoned, forced_idx).any()
