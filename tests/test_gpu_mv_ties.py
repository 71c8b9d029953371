"""Mask voting where one pixel's aggregate sits on the 0.4 threshold or a few ulps from it
(tests/mv_ties.py): every entry point must give the tight boxes and the resampled masks of the
reference `_mv` as nvcc builds it (the `ref` emulation) bit for bit.  When oracle/_ref holds the
reference's own `_mv`, it must give the `ref` emulation too, and its -fmad=false build the `nofma`
one.  Also: candidate lists at IoU = 0.5 exactly and the nearest float32 boxes either side."""
import ctypes
import os

import numpy as np
import pytest

from tests import mv_ties as T

pytestmark = pytest.mark.gpu
IMAGES = range(len(T.IMAGES))
REF_SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref",
                      "libmnc_ref.so")


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _same(got_box, got_mask, cases, rounding="ref"):
    eb, em = T.expected(cases, rounding)
    bad = np.flatnonzero((np.asarray(got_box)[:, :4] != eb).any(1))
    assert len(bad) == 0, [(cases[i]["plan"], cases[i]["offset"], list(got_box[i]), list(eb[i])) for i in bad[:5]]
    assert np.array_equal(np.asarray(got_mask, dtype=np.float32).view(np.int32), em.view(np.int32))


@pytest.mark.parametrize("img", IMAGES)
def test_mv_host_ties(img):
    """mnc_mv_host, the `_mv` drop-in, and nms.mv.mv over it."""
    from mnc_b200._lib import lib, check
    import mnc_b200.lib as L
    L.install()
    from nms.mv import mv
    H, W, _, cases = T.image_cases(img)
    boxes, masks, inds, start, wts = T.pack(cases)
    k = len(start)
    rm = np.zeros((k, 1, T.M, T.M), np.float32)
    rb = np.zeros((k, 4), np.int32)
    check(lib.mnc_mv_host(_p(boxes), _p(masks), len(boxes), _p(inds), _p(start), _p(wts), len(inds),
                          H, W, 4, T.M, k, _p(rm), _p(rb), 0), "mnc_mv_host")
    _same(rb, rm, cases)
    rm2, rb2 = mv(boxes, masks, inds, start, wts, H, W)
    _same(rb2, rm2, cases)


@pytest.mark.parametrize("two_pass", [True, False])
def test_mv_device_ties(two_pass):
    """mnc_mv_device (the kernels of ops.mask_voting) on all images in one batch: two image sizes,
    unit range (early exit, region cut) and not (full sums), coarse + border pass or one sweep."""
    import torch
    from mnc_b200 import ops
    from mnc_b200._lib import lib, check
    packs = [(T.image_cases(i), T.pack(T.image_cases(i)[3])) for i in IMAGES]
    B = len(packs)
    nb = max(len(p[1][0]) for p in packs)
    R = max(len(p[1][3]) for p in packs)
    boxes = np.zeros((B, nb, 4), np.float32)
    masks = np.zeros((B, nb, 1, T.M, T.M), np.float32)
    stride = R * nb
    cinds = np.zeros((B, stride), np.int32)
    cw = np.zeros((B, stride), np.float32)
    beg = np.zeros((B, R), np.int32)
    end = np.zeros((B, R), np.int32)
    n_res = np.zeros(B, np.int32)
    hw = np.zeros((B, 2), np.int32)
    for b, ((H, W, _, cases), (bx, mk, ii, st, ww)) in enumerate(packs):
        boxes[b, :len(bx)], masks[b, :len(bx)] = bx, mk
        # lists placed with gaps between them, as ops.mask_voting lays them out
        s0 = np.concatenate([[0], st[:-1]])
        for t, (lo, hi) in enumerate(zip(s0, st)):
            beg[b, t], end[b, t] = t * nb, t * nb + (hi - lo)
            cinds[b, t * nb:t * nb + hi - lo] = ii[lo:hi]
            cw[b, t * nb:t * nb + hi - lo] = ww[lo:hi]
        n_res[b] = len(st)
        hw[b] = (H, W)
    d = {k: torch.from_numpy(v).cuda() for k, v in dict(boxes=boxes, masks=masks, cinds=cinds, cw=cw,
                                                          beg=beg, end=end, n_res=n_res, hw=hw).items()}
    ws = torch.zeros(B * R * 4 + B, dtype=torch.int32, device="cuda")
    om = torch.zeros((B, R, 1, T.M, T.M), dtype=torch.float32, device="cuda")
    ob = torch.zeros((B, R, 4), dtype=torch.int32, device="cuda")
    prev = ops.mv_set_two_pass(two_pass)
    try:
        check(lib.mnc_mv_device(d["boxes"].data_ptr(), d["masks"].data_ptr(), nb, 4, T.M,
                                d["cinds"].data_ptr(), d["cw"].data_ptr(), stride, d["beg"].data_ptr(),
                                d["end"].data_ptr(), d["n_res"].data_ptr(), R, B, d["hw"].data_ptr(),
                                ws.data_ptr(), om.data_ptr(), ob.data_ptr(), None), "mnc_mv_device")
        torch.cuda.synchronize()
    finally:
        ops.mv_set_two_pass(prev)
    unit = ws[B * R * 4:].cpu().numpy()
    assert list(unit) == [int(T.IMAGES[i][2]) for i in IMAGES]      # which path each image took
    for b, ((H, W, _, cases), _) in enumerate(packs):
        k = len(cases)
        _same(ob[b, :k].cpu().numpy(), om[b, :k].cpu().numpy(), cases)


@pytest.mark.parametrize("img", IMAGES)
def test_reference_mv_ties(img):
    """The reference's `_mv` (lib/nms/mv_kernel.cu compiled unmodified) gives the `ref` emulation,
    and the same source built with -fmad=false gives the `nofma` one."""
    if not os.path.exists(REF_SO):
        pytest.skip("oracle/_ref/libmnc_ref*.so not built (needs the reference's sources at build time)")
    H, W, _, cases = T.image_cases(img)
    boxes, masks, inds, start, wts = T.pack(cases)
    k = len(start)
    for so, rounding in ((REF_SO, "ref"), (REF_SO.replace(".so", "_nofma.so"), "nofma")):
        rm = np.zeros((k, 1, T.M, T.M), np.float32)
        rb = np.zeros((k, 4), np.int32)
        ctypes.CDLL(so)._Z3_mvPKfS0_iPKiS2_S0_iiiiiiPfPii(
            _p(boxes), _p(masks), len(boxes), _p(inds), _p(start), _p(wts), len(inds), H, W, 4, T.M, k,
            _p(rm), _p(rb), 0)
        _same(rb, rm, cases, rounding)


def _iou_tie_boxes():
    """Query box 0 and boxes whose float64 IoU with it is 0.5 exactly (integer boxes), or whose
    x2 is the float32 next to such a box's either way (the IoU is then just off 0.5)."""
    q = np.array([[10, 20, 109, 39]], np.float32)                     # 100 x 20
    out = [q[0]]
    out.append(np.array([10, 20, 59, 39], np.float32))                # left half: I / U = 1/2
    out.append(np.array([60, 20, 109, 39], np.float32))               # right half
    out.append(np.array([10, 20, 109, 59], np.float32))               # double height: 2000/4000
    out.append(np.array([-40, 20, 159, 39], np.float32))              # double width, centred
    base = list(out[1:])
    for b in base:
        for direction in (-np.inf, np.inf):
            for k in (1, 2):
                c = b.copy()
                for _ in range(k):
                    c[2] = np.nextafter(c[2], np.float32(direction))
                out.append(c)
    return np.array(out, np.float32)


def _iou64(b, q):
    iw = min(b[2], q[2]) - max(b[0], q[0]) + 1.0
    ih = min(b[3], q[3]) - max(b[1], q[1]) + 1.0
    if iw <= 0 or ih <= 0:
        return 0.0
    return iw * ih / ((b[2] - b[0] + 1.0) * (b[3] - b[1] + 1.0) + (q[2] - q[0] + 1.0) * (q[3] - q[1] + 1.0) - iw * ih)


def test_candidate_lists_at_iou_half():
    """mnc_bbox_overlaps_host equals the float64 IoU bit for bit, and mnc_vote_candidates keeps
    exactly the boxes with IoU >= 0.5 (ties included) in index order, with the reference's weights."""
    import torch
    from mnc_b200._lib import lib, check
    boxes = _iou_tie_boxes()
    nb = len(boxes)
    b64, q64 = boxes.astype(np.float64), boxes[:1].astype(np.float64)
    want = np.array([_iou64(b, q64[0]) for b in b64])
    assert (want == 0.5).sum() == 4 and ((want > 0.5) & (want < 0.5 + 1e-6)).any() and \
        ((want < 0.5) & (want > 0.5 - 1e-6)).any()
    out = np.zeros((nb, 1), np.float64)
    check(lib.mnc_bbox_overlaps_host(_p(np.ascontiguousarray(b64)), nb, _p(np.ascontiguousarray(q64)), 1,
                                     _p(out)), "mnc_bbox_overlaps_host")
    assert np.array_equal(out[:, 0], want)
    rng = np.random.default_rng(3)
    ncls = 3
    scores = rng.uniform(0.05, 1, (1, nb, ncls)).astype(np.float32)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()            # noqa: E731
    R = 1
    res_idx, res_cls, n_res = dev(np.zeros((1, R), np.int32)), dev(np.full((1, R), 2, np.int32)), \
        dev(np.ones(1, np.int32))
    ci = torch.zeros((1, R, nb), dtype=torch.int32, device="cuda")
    cw = torch.zeros((1, R, nb), dtype=torch.float32, device="cuda")
    cb = torch.zeros((1, R), dtype=torch.int32, device="cuda")
    ce = torch.zeros((1, R), dtype=torch.int32, device="cuda")
    db, ds = dev(boxes[None]), dev(scores)
    check(lib.mnc_vote_candidates(db.data_ptr(), ds.data_ptr(), None, nb, ncls, res_idx.data_ptr(),
                                  res_cls.data_ptr(), n_res.data_ptr(), R, 1, 0.5, ci.data_ptr(),
                                  cw.data_ptr(), cb.data_ptr(), ce.data_ptr(), None), "mnc_vote_candidates")
    torch.cuda.synchronize()
    keep = np.flatnonzero(want >= 0.5)
    n = int(ce[0, 0].item() - cb[0, 0].item())
    assert n == len(keep) and np.array_equal(ci[0, 0, :n].cpu().numpy(), keep)
    s = scores[0, keep, 2]
    total = np.float32(sum(float(v) for v in s))
    assert np.array_equal(cw[0, 0, :n].cpu().numpy(), s / total)
