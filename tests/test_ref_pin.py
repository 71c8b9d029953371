"""Pin the oracle AND the CUDA path against the reference's own kernels: lib/nms/nms_kernel.cu and
lib/nms/mv_kernel.cu compiled unmodified into oracle/_ref/libmnc_ref.so (oracle/Makefile `ref`).
The .so is built in the build container and travels with the snapshot; /root/reference itself is
not needed at run time."""
import ctypes
import os

import numpy as np
import pytest

from tests import util

pytestmark = pytest.mark.gpu
REF_SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref",
                      "libmnc_ref.so")


def _ref(nofma=False):
    so = REF_SO.replace(".so", "_nofma.so") if nofma else REF_SO
    if not os.path.exists(so):
        pytest.skip("oracle/_ref/libmnc_ref*.so not built (needs /root/reference at build time)")
    return ctypes.CDLL(so)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.mark.parametrize("n,thresh,seed", [(600, 0.3, 1), (6000, 0.7, 2), (10000, 0.7, 10)])
def test_nms_three_way(n, thresh, seed):
    """reference `_nms` == oracle orc_nms == mnc_nms_host, float boxes, no margin nudging."""
    from oracle import oracle as O
    from mnc_b200._lib import lib, check
    ref = _ref()
    boxes = util.random_boxes(n, seed=seed)
    scores = util.tie_free_scores(n, seed=seed + 1)
    dets = np.hstack([boxes, scores[:, None]]).astype(np.float32)
    sorted_dets = np.ascontiguousarray(dets[O.order_desc(scores)])
    keep_ref = np.zeros(n, dtype=np.int32)
    num_ref = ctypes.c_int(0)
    ref._Z4_nmsPiS_PKfiifi(_p(keep_ref), ctypes.byref(num_ref), _p(sorted_dets), n, 5,
                           ctypes.c_float(thresh), 0)
    keep_ref = keep_ref[:num_ref.value]
    keep = np.zeros(n, dtype=np.int32)
    num = ctypes.c_int(0)
    check(lib.mnc_nms_host(_p(keep), ctypes.byref(num), _p(sorted_dets), n, 5,
                           ctypes.c_float(thresh), 0), "mnc_nms_host")
    assert np.array_equal(keep[:num.value], keep_ref), "CUDA path differs from reference _nms"
    assert np.array_equal(O.nms_sorted(sorted_dets, thresh), keep_ref), "oracle differs from reference _nms"


def _voting_inputs(nb, H, W, seed):
    rng = np.random.default_rng(seed)
    boxes = util.random_boxes(nb, seed=seed, width=W, height=H, smin=12, smax=min(H, W) * 0.8)
    masks = (1.0 / (1.0 + np.exp(-rng.normal(0, 2, size=(nb, 1, 21, 21))))).astype(np.float32)
    logits = rng.normal(0, 1, size=(nb, 21))
    scores = (np.exp(logits) / np.exp(logits).sum(1, keepdims=True)).astype(np.float32)
    return boxes, masks, scores


def test_mv_three_way():
    """reference `_mv` vs oracle orc_mv vs mnc_mv_host on gpu_mask_voting's candidate lists
    (small image so the reference's nb*H*W render buffer stays small)."""
    from oracle import oracle as O
    from mnc_b200._lib import lib, check
    ref = _ref()
    nb, H, W = 120, 150, 200
    boxes, masks, scores = _voting_inputs(nb, H, W, seed=21)
    inds, start, weights, cscores, _ = O.mask_voting_candidates(boxes, scores, 21, 100)
    k = len(start)
    assert k > 10
    rm_ref = np.zeros((k, 1, 21, 21), dtype=np.float32)
    rb_ref = np.zeros((k, 4), dtype=np.int32)
    ref._Z3_mvPKfS0_iPKiS2_S0_iiiiiiPfPii(_p(boxes), _p(masks), nb, _p(inds), _p(start), _p(weights),
                                          len(inds), H, W, 4, 21, k, _p(rm_ref), _p(rb_ref), 0)
    rm_o, rb_o = O.mv(boxes, masks, inds, start, weights, H, W)
    rm = np.zeros_like(rm_ref)
    rb = np.zeros_like(rb_ref)
    check(lib.mnc_mv_host(_p(boxes), _p(masks), nb, _p(inds), _p(start), _p(weights), len(inds), H,
                          W, 4, 21, k, _p(rm), _p(rb), 0), "mnc_mv_host")
    # boxes: int-exact unless an aggregate value sits within an ulp of 0.4 (FMA contraction);
    # allow no mismatch on this seeded input
    assert np.array_equal(rb_o, rb_ref), "oracle boxes differ from reference _mv"
    assert np.array_equal(rb, rb_ref), "CUDA boxes differ from reference _mv"
    # mask values: the reference binary contracts a*b+c into FMA, the C oracle does not
    assert util.rel_err(rm_o, rm_ref) < 1e-4
    assert util.rel_err(rm, rm_ref) < 1e-4
    # ... and with contraction off (-fmad=false build of the same source) the reference equals the
    # oracle bit for bit
    nf = _ref(True)
    rm_nf = np.zeros_like(rm_ref)
    rb_nf = np.zeros_like(rb_ref)
    nf._Z3_mvPKfS0_iPKiS2_S0_iiiiiiPfPii(_p(boxes), _p(masks), nb, _p(inds), _p(start), _p(weights),
                                         len(inds), H, W, 4, 21, k, _p(rm_nf), _p(rb_nf), 0)
    assert np.array_equal(rb_nf, rb_o) and np.array_equal(rm_nf, rm_o)


# ------------------------------------------------------------------------------------------------
# Replay of the native calls the reference's Python made while scripts/make_ref_fixtures.py produced
# tests/golden/ref_*.npz.  There (no GPU) `gpu_nms` was answered by the reference's py_cpu_nms.py
# and `mv` by the C oracle; here the recorded inputs go through the reference's REAL CUDA
# extensions (`_nms`, `_mv`, compiled unmodified) and must reproduce the recorded outputs -- which
# closes the chain fixture == reference-with-its-own-extensions.
def _ref_gpu_nms(ref, dets, thresh):
    """lib/nms/gpu_nms.pyx:16-31 around the reference's `_nms`."""
    n = dets.shape[0]
    keep = np.zeros(n, dtype=np.int32)
    num = ctypes.c_int(0)
    order = dets[:, 4].argsort()[::-1]
    sorted_dets = np.ascontiguousarray(dets[order, :])
    ref._Z4_nmsPiS_PKfiifi(_p(keep), ctypes.byref(num), _p(sorted_dets), n, dets.shape[1],
                           ctypes.c_float(thresh), 0)
    return order[keep[:num.value]]


def test_recorded_native_calls_replay():
    from tests.test_ref_fixtures import load, voting_case
    ref = _ref()
    f = load("ref_native_calls.npz")
    for tag in f["cases"]:                        # ProposalLayer.forward -> nms(dets, 0.7)
        got = _ref_gpu_nms(ref, f["dets_" + tag], float(f["thresh_" + tag]))
        assert np.array_equal(got, f["keep_" + tag]), tag
    v = load("ref_voting.npz")
    for tag in ("a", "b", "c"):
        boxes, masks, scores, H, W = voting_case(v, tag)
        for c in range(1, 21):                    # gpu_mask_voting -> nms(dets, 0.3) per class
            dets = np.hstack((boxes.astype(np.float32), scores[:, c:c + 1]))
            assert np.array_equal(_ref_gpu_nms(ref, dets, 0.3), v["nms_keep_%s_c%d" % (tag, c)]), (tag, c)
        for variant in ("np1", "np2"):            # gpu_mask_voting -> mv(...)
            sfx = "_%s_%s" % (tag, variant)
            inds, start, w = v["cand_inds" + sfx], v["cand_start" + sfx], v["cand_weights" + sfx]
            k = len(start)
            rm = np.zeros((k, 1, 21, 21), dtype=np.float32)
            rb = np.zeros((k, 4), dtype=np.int32)
            ref._Z3_mvPKfS0_iPKiS2_S0_iiiiiiPfPii(_p(boxes), _p(masks), boxes.shape[0], _p(inds),
                                                  _p(start), _p(w), len(inds), H, W, 4, 21, k,
                                                  _p(rm), _p(rb), 0)
            assert np.array_equal(rb, v["result_box" + sfx][:, :4].astype(np.int32)), (tag, variant)
            # the reference binary contracts a*b+c into FMA, the C oracle that recorded the masks
            # does not: values agree to fp32 rounding of one product, not bit for bit
            assert util.rel_err(rm, v["result_mask" + sfx]) < 1e-4
            rm_nf = np.zeros_like(rm)         # same source, -fmad=false: bit for bit
            rb_nf = np.zeros_like(rb)
            _ref(True)._Z3_mvPKfS0_iPKiS2_S0_iiiiiiPfPii(_p(boxes), _p(masks), boxes.shape[0], _p(inds),
                                                         _p(start), _p(w), len(inds), H, W, 4, 21, k,
                                                         _p(rm_nf), _p(rb_nf), 0)
            assert np.array_equal(rb_nf, rb) and np.array_equal(rm_nf, v["result_mask" + sfx])


# ------------------------------------------------------------------------------------------------
# The reference's Caffe layers for this path, compiled UNMODIFIED (.cu kernels and .cpp
# LayerSetUp/Reshape, class declarations from the reference's own headers) against the Caffe-runtime
# stand-in oracle/ref_stub into oracle/_ref/libmnc_ref_layers.so: reference == oracle == CUDA path.
LAYERS_SO = os.path.join(os.path.dirname(REF_SO), "libmnc_ref_layers.so")


def _layers(nofma=False):
    so = LAYERS_SO.replace(".so", "_nofma.so") if nofma else LAYERS_SO
    if not os.path.exists(so):
        pytest.skip("oracle/_ref/libmnc_ref_layers*.so not built (needs /root/reference at build time)")
    return ctypes.CDLL(so)


def _warp_inputs(R, seed, B=2, C=24, H=38, W=63):
    rng = np.random.default_rng(seed)
    feat = np.maximum(rng.standard_normal((B, C, H, W)), 0).astype(np.float32)
    x1, y1 = rng.uniform(0, 16 * W - 17, R), rng.uniform(0, 16 * H - 17, R)
    rois = np.stack([rng.integers(0, B, R), x1, y1, np.minimum(x1 + rng.uniform(16, 600, R), 16 * W - 1),
                     np.minimum(y1 + rng.uniform(16, 600, R), 16 * H - 1)], 1).astype(np.float32)
    edge = np.array([[0, 0, 0, 0, 0],                       # degenerate: one sample point
                     [0, 0, 0, 16 * W - 1, 16 * H - 1],     # whole map
                     [1, 16 * W - 9, 16 * H - 9, 16 * W - 1, 16 * H - 1],   # bottom-right corner
                     [0, 8, 8, 8, 300], [1, 8, 8, 300, 8],  # zero width / zero height after rounding
                     [0, 500, 300, 400, 200],               # inverted (end < start): clamped to 0 size
                     [1, 7.99, 24.0, 600.5, 424.01]], dtype=np.float32)   # .5 rounding cases
    return feat, np.vstack([edge, rois]).astype(np.float32)


# (ph, pw, C): the three fast paths at 24 channels, the generic kernel at a non-square and at the
# largest size, and a channel count that is no multiple of the row walk's 32-channel CTAs
WARP_PIN_SIZES = [pytest.param(P, P, 24, id=str(P)) for P in (28, 14, 7)] + [
    pytest.param(9, 5, 24, id="9x5"), pytest.param(32, 32, 24, id="32x32"), pytest.param(28, 28, 72, id="C72-28")]


def _pin_seed(P, PW, C):
    return P if (PW, C) == (P, 24) else 1000 * C + 10 * P + PW


@pytest.mark.parametrize("P,PW,C", WARP_PIN_SIZES)
def test_roi_warping_three_way(P, PW, C):
    """ROIWarpingLayer::Forward_gpu (roi_warping_layer.cu:67-122) == oracle == mnc_roi_warp_nchw."""
    import torch
    from oracle import oracle as O
    from mnc_b200 import ops
    L = _layers()
    feat, rois = _warp_inputs(120, seed=_pin_seed(P, PW, C), C=C)
    B, C, H, W = feat.shape
    R = rois.shape[0]
    ref_out = np.zeros((R, C, P, PW), np.float32)
    assert L.ref_roi_warp(_p(feat), B, C, H, W, _p(rois), R, P, PW, ctypes.c_float(0.0625), _p(ref_out)) == 0
    assert np.abs(ref_out).max() > 0
    orc = O.roi_warp(feat, rois, P, PW)
    got = ops.roi_warp_nchw(torch.from_numpy(feat).cuda(), torch.from_numpy(rois).cuda(), P, PW).cpu().numpy()
    # nvcc fuses `start + p * bin` and the 4-tap sum of the reference source into FMAs; a 1-ulp
    # sample coordinate moves a value by ~1e-5 of the map's range.  The oracle and our kernel keep
    # every operation separately rounded, and equal the reference compiled with -fmad=false bit
    # for bit.
    assert util.rel_err(orc, ref_out) < 2e-5, "oracle differs from reference ROIWarping"
    assert util.rel_err(got, ref_out) < 2e-5, "CUDA path differs from reference ROIWarping"
    assert np.array_equal(ref_out == 0, orc == 0)      # out-of-map samples in the same places
    nofma = np.zeros_like(ref_out)
    assert _layers(True).ref_roi_warp(_p(feat), B, C, H, W, _p(rois), R, P, PW, ctypes.c_float(0.0625),
                                      _p(nofma)) == 0
    assert np.array_equal(orc, nofma), "oracle != reference ROIWarping built with -fmad=false"
    assert np.array_equal(got, nofma), "CUDA path != reference ROIWarping built with -fmad=false"


def test_mask_resize_and_pooling_three_way():
    """MaskResizeLayer / MaskPoolingLayer Forward_gpu (mask_resize_layer.cu:57-84,
    mask_pooling_layer.cu:13-41) == oracle == mnc_mask_resize_nchw / mnc_mask_pool_nchw."""
    import torch
    from oracle import oracle as O
    from mnc_b200 import ops
    L = _layers()
    rng = np.random.default_rng(5)
    m = rng.uniform(0, 1, size=(37, 1, 21, 21)).astype(np.float32)
    for oh, ow in ((14, 14), (7, 9), (21, 21), (28, 28)):
        ref_out = np.zeros((37, 1, oh, ow), np.float32)
        assert L.ref_mask_resize(_p(m), 37, 1, 21, 21, oh, ow, _p(ref_out)) == 0
        orc = O.mask_resize(m, oh, ow)
        got = ops.mask_resize_nchw(torch.from_numpy(m).cuda(), oh, ow).cpu().numpy()
        assert util.rel_err(orc, ref_out) < 2e-6 and util.rel_err(got, ref_out) < 2e-6
        nofma = np.zeros_like(ref_out)
        assert _layers(True).ref_mask_resize(_p(m), 37, 1, 21, 21, oh, ow, _p(nofma)) == 0
        assert np.array_equal(orc, nofma) and np.array_equal(got, nofma)
    feat = rng.standard_normal((37, 24, 14, 14)).astype(np.float32)
    mask = rng.uniform(0, 1, size=(37, 1, 14, 14)).astype(np.float32)
    ref_out = np.zeros_like(feat)
    assert L.ref_mask_pool(_p(feat), _p(mask), 37, 24, 14, 14, _p(ref_out)) == 0
    got = ops.mask_pool_nchw(torch.from_numpy(feat).cuda(), torch.from_numpy(mask).cuda()).cpu().numpy()
    assert np.array_equal(O.mask_pool(feat, mask), ref_out)      # one multiply: bit-exact
    assert np.array_equal(got, ref_out)


@pytest.mark.parametrize("P", [7, 14])
def test_roi_pooling_three_way(P):
    """ROIPoolingLayer Forward_gpu and Forward_cpu (roi_pooling_layer.cu:17-92, .cpp:46-132) ==
    oracle == mnc_roi_pool_nchw (max over integer bins: bit-exact)."""
    import torch
    from oracle import oracle as O
    from mnc_b200 import ops
    L = _layers()
    feat, rois = _warp_inputs(100, seed=40 + P)
    B, C, H, W = feat.shape
    R = rois.shape[0]
    outs = []
    for use_gpu in (1, 0):
        o = np.zeros((R, C, P, P), np.float32)
        assert L.ref_roi_pool(_p(feat), B, C, H, W, _p(rois), R, P, P, ctypes.c_float(0.0625), use_gpu, _p(o)) == 0
        outs.append(o)
    assert np.array_equal(outs[0], outs[1])
    assert np.array_equal(O.roi_pool(feat, rois, P, P), outs[0])
    got = ops.roi_pool_nchw(torch.from_numpy(feat).cuda(), torch.from_numpy(rois).cuda(), P, P).cpu().numpy()
    assert np.array_equal(got, outs[0])
