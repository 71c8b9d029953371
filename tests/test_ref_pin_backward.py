"""Pin the backward passes three ways: the reference's own Backward_gpu (caffe-mnc layer sources
compiled unmodified into oracle/_ref/libmnc_ref_backward*.so by oracle/backward.mk, driven by
oracle/ref_backward_driver.cu)
== oracle == CUDA path.  Against the -fmad=false build every feature and mask gradient is
bit-exact; against the default build they agree to the FMA-rounding tolerance of the forward pins.
RoI coordinate gradients: within 1e-5 of the sum of their terms' magnitudes (thrust's reduction
order is unspecified).

The reference is only ever fed inputs that keep it inside its buffers: its coordinate kernel reads
outside the sampled plane for a sample outside the map and asserts on end < start, so
propagate_down[1] is set only for RoIs free of both (selected on the host with the oracle's
geometry), and every MaskResize shape is checked for reads past top_diff first."""
import ctypes
import os

import numpy as np
import pytest

from tests import util
from tests.test_ref_pin import _p, _warp_inputs
from tests.test_oracle_backward import _roundf, _warp_geometry

pytestmark = pytest.mark.gpu
SS = 0.0625
BACKWARD_SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref",
                           "libmnc_ref_backward.so")


def _layers(nofma=False):
    so = BACKWARD_SO.replace(".so", "_nofma.so") if nofma else BACKWARD_SO
    if not os.path.exists(so):
        pytest.skip("oracle/_ref/libmnc_ref_backward*.so not built (needs a reference checkout at build time)")
    return ctypes.CDLL(so)


def _coord_safe(rois, P, H, W):
    """RoIs the reference's coordinate kernel handles inside its buffers."""
    ok = np.zeros(len(rois), bool)
    for i, roi in enumerate(rois):
        sw, sh, ew, eh = (int(v) for v in _roundf(roi[1:5] * np.float32(SS)))
        _, _, ((_, okh), (_, okw)) = _warp_geometry(roi, P, H, W)
        ok[i] = okh.all() and okw.all() and sh <= eh and sw <= ew
    return ok


def _ref_warp(L, feat, rois, top, P, pd1):
    B, C, H, W = feat.shape
    R = rois.shape[0]
    fd = np.zeros_like(feat)
    rd = np.zeros((R, 5), np.float32)
    assert L.ref_roi_warp_backward(_p(feat), B, C, H, W, _p(rois), R, P, P, ctypes.c_float(SS),
                                   _p(top), 1, int(pd1), _p(fd), _p(rd), 0, None) == 0
    return fd, rd


@pytest.mark.parametrize("P", [28, 14, 7])
def test_roi_warping_backward_three_way(P):
    import torch
    from oracle import oracle_backward as OB
    from mnc_b200 import ops
    feat, rois = _warp_inputs(60, seed=P)
    B, C, H, W = feat.shape
    rng = np.random.default_rng(P)
    top = rng.standard_normal((rois.shape[0], C, P, P)).astype(np.float32)
    want_f, want_r, mag = OB.roi_warp_backward(feat, rois, top, P, P, want_abs=True)
    fd, rd = ops.roi_warp_backward_nchw(torch.from_numpy(feat).cuda(), torch.from_numpy(rois).cuda(),
                                        torch.from_numpy(top).cuda(), P, P)
    fd, rd = fd.cpu().numpy(), rd.cpu().numpy()
    # feature gradient, every RoI (edge RoIs included), propagate_down = (1, 0)
    nf_f, _ = _ref_warp(_layers(True), feat, rois, top, P, False)
    assert np.array_equal(nf_f, want_f), "oracle != reference ROIWarping backward (-fmad=false)"
    assert np.array_equal(nf_f, fd), "CUDA != reference ROIWarping backward (-fmad=false)"
    df_f, _ = _ref_warp(_layers(), feat, rois, top, P, False)
    assert util.rel_err(fd, df_f) < 1e-4
    # coordinate gradient on the RoIs the reference's kernel handles inside its buffers
    safe = _coord_safe(rois, P, H, W)
    assert safe.sum() >= 30
    sr, st = np.ascontiguousarray(rois[safe]), np.ascontiguousarray(top[safe])
    for L in (_layers(True), _layers()):
        f2, r2 = _ref_warp(L, feat, sr, st, P, True)
        assert np.all(r2[:, 0] == 0)
        assert np.all(np.abs(r2 - want_r[safe]) <= 1e-5 * mag[safe] + 1e-30)
        assert np.all(np.abs(r2 - rd[safe]) <= 1e-5 * mag[safe] + 1e-30)


def _resize_reads_in_bounds(ih, iw, oh, ow):
    """Every top_diff element MaskResizeBackward reads (mask_resize_layer.cu:151-168) lies in its
    plane, so the last plane's reads stay inside the blob."""
    rh, rw = np.float32(ih) / np.float32(oh), np.float32(iw) / np.float32(ow)
    for h in range(ih):
        for w in range(iw):
            hs, ws = int(np.floor(np.float32(h) / rh)), int(np.floor(np.float32(w) / rw))
            for ph in (hs, hs + 1):
                for pw in (ws, ws + 1):
                    if abs(np.float32(pw) * rw - np.float32(w)) < 1 and abs(np.float32(ph) * rh - np.float32(h)) < 1:
                        if ph * ow + pw >= oh * ow:
                            return False
    return True


def test_mask_resize_and_pooling_backward_three_way():
    import torch
    from oracle import oracle_backward as OB
    from mnc_b200 import ops
    rng = np.random.default_rng(6)
    m = rng.uniform(0, 1, size=(37, 1, 21, 21)).astype(np.float32)
    for oh, ow in ((14, 14), (7, 9), (21, 21), (28, 28)):
        assert _resize_reads_in_bounds(21, 21, oh, ow)
        g = rng.standard_normal((37, 1, oh, ow)).astype(np.float32)
        want = OB.mask_resize_backward(g, 21, 21)
        got = ops.mask_resize_backward_nchw(torch.from_numpy(g).cuda(), 21, 21).cpu().numpy()
        outs = []
        for L in (_layers(True), _layers()):
            o = np.zeros_like(m)
            assert L.ref_mask_resize_backward(_p(m), 37, 1, 21, 21, oh, ow, _p(g), _p(o), 0, None) == 0
            outs.append(o)
        assert np.array_equal(outs[0], want) and np.array_equal(got, want)
        assert util.rel_err(got, outs[1]) < 2e-5
    feat = rng.standard_normal((37, 24, 14, 14)).astype(np.float32)
    mask = rng.uniform(0, 1, size=(37, 1, 14, 14)).astype(np.float32)
    g = rng.standard_normal(feat.shape).astype(np.float32)
    wf, wm = OB.mask_pool_backward(feat, mask, g)
    fd, md = ops.mask_pool_backward_nchw(torch.from_numpy(feat).cuda(), torch.from_numpy(mask).cuda(),
                                         torch.from_numpy(g).cuda())
    for i, L in enumerate((_layers(True), _layers())):
        rf, rm = np.zeros_like(feat), np.zeros_like(mask)
        assert L.ref_mask_pool_backward(_p(feat), _p(mask), 37, 24, 14, 14, _p(g), 1, 1, _p(rf), _p(rm), 0, None) == 0
        assert np.array_equal(rf, wf) and np.array_equal(fd.cpu().numpy(), wf)
        if i == 0:
            assert np.array_equal(rm, wm) and np.array_equal(md.cpu().numpy(), wm)
        else:
            assert util.rel_err(md.cpu().numpy(), rm) < 1e-4


@pytest.mark.parametrize("P", [7, 14])
def test_roi_pooling_backward_three_way(P):
    import torch
    from oracle import oracle as O
    from oracle import oracle_backward as OB
    from mnc_b200 import ops
    feat, rois = _warp_inputs(80, seed=50 + P)
    B, C, H, W = feat.shape
    R = rois.shape[0]
    rng = np.random.default_rng(P)
    top = rng.standard_normal((R, C, P, P)).astype(np.float32)
    _, arg = O.roi_pool(feat, rois, P, P, return_argmax=True)
    want = OB.roi_pool_backward(top, arg, feat.shape, rois, P, P)
    got = ops.roi_pool_backward_nchw(torch.from_numpy(top).cuda(), torch.from_numpy(arg).cuda(),
                                     feat.shape, torch.from_numpy(rois).cuda(), P, P).cpu().numpy()
    assert np.array_equal(got, want)
    for L in (_layers(True), _layers()):
        o = np.zeros_like(feat)
        assert L.ref_roi_pool_backward(_p(feat), B, C, H, W, _p(rois), R, P, P, ctypes.c_float(SS),
                                       _p(top), 1, _p(o), 0, None) == 0
        assert np.array_equal(o, want)      # float adds in the same order, no products: exact
