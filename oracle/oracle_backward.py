"""oracle/oracle_backward.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

ctypes bindings of oracle/mnc_oracle_backward.c: the C restatements of the backward passes of the
reference's ROIWarping, MaskResize, MaskPooling and ROIPooling layers.  Only tests/ and scripts/
import this module; nothing under mnc_b200/ does.  Pinned to the reference's own Backward_gpu by
tests/test_ref_pin_backward.py.
"""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build_c():
    """Compile oracle/mnc_oracle_backward.c -> oracle/liboracle_backward.so (gcc, no FMA
    contraction) unless it is up to date; __graft_entry__.build() runs this."""
    import subprocess
    src = os.path.join(_HERE, "mnc_oracle_backward.c")
    out = os.path.join(_HERE, "liboracle_backward.so")
    if (not os.path.exists(out)) or os.path.getmtime(out) < os.path.getmtime(src):
        subprocess.check_call(["gcc", "-O2", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-shared",
                               "-fPIC", "-o", out, src, "-lm"])
    return out


def _lib():
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(build_c())
    return _LIB


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def roi_warp_backward(feat, rois, top_diff, pooled_h, pooled_w, spatial_scale=0.0625,
                      want_abs=False):
    """ROIWarpingLayer backward -- roi_warping_layer.cu:175-245, :306-361, :409-434.
    -> (feat_diff (B,C,H,W), rois_diff (R,5)) [+ rois_abs (R,5) float64: sums of |term|]."""
    feat = np.ascontiguousarray(feat, dtype=np.float32)
    rois = np.ascontiguousarray(rois, dtype=np.float32)
    top_diff = np.ascontiguousarray(top_diff, dtype=np.float32)
    B, C, H, W = feat.shape
    R = rois.shape[0]
    fd = np.zeros_like(feat)
    rd = np.zeros((R, 5), dtype=np.float32)
    ra = np.zeros((R, 5), dtype=np.float64)
    _lib().orc_roi_warp_backward(_p(feat), ctypes.c_int(B), ctypes.c_int(C), ctypes.c_int(H),
                                 ctypes.c_int(W), _p(rois), ctypes.c_int(R), ctypes.c_int(pooled_h),
                                 ctypes.c_int(pooled_w), ctypes.c_float(spatial_scale), _p(top_diff),
                                 _p(fd), _p(rd), _p(ra))
    return (fd, rd, ra) if want_abs else (fd, rd)


def mask_resize_backward(top_diff, in_h, in_w):
    """MaskResizeLayer backward -- mask_resize_layer.cu:135-173.  top_diff (N,C,oh,ow)."""
    top_diff = np.ascontiguousarray(top_diff, dtype=np.float32)
    N, C, oh, ow = top_diff.shape
    out = np.zeros((N, C, in_h, in_w), dtype=np.float32)
    _lib().orc_mask_resize_backward(_p(top_diff), ctypes.c_int(N), ctypes.c_int(C), ctypes.c_int(in_h),
                                    ctypes.c_int(in_w), ctypes.c_int(oh), ctypes.c_int(ow), _p(out))
    return out


def mask_pool_backward(feat, mask, top_diff):
    """MaskPoolingLayer backward -- mask_pooling_layer.cu:43-76.  -> (feat_diff, mask_diff)."""
    feat = np.ascontiguousarray(feat, dtype=np.float32)
    mask = np.ascontiguousarray(mask, dtype=np.float32)
    top_diff = np.ascontiguousarray(top_diff, dtype=np.float32)
    N, C, H, W = feat.shape
    fd = np.zeros_like(feat)
    md = np.zeros_like(mask)
    _lib().orc_mask_pool_backward(_p(feat), _p(mask), _p(top_diff), ctypes.c_int(N), ctypes.c_int(C),
                                  ctypes.c_int(H), ctypes.c_int(W), _p(fd), _p(md))
    return fd, md


def roi_pool_backward(top_diff, argmax, feat_shape, rois, pooled_h, pooled_w, spatial_scale=0.0625):
    """ROIPoolingLayer backward -- roi_pooling_layer.cu:94-165.  -> feat_diff of feat_shape."""
    top_diff = np.ascontiguousarray(top_diff, dtype=np.float32)
    argmax = np.ascontiguousarray(argmax, dtype=np.int32)
    rois = np.ascontiguousarray(rois, dtype=np.float32)
    B, C, H, W = feat_shape
    out = np.zeros(feat_shape, dtype=np.float32)
    _lib().orc_roi_pool_backward(_p(top_diff), _p(argmax), ctypes.c_int(B), ctypes.c_int(C),
                                 ctypes.c_int(H), ctypes.c_int(W), _p(rois), ctypes.c_int(rois.shape[0]),
                                 ctypes.c_int(pooled_h), ctypes.c_int(pooled_w),
                                 ctypes.c_float(spatial_scale), _p(out))
    return out
