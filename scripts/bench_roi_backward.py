"""Times the backward entry points of ROIWarping, MaskResize, MaskPooling and ROIPooling with CUDA
events (warm-up, then --iters launches each; the median is reported) at two shapes:

  train  the VGG16 mnc_5stage training net: one 600x1000 image, conv5_3 1x512x38x63, 64 RoIs
         (cfg.TRAIN.BATCH_SIZE), ROIWarping 28x28, MaskResize 21->14, MaskPooling 64x512x14x14
  infer  the inference batch: 8 images, conv5_3 8x512x38x63, 2400 RoIs (300 per image)

ROIPooling runs at 7x7 (the CFM net's pooled size) on the same RoIs.  When
oracle/_ref/libmnc_ref_backward.so exists (oracle/Makefile), the reference's own Backward_gpu is timed on the same
inputs through the driver's timed entry points (Backward between events on one set-up layer).
Our calls are timed as CUDA-graph replays; the reference's as events around its Backward call.
Prints one JSON line with the card's name and power limit.

    python scripts/bench_roi_backward.py [--iters 50] [--warmup 5] [--no-ref]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from mnc_b200 import ops  # noqa: E402

SS = 0.0625
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libmnc_ref_backward.so")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True,
                             timeout=30).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1])}
    except Exception:
        return {"name": torch.cuda.get_device_name(0), "power_limit_w": None}


def rois_for(B, per_img, H, W, seed):
    """Proposals inside the map: x2 <= 16 (W - 1), so every ROIWarping sample lies on the map (the
    reference's coordinate kernel reads outside the sampled plane otherwise)."""
    rng = np.random.default_rng(seed)
    R = B * per_img
    w = rng.uniform(32, 400, R)
    h = rng.uniform(32, 300, R)
    x1 = rng.uniform(0, 16 * (W - 1) - w)
    y1 = rng.uniform(0, 16 * (H - 1) - h)
    return np.stack([np.repeat(np.arange(B), per_img), x1, y1, x1 + w, y1 + h], 1).astype(np.float32)


def log(msg):
    print(msg, file=sys.stderr, flush=True)


def median_ms(fn, iters, warmup):
    """One call of fn is captured into a CUDA graph and each replay is timed with events, so the
    Python wrapper's host time (allocation, ctypes) is not counted as device time."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(warmup):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    for _ in range(warmup):
        g.replay()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def ref_ms(call, iters):
    times = np.zeros(iters, np.float32)
    assert call(iters, times.ctypes.data_as(ctypes.c_void_p)) == 0
    return float(np.median(times))


class Timings(dict):
    """A dict of medians that reports each one as it is taken."""

    def __init__(self, tag):
        super().__init__()
        self.tag = tag

    def __setitem__(self, k, v):
        log("%s %s %.4f ms" % (self.tag, k, v))
        super().__setitem__(k, v)


def run_shape(name, B, per_img, iters, warmup, L):
    C, H, W, P, PP = 512, 38, 63, 28, 7
    rng = np.random.default_rng(1)
    feat_h = np.maximum(rng.standard_normal((B, C, H, W)), 0).astype(np.float32)
    rois_h = rois_for(B, per_img, H, W, 2)
    R = rois_h.shape[0]
    top_h = rng.standard_normal((R, C, P, P)).astype(np.float32)
    mtop_h = rng.standard_normal((R, 1, 14, 14)).astype(np.float32)
    mfeat_h = rng.standard_normal((R, C, 14, 14)).astype(np.float32)
    mask_h = rng.uniform(0, 1, (R, 1, 14, 14)).astype(np.float32)
    ptop_h = rng.standard_normal((R, C, PP, PP)).astype(np.float32)
    feat, rois, top = (torch.from_numpy(a).cuda() for a in (feat_h, rois_h, top_h))
    mtop, mfeat, mask, ptop = (torch.from_numpy(a).cuda() for a in (mtop_h, mfeat_h, mask_h, ptop_h))
    arg = torch.empty((R, C, PP, PP), dtype=torch.int32, device="cuda")
    ops.roi_pool_nchw(feat, rois, PP, PP, argmax=arg)
    res = {"B": B, "R": R, "C": C, "H": H, "W": W, "pooled": P}
    ms = res["ms"] = Timings(name)
    ms["roi_warp_feat"] = median_ms(lambda: ops.roi_warp_backward_nchw(feat, rois, top, P, P, want_rois=False), iters, warmup)
    ms["roi_warp_coord"] = median_ms(lambda: ops.roi_warp_backward_nchw(feat, rois, top, P, P, want_feat=False), iters, warmup)
    ms["roi_warp_both"] = median_ms(lambda: ops.roi_warp_backward_nchw(feat, rois, top, P, P), iters, warmup)
    ms["mask_resize_21_14"] = median_ms(lambda: ops.mask_resize_backward_nchw(mtop, 21, 21), iters, warmup)
    ms["mask_pool_both"] = median_ms(lambda: ops.mask_pool_backward_nchw(mfeat, mask, mfeat), iters, warmup)
    ms["roi_pool_7"] = median_ms(lambda: ops.roi_pool_backward_nchw(ptop, arg, feat.shape, rois, PP, PP), iters, warmup)
    if L is not None:
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
        ref = res["ref_ms"] = Timings(name + " reference")
        # the reference's feature kernels loop over every RoI of the batch per element: at the
        # inference shape one ROIWarping call takes minutes, so it is not timed there, and fewer
        # calls of the others are
        ri = res["ref_iters"] = iters if name == "train" else min(iters, 5)
        fd = np.zeros_like(feat_h)
        rd = np.zeros((R, 5), np.float32)
        common = (p(feat_h), B, C, H, W, p(rois_h), R, P, P, ctypes.c_float(SS), p(top_h))
        if name == "train":
            ref["roi_warp_feat"] = ref_ms(lambda n, t: L.ref_roi_warp_backward(*common, 1, 0, p(fd), p(rd), n, t), ri)
            # the coordinate pass materialises R*5*C*P*P floats twice (0.5 GB each here, 19 GB
            # each at the inference shape)
            ref["roi_warp_both"] = ref_ms(lambda n, t: L.ref_roi_warp_backward(*common, 1, 1, p(fd), p(rd), n, t), ri)
        mi = np.zeros((R, 1, 21, 21), np.float32)
        ref["mask_resize_21_14"] = ref_ms(lambda n, t: L.ref_mask_resize_backward(p(mi), R, 1, 21, 21, 14, 14, p(mtop_h), p(mi), n, t), ri)
        mf, mm = np.zeros_like(mfeat_h), np.zeros_like(mask_h)
        ref["mask_pool_both"] = ref_ms(lambda n, t: L.ref_mask_pool_backward(p(mfeat_h), p(mask_h), R, C, 14, 14, p(mfeat_h), 1, 1, p(mf), p(mm), n, t), ri)
        ref["roi_pool_7"] = ref_ms(lambda n, t: L.ref_roi_pool_backward(p(feat_h), B, C, H, W, p(rois_h), R, PP, PP, ctypes.c_float(SS), p(ptop_h), 1, p(fd), n, t), ri)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-ref", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_roi_backward.py needs a CUDA device")
    L = None if (a.no_ref or not os.path.exists(REF_SO)) else ctypes.CDLL(REF_SO)
    out = {"card": card(), "iters": a.iters, "warmup": a.warmup,
           "train": run_shape("train", 1, 64, a.iters, a.warmup, L),
           "infer": run_shape("infer", 8, 300, a.iters, a.warmup, L)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
