"""Times the TRAIN phase of StageBridgeLayer and MaskLayer, forward + backward of both, as the
median of CUDA-graph replays, at two shapes:

  train    one 600x1000 image at im_scale 1.6, 64 RoIs (cfg.TRAIN.BATCH_SIZE) and 3..20 gt
  many_gt  the same image with 200 RoIs and 100 gt

and the numpy oracle (oracle/oracle_train.py, the reference's arithmetic with cv2) on the host for
the same work, including the device->host and host->device copies of the blobs the reference's
Python layers force.  Prints one JSON line with the card's name and power limit.

    python scripts/bench_train_bridge.py [--iters 50] [--warmup 5] [--host-iters 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from mnc_b200 import ops  # noqa: E402
from oracle import oracle_train as T  # noqa: E402
from scripts.bench_roi_backward import card  # noqa: E402

SHAPES = {"train_G3": dict(n=64, G=3), "train_G20": dict(n=64, G=20), "many_gt": dict(n=200, G=100)}


def device_step(t, td, mtd, G):
    o = ops.stage_bridge_train(*t, means=T.BBOX_NORMALIZE_MEANS, stds=T.BBOX_NORMALIZE_STDS)
    ops.stage_bridge_train_backward(td, o["state"], t[0], t[1], G, 1.0 / 512)
    lab = ops.mask_layer_train(o["mask_targets"], t[4], o["gt_mask_info"])
    ops.mask_layer_train_backward(mtd, lab)


def host_step(case, t, td, mtd):
    # the Python layers read bottom blobs on the host and write tops back to the device
    c = {k: v.cpu().numpy() for k, v in zip(("rois", "bbox_pred", "seg_cls_prob", "gt_boxes",
                                             "gt_masks", "im_info", "mask_info"), t)}
    out = T.stage_bridge_forward(**c, num_classes=21)
    tops = [torch.from_numpy(out[k]).cuda() for k in ("rois", "labels", "mask_targets", "mask_weight",
                                                      "gt_mask_info", "bbox_targets",
                                                      "bbox_inside_weights", "bbox_outside_weights")]
    rd, bd = T.stage_bridge_backward(td.cpu().numpy(), out, c["rois"], c["bbox_pred"], 1.0 / 512)
    torch.from_numpy(rd).cuda(), torch.from_numpy(bd).cuda()
    pred = tops[2].cpu().numpy().reshape(tops[2].shape[0], -1)
    lab = T.mask_layer_forward(pred, c["gt_masks"], tops[4].cpu().numpy())
    torch.from_numpy(lab).cuda()
    g = T.mask_layer_backward(mtd.cpu().numpy(), lab)
    torch.from_numpy(g).cuda()
    torch.cuda.synchronize()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--host-iters", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_bridge.py needs a CUDA device")
    res = {"gpu": card(), "unit": "ms"}
    for label, kw in SHAPES.items():
        case = T.make_case(7, H=600, W=1000, im_scale=1.6, **kw)
        case["gt_masks"] = case["gt_masks"].astype(np.float32)
        t = [torch.from_numpy(np.ascontiguousarray(case[k])).cuda() for k in
             ("rois", "bbox_pred", "seg_cls_prob", "gt_boxes", "gt_masks", "im_info", "mask_info")]
        K = kw["n"] + kw["G"]
        td = torch.randn(K, 5, device="cuda") * 1e-5
        mtd = torch.randn(K, 1, 21, 21, device="cuda")
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(a.warmup):
                device_step(t, td, mtd, kw["G"])
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            device_step(t, td, mtd, kw["G"])
        for _ in range(a.warmup):
            g.replay()
        times = []
        for _ in range(a.iters):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            g.replay()
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        host_step(case, t, td, mtd)                       # warm-up (imports, cv2)
        ht = []
        for _ in range(a.host_iters):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            host_step(case, t, td, mtd)
            ht.append((time.perf_counter() - t0) * 1e3)
        res[label] = {"rois": kw["n"], "gt": kw["G"], "device_fwd_bwd_ms": float(np.median(times)),
                      "host_oracle_ms": float(np.median(ht))}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
