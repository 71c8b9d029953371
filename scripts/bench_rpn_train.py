"""Times the TRAIN phase of the three RPN-stage layers -- ProposalLayer forward + backward,
ProposalTargetLayer forward + backward, AnchorTargetLayer forward -- as the median of CUDA-graph
replays, at the training shape (one 600x1000 image at im_scale 1.6, 38x63 feature map, 300
proposals) with 3, 20 and 100 gt boxes, and the numpy mirror of the same work on the host
(oracle/oracle_rpn_train.py, the reference's arithmetic) including the device->host and
host->device copies of the blobs the reference's Python layers force.  Prints one JSON line with
the card's name and power limit.

    python scripts/bench_rpn_train.py [--iters 50] [--warmup 5] [--host-iters 3]
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
from oracle import oracle_rpn_train as R  # noqa: E402
from scripts.bench_roi_backward import card  # noqa: E402

H, W, INFO = 38, 63, (600, 1000, 1.6)
SHAPES = {"train_G3": 3, "train_G20": 20, "train_G100": 100}


def device_step(t, keys, akeys, td, G):
    prob, deltas, info, gt, gm, mi = t
    rois, index, count, state = ops.proposal_train(prob, deltas, info, H, W)
    o = ops.proposal_target(rois, index, gt, gm, mi, info, keys, n_valid=count)
    rd = ops.proposal_target_backward(td, o["state"], rois.shape[0], G)
    ops.proposal_backward(rd, state, deltas, 1.0 / 512)
    ops.anchor_target(H, W, gt, info, akeys, o["fg_inds"], o["bg_inds"], o["counts"])


def host_step(t, keys, akeys, td):
    c = [x.cpu().numpy() for x in t]
    prob, deltas, info, gt, gm, mi = c
    rois, index, st = R.proposal_train_forward(prob, deltas, info)
    torch.from_numpy(rois).cuda(), torch.from_numpy(index).cuda()
    pt = R.proposal_target_forward(rois, index, gt, gm, mi, info, keys)
    tops = [torch.from_numpy(np.ascontiguousarray(pt[k])).cuda() for k in (
        "rois", "labels", "bbox_targets", "bbox_inside_weights", "bbox_outside_weights",
        "mask_targets", "mask_weight", "gt_masks_info", "fg_inds", "bg_inds")]
    at = R.anchor_target_forward(H, W, gt, info, akeys, tops[8].cpu().numpy(), tops[9].cpu().numpy())
    [torch.from_numpy(x).cuda() for x in at]
    K = pt["labels"].shape[0]
    rd = R.proposal_target_backward(td[:K].cpu().numpy(), pt["keep_ind"], rois.shape[0])
    torch.from_numpy(rd).cuda()
    bd = R.proposal_backward(rd, st, deltas, 1.0 / 512)
    torch.from_numpy(bd).cuda()
    torch.cuda.synchronize()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--host-iters", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rpn_train.py needs a CUDA device")
    res = {"gpu": card(), "unit": "ms"}
    for label, G in SHAPES.items():
        cs = R.make_case(11, H, W, INFO, G, n=0)
        t = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (
            cs["prob"], cs["deltas"], cs["im_info"].ravel(), cs["gt_boxes"],
            cs["gt_masks"].astype(np.float32), cs["mask_info"])]
        rng = np.random.default_rng(G)
        keys_np = rng.integers(0, 2 ** 32, (3, 300 + G), dtype=np.uint64).astype(np.uint32)
        akeys_np = rng.integers(0, 2 ** 32, H * W * 9, dtype=np.uint64).astype(np.uint32)
        keys = torch.from_numpy(keys_np.view(np.int32)).cuda()
        akeys = torch.from_numpy(akeys_np.view(np.int32)).cuda()
        Kmax = ops.proposal_target_capacity(64, (0.3,), (0.85, 0.15))
        td = torch.randn(Kmax, 5, device="cuda") * 1e-3
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(a.warmup):
                device_step(t, keys, akeys, td, G)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            device_step(t, keys, akeys, td, G)
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
        host_step(t, keys_np, akeys_np, td)                # warm-up
        ht = []
        for _ in range(a.host_iters):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            host_step(t, keys_np, akeys_np, td)
            ht.append((time.perf_counter() - t0) * 1e3)
        res[label] = {"proposals": 300, "gt": G, "device_fwd_bwd_ms": float(np.median(times)),
                      "host_numpy_ms": float(np.median(ht))}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
