"""Times the 14 loss and accuracy layers of one step of models/VGG16/mnc_5stage/train.prototxt
(rpn_loss_cls, rpn_loss_bbox; loss_cls, loss_seg_cls, loss_bbox, loss_mask, accuracy_det,
accuracy_seg and their _ext copies), forward and backward, as the median of CUDA-graph replays, at
the training shapes: a 38x63 feature map with A = 9 anchors, stage 1 at the ProposalTargetLayer
capacity of 64 + 3 rows with a device row count of 64, stage 2 at 67 rows (a StageBridge count of
64 RoIs + 3 gt boxes).  Targets are synthetic with the target layers' value sets.  When
oracle/_ref/libmnc_ref_loss.so is built (oracle/loss.mk), the same 14 layers are timed through the
reference's own Forward + Backward (CUDA events; its device->host round trips and host loops
included; Accuracy, CPU-only there, by the host clock).  Prints one JSON line with the card's name
and power limit.

    python scripts/bench_losses.py [--iters 200] [--warmup 10]
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

from mnc_b200 import autograd as AG  # noqa: E402
from scripts.bench_roi_backward import card  # noqa: E402

H, W, A = 38, 63, 9
KMAX, K, K2 = 67, 64, 67
LOSS_WEIGHTS = (1, 1, 2, 1, 1, 1, 2, 1, 1, 1)


def inputs(seed=0):
    g = torch.Generator("cuda").manual_seed(seed)
    n = lambda *s: torch.randn(*s, device="cuda", generator=g)
    i = lambda lo, hi, *s: torch.randint(lo, hi, s, device="cuda", generator=g).float()
    p = {"rpn_cls": n(1, 2, A * H, W), "rpn_bbox": n(1, 4 * A, H, W), "cls": n(KMAX, 21),
         "seg_cls": n(KMAX, 21), "bbox": n(KMAX, 84), "mask": n(KMAX, 1, 21, 21),
         "cls_ext": n(K2, 21), "seg_cls_ext": n(K2, 21), "bbox_ext": n(K2, 84),
         "mask_ext": n(K2, 1, 21, 21)}
    for v in p.values():
        v.requires_grad_()
    t = {"rpn_labels": i(-1, 2, 1, 1, A * H, W), "rpn_t": n(1, 4 * A, H, W),
         "rpn_in": i(0, 2, 1, 4 * A, H, W), "rpn_out": i(0, 2, 1, 4 * A, H, W) / 256,
         "n_valid": torch.tensor([K], dtype=torch.int32, device="cuda")}
    for s, rows in (("", KMAX), ("_ext", K2)):
        t["labels" + s] = i(-1, 21, rows)
        t["seg_labels" + s] = i(0, 21, rows)
        t["bbox_t" + s] = n(rows, 84)
        t["bbox_in" + s] = i(0, 2, rows, 84)
        t["bbox_out" + s] = t["bbox_in" + s].clone()
        t["mask_t" + s] = i(0, 2, rows, 1, 21, 21)
        t["mask_w" + s] = i(0, 2, rows, 1, 1, 1).expand(rows, 1, 21, 21).contiguous()
    return p, t


def step(p, t, weights):
    nv = t["n_valid"]
    losses = [AG.softmax_loss(p["rpn_cls"], t["rpn_labels"]),
              AG.smooth_l1_loss(p["rpn_bbox"], t["rpn_t"], t["rpn_in"], t["rpn_out"], sigma=3.0)]
    for s in ("", "_ext"):
        v = nv if s == "" else None
        losses += [AG.sigmoid_ce_loss(p["mask" + s], t["mask_t" + s], t["mask_w" + s], n_valid=v),
                   AG.softmax_loss(p["cls" + s], t["labels" + s], n_valid=v),
                   AG.softmax_loss(p["seg_cls" + s], t["seg_labels" + s], n_valid=v),
                   AG.smooth_l1_loss(p["bbox" + s], t["bbox_t" + s], t["bbox_in" + s],
                                     t["bbox_out" + s], n_valid=v)]
        AG.accuracy(p["cls" + s], t["labels" + s], n_valid=v)
        AG.accuracy(p["seg_cls" + s], t["seg_labels" + s], n_valid=v)
    keys = ["rpn_cls", "rpn_bbox", "mask", "cls", "seg_cls", "bbox", "mask_ext", "cls_ext",
            "seg_cls_ext", "bbox_ext"]
    return torch.autograd.grad(losses, [p[k] for k in keys], weights)


def reference_ms(p, t, reps=5):
    """Median over `reps` of the summed Forward + Backward time of the 14 layers in the reference's
    own code, or None when the library is not built."""
    path = os.path.join(ROOT, "oracle", "_ref", "libmnc_ref_loss.so")
    if not os.path.exists(path):
        return None
    from tests.test_ref_pin_loss import _lib, _c
    lib = _lib(path)
    h = {k: _c(v.detach().cpu().numpy()) for k, v in list(p.items()) + list(t.items())
         if v.dtype == torch.float32}
    K = int(t["n_valid"].item())
    ms = np.zeros(1, np.float32)
    f = lambda a: None if a is None else a.ctypes.data
    out = [np.zeros(a.size, np.float32) for a in (h["rpn_cls"], h["mask"])]
    totals = []
    for _ in range(reps):
        tot = 0.0
        x = h["rpn_cls"]
        lib.ref_softmax_loss(f(x), f(h["rpn_labels"]), 1, 2, x.size // 2, 1, -1, -1, 1, 1.0,
                             f(out[0]), None, None, f(ms)); tot += ms[0]
        lib.ref_smooth_l1_loss(f(h["rpn_bbox"]), f(h["rpn_t"]), f(h["rpn_in"]), f(h["rpn_out"]),
                               1, 4 * A, H, W, 3.0, 1.0, f(out[0]), None, f(ms)); tot += ms[0]
        for s, rows in (("", K), ("_ext", K2)):
            g = lambda k: np.ascontiguousarray(h[k + s][:rows])
            lib.ref_sigmoid_ce_loss(f(g("mask")), f(g("mask_t")), f(g("mask_w")), rows, 441, 2.0,
                                    f(out[1]), None, f(ms)); tot += ms[0]
            for sc, lab in (("cls", "labels"), ("seg_cls", "seg_labels")):
                lib.ref_softmax_loss(f(g(sc)), f(g(lab)), rows, 21, 1, 1, -1, -1, 1, 1.0,
                                     f(out[0]), None, None, f(ms)); tot += ms[0]
            lib.ref_smooth_l1_loss(f(g("bbox")), f(g("bbox_t")), f(g("bbox_in")), f(g("bbox_out")),
                                   rows, 84, 1, 1, 1.0, 1.0, f(out[0]), None, f(ms)); tot += ms[0]
            for sc, lab in (("cls", "labels"), ("seg_cls", "seg_labels")):
                t0 = time.perf_counter()
                lib.ref_accuracy(f(g(sc)), f(g(lab)), rows, 21, 1, 1, 0, 0, f(out[0]))
                tot += (time.perf_counter() - t0) * 1e3
        totals.append(tot)
    return float(np.median(totals))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_losses.py needs a CUDA device")
    p, t = inputs()
    weights = [torch.full((), float(w), device="cuda") for w in LOSS_WEIGHTS]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(a.warmup):
            step(p, t, weights)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step(p, t, weights)
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
    print(json.dumps({"gpu": card(), "unit": "ms", "layers": 14, "graph_replays": a.iters,
                      "device_fwd_bwd_ms": float(np.median(times)),
                      "p10_ms": float(np.percentile(times, 10)),
                      "p90_ms": float(np.percentile(times, 90)),
                      "reference_fwd_bwd_ms": reference_ms(p, t)}))


if __name__ == "__main__":
    main()
