"""Times the head layers of both stages of models/VGG16/mnc_5stage/train.prototxt, forward and
backward, at the training shapes (67 RoI rows per stage: stage 1 at the ProposalTargetLayer capacity
of 64 + 3, stage 2 at 64 RoIs + 3 gt boxes): the pools 28 -> 14 -> 7, the 18 InnerProducts (9
shared parameter pairs), the ReLUs and the Sigmoids, through mnc_b200.autograd, as the median of
CUDA-graph replays.  Then each InnerProduct's forward and backward (dW + db + dX) alone, CUDA events
over many launches, with the bytes each must move (fp32 weights read, dW read and written,
activations) and their share of 3.35 TB/s, next to the same products through cuBLAS in fp32
(torch.addmm / matmul, TF32 off), which is what the reference's sgemm / sgemv run.  Prints one JSON line with the card's name and power
limit.

    python scripts/bench_heads_train.py [--iters 50] [--warmup 5]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from mnc_b200 import autograd as AG, ops  # noqa: E402
from scripts.bench_roi_backward import card  # noqa: E402
from tests.fc_bound import MNC_FC_SHAPES  # noqa: E402

ROWS = 67
HBM = 3.35e12


def params(g):
    P = {}
    for name, N, K in MNC_FC_SHAPES:
        P[name] = ((torch.randn(N, K, device="cuda", generator=g) * (2.0 / K) ** 0.5).requires_grad_(),
                   (torch.randn(N, device="cuda", generator=g) * 0.01).requires_grad_())
    return P


def stage(P, premax):
    """One stage's heads from the 28 x 28 ROIWarping output; -> the outputs the losses read."""
    ip = lambda x, n: AG.inner_product(x, *P[n])
    r5 = AG.max_pool(premax)
    mask_out = AG.sigmoid(ip(AG.relu(ip(r5, "fc6_maskest")), "mask_pred"))
    h7 = AG.relu(ip(AG.relu(ip(AG.max_pool(r5), "fc6")), "fc7"))
    m7 = AG.relu(ip(AG.relu(ip(AG.max_pool(r5), "fc6_mask")), "fc7_mask"))
    join = torch.cat([m7, h7], 1)
    return [mask_out, ip(join, "cls_score"), ip(join, "seg_cls_score"), ip(join, "bbox_pred")]


def median_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_heads_train.py measures on a CUDA device; none is present")
    g = torch.Generator(device="cuda").manual_seed(0)
    P = params(g)
    leaves = [t for pair in P.values() for t in pair]
    x1 = torch.randn(ROWS, 512, 28, 28, device="cuda", generator=g).requires_grad_()
    x2 = torch.randn(ROWS, 512, 28, 28, device="cuda", generator=g).requires_grad_()
    dys = [torch.randn_like(o) for o in (stage(P, x1) + stage(P, x2))]

    def step():
        outs = stage(P, x1) + stage(P, x2)
        loss = sum((o * d).sum() for o, d in zip(outs, dys))   # top diffs dys
        return torch.autograd.grad(loss, [x1, x2] + leaves)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    step_ms = median_ms(graph.replay, a.iters, a.warmup)

    torch.backends.cuda.matmul.allow_tf32 = False
    per_layer, fc_total, cublas_total = [], 0.0, 0.0
    for name, N, K in MNC_FC_SHAPES:
        w, b = (t.detach() for t in P[name])
        x = torch.randn(ROWS, K, device="cuda", generator=g)
        dy = torch.randn(ROWS, N, device="cuda", generator=g)
        dw, db = torch.zeros_like(w), torch.zeros_like(b)
        f_ms = median_ms(lambda: ops.fc_forward(x, w, b), a.iters, a.warmup)
        b_ms = median_ms(lambda: ops.fc_backward(x, w, dy, dw=dw, db=db), a.iters, a.warmup)
        # the same products through cuBLAS fp32 (torch, TF32 off): Caffe's sgemm / sgemv
        tf = median_ms(lambda: torch.addmm(b, x, w.T), a.iters, a.warmup)
        tb = median_ms(lambda: (dw.addmm_(dy.T, x), db.add_(dy.sum(0)), dy @ w), a.iters, a.warmup)
        cublas_total += 2 * (tf + tb)
        f_bytes = 4 * (N * K + ROWS * K + ROWS * N + N)
        b_bytes = 4 * (3 * N * K + 2 * ROWS * K + ROWS * N + 2 * N)   # W read, dW read + write
        fc_total += 2 * (f_ms + b_ms)
        per_layer.append({"layer": name, "N": N, "K": K, "fwd_ms": round(f_ms, 4),
                          "cublas_fp32_fwd_ms": round(tf, 4), "cublas_fp32_bwd_ms": round(tb, 4),
                          "fwd_bytes": f_bytes, "fwd_hbm_share": round(f_bytes / HBM / (f_ms * 1e-3), 3),
                          "bwd_ms": round(b_ms, 4), "bwd_bytes": b_bytes,
                          "bwd_hbm_share": round(b_bytes / HBM / (b_ms * 1e-3), 3)})
    step_bytes = sum(2 * (l["fwd_bytes"] + l["bwd_bytes"]) for l in per_layer)
    print(json.dumps({"bench": "heads_train", "card": card(), "rows_per_stage": ROWS,
                      "step_graph_median_ms": round(step_ms, 4),
                      "fc_sum_of_launches_ms": round(fc_total, 4),
                      "cublas_fp32_sum_ms": round(cublas_total, 4),
                      "fc_step_bytes": step_bytes,
                      "fc_step_hbm_floor_ms": round(step_bytes / HBM * 1e3, 4),
                      "reference_arm": "cublas_fp32_*: the sgemm / sgemv the reference's "
                                       "InnerProduct runs, without its host round trips",
                      "fc": per_layer}))


if __name__ == "__main__":
    main()
