"""Times the 16 convolutions of models/VGG16/mnc_5stage/train.prototxt (the VGG-16 trunk, rpn_conv_3x3
and the two 1x1 RPN heads) for training at batch 1 on a 600x1000 image (TRAIN.SCALES 600,
MAX_SIZE 1000): per layer the forward, dX and dW + db, each the median of CUDA-event-timed launches
after warm-up; then the trunk + RPN training step (frozen conv1_x / conv2_x forward only, no dX
below conv3_1, ReLUs, pools, backward from seeded diffs of the two RPN heads and of conv5_3's head
side) as one CUDA graph, the median of its replays.  Next to
each, the same work through torch conv2d in fp32 with TF32 off (cuDNN), which is what a cuDNN build
of the reference runs.  Each figure carries the algorithmic FLOP from the shapes, the achieved
TFLOP/s and, for ours, the share of the 989 TFLOP/s bf16 pipe at three bf16 products per MAC.
Prints one JSON line with the card's name and power limit, read in the same run.

    python scripts/bench_conv_train.py [--iters 30] [--warmup 5]
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as TF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from mnc_b200 import autograd as AG, ops  # noqa: E402
from scripts.bench_heads_train import median_ms  # noqa: E402
from scripts.bench_roi_backward import card  # noqa: E402
from mnc_b200.weights import POOL_AFTER, TRAIN_CONVS as CONV_LAYERS, train_conv_size as spatial  # noqa: E402

IMAGE = (600, 1000)
BF16_PEAK = 989e12


def tflops(flop, ms):
    return round(flop / (ms * 1e-3) / 1e12, 2)


def step_fn(P, data, grad_out, conv, relu, pool):
    """The trunk + RPN step with the given layer functions: forward to rpn_cls_score /
    rpn_bbox_pred, backward from seeded top diffs of the two RPN heads and of conv5_3's head side."""
    learn = [t for name, *_, learns in CONV_LAYERS if learns for t in P[name]]

    def step():
        h = data
        for name, *_ in CONV_LAYERS[:13]:
            h = relu(conv(h, *P[name]))
            if name in POOL_AFTER:
                h = pool(h)
        r = relu(conv(h, *P["rpn_conv_3x3"]))
        outs = [conv(r, *P["rpn_cls_score"]), conv(r, *P["rpn_bbox_pred"]), h]
        return torch.autograd.grad(outs, learn, grad_out)
    return step


def graph_ms(step, iters, warmup):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    return median_ms(graph.replay, iters, warmup)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_conv_train.py measures on a CUDA device; none is present")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator(device="cuda").manual_seed(0)

    per_layer, step_flop = [], 0
    tot = {"ours": 0.0, "cudnn": 0.0}
    for name, Cin, Cout, k, level, learns in CONV_LAYERS:
        H, W = spatial(*IMAGE, level)
        pad = (k - 1) // 2
        x = torch.randn(1, Cin, H, W, device="cuda", generator=g)
        w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) * (2.0 / (Cin * k * k)) ** 0.5
        b = torch.randn(Cout, device="cuda", generator=g) * 0.01
        dy = torch.randn(1, Cout, H, W, device="cuda", generator=g)
        dw, db = torch.zeros_like(w), torch.zeros_like(b)
        flop = 2 * Cout * Cin * k * k * H * W     # one product
        wants_dx = learns and name != "conv3_1"
        step_flop += flop * (1 + learns + wants_dx)     # forward, dW, dX
        t = {
            "fwd": median_ms(lambda: ops.conv_forward(x, w, b), a.iters, a.warmup),
            "dx": median_ms(lambda: ops.conv_backward(x, w, dy), a.iters, a.warmup),
            "dw_db": median_ms(lambda: ops.conv_backward(x, w, dy, dw=dw, db=db, want_dx=False),
                               a.iters, a.warmup),
            "cudnn_fwd": median_ms(lambda: TF.conv2d(x, w, b, padding=pad), a.iters, a.warmup),
            "cudnn_dx": median_ms(lambda: torch.nn.grad.conv2d_input(x.shape, w, dy, padding=pad),
                                  a.iters, a.warmup),
            "cudnn_dw_db": median_ms(lambda: (dw.add_(torch.nn.grad.conv2d_weight(x, w.shape, dy, padding=pad)),
                                              db.add_(dy.sum((0, 2, 3)))), a.iters, a.warmup),
        }
        row = {"layer": name, "Cin": Cin, "Cout": Cout, "k": k, "H": H, "W": W,
               "gflop_per_product": round(flop / 1e9, 3)}
        for key, ms in t.items():
            row[key + "_ms"] = round(ms, 4)
            row[key + "_tflops"] = tflops(flop, ms)
            if not key.startswith("cudnn"):
                row[key + "_bf16_pipe_share"] = round(3 * flop / (ms * 1e-3) / BF16_PEAK, 3)
        per_layer.append(row)
        tot["ours"] += t["fwd"] + (t["dw_db"] if learns else 0) + (t["dx"] if wants_dx else 0)
        tot["cudnn"] += t["cudnn_fwd"] + (t["cudnn_dw_db"] if learns else 0) + \
            (t["cudnn_dx"] if wants_dx else 0)
        del x, w, b, dy, dw, db

    # the whole step in one CUDA graph, ours and the cuDNN fp32 arm on the same parameters
    P = {}
    for name, Cin, Cout, k, level, learns in CONV_LAYERS:
        P[name] = ((torch.randn(Cout, Cin, k, k, device="cuda", generator=g) *
                    (2.0 / (Cin * k * k)) ** 0.5).requires_grad_(learns),
                   (torch.randn(Cout, device="cuda", generator=g) * 0.01).requires_grad_(learns))
    data = torch.randn(1, 3, *IMAGE, device="cuda", generator=g) * 50
    H5, W5 = spatial(*IMAGE, 4)
    grad_out = [torch.randn(1, c, H5, W5, device="cuda", generator=g) * 1e-3 for c in (18, 36, 512)]
    ours = step_fn(P, data, grad_out, AG.convolution, AG.relu, AG.max_pool)
    ref = step_fn(P, data, grad_out, lambda x, w, b: TF.conv2d(x, w, b, padding=(w.shape[-1] - 1) // 2),
                  TF.relu, lambda x: TF.max_pool2d(x, 2, 2, ceil_mode=True))
    step = {"ours": graph_ms(ours, a.iters, a.warmup), "cudnn": graph_ms(ref, a.iters, a.warmup)}

    print(json.dumps({
        "bench": "conv_train", "card": card(), "image": IMAGE, "batch": 1,
        "step_conv_gflop": round(step_flop / 1e9, 1),
        "step_graph_median_ms": {k: round(v, 3) for k, v in step.items()},
        "step_conv_tflops": {k: tflops(step_flop, v) for k, v in step.items()},
        "step_conv_sum_of_launches_ms": {k: round(v, 3) for k, v in tot.items()},
        "step_bf16_pipe_share": round(3 * step_flop / (step["ours"] * 1e-3) / BF16_PEAK, 3),
        "reference_arm": "cudnn_*: torch conv2d / conv2d_input / conv2d_weight in fp32 with TF32 "
                         "off, what a cuDNN build of the reference runs",
        "conv": per_layer}))


if __name__ == "__main__":
    main()
