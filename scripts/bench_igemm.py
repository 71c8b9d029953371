"""Per-launch-site timing of the implicit-GEMM kernel (igemm_tc_kernel) in the flagship step.

Builds the engine at batch 8, 600x1000 (bench.py's shape), runs one eager step with the launches
of dense.igemm2 recorded, then re-times every distinct launch 20x with CUDA events (median) on the
step's own buffers.  Per site: ms, algorithmic TFLOP/s (2*M*N*K over the time) and the tensor-pipe
fraction (issued tensor work -- 2 units per MAC with tri-plane operands, 3 with split-bf16 -- over
the H100 SXM data-sheet 989 TFLOP/s dense fp16/bf16, which a card at a lower power limit cannot
reach).  Two diagnostics on synthetic operands:
  * fc7 (M 2400, K 4096, N 4096) at bn = 64 and bn = 128: ring depth against operand bytes/MAC;
  * a conv4_2-shaped launch (8 x 75 x 125, 512 -> 512) on 132 and on 66 CTAs: whether the shared
    L2 / HBM path or the per-CTA pipeline bounds the rate.
Writes one JSON file (card name and power limit included) into --out-dir.

    python scripts/bench_igemm.py --out-dir DIR [--iters 20] [--tag NAME]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from mnc_b200 import dense, weights as Wt, ops  # noqa: E402
from mnc_b200.engine import MNCEngine  # noqa: E402
from bench import gpu_identity  # noqa: E402

B, H, W = 8, 600, 1000
PEAK_TFLOPS = 989.0   # H100 SXM data sheet, dense fp16 / bf16, 700 W


def median_ms(fn, iters, warm=3):
    for _ in range(warm):
        fn()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(iters + 1)]
    torch.cuda.synchronize()
    ev[0].record()
    for k in range(iters):
        fn()
        ev[k + 1].record()
    torch.cuda.synchronize()
    t = sorted(ev[k].elapsed_time(ev[k + 1]) for k in range(iters))
    return t[iters // 2]


def site_key(args, kw):
    a, batch, h, w, cin, _, cout, taps = args[:8]
    tri = isinstance(a, dense.Tri)
    return (batch, h, w, cin, cout, taps, kw.get("bn", 0), kw.get("split_k", 1), bool(kw.get("pool", False)),
            kw.get("out_f32") is not None, tri)


def row(key, ms, count):
    batch, h, w, cin, cout, taps, bn, split, pool, f32, tri = key
    flops = 2.0 * batch * h * w * cout * taps * cin
    tf = flops / (ms * 1e-3) / 1e12
    units = 2 if tri else 3
    return {"M": batch * h * w, "N": cout, "K": taps * cin, "taps": taps, "bn": bn, "split_k": split,
            "pooled": pool, "fp32_out": f32, "tri": tri, "launches_per_step": count,
            "ms": round(ms, 4), "ms_per_step": round(ms * count, 4), "tflops": round(tf, 1),
            "frac_tensor_pipe": round(units * tf / PEAK_TFLOPS, 3)}


def diagnostics(iters):
    out = {}
    torch.manual_seed(0)
    # fc7: M 2400, K 4096, N 4096, tri operands, tri output
    M, K, N = 2400, 4096, 4096
    x = dense.tri_from_f32(torch.relu(torch.randn(M, K, device="cuda")))
    wt = dense.tri_from_f32(torch.randn(N, K, device="cuda") / K ** 0.5, weight=True)
    o = dense.tri_alloc((M, N), "cuda")
    flops = 2.0 * M * N * K
    for bn in (64, 128):
        ms = median_ms(lambda: dense.igemm2(x.view(1, 1, M, K), 1, 1, M, K, wt, N, 1, relu=True, out=o,
                                            bn=bn), iters)
        out["fc7_bn%d" % bn] = {"ms": round(ms, 4), "tflops": round(flops / (ms * 1e-3) / 1e12, 1)}
    del x, wt, o
    # conv4_2: 8 x 75 x 125, 512 -> 512, 3x3
    b, h, w, c = 8, 75, 125, 512
    xa = dense.tri_from_f32(torch.relu(torch.randn(b, h, w, c, device="cuda")))
    wc = dense.conv_weight_to_tri(torch.randn(c, c, 3, 3, device="cuda") / (9 * c) ** 0.5)
    oc = dense.tri_alloc((b, h, w, c), "cuda")
    flops = 2.0 * b * h * w * c * 9 * c
    for ctas in (132, 66):
        ms = median_ms(lambda: dense.igemm2(xa, b, h, w, c, wc, c, 9, relu=True, out=oc, max_ctas=ctas), iters)
        out["conv4_2_ctas%d" % ctas] = {"ms": round(ms, 4), "tflops": round(flops / (ms * 1e-3) / 1e12, 1)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--tag", default="igemm")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_igemm.py needs a CUDA device"
    dev = torch.device("cuda", 0)
    eng = MNCEngine(Wt.make_weights(Wt.FULL_ARCH), device=dev)
    eng.overlap_heads = False
    data = ops.prep_images(torch.randint(0, 256, (B, H, W, 3), dtype=torch.uint8,
                                         generator=torch.Generator().manual_seed(1234)).to(dev), 1.0)
    im_info = torch.tensor([[H, W, 1.0]] * B, dtype=torch.float32, device=dev)
    eng.forward(data, im_info)    # warm-up: modules, tensor maps, buffers
    torch.cuda.synchronize()

    # one eager step with every dense.igemm2 launch recorded (arguments kept for the re-timing)
    calls = []
    orig = dense.igemm2

    def rec(*a, **kw):
        calls.append((a, kw))
        return orig(*a, **kw)

    dense.igemm2, dense.timer = rec, dense.KernelTimer()
    eng.forward(data, im_info)
    torch.cuda.synchronize()
    ktimer, dense.igemm2, dense.timer = dense.timer, orig, None
    step_ms = sum(s.elapsed_time(e) for s, e, _, _ in ktimer.records)

    sites, order = {}, []
    for a, kw in calls:
        k = site_key(a, kw)
        if k not in sites:
            sites[k] = [a, kw, 0]
            order.append(k)
        sites[k][2] += 1
    table = []
    for k in order:
        a, kw, n = sites[k]
        ms = median_ms(lambda: orig(*a, **kw), args.iters)
        table.append(row(k, ms, n))
    total = sum(r["ms_per_step"] for r in table)
    res = {"tag": args.tag, "gpu": gpu_identity(0), "batch": B, "shape": [H, W],
           "igemm_launches_per_step": len(calls), "igemm_ms_per_step_eager_events": round(step_ms, 3),
           "igemm_ms_per_step_retimed": round(total, 3), "sites": table,
           "diagnostics": diagnostics(args.iters),
           "note": "frac_tensor_pipe: issued tensor work (2 units/MAC tri-plane, 3 split-bf16) over the "
                   "989 TFLOP/s data-sheet rate of the H100 SXM at 700 W"}
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "bench_igemm_%s.json" % args.tag)
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"tag": args.tag, "gpu": res["gpu"], "retimed_ms": res["igemm_ms_per_step_retimed"],
                      "diagnostics": res["diagnostics"]}))


if __name__ == "__main__":
    main()
