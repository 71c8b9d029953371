"""Times mnc_mv_device -- the tight boxes and resampled masks of mask voting -- in two builds of
the library, alternated in one process, and checks that both give the same bytes.  Inputs: the
seeded voting inputs of bench.py's mask voting microbenchmark (600 boxes x 21 classes at 600x1000),
one seed per image, batch 8; the candidate lists come from ops.mask_voting of the in-tree build.
Prints one JSON line with the card's name and power limit.

    python scripts/bench_mask_voting.py --lib-a OLD.so --lib-b NEW.so [--iters 50] [--rounds 6]
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from mnc_b200 import ops  # noqa: E402
from scripts.bench_roi_backward import card  # noqa: E402
from tests.test_ref_pin import _voting_inputs  # noqa: E402

B, NB, H, W, M = 8, 600, 600, 1000, 21


def load(path):
    lib = ctypes.CDLL(os.path.abspath(path))
    f = lib.mnc_mv_device
    f.restype = ctypes.c_int
    f.argtypes = ([ctypes.c_void_p] * 2 + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 2 +
                  [ctypes.c_longlong] + [ctypes.c_void_p] * 3 + [ctypes.c_int] * 2 +
                  [ctypes.c_void_p] * 5)
    return f


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib-a", required=True)
    ap.add_argument("--lib-b", required=True)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=6)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    ins = [_voting_inputs(NB, H, W, 11 + b) for b in range(B)]
    boxes = torch.from_numpy(np.stack([i[0] for i in ins])).cuda()
    masks = torch.from_numpy(np.stack([i[1] for i in ins])).cuda()
    scores = torch.from_numpy(np.stack([i[2] for i in ins])).cuda()
    hw = torch.tensor([[H, W]] * B, dtype=torch.int32, device="cuda")
    r = ops.mask_voting(boxes, masks, scores, hw)
    R = r["cand_begin"].shape[1]
    libs = {"a": load(args.lib_a), "b": load(args.lib_b)}
    ws = torch.zeros(B * R * 4 + B, dtype=torch.int32, device="cuda")
    outs = {k: (torch.zeros((B, R, 1, M, M), device="cuda"), torch.zeros((B, R, 4), dtype=torch.int32, device="cuda"))
            for k in libs}
    stream = torch.cuda.current_stream().cuda_stream

    def call(k):
        om, ob = outs[k]
        rc = libs[k](boxes.data_ptr(), masks.data_ptr(), NB, 4, M, r["cand_inds"].data_ptr(),
                     r["cand_weights"].data_ptr(), R * NB, r["cand_begin"].data_ptr(),
                     r["cand_end"].data_ptr(), r["n_res"].data_ptr(), R, B, hw.data_ptr(),
                     ws.data_ptr(), om.data_ptr(), ob.data_ptr(), stream)
        assert rc == 0, rc

    for k in libs:
        for _ in range(3):
            call(k)
    torch.cuda.synchronize()
    n = r["n_res"].cpu().numpy()
    same = all(torch.equal(outs["a"][j][b, :n[b]], outs["b"][j][b, :n[b]]) for j in (0, 1) for b in range(B))
    times = {k: [] for k in libs}
    for _ in range(args.rounds):
        for k in libs:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                call(k)
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) * 1000.0 / args.iters)
    print(json.dumps({"card": card(), "batch": B, "image": [H, W], "results": [int(v) for v in n],
                      "outputs_identical": bool(same),
                      "us_per_call": {k: {"median": float(np.median(v)), "all": [round(x, 1) for x in v]}
                                      for k, v in times.items()},
                      "libs": {"a": args.lib_a, "b": args.lib_b}}))


if __name__ == "__main__":
    main()
