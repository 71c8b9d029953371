"""Precision contract of the split-bf16 InnerProduct GEMMs (mnc_fc_forward / mnc_fc_backward) and a
float64 model of their arithmetic.

Each fp32 operand x is split into hi = rn_bf16(x) and lo = rn_bf16(x - hi), so |x - hi - lo| <=
2^-16 |x|; the product is hi*hi + hi*lo + lo*hi, which drops lo*lo (<= 2^-16 |ab|).  One product
is therefore within 3 * 2^-16 |ab| of the exact one.  The float32 accumulation adds the same again
for the ~10^3 roundings of the longest reduction (e.g. fc6_maskest: 49 k-steps x 12 wgmma per
split, then 32 partials), so every output element obeys

    |got - ref64| <= TAU * (|A| |B|)_ij + OUT_ROUND * |ref64|_ij,   TAU = 2^-13

where ref64 is the float64 product of the same fp32 operands, and OUT_ROUND covers the rounding of
the result (and of the bias add or the beta-1 add) to float32.  A kernel that drops the two lo
products is off by up to 2^-8 |ab| per product and fails this bound by an order of magnitude on
operands whose bf16 rounding errors share a sign.
"""
import numpy as np

TAU = 2.0 ** -13
OUT_ROUND = 2.0 ** -23

# (name, N, K) of the 9 InnerProduct parameter pairs of models/VGG16/mnc_5stage/train.prototxt
MNC_FC_SHAPES = [
    ("fc6_maskest", 256, 512 * 14 * 14),
    ("mask_pred", 441, 256),
    ("fc6", 4096, 512 * 7 * 7),
    ("fc7", 4096, 4096),
    ("fc6_mask", 4096, 512 * 7 * 7),
    ("fc7_mask", 4096, 4096),
    ("cls_score", 21, 8192),
    ("seg_cls_score", 21, 8192),
    ("bbox_pred", 84, 8192),
]
BATCHES = (1, 64, 67, 300)
# K and N off every multiple of 4, 8 and 64, M off 64
TAIL_SHAPES = [(1, 1, 1), (3, 5, 7), (67, 21, 99), (65, 129, 1001), (130, 77, 130), (7, 250, 4099)]


def bf16_rn(x):
    """float32 -> nearest-even bfloat16, returned as float32."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)


def bf16_rz(x):
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32) & np.uint32(0xFFFF0000)
    return u.view(np.float32)


def split(x):
    """hi = rn_bf16(x) (toward zero where that overflows a finite x), lo = rn_bf16(x - hi)."""
    x = np.asarray(x, dtype=np.float32)
    hi = bf16_rn(x)
    big = np.isinf(hi) & np.isfinite(x)
    hi = np.where(big, bf16_rz(x), hi)
    lo = bf16_rn(x - hi)
    return hi, lo


def model_gemm(A, B, splits=1, drop_lo=False, bk=64):
    """C[p, q] = sum_r A[p, r] B[q, r] as the kernel computes it: per 16-wide slice the three bf16
    products lo*hi, hi*lo, hi*hi (each an exact 16-term dot product) are added to a float32
    accumulator, slices in order; `splits` contiguous ranges of whole 64-wide k-steps give float32
    partials that are added in split order.  drop_lo: hi*hi only (the mutant)."""
    P, R = A.shape
    Q = B.shape[0]
    ksteps = -(-R // bk)
    per = -(-ksteps // splits)
    Rp = ksteps * bk
    Ap = np.zeros((P, Rp), np.float32)
    Bp = np.zeros((Q, Rp), np.float32)
    Ap[:, :R], Bp[:, :R] = A, B
    ah, al = split(Ap)
    bh, bl = split(Bp)
    G = Rp // 16

    def slices(x, y):
        return np.einsum("pgk,qgk->pqg", x.astype(np.float64).reshape(P, G, 16),
                         y.astype(np.float64).reshape(Q, G, 16))

    terms = [slices(ah, bh)] if drop_lo else [slices(al, bh), slices(ah, bl), slices(ah, bh)]
    out = None
    for s in range(0, ksteps, per):
        acc = np.zeros((P, Q), np.float32)
        for g in range(s * bk // 16, min(ksteps, s + per) * bk // 16):
            for t in terms:
                acc = (acc.astype(np.float64) + t[:, :, g]).astype(np.float32)
        out = acc if out is None else (out + acc).astype(np.float32)
    return out


def ratio(got, ref64, absprod):
    """max over elements of |got - ref64| / (TAU-side scale): <= 1 means within the bound."""
    err = np.abs(np.asarray(got, np.float64) - ref64)
    return float((err / (TAU * absprod + OUT_ROUND * np.abs(ref64) + 1e-300)).max())


def excess(got, ref64, absprod):
    """max |got - ref64| / (|A||B|) -- the measured counterpart of TAU (outputs with |A||B| > 0)."""
    err = np.abs(np.asarray(got, np.float64) - ref64) - OUT_ROUND * np.abs(ref64)
    m = absprod > 0
    return float((np.maximum(err[m], 0) / absprod[m]).max()) if m.any() else 0.0
