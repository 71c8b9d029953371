"""The convolutions of models/VGG16/mnc_5stage/train.prototxt and a float64 model of the arithmetic of
mnc_conv_forward / mnc_conv_backward on their gathered operands.

Each product is the InnerProduct GEMM (tests/fc_bound.py) with an image operand gathered in the
loader (DESIGN.md "Trunk and RPN convolutions for training"), so the InnerProduct contract holds
with the convolution's operands:

    |got - ref64| <= TAU * (|A| |B|)_ij + OUT_ROUND * (|ref64| + |product|)_ij

where |A| |B| is the same convolution in float64 on |W| and |X| (or |dY|).  db is a sum of dY:
per image, thread j of 256 adds pixels j, j + 256, ... in order, a binary tree adds the 256
partials, and the images' sums are added in order.
"""
import numpy as np

from mnc_b200 import weights as Wt
from tests import fc_bound as F

CONV_LAYERS = Wt.TRAIN_CONVS
POOL_AFTER = Wt.POOL_AFTER
spatial = Wt.train_conv_size

# (N, Cin, H, W, Cout, kernel): Cin 3, Cout 18 / 36, H or W of 1 or 2, H * W off every multiple of
# 128, Cin off 64, N = 2
TAIL_SHAPES = [(1, 3, 1, 1, 64, 3), (2, 3, 2, 7, 18, 3), (1, 67, 5, 130, 36, 1),
               (2, 100, 13, 11, 70, 3), (1, 512, 2, 1, 36, 1), (2, 65, 9, 9, 18, 3),
               (1, 1, 1, 1, 1, 1), (2, 130, 37, 62, 129, 3), (2, 512, 1, 2, 18, 1)]


def products(Cin, H, W, Cout, k):
    """(name, rows, cols, red) of the per-image forward, dX and dW products."""
    t = k * k
    return [("fwd", Cout, H * W, Cin * t), ("dx", Cin, H * W, Cout * t), ("dw", Cout, Cin * t, H * W)]


def gather(img, k, sign, pix, r_idx):
    """Rows `pix` of the gathered image operand, element (pix, c * k * k + t) =
    img[c, y + sign * (kh - p), x + sign * (kw - p)], zero outside the image (p = (k - 1) / 2)."""
    C, H, W = img.shape
    p = (k - 1) // 2
    pix = np.asarray(pix)[:, None]
    c, t = np.divmod(np.asarray(r_idx)[None, :], k * k)
    kh, kw = np.divmod(t, k)
    y = pix // W + sign * (kh - p)
    x = pix % W + sign * (kw - p)
    ok = (y >= 0) & (y < H) & (x >= 0) & (x < W)
    return np.where(ok, img[c, np.clip(y, 0, H - 1), np.clip(x, 0, W - 1)], 0).astype(np.float32)


def model_bias_grad(dy):
    """db of mnc_conv_backward from zero, in float32: dy (N, Cout, HW)."""
    N, Cout, HW = dy.shape
    total = None
    for n in range(N):
        lanes = np.zeros((Cout, 256), np.float32)
        for i in range(0, HW, 256):
            chunk = dy[n, :, i:i + 256]
            lanes[:, :chunk.shape[1]] = (lanes[:, :chunk.shape[1]] + chunk).astype(np.float32)
        h = 128
        while h:
            lanes[:, :h] = (lanes[:, :h] + lanes[:, h:2 * h]).astype(np.float32)
            h //= 2
        s = lanes[:, 0].copy()
        total = s if total is None else (total + s).astype(np.float32)
    return total


def ratio(got, ref64, absprod):
    """max |got - ref64| / (TAU |A||B| + OUT_ROUND (|ref| + |product|)), product = ref here."""
    err = np.abs(np.asarray(got, np.float64) - ref64)
    return float((err / (F.TAU * absprod + 2 * F.OUT_ROUND * np.abs(ref64) + 1e-300)).max())
