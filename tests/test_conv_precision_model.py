"""CPU checks of the Convolution precision contract (tests/conv_bound.py): the float64 model of the
split-bf16 GEMM (tests/fc_bound.py) on gathered operands, with the split-K factor the library picks,
meets TAU at every layer's products for a 600x1000 image, dW's 37,500-pixel reduction at conv3_x
included, and so does the fixed-order db; a kernel that drops the two lo products fails it.  The
workspace size and the split choice are pure functions of the shape."""
import zlib

import numpy as np
import pytest

from tests import conv_bound as C
from tests import fc_bound as F


def _lib():
    from mnc_b200._lib import lib
    return lib


def _image(rng, shape, biased):
    if biased:   # bf16 rounding errors all of one sign: 1 + f, f < half a bf16 ulp
        return (1 + rng.uniform(0, 2 ** -9, shape)).astype(np.float32)
    return rng.standard_normal(shape, dtype=np.float32)


def _pixels(rng, H, W, n=8):
    """Corner and edge pixels (whose gathers read the zero padding) and random ones."""
    fixed = [0, W - 1, (H - 1) * W, H * W - 1]
    return np.unique(np.concatenate([fixed, rng.integers(0, H * W, n - len(fixed))]))[:n]


def _operands(rng, prod, Cin, H, W, Cout, k, biased):
    """Rows of A and B (the full reduction each) for a sample of a product's outputs."""
    t = k * k
    if prod == "fwd":
        A = _image(rng, (8, Cin * t), biased)
        x = _image(rng, (Cin, H, W), biased)
        B = C.gather(x, k, 1, _pixels(rng, H, W), np.arange(Cin * t))
    elif prod == "dx":
        A = _image(rng, (8, Cout * t), biased)
        dy = _image(rng, (Cout, H, W), biased)
        B = C.gather(dy, k, -1, _pixels(rng, H, W), np.arange(Cout * t))
    else:
        A = _image(rng, (8, H * W), biased)
        x = _image(rng, (min(Cin, 3), H, W), biased)
        q = rng.integers(0, min(Cin, 3) * t, 8)
        B = np.ascontiguousarray(C.gather(x, k, 1, np.arange(H * W), q).T)
    return A, B


@pytest.mark.parametrize("name,Cin,Cout,k,level,learns", C.CONV_LAYERS)
def test_model_within_tau_at_layer_shapes(name, Cin, Cout, k, level, learns):
    H, W = C.spatial(600, 1000, level)
    for i, (prod, rows, cols, red) in enumerate(C.products(Cin, H, W, Cout, k)):
        if prod == "dw" and not learns:
            continue
        rng = np.random.default_rng(zlib.crc32(name.encode()) + i)
        s = _lib().mnc_fc_split_k(rows, cols, red)
        for biased in (False, True):
            A, B = _operands(rng, prod, Cin, H, W, Cout, k, biased)
            assert A.shape[1] == B.shape[1] == red
            ref = A.astype(np.float64) @ B.astype(np.float64).T
            absprod = np.abs(A.astype(np.float64)) @ np.abs(B.astype(np.float64)).T
            good = F.ratio(F.model_gemm(A, B, s), ref, absprod)
            print("MODEL %s %s split %d biased %d: %.3g" % (name, prod, s, biased, good))
            assert good <= 0.5, (name, prod, s, biased, good)
            if biased:
                bad = F.ratio(F.model_gemm(A, B, s, drop_lo=True), ref, absprod)
                assert bad >= 8.0, (name, prod, s, bad)


@pytest.mark.parametrize("N,HW", [(1, 150 * 250), (2, 38 * 63), (1, 600 * 1000), (2, 1), (1, 257)])
def test_bias_grad_model_within_tau(N, HW):
    """db at conv3_x's 37,500 pixels and conv1_x's 600,000: the fixed-order sum is within TAU of
    float64; a running float32 sum over all pixels is not, on operands of one sign."""
    rng = np.random.default_rng(N * HW)
    for biased in (False, True):
        dy = _image(rng, (N, 4, HW), biased)
        ref = dy.astype(np.float64).sum((0, 2))
        absum = np.abs(dy.astype(np.float64)).sum((0, 2))
        got = C.model_bias_grad(dy)
        assert C.ratio(got, ref, absum) <= 0.5, (N, HW, biased)
    if N * HW >= 37500:
        run = np.zeros(4, np.float32)
        for v in dy.transpose(0, 2, 1).reshape(-1, 4):
            run = (run + v).astype(np.float32)
        assert C.ratio(run, ref, absum) > 1.0


def test_workspace_and_split_are_pure_functions_of_the_shape():
    lib = _lib()
    # a 3x3 layer: the transposed weight of dX (Cin * Cout * 9 floats) after the largest split-K
    # partials of the three per-image products, 256-byte aligned
    for name, Cin, Cout, k, level, _ in C.CONV_LAYERS:
        for image in ((600, 1000), (601, 999)):
            H, W = C.spatial(*image, level)
            part = 0
            for _, rows, cols, red in C.products(Cin, H, W, Cout, k):
                s = lib.mnc_fc_split_k(rows, cols, red)
                if s > 1:
                    part = max(part, s * rows * cols * 4)
            part = -(-part // 256) * 256
            want = part + (Cin * Cout * 9 * 4 if k == 3 else 0)
            for N in (1, 2):
                assert lib.mnc_conv_workspace_bytes(N, Cin, H, W, Cout, k) == want, (name, image)
    # the split of the 37,500-pixel dW at conv3_x: 72 tiles on 264 slots -> 4 splits
    assert lib.mnc_fc_split_k(256, 256 * 9, 150 * 250) == 4
    # conv5 forward at 600x1000 (8 x 19 tiles) splits; conv3 forward (4 x 293 tiles) does not
    assert lib.mnc_fc_split_k(512, 38 * 63, 512 * 9) == 2
    assert lib.mnc_fc_split_k(256, 150 * 250, 256 * 9) == 1
    # no workspace for shapes the kernel rejects
    assert lib.mnc_conv_workspace_bytes(1, 8, 6, 6, 4, 5) == 0
    assert lib.mnc_conv_workspace_bytes(0, 8, 6, 6, 4, 3) == 0
    assert lib.mnc_conv_workspace_bytes(1, 8, 0, 6, 4, 3) == 0
