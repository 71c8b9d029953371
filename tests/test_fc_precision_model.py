"""CPU checks of the InnerProduct precision contract (tests/fc_bound.py): the float64 model of the
split-bf16 arithmetic meets TAU at every MNC layer shape and product orientation, with the split-K
factor the library picks, and a kernel that drops the two lo products fails it by a wide margin."""
import zlib

import numpy as np
import pytest

from tests import fc_bound as F


def _split_k(rows, cols, red):
    from mnc_b200._lib import lib
    return lib.mnc_fc_split_k(rows, cols, red)


def _products(M, N, K):
    """(name, rows, cols, red) of forward, dX and dW."""
    return [("fwd", N, M, K), ("dx", K, M, N), ("dw", N, K, M)]


def _sampled(rng, rows, cols, red, biased, n_rows=8, n_cols=8):
    """Operands of a sample of the output: n_rows x n_cols elements, the full reduction each."""
    if biased:   # bf16 rounding errors all of one sign: 1 + f, f < half a bf16 ulp
        A = (1 + rng.uniform(0, 2 ** -9, (min(rows, n_rows), red))).astype(np.float32)
        B = (1 + rng.uniform(0, 2 ** -9, (min(cols, n_cols), red))).astype(np.float32)
    else:
        A = rng.standard_normal((min(rows, n_rows), red)).astype(np.float32)
        B = rng.standard_normal((min(cols, n_cols), red)).astype(np.float32)
    return A, B


def _check(rows, cols, red, seed):
    rng = np.random.default_rng(seed)
    s = _split_k(rows, cols, red)
    for biased in (False, True):
        A, B = _sampled(rng, rows, cols, red, biased)
        ref = A.astype(np.float64) @ B.astype(np.float64).T
        absprod = np.abs(A.astype(np.float64)) @ np.abs(B.astype(np.float64)).T
        good = F.ratio(F.model_gemm(A, B, s), ref, absprod)
        assert good <= 0.5, (rows, cols, red, s, biased, good)
        if biased:
            bad = F.ratio(F.model_gemm(A, B, s, drop_lo=True), ref, absprod)
            assert bad >= 8.0, (rows, cols, red, s, bad)


@pytest.mark.parametrize("name,N,K", F.MNC_FC_SHAPES)
@pytest.mark.parametrize("M", F.BATCHES)
def test_model_within_tau_at_mnc_shapes(name, N, K, M):
    for i, (_, rows, cols, red) in enumerate(_products(M, N, K)):
        _check(rows, cols, red, seed=zlib.crc32(name.encode()) + 10 * M + i)


@pytest.mark.parametrize("M,N,K", F.TAIL_SHAPES)
def test_model_within_tau_at_tail_shapes(M, N, K):
    for i, (_, rows, cols, red) in enumerate(_products(M, N, K)):
        _check(rows, cols, red, seed=M * 7919 + N * 31 + K + i)


def test_bf16_split_is_exact_to_2e16():
    x = np.random.default_rng(0).standard_normal(100000).astype(np.float32)
    hi, lo = F.split(x)
    assert np.all(np.abs(x.astype(np.float64) - hi - lo) <= 2.0 ** -16 * np.abs(x))
    assert F.bf16_rn(np.float32([1 + 2 ** -8]))[0] == 1.0          # tie to even
    assert F.bf16_rn(np.float32([1 + 3 * 2 ** -8]))[0] == 1 + 2 ** -6


def test_split_k_is_a_pure_function_of_the_shape():
    """Split-K only where the tiles (64 x 128) cannot fill 264 resident CTAs; never an empty split;
    at most 32."""
    assert _split_k(4096, 25088, 67) == 1                 # dW of fc6: 12544 tiles
    assert _split_k(25088, 67, 4096) == 1                 # dX of fc6: 392 tiles
    assert _split_k(256, 67, 100352) == 32                # forward fc6_maskest: 4 tiles
    assert _split_k(4096, 67, 25088) == 5                 # forward fc6: 64 tiles
    assert _split_k(1, 1, 1) == 1
    for rows, cols, red in [(21, 300, 8192), (441, 64, 256), (7, 3, 4099), (84, 1, 130)]:
        s = _split_k(rows, cols, red)
        ksteps = -(-red // 64)
        per = -(-ksteps // s)
        assert 1 <= s <= 32 and (s - 1) * per < ksteps, (rows, cols, red, s)
        assert _split_k(rows, cols, red) == s
