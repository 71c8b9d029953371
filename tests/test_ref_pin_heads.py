"""Pin of the head layers against the reference's own InnerProduct, Pooling, ReLU and Sigmoid
(compiled unmodified into oracle/_ref/libmnc_ref_heads*.so by oracle/heads.mk, run as Caffe runs
them in GPU mode).  Pooling, ReLU and Sigmoid, forward and backward, equal both reference builds bit
for bit.  The reference's InnerProduct (cuBLAS sgemm / sgemv) and ours are each held to float64 of
the same operands; ours must meet the split-bf16 bound of tests/fc_bound.py, and both max ratios
are reported."""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import fc_bound as F
from tests.test_gpu_heads_train import _pool_input, _same, _special

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBS = [os.path.join(ROOT, "oracle", "_ref", n) for n in
        ("libmnc_ref_heads_nofma.so", "libmnc_ref_heads.so")]
if not all(os.path.exists(p) for p in LIBS):
    pytest.skip("reference head-layer library not built (oracle/heads.mk needs a reference checkout)",
                allow_module_level=True)
F32 = np.float32


def _lib(path):
    lib = ctypes.CDLL(path)
    P, I = ctypes.c_void_p, ctypes.c_int
    lib.ref_inner_product.argtypes = [P, P, P, P, I, I, I, P, P, P, P]
    lib.ref_max_pool.argtypes = [P, I, I, I, I, P, P, P, P]
    lib.ref_neuron.argtypes = [I, P, I, P, P, P]
    return lib


REFS = [_lib(p) for p in LIBS]


def _p(a):
    return None if a is None else a.ctypes.data


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("shape", [(67, 512, 28, 28), (67, 512, 14, 14), (2, 5, 7, 9), (1, 3, 1, 1)])
def test_max_pool_equals_both_reference_builds(shape):
    from mnc_b200 import ops
    rng = np.random.default_rng(sum(shape) + 1)
    x = _pool_input(rng, shape)
    y, m = ops.max_pool_nchw(_cuda(x))
    dy = rng.standard_normal(tuple(y.shape)).astype(F32)
    dx = ops.max_pool_backward_nchw(_cuda(dy), m, shape)
    for lib in REFS:
        ry, rm, rdx = np.empty(y.shape, F32), np.empty(y.shape, np.int32), np.empty(shape, F32)
        lib.ref_max_pool(_p(x), *shape, _p(dy), _p(ry), _p(rm), _p(rdx))
        assert np.array_equal(m.cpu().numpy(), rm)
        assert _same(y.cpu().numpy(), ry)
        assert _same(dx.cpu().numpy(), rdx)


@pytest.mark.parametrize("kind", ["relu", "sigmoid"])
def test_neurons_equal_both_reference_builds(kind):
    from mnc_b200 import ops
    rng = np.random.default_rng(9)
    n = 67 * 4096 + 3
    x, dy = _special(rng, n), _special(rng, n)
    dy[11:22] = np.array([np.nan, np.inf, -np.inf] * 3 + [1.0, -0.0], F32)
    x[11:22] = np.array([-1.0, -2.0, 0.0, -0.0, 3.0, 5.0, np.nan, -3.0, -0.0, np.nan, 2.0], F32)
    if kind == "relu":
        y = ops.relu(_cuda(x))
        dx = ops.relu_backward(_cuda(x), _cuda(dy))
    else:
        y = ops.sigmoid(_cuda(x))
        dx = ops.sigmoid_backward(y, _cuda(dy))
    for lib in REFS:
        ry, rdx = np.empty(n, F32), np.empty(n, F32)
        lib.ref_neuron(0 if kind == "relu" else 1, _p(x), n, _p(dy), _p(ry), _p(rdx))
        assert _same(y.cpu().numpy(), ry), kind
        assert _same(dx.cpu().numpy(), rdx), kind


def _ratio(got, ref64, absprod, extra64):
    err = np.abs(got.astype(np.float64) - ref64)
    return float((err / (F.TAU * absprod + F.OUT_ROUND * (np.abs(ref64) + np.abs(extra64)) + 1e-300)).max())


@pytest.mark.parametrize("name,N,K,M", [(n, N, K, 67) for n, N, K in F.MNC_FC_SHAPES] +
                         [("fc7", 4096, 4096, 1), ("tail", 77, 1001, 65)])
def test_inner_product_reference_and_device_against_float64(name, N, K, M):
    from mnc_b200 import ops
    rng = np.random.default_rng(N + K + M)
    x = rng.standard_normal((M, K)).astype(F32)
    w = (rng.standard_normal((N, K)) * 0.01).astype(F32)
    b = rng.standard_normal(N).astype(F32)
    dy = rng.standard_normal((M, N)).astype(F32)
    dw0 = rng.standard_normal((N, K)).astype(F32)
    db0 = rng.standard_normal(N).astype(F32)

    dwt, dbt = _cuda(dw0), _cuda(db0)
    ours = {"fwd": ops.fc_forward(_cuda(x), _cuda(w), _cuda(b)).cpu().numpy(),
            "dx": ops.fc_backward(_cuda(x), _cuda(w), _cuda(dy), dw=dwt, db=dbt).cpu().numpy()}
    ours["dw"], ours["db"] = dwt.cpu().numpy(), dbt.cpu().numpy()

    x64, w64, dy64 = (torch.from_numpy(a).cuda().double() for a in (x, w, dy))
    prods = {"fwd": x64 @ w64.T, "dx": dy64 @ w64, "dw": dy64.T @ x64, "db": dy64.sum(0)}
    absp = {"fwd": x64.abs() @ w64.abs().T, "dx": dy64.abs() @ w64.abs(),
            "dw": dy64.abs().T @ x64.abs(), "db": dy64.abs().sum(0)}
    base = {"fwd": torch.from_numpy(b).cuda().double(), "dx": 0.0,
            "dw": torch.from_numpy(dw0).cuda().double(), "db": torch.from_numpy(db0).cuda().double()}
    ref64 = {k: (prods[k] + base[k]).cpu().numpy() for k in prods}
    prods = {k: v.cpu().numpy() for k, v in prods.items()}
    absp = {k: v.cpu().numpy() for k, v in absp.items()}

    for lib, build in zip(REFS, ("nofma", "fma")):
        ry, rdx = np.empty((M, N), F32), np.empty((M, K), F32)
        rdw, rdb = dw0.copy(), db0.copy()
        lib.ref_inner_product(_p(x), _p(w), _p(b), _p(dy), M, N, K, _p(ry), _p(rdx), _p(rdw), _p(rdb))
        theirs = {"fwd": ry, "dx": rdx, "dw": rdw, "db": rdb}
        line = []
        for k in ("fwd", "dx", "dw", "db"):
            r_ref = _ratio(theirs[k], ref64[k], absp[k], prods[k])
            r_our = _ratio(ours[k], ref64[k], absp[k], prods[k])
            line.append("%s ref=%.3g ours=%.3g" % (k, r_ref, r_our))
            assert r_our <= 1.0, (name, k, r_our)
        print("REF_PIN_FC %s M=%d %s: %s" % (name, M, build, ", ".join(line)))
