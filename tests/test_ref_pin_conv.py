"""Pin of the convolution against the reference's own ConvolutionLayer (conv_layer, base_conv_layer
and im2col compiled unmodified into oracle/_ref/libmnc_ref_conv*.so by oracle/conv.mk, run as Caffe
runs it in GPU mode: im2col + sgemm per image, the bias by a gemm / gemv with beta 1).  At the 16
layer shapes of the training net, for a reduced 150x250 image, and at tail shapes with two images,
the reference and ours are each held to float64 of the same operands, and ours to the reference
directly, within the split-bf16 bound of tests/conv_bound.py; the reference's and our fractions of
the bound are reported.  A tap order, a dX flip, a dW layout or a bias handling that differed from
Caffe's would put ours far outside the bound from the reference."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

from tests import conv_bound as C
from tests import fc_bound as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBS = [os.path.join(ROOT, "oracle", "_ref", n) for n in
        ("libmnc_ref_conv_nofma.so", "libmnc_ref_conv.so")]
if not all(os.path.exists(p) for p in LIBS):
    pytest.skip("reference convolution library not built (oracle/conv.mk needs a reference checkout)",
                allow_module_level=True)
F32 = np.float32
IMAGE = (150, 250)


def _lib(path):
    lib = ctypes.CDLL(path)
    P, I = ctypes.c_void_p, ctypes.c_int
    lib.ref_convolution.argtypes = [P, P, P, P] + [I] * 7 + [P, P, P, P]
    return lib


REFS = [_lib(p) for p in LIBS]


def _p(a):
    return None if a is None else a.ctypes.data


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _ratio(got, ref64, absprod, extra64):
    err = np.abs(got.astype(np.float64) - ref64)
    return float((err / (F.TAU * absprod + F.OUT_ROUND * (np.abs(ref64) + np.abs(extra64)) + 1e-300)).max())


def _case(name, N, Cin, H, W, Cout, k):
    from mnc_b200 import ops
    pad = (k - 1) // 2
    rng = np.random.default_rng(N + Cin * 7 + H * 131 + W + Cout * 17 + k)
    x = rng.standard_normal((N, Cin, H, W)).astype(F32)
    w = (rng.standard_normal((Cout, Cin, k, k)) * (2.0 / (Cin * k * k)) ** 0.5).astype(F32)
    b = rng.standard_normal(Cout).astype(F32)
    dy = rng.standard_normal((N, Cout, H, W)).astype(F32)
    dw0 = rng.standard_normal((Cout, Cin, k, k)).astype(F32)
    db0 = rng.standard_normal(Cout).astype(F32)

    dwt, dbt = _cuda(dw0), _cuda(db0)
    ours = {"fwd": ops.conv_forward(_cuda(x), _cuda(w), _cuda(b)).cpu().numpy(),
            "dx": ops.conv_backward(_cuda(x), _cuda(w), _cuda(dy), dw=dwt, db=dbt).cpu().numpy()}
    ours["dw"], ours["db"] = dwt.cpu().numpy(), dbt.cpu().numpy()

    x64, w64, dy64 = (_cuda(a).double() for a in (x, w, dy))
    G = torch.nn.grad
    prods = {"fwd": TF.conv2d(x64, w64, padding=pad), "dx": G.conv2d_input(x.shape, w64, dy64, padding=pad),
             "dw": G.conv2d_weight(x64, w.shape, dy64, padding=pad), "db": dy64.sum((0, 2, 3))}
    absp = {"fwd": TF.conv2d(x64.abs(), w64.abs(), padding=pad),
            "dx": G.conv2d_input(x.shape, w64.abs(), dy64.abs(), padding=pad),
            "dw": G.conv2d_weight(x64.abs(), w.shape, dy64.abs(), padding=pad),
            "db": dy64.abs().sum((0, 2, 3))}
    base = {"fwd": _cuda(b).double()[:, None, None], "dx": 0.0, "dw": _cuda(dw0).double(),
            "db": _cuda(db0).double()}
    ref64 = {k: (prods[k] + base[k]).cpu().numpy() for k in prods}
    prods = {k: v.cpu().numpy() for k, v in prods.items()}
    absp = {k: v.cpu().numpy() for k, v in absp.items()}

    worst = {}
    for lib, build in zip(REFS, ("nofma", "fma")):
        ry, rdx = np.empty((N, Cout, H, W), F32), np.empty((N, Cin, H, W), F32)
        rdw, rdb = dw0.copy(), db0.copy()
        lib.ref_convolution(_p(x), _p(w), _p(b), _p(dy), N, Cin, H, W, Cout, k, pad, _p(ry), _p(rdx),
                            _p(rdw), _p(rdb))
        theirs = {"fwd": ry, "dx": rdx, "dw": rdw, "db": rdb}
        line = []
        for key in ("fwd", "dx", "dw", "db"):
            r_ref = _ratio(theirs[key], ref64[key], absp[key], prods[key])
            r_our = _ratio(ours[key], ref64[key], absp[key], prods[key])
            # ours against the reference's own result, with the same bound
            r_dir = _ratio(ours[key], theirs[key].astype(np.float64), absp[key], prods[key])
            line.append("%s ref=%.3g ours=%.3g ours-vs-ref=%.3g" % (key, r_ref, r_our, r_dir))
            assert r_our <= 1.0, (name, build, key, r_our)
            assert r_ref <= 1.0, (name, build, key, r_ref)
            assert r_dir <= 1.0, (name, build, key, r_dir)
            worst[key] = max(worst.get(key, 0.0), r_dir)
        print("REF_PIN_CONV %s %s %s: %s" % (name, (N, Cin, H, W, Cout, k), build, ", ".join(line)))
    return worst


@pytest.mark.parametrize("name,Cin,Cout,k,level,learns", C.CONV_LAYERS)
def test_convolution_reference_and_device_against_float64(name, Cin, Cout, k, level, learns):
    H, W = C.spatial(*IMAGE, level)
    _case(name, 1, Cin, H, W, Cout, k)


@pytest.mark.parametrize("N,Cin,H,W,Cout,k", [(2, 3, 2, 7, 18, 3), (2, 65, 9, 9, 18, 3),
                                              (2, 512, 1, 2, 36, 1), (2, 67, 5, 13, 36, 1)])
def test_convolution_reference_and_device_at_tail_shapes(N, Cin, H, W, Cout, k):
    _case("tail", N, Cin, H, W, Cout, k)
