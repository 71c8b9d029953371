"""Three-way pin of the loss layers: the reference's own SoftmaxWithLoss, SmoothL1Loss,
SigmoidCrossEntropyLoss and Accuracy (compiled unmodified into oracle/_ref/libmnc_ref_loss*.so by
oracle/loss.mk, run as Caffe runs them in GPU mode) == the numpy oracle == the device, at the
training-net shapes with the targets of the device's own target layers.  Diffs and prob are held
bit for bit against both builds (the kernels involved contract nothing: no multiply feeds an add),
accuracy exactly, loss scalars to the error bound of the reference's unordered float sum
(n 2^-24 sum |terms|) plus 4 float32 ulp per term where exp / log enter."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import oracle_loss as L

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBS = [os.path.join(ROOT, "oracle", "_ref", n) for n in
        ("libmnc_ref_loss_nofma.so", "libmnc_ref_loss.so")]
if not all(os.path.exists(p) for p in LIBS):
    pytest.skip("reference loss library not built (oracle/loss.mk needs a reference checkout)",
                allow_module_level=True)
F32 = np.float32


def _lib(path):
    lib = ctypes.CDLL(path)
    P, I, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    lib.ref_softmax_loss.argtypes = [P, P, I, I, I, I, I, I, I, F, P, P, P, P]
    lib.ref_smooth_l1_loss.argtypes = [P, P, P, P, I, I, I, I, F, F, P, P, P]
    lib.ref_sigmoid_ce_loss.argtypes = [P, P, P, I, I, F, P, P, P]
    lib.ref_accuracy.argtypes = [P, P, I, I, I, I, I, I, P]
    return lib


REFS = [_lib(p) for p in LIBS]


def _p(a):
    return None if a is None else a.ctypes.data


def _c(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def ref_softmax(lib, x, lab, ignore, mode, lw):
    x, lab = _c(x), _c(lab)
    outer, C = x.shape[0], x.shape[1]
    inner = x.size // (outer * C)
    loss, prob, diff = np.zeros(1, F32), np.zeros_like(x), np.zeros_like(x)
    lib.ref_softmax_loss(_p(x), _p(lab), outer, C, inner, int(ignore is not None), ignore or 0,
                         L.NORMALIZATION[mode], 0, lw, _p(loss), _p(prob), _p(diff), None)
    return loss[0], prob, diff


def ref_smooth_l1(lib, p, t, wi, wo, sigma, lw):
    p, t = _c(p), _c(t)
    wi, wo = (None, None) if wi is None else (_c(wi), _c(wo))
    s = p.shape + (1,) * (4 - p.ndim)
    loss, diff = np.zeros(1, F32), np.zeros_like(p)
    lib.ref_smooth_l1_loss(_p(p), _p(t), _p(wi), _p(wo), *s, sigma, lw, _p(loss), _p(diff), None)
    return loss[0], diff


def ref_sigmoid_ce(lib, x, t, w, lw, before=0.0):
    x, t = _c(x), _c(t)
    w = None if w is None else _c(w)
    loss, diff = np.full(1, before, F32), np.zeros_like(x)
    lib.ref_sigmoid_ce_loss(_p(x), _p(t), _p(w), x.shape[0], x.size // x.shape[0], lw, _p(loss),
                            _p(diff), None)
    return loss[0], diff


def ref_accuracy(lib, x, lab, top_k, ignore):
    x, lab = _c(x), _c(lab)
    outer, C = x.shape[0], x.shape[1]
    out = np.zeros(1, F32)
    lib.ref_accuracy(_p(x), _p(lab), outer, C, x.size // (outer * C), top_k,
                     int(ignore is not None), ignore or 0, _p(out))
    return out[0]


def _np(t):
    return t.detach().cpu().numpy()


def _sum_bound(terms, norm):
    t = np.abs(np.asarray(terms, np.float64))
    return len(t.ravel()) * 2.0 ** -24 * t.sum() / float(norm)


@pytest.fixture(scope="module")
def step():
    """Predictions and the targets of the device's target layers, trimmed to the K real rows."""
    from tests.test_gpu_loss import _targets, _preds
    o, at, seg = _targets()
    K = int(o["counts"][0])
    p = {k: _np(v) for k, v in _preds(o["labels"].shape[0], 67).items()}
    return p, {k: _np(v) for k, v in o.items()}, [_np(a) for a in at], _np(seg), K


def test_softmax_loss_three_way(step):
    from mnc_b200 import ops
    p, o, at, seg, K = step
    r = np.random.default_rng(5)
    cases = [(p["rpn_cls"], at[0], "VALID"), (p["cls"][:K], o["labels"][:K], "VALID"),
             (p["seg_cls"][:K], seg[:K], "VALID"),
             (p["cls"][:K], r.integers(-1, 21, K).astype(F32), "FULL"),
             (p["cls"][:K], r.integers(-1, 21, K).astype(F32), "BATCH_SIZE"),
             (p["cls"][:K], r.integers(-1, 21, K).astype(F32), "NONE")]
    for x, lab, mode in cases:
        dl, dp = ops.softmax_loss(torch.from_numpy(_c(x)).cuda(), torch.from_numpy(_c(lab)).cuda(),
                                  -1, mode)
        dd = _np(ops.softmax_loss_backward(dp, torch.from_numpy(_c(lab)).cuda(),
                                           torch.ones((), device="cuda"), -1, mode))
        dp = _np(dp)
        ol, _ = L.softmax_loss(x, lab, -1, mode)
        for lib in REFS:
            rl, rp, rd = ref_softmax(lib, x, lab, -1, mode, 1.0)
            assert np.array_equal(rp.reshape(dp.shape), dp), mode
            assert np.array_equal(rd.reshape(dd.shape), dd), mode
            lab_i = np.trunc(_c(lab)).astype(int).reshape(x.shape[0], -1)
            pl = np.take_along_axis(dp.reshape(x.shape[0], x.shape[1], -1),
                                    np.clip(lab_i, 0, None)[:, None, :], 1)[:, 0]
            terms = np.where(lab_i >= 0, -L.logf(np.maximum(pl, L.FLT_MIN)), 0)
            norm = L.normalizer(mode, x.shape[0], lab_i.shape[1], int((lab_i >= 0).sum()))
            assert abs(float(rl) - float(_np(dl))) <= _sum_bound(terms, norm) + 2 * np.spacing(rl)
            assert abs(float(ol) - float(_np(dl))) <= 4 * float(np.spacing(np.abs(terms).astype(F32)).sum()) / float(norm) + 4 * np.spacing(ol)


def test_smooth_l1_loss_three_way(step):
    from mnc_b200 import ops
    p, o, at, seg, K = step
    cases = [(p["rpn_bbox"], at[1], at[2], at[3], 3.0),
             (p["bbox"][:K], o["bbox_targets"][:K], o["bbox_inside_weights"][:K],
              o["bbox_outside_weights"][:K], 1.0),
             (p["bbox"][:K], o["bbox_targets"][:K], None, None, 1.0)]
    for x, t, wi, wo, sigma in cases:
        dev = [None if a is None else torch.from_numpy(_c(a)).cuda() for a in (x, t, wi, wo)]
        dl = _np(ops.smooth_l1_loss(*dev, sigma=sigma))
        dd = _np(ops.smooth_l1_loss_backward(*dev, sigma=sigma, top_diff=torch.ones((), device="cuda")))
        assert dl == L.smooth_l1_loss(x, t, wi, wo, sigma)
        assert np.array_equal(dd, L.smooth_l1_loss_backward(x, t, wi, wo, sigma, 1.0))
        val = _c(x) - _c(t) if wi is None else _c(wi) * (_c(x) - _c(t))
        for lib in REFS:
            rl, rd = ref_smooth_l1(lib, x, t, wi, wo, sigma, 1.0)
            assert np.array_equal(rd.reshape(dd.shape), dd)
            assert abs(float(rl) - float(dl)) <= _sum_bound(np.abs(val) * 4, x.shape[0]) + 2 * np.spacing(rl)


def test_sigmoid_ce_loss_three_way(step):
    from mnc_b200 import ops
    p, o, at, seg, K = step
    cases = [(p["mask"][:K], o["mask_targets"][:K], o["mask_weight"][:K]),
             (p["mask"][:K], o["mask_targets"][:K], None),
             (p["mask"][:K], o["mask_targets"][:K], np.zeros_like(o["mask_weight"][:K]))]
    for x, t, w in cases:
        dev = [None if a is None else torch.from_numpy(_c(a)).cuda() for a in (x, t, w)]
        out = torch.full((), 3.5, device="cuda")
        dl = _np(ops.sigmoid_ce_loss(*dev, out=out))
        dd = _np(ops.sigmoid_ce_loss_backward(*dev, top_diff=torch.full((), 2.0, device="cuda")))
        terms = L.sigmoid_ce_terms(x, t, w)
        norm = x.shape[0] if w is None else max(float(L.fixed_sum(w)), 1.0)
        ol = L.sigmoid_ce_loss(x, t, w, untouched=F32(3.5))
        assert abs(float(ol) - float(dl)) <= 4 * float(np.spacing(np.abs(terms)).sum()) / norm + 4 * np.spacing(ol)
        for lib in REFS:
            rl, rd = ref_sigmoid_ce(lib, x, t, w, 2.0, before=3.5)
            assert np.array_equal(rd.reshape(dd.shape), dd)
            bound = _sum_bound(terms, norm) + 4 * float(np.spacing(np.abs(terms)).sum()) / norm
            assert abs(float(rl) - float(dl)) <= bound + 2 * np.spacing(rl)
        if w is not None and not w.any():
            assert float(dl) == 3.5


def test_accuracy_three_way(step):
    from mnc_b200 import ops
    p, o, at, seg, K = step
    r = np.random.default_rng(6)
    tied = r.integers(0, 3, (K, 21)).astype(F32)
    cases = [(p["cls"][:K], o["labels"][:K], 1, None), (p["seg_cls"][:K], seg[:K], 1, None),
             (tied, o["labels"][:K], 1, None), (tied, o["labels"][:K], 3, -1),
             (p["rpn_cls"], at[0], 1, -1)]
    for x, lab, k, ign in cases:
        d = _np(ops.accuracy(torch.from_numpy(_c(x)).cuda(), torch.from_numpy(_c(lab)).cuda(), k, ign))
        assert d == L.accuracy(x, lab, k, ign)
        for lib in REFS:
            assert ref_accuracy(lib, x, lab, k, ign) == d
