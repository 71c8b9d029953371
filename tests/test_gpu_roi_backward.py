"""Backward passes of ROIWarping / MaskResize / MaskPooling / ROIPooling (mnc_*_backward_nchw) vs
the C oracle: feature and mask gradients bit-exact, RoI coordinate gradients to 1e-5 of the sum of
their terms' magnitudes; determinism, NULL outputs, the layer mirrors' Backward_gpu and the autograd
Functions."""
import numpy as np
import pytest
import torch

from tests import roi_shapes as RS
from tests.test_gpu_roi import _rois, table_params

pytestmark = pytest.mark.gpu


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _warp_case(P, PW=None, seed=0):
    PW = PW or P
    rng = np.random.default_rng(100 + P + seed)
    feat = rng.normal(size=(2, 40, 38, 63)).astype(np.float32)
    rois = _rois(64, 8 + P)                 # edge RoIs of test_gpu_roi: whole map, degenerate,
    rois[10:30, 0] = 1                      # off-map, past the edge, round-half, inverted
    top = rng.normal(size=(rois.shape[0], 40, P, PW)).astype(np.float32)
    return feat, rois, top


def _table_case(case, ph, pw):
    """feat, rois, top_diff and spatial scale of a case of tests/roi_shapes.py."""
    return RS.feat(case), RS.rois(case), RS.top_diff(case, ph, pw), RS.BY_NAME[case].scale


def _images_without_rois(feat, rois):
    return sorted(set(range(feat.shape[0])) - set(rois[:, 0].astype(int).tolist()))


def _same_bits(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


@pytest.mark.parametrize("case,size", [pytest.param(None, (P, PW), id="%d-%d" % (P, PW))
                                       for P, PW in [(28, 28), (14, 14), (7, 7), (9, 5)]] + table_params())
def test_roi_warp_backward_matches_oracle(case, size):
    from oracle import oracle_backward as OB
    from mnc_b200 import ops
    P, PW = size
    if case is None:
        feat, rois, top = _warp_case(P, PW)
        ss = 0.0625
    else:
        feat, rois, top, ss = _table_case(case, P, PW)
    want_f, want_r, mag = OB.roi_warp_backward(feat, rois, top, P, PW, ss, want_abs=True)
    fd, rd = ops.roi_warp_backward_nchw(_cuda(feat), _cuda(rois), _cuda(top), P, PW, ss)
    fd, rd = fd.cpu().numpy(), rd.cpu().numpy()
    assert np.array_equal(fd, want_f)
    assert np.abs(want_f).max() > 0
    assert np.all(rd[:, 0] == 0)
    assert np.all(np.abs(rd - want_r) <= 1e-5 * mag + 1e-30)
    H, W = feat.shape[2:]
    if H > 1 and W > 1:
        # (on a single row or column every sample's second tap lies past the map: no term)
        assert np.abs(want_r).max() > 0
    # RoI 3 lies entirely outside the map: every sample is out of range and contributes 0
    for r in ([3] if case is None else RS.outside_rows(case)):
        assert np.all(rd[r] == 0)
    # an image no RoI points at gets exact +0.0 (the output comes from torch.empty)
    for n in _images_without_rois(feat, rois):
        assert _same_bits(fd[n], np.zeros_like(fd[n]))
    # a second call gives the same bits
    fd2, rd2 = ops.roi_warp_backward_nchw(_cuda(feat), _cuda(rois), _cuda(top), P, PW, ss)
    assert _same_bits(fd2.cpu().numpy(), fd) and _same_bits(rd2.cpu().numpy(), rd)


def test_roi_warp_backward_null_outputs_and_limits():
    from mnc_b200 import ops
    from mnc_b200._lib import lib, ptr, cur_stream, MncError
    feat, rois, top = _warp_case(7)
    f, r, t = _cuda(feat), _cuda(rois), _cuda(top)
    fd_only, none = ops.roi_warp_backward_nchw(f, r, t, 7, 7, want_rois=False)
    assert none is None
    none, rd_only = ops.roi_warp_backward_nchw(f, r, t, 7, 7, want_feat=False)
    assert none is None
    fd, rd = ops.roi_warp_backward_nchw(f, r, t, 7, 7)
    assert torch.equal(fd_only, fd) and torch.equal(rd_only, rd)
    # NULL rois_diff leaves nothing else written; R = 0 touches nothing
    sentinel = torch.full_like(f, 7.0)
    rc = lib.mnc_roi_warp_backward_nchw(ptr(f), 2, 40, 38, 63, ptr(r), 0, 7, 7, 0.0625, ptr(t),
                                        ptr(sentinel), ptr(None), cur_stream())
    torch.cuda.synchronize()
    assert rc == 0 and bool((sentinel == 7.0).all())
    with pytest.raises(MncError):
        ops.roi_warp_backward_nchw(f, r, torch.zeros(r.shape[0], 40, 33, 33, device="cuda"), 33, 33)
    with pytest.raises(MncError):
        ops.roi_warp_backward_nchw(f, r, torch.zeros(r.shape[0], 40, 7, 40, device="cuda"), 7, 40)
    z = ops.roi_warp_backward_nchw(f, r[:0], t[:0], 7, 7)
    assert not z[0].any() and z[1].shape == (0, 5)


@pytest.mark.parametrize("oh,ow,planes", [pytest.param(oh, ow, (37, 2), id="%d-%d" % (oh, ow))
                                           for oh, ow in [(14, 14), (7, 9), (21, 21), (28, 28)]] +
                         [pytest.param(o[0], o[1], s[:2], id=k) for k, (s, o) in RS.MASK_RESIZE_BWD.items()])
def test_mask_resize_backward_matches_oracle(oh, ow, planes):
    from oracle import oracle_backward as OB
    from mnc_b200 import ops
    rng = np.random.default_rng(oh + ow)
    g = rng.normal(size=planes + (oh, ow)).astype(np.float32)
    got = ops.mask_resize_backward_nchw(_cuda(g), 21, 21).cpu().numpy()
    want = OB.mask_resize_backward(g, 21, 21)
    assert np.array_equal(got, want) and np.abs(want).max() > 0


@pytest.mark.parametrize("shape", [pytest.param(s, id="shape%d" % i) for i, s in enumerate([(64, 24, 14, 14), (3, 5, 7, 9)])] +
                         [pytest.param(s, id=k) for k, s in RS.MASK_POOL.items()])
def test_mask_pool_backward_matches_oracle(shape):
    from oracle import oracle_backward as OB
    from mnc_b200 import ops
    rng = np.random.default_rng(5)
    N, C, H, W = shape
    feat = rng.normal(size=shape).astype(np.float32)
    mask = rng.uniform(size=(N, 1, H, W)).astype(np.float32)
    g = rng.normal(size=shape).astype(np.float32)
    wf, wm = OB.mask_pool_backward(feat, mask, g)
    fd, md = ops.mask_pool_backward_nchw(_cuda(feat), _cuda(mask), _cuda(g))
    assert np.array_equal(fd.cpu().numpy(), wf) and np.array_equal(md.cpu().numpy(), wm)
    none, md2 = ops.mask_pool_backward_nchw(_cuda(feat), _cuda(mask), _cuda(g), want_feat=False)
    assert none is None and torch.equal(md2, md)


@pytest.mark.parametrize("case,size", [pytest.param(None, (P, P), id=str(P)) for P in (7, 14)] + table_params())
def test_roi_pool_backward_matches_oracle(case, size):
    from oracle import oracle_backward as OB
    from mnc_b200 import ops
    P, PW = size
    if case is None:
        feat, rois, _ = _warp_case(P, seed=3)
        g = np.random.default_rng(P).normal(size=(rois.shape[0], 40, P, P)).astype(np.float32)
        ss = 0.0625
    else:
        feat, rois, g, ss = _table_case(case, P, PW)
    arg = torch.empty(g.shape, dtype=torch.int32, device="cuda")
    ops.roi_pool_nchw(_cuda(feat), _cuda(rois), P, PW, ss, argmax=arg)
    want = OB.roi_pool_backward(g, arg.cpu().numpy(), feat.shape, rois, P, PW, ss)
    got = ops.roi_pool_backward_nchw(_cuda(g), arg, feat.shape, _cuda(rois), P, PW, ss)
    assert np.array_equal(got.cpu().numpy(), want) and np.abs(want).max() > 0
    for n in _images_without_rois(feat, rois):
        assert _same_bits(got[n].cpu().numpy(), np.zeros_like(want[n]))
    again = ops.roi_pool_backward_nchw(_cuda(g), arg, feat.shape, _cuda(rois), P, PW, ss)
    assert _same_bits(again.cpu().numpy(), got.cpu().numpy())


def test_layer_mirrors_backward():
    import mnc_b200.lib as L
    L.install()
    import caffe
    from caffe.layers import ROIWarpingLayer, MaskResizeLayer, MaskPoolingLayer, ROIPoolingLayer
    from oracle import oracle_backward as OB
    rng = np.random.default_rng(2)
    feat, rois, top = caffe.Blob(), caffe.Blob(), caffe.Blob()
    feat.data = rng.normal(size=(1, 16, 20, 30)).astype(np.float32)
    rois.data = _rois(12, 2, W=480, H=320)
    layer = ROIWarpingLayer(dict(roi_warping_param=dict(pooled_w=14, pooled_h=14, spatial_scale=0.0625)))
    layer.LayerSetUp([feat, rois], [top])
    layer.Forward([feat, rois], [top])
    top.diff = rng.normal(size=top.shape).astype(np.float32)
    wf, wr, mag = OB.roi_warp_backward(feat.data, rois.data, top.diff, 14, 14, want_abs=True)
    layer.Backward([top], [True, True], [feat, rois])
    assert np.array_equal(feat.diff, wf) and np.all(np.abs(rois.diff - wr) <= 1e-5 * mag + 1e-30)
    rois.diff[...] = 5
    layer.Backward([top], [True, False], [feat, rois])       # both diffs zeroed unconditionally
    assert np.array_equal(feat.diff, wf) and not rois.diff.any()
    layer.Backward([top], [False, False], [feat, rois])
    assert not feat.diff.any()
    with pytest.raises(NotImplementedError):
        layer.Backward_cpu([top], [True, True], [feat, rois])

    m, mt = caffe.Blob(), caffe.Blob()
    m.data = rng.uniform(size=(4, 1, 21, 21)).astype(np.float32)
    mr = MaskResizeLayer(dict(mask_resize_param=dict(output_height=14, output_width=14)))
    mr.LayerSetUp([m], [mt])
    mr.Forward([m], [mt])
    mt.diff = rng.normal(size=mt.shape).astype(np.float32)
    m.diff = np.ones((3, 3), np.float32)                     # wrong shape: reallocated
    mr.Backward([mt], [False], [m])                          # MaskResize always writes
    assert np.array_equal(m.diff, OB.mask_resize_backward(mt.diff, 21, 21))

    f, k, pt = caffe.Blob(), caffe.Blob(), caffe.Blob()
    f.data = rng.normal(size=(4, 6, 14, 14)).astype(np.float32)
    k.data = rng.uniform(size=(4, 1, 14, 14)).astype(np.float32)
    mp = MaskPoolingLayer()
    mp.Forward([f, k], [pt])
    pt.diff = rng.normal(size=pt.shape).astype(np.float32)
    wf, wm = OB.mask_pool_backward(f.data, k.data, pt.diff)
    mp.Backward([pt], [True, True], [f, k])
    assert np.array_equal(f.diff, wf) and np.array_equal(k.diff, wm)
    k.diff[...] = 3
    mp.Backward([pt], [False, False], [f, k])                # feature diff zeroed, mask untouched
    assert not f.diff.any() and bool((k.diff == 3).all())

    rp = ROIPoolingLayer(dict(roi_pooling_param=dict(pooled_w=7, pooled_h=7, spatial_scale=0.0625)))
    rp.LayerSetUp([feat, rois], [top])
    rp.Forward([feat, rois], [top])
    top.diff = rng.normal(size=top.shape).astype(np.float32)
    feat.diff[...] = 9
    rp.Backward([top], [False, False], [feat, rois])         # nothing touched
    assert bool((feat.diff == 9).all())
    rp.Backward([top], [True, False], [feat, rois])
    assert np.array_equal(feat.diff, OB.roi_pool_backward(top.diff, rp.max_idx_, feat.shape, rois.data, 7, 7))


def test_autograd_equals_ops():
    from mnc_b200 import autograd as A, ops
    feat, rois, top = _warp_case(14)
    f = _cuda(feat).requires_grad_()
    r = _cuda(rois).requires_grad_()
    out = A.roi_warp(f, r, 14, 14)
    assert torch.equal(out.detach(), ops.roi_warp_nchw(_cuda(feat), _cuda(rois), 14, 14))
    out.backward(_cuda(top))
    fd, rd = ops.roi_warp_backward_nchw(_cuda(feat), _cuda(rois), _cuda(top), 14, 14)
    assert torch.equal(f.grad, fd) and torch.equal(r.grad, rd)

    rng = np.random.default_rng(8)
    x = _cuda(rng.uniform(size=(5, 1, 21, 21)).astype(np.float32)).requires_grad_()
    g = _cuda(rng.normal(size=(5, 1, 14, 14)).astype(np.float32))
    A.mask_resize(x, 14, 14).backward(g)
    assert torch.equal(x.grad, ops.mask_resize_backward_nchw(g, 21, 21))

    fe = _cuda(rng.normal(size=(5, 8, 14, 14)).astype(np.float32)).requires_grad_()
    mk = _cuda(rng.uniform(size=(5, 1, 14, 14)).astype(np.float32)).requires_grad_()
    g = _cuda(rng.normal(size=(5, 8, 14, 14)).astype(np.float32))
    A.mask_pool(fe, mk).backward(g)
    wf, wm = ops.mask_pool_backward_nchw(fe.detach(), mk.detach(), g)
    assert torch.equal(fe.grad, wf) and torch.equal(mk.grad, wm)

    f = _cuda(feat).requires_grad_()
    out = A.roi_pool(f, _cuda(rois), 7, 7)
    g = torch.randn_like(out)
    out.backward(g)
    arg = torch.empty(out.shape, dtype=torch.int32, device="cuda")
    ops.roi_pool_nchw(_cuda(feat), _cuda(rois), 7, 7, argmax=arg)
    assert torch.equal(f.grad, ops.roi_pool_backward_nchw(g, arg, feat.shape, _cuda(rois), 7, 7))
