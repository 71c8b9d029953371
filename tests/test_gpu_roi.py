"""ROIWarping / MaskResize / MaskPooling (layer contract, fp32 NCHW) vs the C oracle: bit-exact,
since the kernels use the same un-fused fp32 operation order; fused split-bf16 forms: 1e-3 rel."""
import numpy as np
import pytest
import torch

from tests import roi_shapes as RS
from tests import util

pytestmark = pytest.mark.gpu


def _rois(n, seed, W=1000, H=600, extra=True):
    b = util.random_boxes(n, seed, width=W, height=H)
    rois = np.hstack([np.zeros((n, 1), np.float32), b])
    if extra and n >= 8:
        rois[0, 1:] = [0, 0, W - 1, H - 1]            # whole image
        rois[1, 1:] = [100, 100, 100, 100]            # degenerate: every cell samples one point
        rois[2, 1:] = [-300, -200, 40, 30]            # partly off the map (negative start)
        rois[3, 1:] = [W + 200, H + 300, W + 400, H + 500]  # entirely outside -> zeros
        rois[4, 1:] = [W - 20, H - 20, W + 300, H + 300]    # runs past the far edge
        rois[5, 1:] = [8, 8, 23.9, 24.1]              # round-half cases at scale 1/16
        rois[6, 1:] = [500, 300, 400, 200]            # malformed (end < start) -> width forced 0
    return rois.astype(np.float32)


def table_params(pool_only=False):
    """(case, size) parameters, size = (ph, pw), over the shape table of tests/roi_shapes.py."""
    return [pytest.param(n, (ph, pw), id=RS.size_id(n, ph, pw)) for n, ph, pw in RS.sizes(pool_only)]


@pytest.mark.parametrize("case,size", [pytest.param(None, (P, P), id=str(P)) for P in (28, 14, 7)] + table_params())
def test_roi_warp_nchw_bit_exact(case, size):
    from oracle import oracle as O
    from mnc_b200 import ops
    ph, pw = size
    if case is None:
        rng = np.random.default_rng(7)
        feat = np.maximum(rng.normal(size=(2, 40, 38, 63)), 0).astype(np.float32)
        rois = _rois(64, 8)
        rois[10:20, 0] = 1  # second image of the batch (roi_warping_layer.cu:79,96)
        ss = 0.0625
    else:
        feat, rois, ss = RS.feat(case), RS.rois(case), RS.BY_NAME[case].scale
    want = O.roi_warp(feat, rois, ph, pw, ss)
    got = ops.roi_warp_nchw(torch.from_numpy(feat).cuda(), torch.from_numpy(rois).cuda(), ph, pw, ss).cpu().numpy()
    assert np.array_equal(got, want)
    for r in ([3] if case is None else RS.outside_rows(case)):
        assert np.abs(want[r]).max() == 0.0
    assert np.abs(want).max() > 0


def test_roi_warp_layer_mirror_contract():
    import mnc_b200.lib as L
    L.install()
    import caffe
    from caffe.layers import ROIWarpingLayer
    from oracle import oracle as O
    rng = np.random.default_rng(1)
    feat, rois = caffe.Blob(), caffe.Blob()
    feat.data = rng.normal(size=(1, 16, 20, 30)).astype(np.float32)
    rois.data = _rois(12, 2, W=480, H=320)
    top = caffe.Blob()
    layer = ROIWarpingLayer(dict(roi_warping_param=dict(pooled_w=14, pooled_h=14, spatial_scale=0.0625)))
    layer.LayerSetUp([feat, rois], [top])
    layer.Forward([feat, rois], [top])
    assert top.shape == (12, 16, 14, 14)
    assert np.array_equal(top.data, O.roi_warp(feat.data, rois.data, 14, 14))
    with pytest.raises(NotImplementedError):
        layer.Forward_cpu([feat, rois], [top])
    with pytest.raises(ValueError):
        ROIWarpingLayer(dict(roi_warping_param=dict(pooled_w=0, pooled_h=14))).LayerSetUp([feat, rois], [top])


def test_mask_resize_and_pool_bit_exact():
    from oracle import oracle as O
    from mnc_b200 import ops
    rng = np.random.default_rng(9)
    masks = rng.uniform(size=(50, 1, 21, 21)).astype(np.float32)
    want = O.mask_resize(masks, 14, 14)
    got = ops.mask_resize_nchw(torch.from_numpy(masks).cuda(), 14, 14).cpu().numpy()
    assert np.array_equal(got, want)
    # Caffe's own test shape (test_mask_resize_layer.cpp: (4,1,21,21) -> 14x14), plus upsampling
    m2 = rng.normal(0, 10, size=(4, 1, 21, 21)).astype(np.float32)
    assert np.array_equal(ops.mask_resize_nchw(torch.from_numpy(m2).cuda(), 30, 17).cpu().numpy(),
                          O.mask_resize(m2, 30, 17))
    feat = rng.normal(size=(50, 24, 14, 14)).astype(np.float32)
    m14 = want
    got = ops.mask_pool_nchw(torch.from_numpy(feat).cuda(), torch.from_numpy(m14).cuda()).cpu().numpy()
    assert np.array_equal(got, O.mask_pool(feat, m14))
    # odd spatial size -> scalar kernel
    f2 = rng.normal(size=(3, 5, 7, 9)).astype(np.float32)
    k2 = rng.uniform(size=(3, 1, 7, 9)).astype(np.float32)
    assert np.array_equal(ops.mask_pool_nchw(torch.from_numpy(f2).cuda(), torch.from_numpy(k2).cuda()).cpu().numpy(),
                          O.mask_pool(f2, k2))
    with pytest.raises(ValueError):
        ops.mask_pool_nchw(torch.from_numpy(f2).cuda(), torch.from_numpy(k2[:, :, :6]).contiguous().cuda())
    # a blob larger than one grid-stride pass, through the vector kernel and, offset by one float
    # (a view: 4-byte aligned only), through the scalar one
    shape = RS.MASK_POOL["pool_64x512"]
    f3 = rng.normal(size=shape).astype(np.float32)
    k3 = rng.uniform(size=(shape[0], 1) + shape[2:]).astype(np.float32)
    want = O.mask_pool(f3, k3)
    d_k3 = torch.from_numpy(k3).cuda()
    assert np.array_equal(ops.mask_pool_nchw(torch.from_numpy(f3).cuda(), d_k3).cpu().numpy(), want)
    store = torch.empty(f3.size + 1, device="cuda")
    d_f3 = store[1:].view(shape)
    d_f3.copy_(torch.from_numpy(f3))
    assert d_f3.data_ptr() % 16 == 4
    assert np.array_equal(ops.mask_pool_nchw(d_f3, d_k3).cpu().numpy(), want)


@pytest.mark.parametrize("sub", [2, 1])
def test_fused_roi_warp_split(sub):
    """warp (+2x2 max) -> 14x14 and 7x7 on split NHWC == oracle warp + F.max_pool2d, on the same
    (hi+lo) feature values."""
    import torch.nn.functional as F
    from oracle import oracle as O
    from mnc_b200 import ops, dense
    rng = np.random.default_rng(3)
    C, H, W = 64, 38, 63
    feat = np.maximum(rng.normal(size=(2, C, H, W)), 0).astype(np.float32)
    fs = dense.split(torch.from_numpy(feat).cuda().permute(0, 2, 3, 1).contiguous())
    feat_q = dense.merge(fs).permute(0, 3, 1, 2).contiguous().cpu().numpy()  # what the kernel sees
    rois = _rois(40, 5)
    rois[20:, 0] = 1
    R = rois.shape[0]
    o14 = torch.zeros(2, R, 14, 14, C, dtype=torch.bfloat16, device="cuda")
    o7 = torch.zeros(2, R, 7, 7, C, dtype=torch.bfloat16, device="cuda")
    ops.roi_warp_split(dense.merge(fs).contiguous(), C, H, W, torch.from_numpy(rois).cuda(), sub, o14, o7)
    want28 = torch.from_numpy(O.roi_warp(feat_q, rois, 14 * sub, 14 * sub))
    want14 = F.max_pool2d(want28, 2, 2) if sub == 2 else want28
    want7 = F.max_pool2d(want14, 2, 2)
    got14 = dense.merge(o14).permute(0, 3, 1, 2).cpu()
    got7 = dense.merge(o7).permute(0, 3, 1, 2).cpu()
    # outputs are re-split to 16 mantissa bits: 2^-16 relative
    assert torch.allclose(got14, want14, rtol=3e-5, atol=1e-6)
    assert torch.allclose(got7, want7, rtol=3e-5, atol=1e-6)


def test_fused_sigmoid_resize_and_mask_pool_split():
    import torch.nn.functional as F
    from oracle import oracle as O
    from mnc_b200 import ops, dense
    rng = np.random.default_rng(4)
    R, C = 37, 64
    logits = rng.normal(0, 2, size=(R, 448)).astype(np.float32)
    mp, m14 = ops.sigmoid_mask_resize(torch.from_numpy(logits).cuda(), R)
    want_mp = torch.sigmoid(torch.from_numpy(logits[:, :441])).numpy().reshape(R, 1, 21, 21)
    assert util.rel_err(mp.cpu().numpy(), want_mp) < 1e-6
    # resize is bit-exact given the kernel's own sigmoid output
    assert np.array_equal(m14.cpu().numpy(), O.mask_resize(mp.cpu().numpy(), 14, 14))
    feat = np.maximum(rng.normal(size=(R, C, 14, 14)), 0).astype(np.float32)
    fs = dense.split(torch.from_numpy(feat).cuda().permute(0, 2, 3, 1).contiguous())
    feat_q = dense.merge(fs).permute(0, 3, 1, 2).contiguous().cpu().numpy()
    o7 = torch.zeros(2, R, 7, 7, C, dtype=torch.bfloat16, device="cuda")
    ops.mask_pool_split(fs, m14, R, C, o7)
    want = F.max_pool2d(torch.from_numpy(O.mask_pool(feat_q, m14.cpu().numpy())), 2, 2)
    assert torch.allclose(dense.merge(o7).permute(0, 3, 1, 2).cpu(), want, rtol=3e-5, atol=1e-6)
