"""TRAIN phase of StageBridgeLayer and MaskLayer on the device (mnc_stage_bridge_train*,
mnc_mask_layer_train*) against the reference's fixtures and the numpy oracle: indices, labels,
weights, mask targets and copied / clamped diffs exact, values derived from exp / log within
4 float32 ulp; determinism, graph replay, NULL diffs, argument errors, the TRAIN mirrors and the
differentiable cascade into ROIWarping."""
import numpy as np
import pytest
import torch

from oracle import oracle_train as T
from tests.test_oracle_train_bridge import fixture, TOPS

pytestmark = pytest.mark.gpu
EXACT = ("labels", "mask_weight", "gt_mask_info", "bbox_inside_weights", "bbox_outside_weights")


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _ulp(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a - b) / np.spacing(np.maximum(np.abs(a), np.abs(b)).astype(np.float32) + np.float32(1e-30))


def _device(f, precomputed, clip):
    from mnc_b200 import ops
    out = ops.stage_bridge_train(
        _cuda(f["rois"]), _cuda(f["bbox_pred"]), _cuda(f["seg_cls_prob"]), _cuda(f["gt_boxes"]),
        _cuda(f["gt_masks"].astype(np.float32)), _cuda(f["im_info"]), _cuda(f["mask_info"]),
        means=T.BBOX_NORMALIZE_MEANS if precomputed else None,
        stds=T.BBOX_NORMALIZE_STDS if precomputed else None)
    rd, bd = ops.stage_bridge_train_backward(_cuda(f["top_diff"]), out["state"], _cuda(f["rois"]),
                                             _cuda(f["bbox_pred"]), f["gt_boxes"].shape[0], clip)
    return out, rd, bd


def _compare(out, rd, bd, want, wrd, wbd, f):
    """Exact where the reference copies, counts or decides; 4 ulp for exp / log values."""
    n = f["rois"].shape[0]
    K = n + f["gt_boxes"].shape[0]
    st = out["state"].cpu().numpy()
    keep = st[:K]
    assert np.array_equal(keep, want["keep_inds"])
    assert np.array_equal(st[K:2 * K][keep], np.arange(K))
    assert np.array_equal(st[2 * K:2 * K + n], want["reg_labels"])
    assert np.array_equal(np.where(st[2 * K + n:2 * K + 2 * n])[0], want["clip_keep"][want["clip_keep"] < n])
    assert st[-1] == int(want["mask_weight"][:, 0, 0, 0].sum())
    got = {k: out[k].cpu().numpy().reshape(want[k].shape) for k in TOPS}
    for k in EXACT:
        assert np.array_equal(got[k], want[k]), k
    assert np.array_equal(got["mask_targets"], want["mask_targets"])
    assert np.all(_ulp(got["rois"], want["rois"]) <= 4)
    assert np.array_equal(got["bbox_targets"] != 0, want["bbox_targets"] != 0)
    assert np.all(_ulp(got["bbox_targets"], want["bbox_targets"]) <= 4)
    rd, bd = rd.cpu().numpy(), bd.cpu().numpy()
    assert np.array_equal(rd[:, :3], wrd[:, :3])               # column 0 and the two copies
    assert np.all(_ulp(rd[:, 3:], wrd[:, 3:]) <= 4)
    assert np.array_equal(bd != 0, wbd != 0)
    clamped = np.abs(wbd) == np.float32(1.0 / 512)
    assert np.array_equal(bd[clamped], wbd[clamped])
    assert np.all(_ulp(bd, wbd) <= 4)
    return got


def _mask_layer(pred, gt_masks, info):
    from mnc_b200 import ops
    return ops.mask_layer_train(_cuda(pred), _cuda(gt_masks.astype(np.float32)), _cuda(info))


@pytest.mark.parametrize("name", ("A", "B", "C"))
def test_matches_reference_fixtures(name):
    f = fixture(name)
    precomputed, use_clip, clip_base, C = (int(v) for v in f["cfg"])
    clip = 1.0 / clip_base if use_clip else 0.0
    out, rd, bd = _device(f, precomputed, clip)
    want = {k: f["top_" + k] for k in TOPS}
    want.update(keep_inds=f["keep_inds"], reg_labels=f["reg_labels"], clip_keep=f["clip_keep"])
    _compare(out, rd, bd, want, f["rois_diff"], f["bbox_pred_diff"], f)
    labels = _mask_layer(f["ml_pred"], f["gt_masks"], f["ml_info"])
    assert np.array_equal(labels.cpu().numpy(), f["ml_labels"].reshape(-1))
    from mnc_b200 import ops
    g = ops.mask_layer_train_backward(_cuda(f["ml_top_diff"]), labels).cpu().numpy()
    assert np.array_equal(g, f["ml_bottom_diff"].reshape(g.shape))


def test_random_cases_match_oracle():
    near = 0
    for seed in range(24):
        kw = dict(H=600, W=1000, im_scale=1.6, n=64, G=3 + seed % 18) if seed % 2 else \
            dict(H=480, W=640, im_scale=1.0 + 0.05 * seed, n=32 + seed, G=2 + seed % 5)
        case = T.make_case(100 + seed, **kw)
        pre = seed % 3 != 0
        want = T.stage_bridge_forward(**case, num_classes=21, normalize=pre)
        K = want["rois"].shape[0]
        td = np.random.default_rng(seed).normal(0, 1e-5, (K, 5)).astype(np.float32)
        clip = 1.0 / 512 if seed % 4 else 0.0
        wrd, wbd = T.stage_bridge_backward(td, want, case["rois"], case["bbox_pred"], clip)
        f = dict(case, top_diff=td)
        out, rd, bd = _device(f, pre, clip)
        tv = T.target_values(case, want)
        near += int(np.sum(np.abs(tv - 0.4) < 1e-6))
        got = out["mask_targets"].cpu().numpy()
        diff = got != want["mask_targets"]
        assert diff.sum() <= near, (seed, diff.sum(), near)
        want["mask_targets"] = got if diff.sum() else want["mask_targets"]
        _compare(out, rd, bd, want, wrd, wbd, case)
        pred = T.mask_predictions(seed, want["mask_targets"], want["gt_mask_info"])
        labels = _mask_layer(pred, case["gt_masks"], want["gt_mask_info"]).cpu().numpy()
        rv = T.resize_values(pred, want["gt_mask_info"])
        wl = T.mask_layer_forward(pred, case["gt_masks"], want["gt_mask_info"]).reshape(-1)
        if np.abs(rv - 0.4).min(initial=1) >= 1e-6:
            assert np.array_equal(labels, wl), seed
    print("random-case mask samples within 1e-6 of BINARIZE_THRESH: %d" % near)


def _case_tensors(seed=3):
    case = T.make_case(seed)
    return case, [_cuda(case[k]) for k in ("rois", "bbox_pred", "seg_cls_prob", "gt_boxes")] + \
        [_cuda(case["gt_masks"].astype(np.float32)), _cuda(case["im_info"]), _cuda(case["mask_info"])]


def test_deterministic_and_graph_replay():
    from mnc_b200 import ops
    case, t = _case_tensors()
    G = case["gt_boxes"].shape[0]
    K = case["rois"].shape[0] + G
    td = _cuda(np.random.default_rng(0).normal(0, 1e-5, (K, 5)).astype(np.float32))
    mtd = torch.randn(K, 1, 21, 21, device="cuda")

    def step():
        o = ops.stage_bridge_train(*t, means=T.BBOX_NORMALIZE_MEANS, stds=T.BBOX_NORMALIZE_STDS)
        rd, bd = ops.stage_bridge_train_backward(td, o["state"], t[0], t[1], G, 1.0 / 512)
        lab = ops.mask_layer_train(o["mask_targets"], t[4], o["gt_mask_info"])
        md = ops.mask_layer_train_backward(mtd, lab)
        return [o[k] for k in TOPS] + [o["state"], rd, bd, lab, md]
    a = [x.clone() for x in step()]
    b = step()
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        c = step()
    g.replay()
    g.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(a, c))
    assert a[-2].gt(0).any()                      # the targets as predictions keep their labels


def test_null_diffs_and_argument_errors():
    from mnc_b200 import ops
    from mnc_b200._lib import MncError
    case, t = _case_tensors()
    G = case["gt_boxes"].shape[0]
    o = ops.stage_bridge_train(*t)
    K = o["rois"].shape[0]
    td = torch.randn(K, 5, device="cuda") * 1e-5
    rd, bd = ops.stage_bridge_train_backward(td, o["state"], t[0], t[1], G, 1.0 / 512)
    r_only, none = ops.stage_bridge_train_backward(td, o["state"], t[0], t[1], G, 1.0 / 512, want_bbox=False)
    none2, b_only = ops.stage_bridge_train_backward(td, o["state"], t[0], t[1], G, 1.0 / 512, want_rois=False)
    assert none is None and none2 is None
    assert torch.equal(r_only, rd) and torch.equal(b_only, bd)
    with pytest.raises(MncError):                 # G = 0
        ops.stage_bridge_train(t[0], t[1], t[2], t[3][:0], t[4][:0], t[5], t[6][:0])
    with pytest.raises(MncError):
        ops.stage_bridge_train_backward(td, o["state"], t[0], t[1], G, -1.0)
    with pytest.raises(MncError):                 # no gt masks
        ops.mask_layer_train(o["mask_targets"], t[4][:0], o["gt_mask_info"])


def test_train_mirrors_propagate_down_and_zeroing():
    import mnc_b200.lib as lib
    lib.install()
    from caffe import Blob, TRAIN, TEST
    from mnc_config import cfg
    from pylayer.stage_bridge_layer import StageBridgeLayer
    from pylayer.mask_layer import MaskLayer
    f = fixture("A")

    def blob(a):
        b = Blob(*a.shape)
        b.data[...] = a
        return b
    bottom = [blob(f[k]) for k in ("rois", "bbox_pred", "seg_cls_prob", "gt_boxes")] + \
        [blob(f["gt_masks"].astype(np.float32)), blob(f["im_info"][None]), blob(f["mask_info"].astype(np.float32))]
    top = [Blob() for _ in range(8)]
    layer = StageBridgeLayer("{ 'feat_stride': 16, 'use_clip': 1, 'clip_base': 512, 'num_classes': 21}", TRAIN)
    old = cfg.TRAIN.BBOX_NORMALIZE_TARGETS_PRECOMPUTED
    cfg.TRAIN.BBOX_NORMALIZE_TARGETS_PRECOMPUTED = True
    try:
        layer.setup(bottom, top)
        layer.forward(bottom, top)
    finally:
        cfg.TRAIN.BBOX_NORMALIZE_TARGETS_PRECOMPUTED = old
    for i, k in enumerate(TOPS):
        assert top[i].data.shape == f["top_" + k].shape, k
    assert np.array_equal(top[1].data, f["top_labels"])
    top[0].diff = f["top_diff"].copy()
    for b in bottom[:2]:
        b.diff = np.full(b.data.shape, 7, np.float32)
    layer.backward(top, [False, True], bottom)
    assert np.all(bottom[0].diff == 7)                   # not propagated: untouched
    assert np.array_equal(bottom[1].diff != 0, f["bbox_pred_diff"] != 0)
    layer.backward(top, [True, False], bottom)
    assert np.array_equal(bottom[0].diff[:, :3], f["rois_diff"][:, :3])

    ml = MaskLayer("", TRAIN)
    mb = [blob(f["ml_pred"]), blob(f["gt_masks"].astype(np.float32)), blob(f["ml_info"])]
    mt = [Blob(), Blob()]
    ml.setup(mb, mt)
    ml.forward(mb, mt)
    assert np.array_equal(mt[1].data, f["ml_labels"])
    mt[0].diff = f["ml_top_diff"].copy()
    mb[0].diff = np.full(mb[0].data.shape, 7, np.float32)
    ml.backward(mt, [False], mb)
    assert np.all(mb[0].diff == 7)
    ml.backward(mt, [True], mb)
    assert np.array_equal(mb[0].diff, f["ml_bottom_diff"].reshape(mb[0].diff.shape))
    # TEST phase: reshape only, and backward still raises
    mt2 = [Blob()]
    tl = MaskLayer("", TEST)
    tl.setup(mb[:1], mt2)
    tl.forward(mb[:1], mt2)
    assert mt2[0].data.shape == (mb[0].data.shape[0], 1, 21, 21)
    with pytest.raises(NotImplementedError):
        tl.backward(mt2, [True], mb[:1])


def test_differentiable_cascade_into_roi_warp():
    from mnc_b200 import autograd
    from oracle import oracle_backward as OB
    f = fixture("A")
    rng = np.random.default_rng(5)
    feat = rng.normal(size=(1, 16, 38, 63)).astype(np.float32)
    rois = _cuda(f["rois"]).requires_grad_()
    bbox_pred = _cuda(f["bbox_pred"]).requires_grad_()
    outs = autograd.stage_bridge_train(
        rois, bbox_pred, _cuda(f["seg_cls_prob"]), _cuda(f["gt_boxes"]),
        _cuda(f["gt_masks"].astype(np.float32)), _cuda(f["im_info"]), _cuda(f["mask_info"]),
        means=T.BBOX_NORMALIZE_MEANS, stds=T.BBOX_NORMALIZE_STDS, clip_thresh=1.0 / 512)
    rois_ext = outs[0]
    assert not any(o.requires_grad for o in outs[1:])
    out = autograd.roi_warp(_cuda(feat), rois_ext, 28, 28, 0.0625)
    g = rng.normal(size=tuple(out.shape)).astype(np.float32) * np.float32(1e-3)
    (out * _cuda(g)).sum().backward()
    # oracle: ROIWarping's coordinate gradient, then StageBridge's backward
    _, coord, mag = OB.roi_warp_backward(feat, rois_ext.detach().cpu().numpy(), g, 28, 28, want_abs=True)
    state = T.stage_bridge_forward(f["rois"], f["bbox_pred"], f["seg_cls_prob"], f["gt_boxes"],
                                   f["gt_masks"].astype(np.float32), f["im_info"], f["mask_info"], 21)
    wrd, wbd = T.stage_bridge_backward(coord, state, f["rois"], f["bbox_pred"], 1.0 / 512)
    # bounds: push the coordinate tolerance 1e-5 * mag through the same products
    rmag, bmag = T.stage_bridge_backward(mag, state, f["rois"], f["bbox_pred"], 0.0)
    rg, bg = rois.grad.cpu().numpy(), bbox_pred.grad.cpu().numpy()
    assert np.all(np.abs(rg - wrd) <= 1e-5 * np.abs(rmag) + 1e-30)
    clamped = np.abs(wbd) == np.float32(1.0 / 512)
    assert np.array_equal(bg[clamped], wbd[clamped])
    assert np.all(np.abs(bg - wbd)[~clamped] <= 1e-5 * np.abs(bmag)[~clamped] + 1e-30)
    assert np.abs(bg).max() > 0 and np.abs(rg).max() > 0
