"""Loss layers of the training net on the device (mnc_softmax_loss*, mnc_smooth_l1_loss*,
mnc_sigmoid_ce_loss*, mnc_accuracy) against the numpy oracle at the training shapes: the backward
arithmetic and SmoothL1 exact, values that exp / log enter within 4 float32 ulp per term, accuracy
exact; padded blobs with the device row count equal the trimmed blobs bit for bit; the 14 loss and
accuracy layers of one training step forward and backward in one CUDA graph, replay-stable and equal
to the layer mirrors' Backward_gpu."""
import numpy as np
import pytest
import torch

from oracle import oracle_loss as L

pytestmark = pytest.mark.gpu
F32 = np.float32
H, W, A = 38, 63, 9


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _np(t):
    return t.detach().cpu().numpy()


def _term_bound(terms, norm):
    """4 float32 ulp per term, over the normaliser, plus the final rounding."""
    t = np.abs(np.asarray(terms, np.float32))
    return 4 * float(np.spacing(t).sum()) / float(norm) + 1e-30


def _rng(seed):
    return np.random.default_rng(seed)


# ------------------------------------------------------------------ device == oracle
@pytest.mark.parametrize("shape,labels_hi,mode", [
    ((1, 2, A * H, W), 2, "VALID"),          # rpn_loss_cls
    ((67, 21), 21, "VALID"),                  # loss_cls / loss_seg_cls
    ((67, 21), 21, "FULL"), ((67, 21), 21, "BATCH_SIZE"), ((67, 21), 21, "NONE")])
def test_softmax_loss_matches_oracle(shape, labels_hi, mode):
    from mnc_b200 import ops
    r = _rng(sum(shape) + len(mode))
    x = (3 * r.standard_normal(shape)).astype(np.float32)
    lab_shape = (shape[0],) + tuple(shape[2:])
    lab = r.integers(-1, labels_hi, lab_shape).astype(np.float32)
    loss, prob = ops.softmax_loss(_cuda(x), _cuda(lab), -1, mode)
    want_loss, want_prob = L.softmax_loss(x, lab, -1, mode)
    p = _np(prob).reshape(want_prob.shape)
    assert np.all(np.abs(p - want_prob) <= 4 * np.spacing(np.maximum(p, want_prob)))
    # the loss from the device's own prob: only logf differs from the oracle
    lab_i = lab.astype(int).reshape(shape[0], -1)
    ok = lab_i >= 0
    pl = np.take_along_axis(p, np.clip(lab_i, 0, None)[:, None, :], 1)[:, 0]
    terms = np.where(ok, -L.logf(np.maximum(pl, L.FLT_MIN)), 0)
    norm = L.normalizer(mode, shape[0], lab_i.shape[1], int(ok.sum()))
    assert abs(float(_np(loss)) - float(want_loss)) <= _term_bound(terms, norm) + 4 * np.spacing(want_loss)
    # the backward from the device prob: bit-exact
    td = F32(0.75)
    d = ops.softmax_loss_backward(prob, _cuda(lab), _cuda(np.array(td)), -1, mode)
    assert np.array_equal(_np(d).reshape(p.shape), L.softmax_loss_backward(p, lab, td, -1, mode))


@pytest.mark.parametrize("shape,sigma", [((1, 4 * A, H, W), 3.0), ((67, 84), 1.0)])
def test_smooth_l1_loss_matches_oracle_bit_for_bit(shape, sigma):
    from mnc_b200 import ops
    r = _rng(int(sigma) + shape[0])
    p = r.standard_normal(shape).astype(np.float32)
    t = r.standard_normal(shape).astype(np.float32)
    # values on the double threshold and on the kink
    p.flat[:4] = [1 / sigma ** 2, -1 / sigma ** 2, 0.0, 2.0]
    t.flat[:4] = 0
    wi = r.integers(0, 2, shape).astype(np.float32)
    wo = (wi / 256).astype(np.float32)
    args = [_cuda(a) for a in (p, t, wi, wo)]
    loss = ops.smooth_l1_loss(*args, sigma=sigma)
    assert _np(loss) == L.smooth_l1_loss(p, t, wi, wo, sigma)
    d = ops.smooth_l1_loss_backward(*args, sigma=sigma, top_diff=_cuda(np.array(1.0)))
    assert np.array_equal(_np(d), L.smooth_l1_loss_backward(p, t, wi, wo, sigma, 1.0))
    # no weights
    assert _np(ops.smooth_l1_loss(args[0], args[1], sigma=sigma)) == L.smooth_l1_loss(p, t, sigma=sigma)


@pytest.mark.parametrize("weighted", [True, False])
def test_sigmoid_ce_loss_matches_oracle(weighted):
    from mnc_b200 import ops
    r = _rng(7 + weighted)
    shape = (67, 1, 21, 21)
    x = (4 * r.standard_normal(shape)).astype(np.float32)
    x.flat[:3] = [0.0, -0.0, 88.0]
    t = r.integers(0, 2, shape).astype(np.float32)
    w = r.integers(0, 2, shape).astype(np.float32) if weighted else None
    loss = ops.sigmoid_ce_loss(_cuda(x), _cuda(t), None if w is None else _cuda(w))
    want = L.sigmoid_ce_loss(x, t, w)
    terms = L.sigmoid_ce_terms(x, t, w)
    norm = L.fixed_sum(w) if weighted else shape[0]
    assert abs(float(_np(loss)) - float(want)) <= _term_bound(terms, norm) + 4 * np.spacing(want)
    td = F32(2.0)
    d = _np(ops.sigmoid_ce_loss_backward(_cuda(x), _cuda(t), None if w is None else _cuda(w),
                                         _cuda(np.array(td))))
    wd = L.sigmoid_ce_loss_backward(x, t, w, td)
    scale = float(td) / float(norm)
    assert np.all(np.abs(d - wd) <= 4 * 2.0 ** -24 * scale + 4 * np.spacing(np.abs(wd)))
    if weighted:
        assert np.array_equal(d == 0, wd == 0)


def test_sigmoid_ce_zero_weight_sum_leaves_loss_untouched():
    from mnc_b200 import ops
    x = _cuda(np.ones((3, 4)))
    out = _cuda(np.array(5.5))
    ops.sigmoid_ce_loss(x, x, _cuda(np.zeros((3, 4))), out=out)
    assert out.item() == 5.5
    assert ops.sigmoid_ce_loss(x, x, _cuda(np.zeros((3, 4)))).item() == 0


@pytest.mark.parametrize("top_k,ignore", [(1, None), (1, -1), (3, None)])
def test_accuracy_matches_oracle_with_ties(top_k, ignore):
    from mnc_b200 import ops
    r = _rng(top_k)
    x = r.integers(0, 4, (67, 21)).astype(np.float32)      # many tied scores
    lab = r.integers(-1, 21, 67).astype(np.float32)
    got = _np(ops.accuracy(_cuda(x), _cuda(lab), top_k, ignore))
    assert got == L.accuracy(x, lab, top_k, ignore)
    x4 = r.standard_normal((1, 2, A * H, W)).astype(np.float32)
    l4 = r.integers(-1, 2, (1, A * H, W)).astype(np.float32)
    assert _np(ops.accuracy(_cuda(x4), _cuda(l4), 1, ignore)) == L.accuracy(x4, l4, 1, ignore)


def test_out_of_range_labels_stay_in_bounds_and_argument_errors():
    """Labels outside [0, C) that are not ignored: counted, no loss term, no -1 in the diff."""
    from mnc_b200 import ops, _lib
    x = _cuda(np.zeros((4, 3)))
    lab_np = np.array([0, 3, 7, -5], np.float32)
    lab = _cuda(lab_np)
    loss, prob = ops.softmax_loss(x, lab, None, "VALID")
    want, _ = L.softmax_loss(np.zeros((4, 3), np.float32), lab_np)
    assert abs(float(_np(loss)) - float(want)) <= 4 * np.spacing(want)
    d = _np(ops.softmax_loss_backward(prob, lab, None, None, "VALID"))
    assert np.array_equal(d[1:], _np(prob)[1:] * (F32(1) / F32(4)))
    with pytest.raises(ValueError):
        ops.softmax_loss(x, _cuda(np.zeros(5)))
    with pytest.raises(ValueError):
        ops.smooth_l1_loss(x, x, x, None)
    with pytest.raises(ValueError):
        ops.accuracy(x, _cuda(np.zeros(4)), top_k=4)
    bad_mode = _lib.lib.mnc_softmax_loss(_lib.ptr(x), _lib.ptr(lab), 4, 3, 1, None, 0, 0, 7,
                                         _lib.ptr(prob), _lib.ptr(loss), _lib.cur_stream())
    assert bad_mode == 1                                     # MNC_ERR_ARG


# ------------------------------------------------------------------ the real targets, padded
def _targets():
    """One training step's targets from the device layers: proposal_train -> proposal_target
    (n_valid = count) -> anchor_target, and mask_layer_train on the padded stage-1 rows."""
    from mnc_b200 import ops
    from oracle import oracle_train as T
    from tests.test_gpu_rpn_train import _chain_inputs, _keys
    f, (prob, deltas, info) = _chain_inputs()
    gt, gm, mi = _cuda(f["gt_boxes"]), _cuda(f["gt_masks"].astype(np.float32)), \
        torch.from_numpy(np.ascontiguousarray(f["mask_info"])).cuda()
    rois, index, count, _ = ops.proposal_train(prob, deltas, info, H, W)
    o = ops.proposal_target(rois, index, gt, gm, mi, info, _keys(f["keys"]), n_valid=count,
                            means=T.BBOX_NORMALIZE_MEANS, stds=T.BBOX_NORMALIZE_STDS)
    at = ops.anchor_target(H, W, gt, info, _keys(f["anchor_keys"]), o["fg_inds"], o["bg_inds"],
                           o["counts"])
    kmax = o["labels"].shape[0]
    mp = torch.rand(kmax, 21, 21, device="cuda", generator=torch.Generator("cuda").manual_seed(3))
    seg = ops.mask_layer_train(mp, gm, o["gt_masks_info"])
    return o, at, seg


def _preds(kmax, k2, seed=0):
    g = torch.Generator("cuda").manual_seed(seed)
    n = lambda *s: torch.randn(*s, device="cuda", generator=g)
    return {"rpn_cls": n(1, 2, A * H, W), "rpn_bbox": n(1, 4 * A, H, W) * 0.3,
            "cls": n(kmax, 21), "seg_cls": n(kmax, 21), "bbox": n(kmax, 84) * 0.3,
            "mask": n(kmax, 1, 21, 21) * 3,
            "cls_ext": n(k2, 21), "seg_cls_ext": n(k2, 21), "bbox_ext": n(k2, 84) * 0.3,
            "mask_ext": n(k2, 1, 21, 21) * 3}


def _ext_targets(k2, seed=1):
    r = _rng(seed)
    return {"labels": _cuda(r.integers(-1, 21, k2)), "seg_labels": _cuda(r.integers(0, 21, k2)),
            "bbox_targets": _cuda(r.standard_normal((k2, 84))),
            "bbox_in": _cuda(r.integers(0, 2, (k2, 84))), "bbox_out": _cuda(r.integers(0, 2, (k2, 84))),
            "mask_targets": _cuda(r.integers(0, 2, (k2, 1, 21, 21))),
            "mask_weight": _cuda(np.repeat(r.integers(0, 2, (k2, 1, 1, 1)), 441).reshape(k2, 1, 21, 21))}


def test_padded_with_device_count_equals_trimmed():
    from mnc_b200 import ops
    o, _, seg = _targets()
    K = int(o["counts"][0])
    kmax = o["labels"].shape[0]
    assert 0 < K <= kmax
    n = o["counts"][:1]
    p = _preds(kmax, 1)
    nz = lambda t: t[K:].abs().max().item() if t.shape[0] > K else 0.0
    one = _cuda(np.array(1.5))
    for scores, labels in ((p["cls"], o["labels"]), (p["seg_cls"], seg)):
        a, pa = ops.softmax_loss(scores, labels, -1, n_valid=n)
        b, pb = ops.softmax_loss(scores[:K], labels[:K], -1)
        assert torch.equal(a, b) and torch.equal(pa[:K], pb) and nz(pa) == 0
        da = ops.softmax_loss_backward(pa, labels, one, -1, n_valid=n)
        db = ops.softmax_loss_backward(pb, labels[:K], one, -1)
        assert torch.equal(da[:K], db) and nz(da) == 0
        assert torch.equal(ops.accuracy(scores, labels, n_valid=n), ops.accuracy(scores[:K], labels[:K]))
    bb = [p["bbox"], o["bbox_targets"], o["bbox_inside_weights"], o["bbox_outside_weights"]]
    a = ops.smooth_l1_loss(*bb, n_valid=n)
    assert torch.equal(a, ops.smooth_l1_loss(*[t[:K] for t in bb]))
    da = ops.smooth_l1_loss_backward(*bb, top_diff=one, n_valid=n)
    assert torch.equal(da[:K], ops.smooth_l1_loss_backward(*[t[:K] for t in bb], top_diff=one))
    assert nz(da) == 0
    mk = [p["mask"], o["mask_targets"], o["mask_weight"]]
    a = ops.sigmoid_ce_loss(*mk, n_valid=n)
    assert torch.equal(a, ops.sigmoid_ce_loss(*[t[:K] for t in mk]))
    da = ops.sigmoid_ce_loss_backward(*mk, top_diff=one, n_valid=n)
    assert torch.equal(da[:K], ops.sigmoid_ce_loss_backward(*[t[:K] for t in mk], top_diff=one))
    assert nz(da) == 0


# ------------------------------------------------------------------ one training step in a graph
def _step(p, o, at, seg, ext):
    """The 14 loss / accuracy layers of train.prototxt, forward and backward, with its loss
    weights passed as grad_outputs (no PyTorch arithmetic)."""
    from mnc_b200 import autograd as AG
    n = o["counts"][:1]
    losses = [
        AG.softmax_loss(p["rpn_cls"], at[0]),
        AG.smooth_l1_loss(p["rpn_bbox"], at[1], at[2], at[3], sigma=3.0),
        AG.sigmoid_ce_loss(p["mask"], o["mask_targets"], o["mask_weight"], n_valid=n),
        AG.softmax_loss(p["cls"], o["labels"], n_valid=n),
        AG.softmax_loss(p["seg_cls"], seg, n_valid=n),
        AG.smooth_l1_loss(p["bbox"], o["bbox_targets"], o["bbox_inside_weights"],
                          o["bbox_outside_weights"], n_valid=n),
        AG.sigmoid_ce_loss(p["mask_ext"], ext["mask_targets"], ext["mask_weight"]),
        AG.softmax_loss(p["cls_ext"], ext["labels"]),
        AG.softmax_loss(p["seg_cls_ext"], ext["seg_labels"]),
        AG.smooth_l1_loss(p["bbox_ext"], ext["bbox_targets"], ext["bbox_in"], ext["bbox_out"]),
    ]
    accs = [AG.accuracy(p["cls"], o["labels"], n_valid=n), AG.accuracy(p["seg_cls"], seg, n_valid=n),
            AG.accuracy(p["cls_ext"], ext["labels"]), AG.accuracy(p["seg_cls_ext"], ext["seg_labels"])]
    keys = ["rpn_cls", "rpn_bbox", "mask", "cls", "seg_cls", "bbox", "mask_ext", "cls_ext",
            "seg_cls_ext", "bbox_ext"]
    weights = [torch.full((), w, device="cuda") for w in (1, 1, 2, 1, 1, 1, 2, 1, 1, 1)]
    grads = torch.autograd.grad(losses, [p[k] for k in keys], weights)
    return losses + accs + list(grads)


def test_training_step_in_a_cuda_graph_equals_the_mirrors():
    from mnc_b200.lib.caffe import Blob
    from mnc_b200.lib.caffe import layers as LY
    o, at, seg = _targets()
    kmax = o["labels"].shape[0]
    k2 = 70
    p = {k: v.requires_grad_() for k, v in _preds(kmax, k2).items()}
    ext = _ext_targets(k2)
    a = [t.detach().clone() for t in _step(p, o, at, seg, ext)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _step(p, o, at, seg, ext)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        c = _step(p, o, at, seg, ext)
    g.replay()
    torch.cuda.synchronize()
    first = [t.detach().clone() for t in c]
    g.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(first, c))
    assert all(torch.equal(x, y) for x, y in zip(a, c))

    # the layer mirrors on host blobs trimmed to K rows
    K = int(o["counts"][0])

    def blob(t, rows=None):
        b = Blob()
        b.data = _np(t if rows is None else t[:rows]).astype(np.float32).copy()
        return b

    def run(layer_cls, param, bottoms, n_diff=1):
        top = [Blob()]
        layer = layer_cls(param)
        layer.LayerSetUp(bottoms, top)
        layer.Forward(bottoms, top)
        if layer_cls is LY.AccuracyLayer:
            return top[0].data, None
        layer.Backward(top, [True] + [False] * (len(bottoms) - 1), bottoms)
        return top[0].data, bottoms[0].diff

    soft = {"loss_param": {"ignore_label": -1, "normalize": True}}
    cases = [
        (LY.SoftmaxWithLossLayer, soft, [blob(p["rpn_cls"]), blob(at[0])], None, 1),
        (LY.SmoothL1LossLayer, {"smooth_l1_loss_param": {"sigma": 3.0}},
         [blob(p["rpn_bbox"])] + [blob(t) for t in at[1:]], None, 1),
        (LY.SigmoidCrossEntropyLossLayer, {"loss_weight": 2},
         [blob(p["mask"], K), blob(o["mask_targets"], K), blob(o["mask_weight"], K)], K, 2),
        (LY.SoftmaxWithLossLayer, soft, [blob(p["cls"], K), blob(o["labels"], K)], K, 1),
        (LY.SoftmaxWithLossLayer, soft, [blob(p["seg_cls"], K), blob(seg, K)], K, 1),
        (LY.SmoothL1LossLayer, {}, [blob(p["bbox"], K)] + [blob(o[k], K) for k in (
            "bbox_targets", "bbox_inside_weights", "bbox_outside_weights")], K, 1),
        (LY.SigmoidCrossEntropyLossLayer, {"loss_weight": 2},
         [blob(p["mask_ext"]), blob(ext["mask_targets"]), blob(ext["mask_weight"])], None, 2),
        (LY.SoftmaxWithLossLayer, soft, [blob(p["cls_ext"]), blob(ext["labels"])], None, 1),
        (LY.SoftmaxWithLossLayer, soft, [blob(p["seg_cls_ext"]), blob(ext["seg_labels"])], None, 1),
        (LY.SmoothL1LossLayer, {}, [blob(p["bbox_ext"])] + [blob(ext[k]) for k in (
            "bbox_targets", "bbox_in", "bbox_out")], None, 1),
    ]
    for i, (cls, param, bottoms, rows, _) in enumerate(cases):
        loss, diff = run(cls, param, bottoms)
        assert np.array_equal(loss, _np(c[i])), i
        grad = _np(c[14 + i])
        n = grad.shape[0] if rows is None else rows
        assert np.array_equal(diff.reshape(grad[:n].shape), grad[:n]), i
        assert not grad[n:].any(), i
    acc = [(p["cls"], o["labels"], K), (p["seg_cls"], seg, K), (p["cls_ext"], ext["labels"], None),
           (p["seg_cls_ext"], ext["seg_labels"], None)]
    for j, (sc, lab, rows) in enumerate(acc):
        val, _ = run(LY.AccuracyLayer, {}, [blob(sc, rows), blob(lab, rows)])
        assert np.array_equal(val, _np(c[10 + j])), j
        assert val == L.accuracy(_np(sc)[:rows], _np(lab)[:rows])
    assert all(float(_np(c[i])) > 0 for i in range(10))


def test_mirror_checks():
    from mnc_b200.lib.caffe import Blob
    from mnc_b200.lib.caffe import layers as LY
    b = [Blob(2, 4), Blob(2, 4), Blob(2, 4)]
    with pytest.raises(ValueError):
        LY.SmoothL1LossLayer({}).LayerSetUp(b, [Blob()])
    layer = LY.SoftmaxWithLossLayer({"loss_param": {"ignore_label": -1}})
    bottoms, top = [Blob(2, 4), Blob(2)], [Blob()]
    layer.LayerSetUp(bottoms, top)
    layer.Forward(bottoms, top)
    with pytest.raises(ValueError):
        layer.Backward(top, [True, True], bottoms)
    with pytest.raises(ValueError):
        LY.SigmoidCrossEntropyLossLayer({}).Reshape([Blob(2, 4), Blob(2, 3)], [Blob()])
    sce = LY.SigmoidCrossEntropyLossLayer({})
    bottoms, top = [Blob(2, 4), Blob(2, 4), Blob(2, 4)], [Blob()]
    sce.LayerSetUp(bottoms, top)
    top[0].reshape()
    top[0].data[...] = 3.25
    sce.Forward(bottoms, top)                   # weights all 0: top untouched
    assert float(top[0].data) == 3.25
