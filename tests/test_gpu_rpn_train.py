"""TRAIN phase of ProposalLayer, ProposalTargetLayer and AnchorTargetLayer on the device
(mnc_proposal_train_state / mnc_proposal_backward, mnc_proposal_target*, mnc_anchor_target) against
the reference's fixtures and the numpy oracle: indices, labels, counts, weights, mask targets and
copied diffs exact, values derived from exp / log within 4 float32 ulp, RoI coordinates within the
proposal tolerance; padded rows, determinism, graph replay, NULL diffs, argument errors, the
mirrors and the differentiable chain rpn_bbox_pred -> ROIWarping."""
import numpy as np
import pytest
import torch

from oracle import oracle_rpn_train as R
from oracle import oracle_train as T
from tests.test_oracle_rpn_train import fixture, config, CASES, PT_TOPS, AT_TOPS

pytestmark = pytest.mark.gpu
PT_EXACT = ("rois", "labels", "bbox_inside_weights", "bbox_outside_weights", "mask_targets",
            "mask_weight", "gt_masks_info", "fg_inds", "bg_inds")


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _ulp(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a - b) / np.spacing(np.maximum(np.abs(a), np.abs(b)).astype(np.float32) + np.float32(1e-30))


def _keys(a):
    return _cuda(np.asarray(a, np.uint32).view(np.int32))


def _pt_device(f, normalize):
    from mnc_b200 import ops
    return ops.proposal_target(
        _cuda(f["rpn_rois"]), _cuda(f["rois_index"]), _cuda(f["gt_boxes"]),
        _cuda(f["gt_masks"].astype(np.float32)), _cuda(f["mask_info"]), _cuda(f["im_info"].ravel()),
        _keys(f["keys"]), means=T.BBOX_NORMALIZE_MEANS if normalize else None,
        stds=T.BBOX_NORMALIZE_STDS if normalize else None)


def _check_pt(out, want, f):
    """Device ProposalTarget tops (padded) against the K-row reference / oracle tops."""
    K = want["labels"].shape[0]
    cnt = out["counts"].cpu().numpy()
    assert cnt[0] == K and cnt[1] == want["fg_inds"].size and cnt[2] == want["bg_inds"].size
    assert cnt[3] == int(want["mask_weight"][:, 0, 0, 0].sum())
    got = {k: out[k].cpu().numpy() for k in PT_TOPS}
    for k in PT_EXACT:
        w = np.asarray(want[k]).reshape(-1, *got[k].shape[1:])
        n = w.shape[0]
        assert np.array_equal(got[k][:n], w), k
    bt, wbt = got["bbox_targets"][:K], want["bbox_targets"]
    assert np.array_equal(bt != 0, wbt != 0) and np.all(_ulp(bt, wbt) <= 4)
    # padded rows: label -1, zero RoI / targets / weights / masks, gt_masks_info -1, lists -1
    Kmax = got["labels"].shape[0]
    assert np.all(got["labels"][K:] == -1) and np.all(got["rois"][K:] == 0)
    for k in ("bbox_targets", "bbox_inside_weights", "bbox_outside_weights", "mask_targets", "mask_weight"):
        assert np.all(got[k][K:] == 0), k
    assert np.all(got["gt_masks_info"][K:] == -1)
    assert np.all(got["fg_inds"][cnt[1]:] == -1) and np.all(got["bg_inds"][cnt[2]:] == -1)
    assert Kmax == 64 + 3
    return got


def _check_at(at, want):
    got = [x.cpu().numpy() for x in at]
    for k, g, w in zip(AT_TOPS, got, want):
        assert g.shape == w.shape, k
        if k == "bbox_targets":
            assert np.all(_ulp(g, w) <= 4), np.max(_ulp(g, w))
        else:
            assert np.array_equal(g, w), k


@pytest.mark.parametrize("name", CASES)
def test_matches_reference_fixtures(name):
    from mnc_b200 import ops
    f = fixture(name)
    c = config(f)
    if c["n"]:
        rois, index, count, state = ops.proposal_train(_cuda(f["prob"]), _cuda(f["deltas"]),
                                                       _cuda(f["im_info"].ravel()), c["H"], c["W"])
        R_ = f["pl_rois"].shape[0]
        assert int(count[0]) == R_
        assert np.array_equal(index.cpu().numpy()[:R_], f["pl_index"].ravel())
        assert np.allclose(rois.cpu().numpy()[:R_], f["pl_rois"], rtol=1e-5, atol=2e-3)
        bd = ops.proposal_backward(_cuda(f["pl_top_diff"]), state, _cuda(f["deltas"]), c["clip"]).cpu().numpy()
        want = f["pl_bbox_diff"]
        assert np.array_equal(bd != 0, want != 0)
        clamped = np.abs(want) == np.float32(c["clip"])
        assert np.array_equal(bd[clamped], want[clamped])
        assert np.all(_ulp(bd, want) <= 4)
    out = _pt_device(f, c["normalize"])
    want = {k: f["pt_" + k] for k in PT_TOPS}
    _check_pt(out, want, f)
    rd = ops.proposal_target_backward(_cuda(np.pad(f["pt_top_diff"], ((0, 67 - f["pt_top_diff"].shape[0]), (0, 0)),
                                                   constant_values=5.0)),
                                      out["state"], c["n"], c["G"], c["bp_all"]).cpu().numpy()
    assert np.array_equal(rd, f["pt_rois_diff"])          # padded rows (5.0) never read
    at = ops.anchor_target(c["H"], c["W"], _cuda(f["gt_boxes"]), _cuda(f["im_info"].ravel()),
                           _keys(f["anchor_keys"]), out["fg_inds"], out["bg_inds"], out["counts"])
    _check_at(at, [f["at_" + k] for k in AT_TOPS])


def test_random_cases_match_oracle():
    from mnc_b200 import ops
    near = 0
    for seed in range(20):
        G = (3, 20, 7, 1, 12)[seed % 5]
        H, W, info = ((38, 63, (600, 1000, 1.6)), (30, 50, (480, 800, 1.0)))[seed % 2]
        n = (300, 120, 0, 2000)[seed % 4]
        cs = R.make_case(500 + seed, H, W, info, G, n, scores=False)
        rng = np.random.default_rng(seed)
        keys = rng.integers(0, 2 ** 32, (3, n + G), dtype=np.uint64).astype(np.uint32)
        akeys = rng.integers(0, 2 ** 32, H * W * 9, dtype=np.uint64).astype(np.uint32)
        if seed % 3 == 0:
            keys[:, : (n + G) // 2] = 7                   # ties: broken by index
        normalize, bp_all = seed % 2 == 0, seed % 3 != 1
        want = R.proposal_target_forward(cs["rpn_rois"], cs["rois_index"], cs["gt_boxes"],
                                         cs["gt_masks"], cs["mask_info"], cs["im_info"], keys,
                                         normalize=normalize, bp_all=bp_all)
        f = dict(cs, keys=keys)
        out = _pt_device(f, normalize)
        tv = T.target_values({"gt_masks": cs["gt_masks"], "mask_info": cs["mask_info"]},
                             {"nfg": int(want["mask_weight"][:, 0, 0, 0].sum()),
                              "gt_mask_info": want["gt_masks_info"]})
        k_near = int(np.sum(np.abs(tv - 0.4) < 1e-6))
        near += k_near
        if k_near:
            K = want["labels"].shape[0]
            got_m = out["mask_targets"].cpu().numpy()[:K]
            assert np.sum(got_m != want["mask_targets"]) <= k_near
            want["mask_targets"] = got_m
        _check_pt(out, want, f)
        Kmax = out["labels"].shape[0]
        td = rng.normal(0, 1, (Kmax, 5)).astype(np.float32)
        rd = ops.proposal_target_backward(_cuda(td), out["state"], n, G, bp_all).cpu().numpy()
        assert np.array_equal(rd, R.proposal_target_backward(td, want["keep_ind"], n))
        pw = -1.0 if seed % 4 else 0.25
        wat = R.anchor_target_forward(H, W, cs["gt_boxes"], cs["im_info"], akeys, want["fg_inds"],
                                      want["bg_inds"], RPN_POSITIVE_WEIGHT=pw,
                                      RPN_CLOBBER_POSITIVES=seed % 5 == 1)
        at = ops.anchor_target(H, W, _cuda(cs["gt_boxes"]), _cuda(cs["im_info"].ravel()), _keys(akeys),
                               out["fg_inds"], out["bg_inds"], out["counts"], positive_weight=pw,
                               clobber_positives=seed % 5 == 1)
        _check_at(at, wat)
    print("random-case mask samples within 1e-6 of BINARIZE_THRESH: %d" % near)


def test_proposal_train_matches_oracle_and_mix_off():
    from mnc_b200 import ops
    for seed in range(3):
        cs = R.make_case(900 + seed)
        rois, index, count, state = ops.proposal_train(_cuda(cs["prob"]), _cuda(cs["deltas"]),
                                                       _cuda(cs["im_info"].ravel()), 38, 63)
        wr, wi, st = R.proposal_train_forward(cs["prob"], cs["deltas"], cs["im_info"])
        n = wr.shape[0]
        assert int(count[0]) == n
        assert np.array_equal(index.cpu().numpy()[:n], wi.ravel())
        assert np.all(index.cpu().numpy()[n:] == -1)
        assert np.allclose(rois.cpu().numpy()[:n], wr, rtol=1e-5, atol=2e-3)
        td = np.random.default_rng(seed).normal(0, 1e-3, (rois.shape[0], 5)).astype(np.float32)
        td[::3] = 0
        bd = ops.proposal_backward(_cuda(td), state, _cuda(cs["deltas"]), 1.0 / 512).cpu().numpy()
        want = R.proposal_backward(td[:n], st, cs["deltas"], 1.0 / 512)
        assert np.array_equal(bd != 0, want != 0) and np.all(_ulp(bd, want) <= 4)
    # AnchorTarget without MIX_INDEX
    f = fixture("A")
    c = config(f)
    at = ops.anchor_target(c["H"], c["W"], _cuda(f["gt_boxes"]), _cuda(f["im_info"].ravel()),
                           _keys(f["anchor_keys"]))
    _check_at(at, R.anchor_target_forward(c["H"], c["W"], f["gt_boxes"], f["im_info"], f["anchor_keys"]))


def _chain_inputs():
    f = fixture("A")
    return f, [_cuda(f[k]) for k in ("prob", "deltas")] + [_cuda(f["im_info"].ravel())]


def test_deterministic_and_graph_replay():
    from mnc_b200 import ops
    f, (prob, deltas, info) = _chain_inputs()
    gt, gm, mi = _cuda(f["gt_boxes"]), _cuda(f["gt_masks"].astype(np.float32)), _cuda(f["mask_info"])
    keys, akeys = _keys(f["keys"]), _keys(f["anchor_keys"])
    td = torch.randn(67, 5, device="cuda") * 1e-3

    def step():
        rois, index, count, state = ops.proposal_train(prob, deltas, info, 38, 63)
        o = ops.proposal_target(rois, index, gt, gm, mi, info, keys, n_valid=count,
                                means=T.BBOX_NORMALIZE_MEANS, stds=T.BBOX_NORMALIZE_STDS)
        rd = ops.proposal_target_backward(td, o["state"], rois.shape[0], 3)
        bd = ops.proposal_backward(rd, state, deltas, 1.0 / 512)
        at = ops.anchor_target(38, 63, gt, info, akeys, o["fg_inds"], o["bg_inds"], o["counts"])
        return [rois, index, count] + [o[k] for k in PT_TOPS] + [o["counts"], rd, bd] + list(at)
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
    assert a[-5].abs().max() > 0                  # bbox_pred diff reached


def test_null_diffs_and_argument_errors():
    from mnc_b200 import ops
    from mnc_b200._lib import MncError, lib, ptr
    f = fixture("A")
    c = config(f)
    out = _pt_device(f, True)
    st = out["state"]
    assert lib.mnc_proposal_target_backward(ptr(out["rois"]), ptr(st), 300, 3, 1, None, None) == 0
    assert lib.mnc_proposal_backward(ptr(out["rois"]), 0, ptr(st), ptr(out["rois"]), 38, 63, 0.0,
                                     None, None) == 0
    gt = _cuda(f["gt_boxes"])
    with pytest.raises(MncError):                  # G = 0
        ops.proposal_target(_cuda(f["rpn_rois"]), _cuda(f["rois_index"]), gt[:0],
                            _cuda(f["gt_masks"][:0].astype(np.float32)), _cuda(f["mask_info"][:0]),
                            _cuda(f["im_info"].ravel()), _keys(f["keys"][:, :300]))
    with pytest.raises(MncError):                  # fractions summing past 1
        ops.proposal_target(_cuda(f["rpn_rois"]), _cuda(f["rois_index"]), gt,
                            _cuda(f["gt_masks"].astype(np.float32)), _cuda(f["mask_info"]),
                            _cuda(f["im_info"].ravel()), _keys(f["keys"]), bg_fraction=(0.85, 0.25))
    with pytest.raises(MncError):
        ops.anchor_target(c["H"], c["W"], gt[:0], _cuda(f["im_info"].ravel()), _keys(f["anchor_keys"]))
    with pytest.raises(MncError):
        ops.anchor_target(c["H"], c["W"], gt, _cuda(f["im_info"].ravel()), _keys(f["anchor_keys"]),
                          positive_weight=1.5)
    with pytest.raises(MncError):
        ops.proposal_backward(torch.zeros(300, 5, device="cuda"), torch.zeros(300, 2, dtype=torch.int32,
                              device="cuda"), _cuda(f["deltas"]), -1.0)


def test_mirrors_follow_the_prototxt():
    """proposal -> roi-data -> rpn-data as caffe.Layer objects, in train.prototxt's order and with
    its propagate_down, reproduce the reference fixture's blobs and diffs."""
    import mnc_b200.lib as lib
    lib.install()
    from caffe import Blob, TRAIN
    from mnc_config import cfg
    from pylayer.proposal_layer import ProposalLayer
    from pylayer.proposal_target_layer import ProposalTargetLayer
    from pylayer.anchor_target_layer import AnchorTargetLayer
    f = fixture("A")
    c = config(f)

    def blob(a):
        b = Blob(*a.shape)
        b.data[...] = a
        return b
    pl = ProposalLayer("{'feat_stride': 16, 'use_clip': 1, 'clip_base': 512}", TRAIN)
    pb = [blob(f["prob"]), blob(f["deltas"]), blob(f["im_info"])]
    ptop = [Blob(), Blob()]
    pl.setup(pb, ptop)
    pl.forward(pb, ptop)
    assert ptop[0].data.shape == f["pl_rois"].shape and np.array_equal(ptop[1].data, f["pl_index"])
    assert np.allclose(ptop[0].data, f["pl_rois"], rtol=1e-5, atol=2e-3)
    tl = ProposalTargetLayer("{'num_classes': 21}", TRAIN)
    tb = [blob(f["rpn_rois"]), blob(f["gt_boxes"]), blob(f["im_info"]),
          blob(f["gt_masks"].astype(np.float32)), blob(f["mask_info"].astype(np.float32)),
          blob(f["rois_index"])]
    ttop = [Blob() for _ in range(10)]
    old = cfg.TRAIN.BBOX_NORMALIZE_TARGETS_PRECOMPUTED
    cfg.TRAIN.BBOX_NORMALIZE_TARGETS_PRECOMPUTED = True
    try:
        tl.setup(tb, ttop)
        tl.keys = _keys(f["keys"])
        tl.forward(tb, ttop)
    finally:
        cfg.TRAIN.BBOX_NORMALIZE_TARGETS_PRECOMPUTED = old
    for i, k in enumerate(PT_TOPS):
        assert ttop[i].data.shape == f["pt_" + k].shape, k
        if k != "bbox_targets":
            assert np.array_equal(ttop[i].data, f["pt_" + k]), k
    al = AnchorTargetLayer("{'feat_stride': 16}", TRAIN)
    ab = [Blob(1, 18, c["H"], c["W"]), blob(f["gt_boxes"]), blob(f["im_info"]), ttop[8], ttop[9]]
    atop = [Blob() for _ in range(4)]
    al.setup(ab, atop)
    al.keys = _keys(f["anchor_keys"])
    al.forward(ab, atop)
    for i, k in enumerate(AT_TOPS):
        assert atop[i].data.shape == f["at_" + k].shape, k
        if k != "bbox_targets":
            assert np.array_equal(atop[i].data, f["at_" + k]), k
    # backward: roi-data propagates to rpn_rois only, proposal to rpn_bbox_pred only
    # diffs are written into the blobs' arrays: pycaffe's Blob.diff cannot be rebound
    ttop[0].diff = f["pt_top_diff"].copy()
    for b in tb:
        b.diff = np.full(b.data.shape, 7, np.float32)
    held = tb[0].diff
    tl.backward(ttop, [True, False, False, False, False, False], tb)
    assert tb[0].diff is held
    assert np.array_equal(tb[0].diff, f["pt_rois_diff"]) and np.all(tb[1].diff == 7)
    tb[0].diff[...] = 7
    tl.backward(ttop, [False] * 6, tb)
    assert np.all(tb[0].diff == 7)
    ptop[0].diff = f["pl_top_diff"].copy()
    for b in pb:
        b.diff = np.full(b.data.shape, 7, np.float32)
    held = pb[1].diff
    pl.backward(ptop, [False, True, False], pb)
    assert pb[1].diff is held
    want = f["pl_bbox_diff"]
    assert np.array_equal(pb[1].diff != 0, want != 0) and np.all(_ulp(pb[1].diff, want) <= 4)
    assert np.all(pb[0].diff == 7)


def test_differentiable_chain_into_roi_warp():
    from mnc_b200 import autograd
    from oracle import oracle_backward as OB
    f = fixture("A")
    rng = np.random.default_rng(5)
    feat = rng.normal(size=(1, 16, 38, 63)).astype(np.float32)
    deltas = _cuda(f["deltas"]).requires_grad_()
    rois, index, count = autograd.proposal_train(_cuda(f["prob"]), deltas, _cuda(f["im_info"].ravel()),
                                                 clip_thresh=1.0 / 512)
    n = int(count[0])
    assert n == rois.shape[0] == 300
    outs = autograd.proposal_target(rois, index, _cuda(f["gt_boxes"]),
                                    _cuda(f["gt_masks"].astype(np.float32)), _cuda(f["mask_info"]),
                                    _cuda(f["im_info"].ravel()), keys=_keys(f["keys"]), count=count)
    rois_pt = outs[0]
    assert not any(o.requires_grad for o in outs[1:])
    out = autograd.roi_warp(_cuda(feat), rois_pt, 14, 14, 0.0625)
    g = (rng.normal(size=tuple(out.shape)) * 1e-3).astype(np.float32)
    (out * _cuda(g)).sum().backward()
    # oracle: ROIWarping's coordinate gradient, then ProposalTarget's and Proposal's backward
    _, coord, mag = OB.roi_warp_backward(feat, rois_pt.detach().cpu().numpy(), g, 14, 14, want_abs=True)
    pt = R.proposal_target_forward(rois.detach().cpu().numpy(), index.cpu().numpy()[None],
                                   f["gt_boxes"], f["gt_masks"], f["mask_info"], f["im_info"], f["keys"])
    K = pt["labels"].shape[0]
    _, _, st = R.proposal_train_forward(f["prob"], f["deltas"], f["im_info"])
    rd = R.proposal_target_backward(coord[:K], pt["keep_ind"], n)
    want = R.proposal_backward(rd, st, f["deltas"], 1.0 / 512)
    # bound: push the coordinate tolerance 1e-5 * mag through the same products; the x/y channels
    # see |d1| + |d3|, the w/h channels (|d3| + |d1|) / 2
    rmag = np.abs(R.proposal_target_backward(mag[:K], pt["keep_ind"], n))
    flip = rmag * np.array([1, -1, -1, 1, 1], np.float32)
    bmag = np.maximum(np.abs(R.proposal_backward(rmag, st, f["deltas"], 0.0)),
                      np.abs(R.proposal_backward(flip, st, f["deltas"], 0.0)))
    got = deltas.grad.cpu().numpy()
    clamped = np.abs(want) == np.float32(1.0 / 512)
    assert np.array_equal(got[clamped], want[clamped])
    assert np.all(np.abs(got - want)[~clamped] <= 1e-5 * np.abs(bmag)[~clamped] + 1e-30)
    assert np.abs(got).max() > 0


def test_padding_rows_past_the_device_count_take_no_part():
    """rpn_rois padded past a device count (ProposalLayer keeping fewer than RPN_POST_NMS_TOP_N)
    give the tops of the unpadded rows; only the gt rows' key index moves by the padding."""
    from mnc_b200 import ops
    for name in ("A", "B"):
        f = fixture(name)
        c = config(f)
        n, G, P = c["n"], c["G"], 37
        rois = np.concatenate([f["rpn_rois"], np.zeros((P, 5), np.float32)])
        index = np.concatenate([f["rois_index"], np.full((1, P), -1, np.float32)], axis=1)
        keys = np.concatenate([f["keys"][:, :n], np.zeros((3, P), np.uint32), f["keys"][:, n:]], axis=1)
        count = torch.tensor([n], dtype=torch.int32, device="cuda")
        out = ops.proposal_target(
            _cuda(rois), _cuda(index), _cuda(f["gt_boxes"]), _cuda(f["gt_masks"].astype(np.float32)),
            _cuda(f["mask_info"]), _cuda(f["im_info"].ravel()), _keys(keys), n_valid=count,
            means=T.BBOX_NORMALIZE_MEANS if c["normalize"] else None,
            stds=T.BBOX_NORMALIZE_STDS if c["normalize"] else None)
        _check_pt(out, {k: f["pt_" + k] for k in PT_TOPS}, f)
        td = np.pad(f["pt_top_diff"], ((0, 67 - f["pt_top_diff"].shape[0]), (0, 0)))
        rd = ops.proposal_target_backward(_cuda(td), out["state"], n + P, G, c["bp_all"]).cpu().numpy()
        assert np.array_equal(rd[:n], f["pt_rois_diff"]) and np.all(rd[n:] == 0)


def test_default_keys_follow_torch_seed():
    """keys=None draws with torch's generator on the device: the same seed, the same sample."""
    from mnc_b200 import autograd
    f = fixture("A")
    args = (_cuda(f["rpn_rois"]), _cuda(f["rois_index"]), _cuda(f["gt_boxes"]),
            _cuda(f["gt_masks"].astype(np.float32)), _cuda(f["mask_info"]), _cuda(f["im_info"].ravel()))
    runs = []
    for seed in (3, 3, 4):
        torch.manual_seed(seed)
        pt = autograd.proposal_target(*args)
        at = autograd.anchor_target(38, 63, args[2], args[5], pt[8], pt[9], pt[10])
        runs.append([x.clone() for x in list(pt) + list(at)])
    assert all(torch.equal(x, y) for x, y in zip(runs[0], runs[1]))
    assert not all(torch.equal(x, y) for x, y in zip(runs[0], runs[2]))
    K = int(runs[0][10][0])
    assert K == 64 and torch.all(runs[0][1][K:] == -1)


def test_config_bounds():
    from mnc_b200 import ops
    from mnc_b200._lib import MncError
    f = fixture("A")
    t = (_cuda(f["rpn_rois"]), _cuda(f["rois_index"]), _cuda(f["gt_boxes"]),
         _cuda(f["gt_masks"].astype(np.float32)), _cuda(f["mask_info"]), _cuda(f["im_info"].ravel()))
    keys = _keys(np.concatenate([f["keys"], f["keys"][:1]]))
    # 0.1 + 0.2 + 0.7 rounds to 1 + 2^-52: accepted, and K stays within the capacity
    out = ops.proposal_target(*t, keys, bg_fraction=(0.1, 0.2, 0.7), bg_thresh_lo=(0.1, 0.0, 0.0),
                              bg_thresh_hi=(0.5, 0.1, 0.5))
    assert int(out["counts"][0]) <= out["labels"].shape[0]
    with pytest.raises(MncError):
        ops.proposal_target(*t, keys, bg_fraction=(0.1, 0.2, 0.71), bg_thresh_lo=(0.1, 0.0, 0.0),
                            bg_thresh_hi=(0.5, 0.1, 0.5))
    with pytest.raises(MncError):           # RPN_FG_FRACTION above 1: a negative bg budget
        ops.anchor_target(38, 63, t[2], t[5], _keys(f["anchor_keys"]), fg_fraction=1.5)
