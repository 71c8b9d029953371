"""SURVEY.md section 8f row 4 -- the sibling test graphs on the same kernels: ROIPooling
(roi_pooling_layer.cu:17-77), the Faster R-CNN test net and the CFM test net, against the oracle
(teacher-forced per stage, as tests/test_gpu_e2e.py)."""
import numpy as np
import pytest
import torch

from tests import roi_shapes as RS
from tests import util
from tests.test_gpu_roi import table_params

pytestmark = pytest.mark.gpu
TOL = 1e-3


def _rois(n, seed, W, H, levels=1):
    rng = np.random.default_rng(seed)
    b = util.random_boxes(n, seed, W, H, smin=8, smax=min(W, H))
    lv = rng.integers(0, levels, n).astype(np.float32)
    r = np.concatenate([lv[:, None], b], axis=1).astype(np.float32)
    if n >= 4:
        r[0, 1:] = [0, 0, W - 1, H - 1]          # whole image
        r[1, 1:] = [40, 30, 41, 31]              # sub-cell RoI: 1x1 after rounding
        r[2, 1:] = [W + 40, H + 40, W + 90, H + 90]  # outside the map: empty bins -> 0 / -1
        r[3, 1:] = [100, 100, 60, 50]            # malformed (x2 < x1): forced to 1x1
    return r


@pytest.mark.parametrize("case,size", [pytest.param(None, (P, P), id=str(P)) for P in (7, 14)] +
                         [pytest.param(None, (6, 3), id="P2")] + table_params(pool_only=True))
def test_roi_pool_nchw_bit_exact(case, size):
    from oracle import oracle as O
    from mnc_b200 import ops
    from mnc_b200._lib import MncError
    ph, pw = size
    if case is None:
        rng = np.random.default_rng(5)
        feat = rng.normal(size=(2, 40, 38, 63)).astype(np.float32)
        rois = _rois(64, 6, 1000, 600, levels=2)
        ss = 0.0625
    else:
        feat, rois, ss = RS.feat(case), RS.rois(case), RS.BY_NAME[case].scale
    want, want_arg = O.roi_pool(feat, rois, ph, pw, ss, return_argmax=True)
    d_feat, d_rois = torch.from_numpy(feat).cuda(), torch.from_numpy(rois).cuda()
    arg = torch.empty(want.shape, dtype=torch.int32, device="cuda")
    got = ops.roi_pool_nchw(d_feat, d_rois, ph, pw, ss, argmax=arg)
    assert np.array_equal(got.cpu().numpy(), want)
    assert np.array_equal(arg.cpu().numpy(), want_arg)
    assert np.array_equal(ops.roi_pool_nchw(d_feat, d_rois, ph, pw, ss).cpu().numpy(), want)  # argmax=NULL
    assert (want_arg >= 0).any()
    if max(ph, pw) > 32:
        # the forward takes any size whose bins fit in shared memory; the backward stages per-RoI
        # tables of at most 32 cells a side and rejects larger ones
        with pytest.raises(MncError):
            ops.roi_pool_backward_nchw(got, arg, feat.shape, d_rois, ph, pw, ss)


def test_roi_pooling_layer_mirror_contract():
    """LayerSetUp / Reshape / Forward_gpu protocol of ROIPoolingLayer (roi_pooling_layer.cpp:20-44)."""
    import mnc_b200.lib as L
    L.install()
    import caffe
    from caffe.layers import ROIPoolingLayer
    from oracle import oracle as O
    rng = np.random.default_rng(2)
    feat, rois, top = caffe.Blob(), caffe.Blob(), caffe.Blob()
    feat.data = rng.normal(size=(2, 16, 20, 30)).astype(np.float32)
    rois.data = _rois(12, 3, 480, 320, levels=2)
    layer = ROIPoolingLayer(dict(roi_pooling_param=dict(pooled_w=7, pooled_h=7, spatial_scale=0.0625)))
    layer.LayerSetUp([feat, rois], [top])
    layer.Forward([feat, rois], [top])
    want, want_arg = O.roi_pool(feat.data, rois.data, 7, 7, return_argmax=True)
    assert top.shape == (12, 16, 7, 7) and np.array_equal(top.data, want)
    assert np.array_equal(layer.max_idx_, want_arg)
    with pytest.raises(ValueError):
        ROIPoolingLayer(dict(roi_pooling_param=dict(pooled_w=7, pooled_h=0))).LayerSetUp([feat, rois], [top])


@pytest.mark.parametrize("C,P", [pytest.param(64, P, id=str(P)) for P in (7, 14)] +
                         [pytest.param(C, P, id="C%d-P%d" % (C, P)) for C in (4, 12, 512) for P in (1, 7, 14, 32)])
def test_roi_pool_and_sample_split_forms(C, P):
    """Engine forms (fp32 NHWC in, split-bf16 rows [r][ph][pw][c] out) vs the NCHW layer kernels'
    oracle.  ROIPooling is a max, so its rows are the split of the oracle's bytes exactly.
    ROIWarping is evaluated with FMAs: per element |got - want| <= 2^-16 |want| + 2^-20 S, with
    S = sum_i w_i |v_i| = roi_warp(|feat|) (the weights are non-negative) -- twice the split
    rounding plus twice the fused-versus-unfused difference of the 4-tap sum."""
    from oracle import oracle as O
    from mnc_b200 import ops, dense
    rng = np.random.default_rng(8 if C == 64 else C + P)
    H, W = 38, 63
    feat = rng.normal(size=(2, C, H, W))
    feat = (np.maximum(feat, 0) if C == 64 else feat).astype(np.float32)
    rois = _rois(50, 9, 1000, 600, levels=2)
    d_nhwc = torch.from_numpy(feat.transpose(0, 2, 3, 1).copy()).cuda()
    d_rois = torch.from_numpy(rois).cuda()
    out = torch.zeros((2, 50, P, P, C), dtype=torch.bfloat16, device="cuda")
    ops.roi_pool_split(d_nhwc, C, H, W, d_rois, P, out)
    want = O.roi_pool(feat, rois, P, P)
    want_split = dense.split(torch.from_numpy(want.transpose(0, 2, 3, 1).copy()))
    assert torch.equal(out.cpu().view(torch.int16), want_split.view(torch.int16))
    assert np.all(want[2] == 0)      # the RoI outside the map
    out.zero_()
    ops.roi_sample_split(d_nhwc, C, H, W, d_rois, P, out)
    got = dense.merge(out).permute(0, 3, 1, 2).cpu().numpy().astype(np.float64)
    want = O.roi_warp(feat, rois, P, P).astype(np.float64)
    bound = 2.0 ** -16 * np.abs(want) + 2.0 ** -20 * O.roi_warp(np.abs(feat), rois, P, P)
    assert np.all(np.abs(got - want) <= bound)
    assert np.abs(want).max() > 0 and np.all(got[2] == 0)


def test_faster_rcnn_engine_stagewise():
    from oracle import oracle as O
    from mnc_b200 import weights as Wt, dense
    from mnc_b200.siblings import FasterRCNNEngine
    w = Wt.make_sibling_weights("faster_rcnn", Wt.TINY_ARCH)
    B, H, W = 2, 224, 320
    ims = [O.synthetic_image(i, H, W) for i in range(B)]
    blobs = [O.prep_blob(im) for im in ims]
    data = np.concatenate([b[0] for b in blobs])
    im_info = np.concatenate([b[1] for b in blobs])
    eng = FasterRCNNEngine(w)
    out = eng.forward(torch.from_numpy(data).cuda(), torch.from_numpy(im_info).cuda(), keep_intermediate=True)
    for img in range(B):
        sl = slice(img * 300, (img + 1) * 300)
        n = int(out["roi_counts"][img].item())
        assert n > 0
        c5 = dense.merge(out["_conv5_3"])[img].permute(2, 0, 1).cpu().numpy()
        rois = out["rois"][sl].cpu().numpy()[:n]
        rois0 = rois.copy()
        rois0[:, 0] = 0
        want5 = O.roi_warp(c5[None], rois0, 7, 7)
        got5 = dense.merge(out["_pool5"])[sl][:n].permute(0, 3, 1, 2).cpu().numpy()
        assert util.rel_err(got5, want5) < 1e-4
        import torch.nn.functional as F
        with torch.no_grad():
            fc6 = F.relu(F.linear(torch.from_numpy(got5).reshape(n, -1), *w["fc6"]))
            fc7 = F.relu(F.linear(fc6, *w["fc7"]))
            want_prob = torch.softmax(F.linear(fc7, *w["cls_score"]), 1).numpy()
            want_bb = F.linear(fc7, *w["bbox_pred"]).numpy()
        assert np.abs(out["cls_prob"][sl][:n].cpu().numpy() - want_prob).max() < TOL
        bb = out["bbox_pred"][sl][:n].cpu().numpy()
        assert np.abs(bb - want_bb).max() < TOL * max(1.0, np.abs(want_bb).max())
    # from pixels, whole net: the oracle's own rois / scores for image 0 (tiny net: no near-ties)
    ob = O.frcnn_net_forward(w, data[0:1], im_info[0:1])
    n0 = int(out["roi_counts"][0].item())
    # (a 1-ulp score difference can legally reorder / swap near-tied proposals, so RoIs are matched
    # as sets and the scores compared on the matched rows)
    assert abs(ob["rois"].shape[0] - n0) <= 2
    got_r = out["rois"][:n0].cpu().numpy()
    d = np.abs(got_r[:, None, 1:] - ob["rois"][None, :, 1:]).max(axis=2)
    match = d.argmin(axis=1)
    hit = d.min(axis=1) < 0.05
    assert hit.mean() > 0.95
    assert np.abs(out["cls_prob"][:n0].cpu().numpy()[hit] - ob["cls_prob"][match[hit]]).max() < 5 * TOL
    # detection tail: per-class decoded + clipped boxes
    info = torch.from_numpy(im_info).cuda()
    hw = torch.tensor([[H, W]] * B, dtype=torch.float32).cuda()
    sc = torch.ones(B).cuda()
    scores, pred, valid, o = eng.detect(torch.from_numpy(data).cuda(), info, hw, sc)
    blobs0 = {"rois": o["rois"][:n0].cpu().numpy(), "bbox_pred": o["bbox_pred"][:n0].cpu().numpy(),
              "cls_prob": o["cls_prob"][:n0].cpu().numpy()}
    blobs0["rois"][:, 0] = 0
    want_scores, want_pred = O.detection_tail(blobs0, (H, W, 3))
    assert pred.shape == (B, 300, 84) and int(valid[0].sum()) == n0
    assert np.abs(pred[0, :n0].cpu().numpy() - want_pred).max() < 1e-3 * W
    assert np.array_equal(scores[0, :n0].cpu().numpy(), want_scores)


def test_cfm_engine_against_oracle():
    """Two pyramid levels, rois assigned to levels by `pred_rois_for_blob`, binary 14x14 masks."""
    from oracle import oracle as O
    from mnc_b200 import weights as Wt, dense
    from mnc_b200.siblings import CFMEngine
    w = Wt.make_sibling_weights("cfm", Wt.TINY_ARCH)
    im = O.synthetic_image(3, 240, 320)
    blob, scales = O.prep_im_for_blob_cfm(im, (200, 300))
    rng = np.random.default_rng(4)
    boxes = util.random_boxes(40, 4, 320, 240, smin=30, smax=320)
    boxes[:6] = [[0, 0, 319, 239], [10, 5, 300, 230], [40, 0, 319, 220], [0, 20, 280, 239],
                 [5, 5, 310, 200], [30, 10, 290, 235]]      # large boxes -> coarser pyramid level
    rois = O.pred_rois_for_blob(boxes, scales).astype(np.float32)
    assert set(np.unique(rois[:, 0])) == {0.0, 1.0}
    masks = (rng.uniform(size=(40, 1, 14, 14)) >= 0.4).astype(np.float32)
    eng = CFMEngine(w)
    out = eng.forward(torch.from_numpy(np.ascontiguousarray(blob)).cuda(), torch.from_numpy(rois).cuda(),
                      torch.from_numpy(masks).cuda(), keep_intermediate=True)
    c5 = dense.merge(out["_conv5_3"]).permute(0, 3, 1, 2).cpu().numpy()
    with torch.no_grad():
        want_c5 = O.trunk_forward(w, blob).numpy()
    assert util.rel_err(c5, want_c5) < TOL
    got7 = dense.merge(out["_box7"]).permute(0, 3, 1, 2).cpu().numpy()
    got14 = dense.merge(out["_feat14"]).permute(0, 3, 1, 2).cpu().numpy()
    assert util.rel_err(got7, O.roi_pool(c5, rois, 7, 7)) < 1e-4
    assert util.rel_err(got14, O.roi_pool(c5, rois, 14, 14)) < 1e-4
    import torch.nn.functional as F
    want_m7 = F.max_pool2d(torch.from_numpy(O.mask_pool(got14, masks)), 2, 2).numpy()
    got_m7 = dense.merge(out["_m7"]).permute(0, 3, 1, 2).cpu().numpy()
    assert util.rel_err(got_m7, want_m7) < 1e-4
    # whole net from pixels (max pooling is selection, FC layers are smooth: no index hazards)
    ob = O.cfm_net_forward(w, blob, rois, masks)
    for k in ("mask_prob", "seg_cls_prob", "cls_prob"):
        got = out[k].cpu().numpy().reshape(ob[k].shape)
        assert np.abs(got - ob[k]).max() < 2 * TOL, k
    bb = out["bbox_pred"].cpu().numpy()
    assert np.abs(bb - ob["bbox_pred"]).max() < 2 * TOL * max(1.0, np.abs(ob["bbox_pred"]).max())


def test_caffe_net_mirror_runs_sibling_graphs():
    """caffe.Net picks the engine from the layer set and exposes the graphs' own blobs."""
    import mnc_b200.lib as L
    L.install()
    import caffe
    from oracle import oracle as O
    from mnc_b200 import weights as Wt
    caffe.set_mode_gpu()
    caffe.set_device(0)
    net = caffe.Net(None, Wt.make_sibling_weights("faster_rcnn", Wt.TINY_ARCH), caffe.TEST)
    assert net.kind == "faster_rcnn" and net.inputs == ["data", "im_info"]
    blob, im_info = O.prep_blob(O.synthetic_image(0, 224, 320))
    net.blobs["data"].reshape(*blob.shape)
    net.blobs["im_info"].reshape(*im_info.shape)
    out = net.forward(data=blob.astype(np.float32, copy=False), im_info=im_info)
    n = net.blobs["rois"].data.shape[0]
    assert set(out) == {"cls_prob", "bbox_pred"} and out["cls_prob"].shape == (n, 21)
    assert out["bbox_pred"].shape == (n, 84) and np.allclose(out["cls_prob"].sum(1), 1, atol=1e-5)
    net = caffe.Net(None, Wt.make_sibling_weights("cfm", Wt.TINY_ARCH), caffe.TEST)
    assert net.kind == "cfm" and net.inputs == ["data", "rois", "masks"]
    im = O.synthetic_image(3, 240, 320)
    blob, scales = O.prep_im_for_blob_cfm(im, (200, 300))
    rois = O.pred_rois_for_blob(util.random_boxes(24, 4, 320, 240, smin=30, smax=320), scales).astype(np.float32)
    masks = (np.random.default_rng(1).uniform(size=(24, 1, 14, 14)) >= 0.4).astype(np.float32)
    net.blobs["data"].reshape(*blob.shape)
    net.blobs["rois"].reshape(*rois.shape)
    net.blobs["masks"].reshape(*masks.shape)
    out = net.forward(data=np.ascontiguousarray(blob), rois=rois, masks=masks)
    ob = O.cfm_net_forward(Wt.make_sibling_weights("cfm", Wt.TINY_ARCH), blob, rois, masks)
    assert out["mask_prob"].shape == (24, 441)          # blobs_out['mask_prob'], TesterWrapper.py:399
    assert np.abs(out["mask_prob"] - ob["mask_prob"]).max() < 2 * TOL
    assert np.abs(out["seg_cls_prob"] - ob["seg_cls_prob"]).max() < 2 * TOL
    with pytest.raises(Exception):
        net.forward(data=blob, rois=rois)               # missing input


class _SiblingImdb:
    def __init__(self, out_dir):
        from oracle import oracle as O
        self.images = [O.synthetic_image(0, 224, 320), O.synthetic_image(1, 200, 300),
                       O.synthetic_image(2, 224, 320)]
        self.image_index = ["a", "b", "c"]
        self.num_classes = 21
        self.output_dir = out_dir
        self.seen = None
        rng = np.random.default_rng(77)
        self.props = []
        for im in self.images:
            H, W = im.shape[:2]
            b = np.round(util.random_boxes(30, int(rng.integers(1000)), W, H, smin=10, smax=min(H, W))).astype(np.float64)
            b[0] = [3, 3, 10, 40]                                    # narrower than 16: filtered out
            b[1] = [0, 0, W - 1, H - 1]                              # large: coarser pyramid level
            b[2] = [5, 5, W - 10, H - 8]
            m = rng.uniform(size=(30, 25, 31)) > 0.45               # arbitrary-size proposal masks
            self.props.append((b, m))

    def image_at(self, i):
        return self.images[i]

    def proposals_at(self, i):
        return self.props[i]

    def evaluate_detections(self, all_boxes, output_dir):
        self.seen = ("det", all_boxes)
        return "det-evaluated"

    def evaluate_segmentation(self, all_boxes, all_masks, output_dir):
        self.seen = ("seg", all_boxes, all_masks)
        return "seg-evaluated"


def test_tester_wrapper_det_task(tmp_path):
    import mnc_b200.lib as L
    L.install()
    from caffeWrapper.TesterWrapper import TesterWrapper
    from nms.nms_wrapper import nms
    from mnc_config import cfg
    from mnc_b200 import weights as Wt
    imdb = _SiblingImdb(str(tmp_path))
    tw = TesterWrapper(None, imdb, Wt.make_sibling_weights("faster_rcnn", Wt.TINY_ARCH), "det", max_batch=2)
    assert tw.get_result() == "det-evaluated" and (tmp_path / "detections.pkl").exists()
    _, dets = imdb.seen
    # the reference's per-image flow (TesterWrapper.py:85-143) on the same engine: per image the
    # 100 best rows per class; the class threshold ends at the (40 * num_images)-th best score
    # pushed (heap of size max_per_set, :113-118) and rows must beat it strictly (:126-129)
    per_image = [tw._detection_forward(im) for im in imdb.images]
    total = 0
    for j in range(1, 21):
        tops = [np.argsort(-sc[:, j])[:100] for sc, _ in per_image]
        pool = np.sort(np.concatenate([sc[t, j] for (sc, _), t in zip(per_image, tops)]))[::-1]
        thresh = pool[tw.max_per_set - 1] if len(pool) > tw.max_per_set else -np.inf
        for i, ((sc, bx), t) in enumerate(zip(per_image, tops)):
            t = t[sc[t, j] > thresh]
            d = np.hstack((bx[t, 4 * j:4 * j + 4], sc[t, j][:, None])).astype(np.float32)
            keep = nms(d, cfg.TEST.NMS) if len(d) else []
            got = np.asarray(dets[j][i]).reshape(-1, 5)
            # (batch-of-2 and batch-of-1 runs may pick different split-K plans: last-bit differences)
            assert got.shape == d[keep].shape and np.allclose(got, d[keep], rtol=1e-4, atol=1e-3)
            total += len(keep)
    assert total > 0
    with pytest.raises(ValueError):
        TesterWrapper(None, imdb, Wt.make_sibling_weights("faster_rcnn", Wt.TINY_ARCH), "seg")


def test_tester_wrapper_cfm_task_multiscale(tmp_path):
    import cv2
    import mnc_b200.lib as L
    L.install()
    from caffeWrapper.TesterWrapper import TesterWrapper
    from mnc_config import cfg
    from oracle import oracle as O
    from mnc_b200 import weights as Wt
    w = Wt.make_sibling_weights("cfm", Wt.TINY_ARCH)
    imdb = _SiblingImdb(str(tmp_path))
    saved = (cfg.TEST.SCALES, cfg.TEST.GROUP_SCALE, cfg.TEST.MAX_ROIS_GPU)
    cfg.TEST.SCALES, cfg.TEST.GROUP_SCALE, cfg.TEST.MAX_ROIS_GPU = (180, 260), 1, [2000, 7]
    try:
        tw = TesterWrapper(None, imdb, w, "cfm")
        masks, boxes, scores = tw.cfm_network_forward(0)
        # oracle flow for the same image: TesterWrapper.py:336-414 restated with oracle pieces
        im = imdb.images[0]
        pb, pm = imdb.props[0]
        keep = np.where((pb[:, 2] - pb[:, 0] + 1 >= 16) & (pb[:, 3] - pb[:, 1] + 1 >= 16))[0]
        pb, pm = pb[keep], pm[keep]
        m14 = np.stack([cv2.resize(m.astype(np.float64), (14, 14)) for m in pm])
        _, sc = O.prep_im_for_blob_cfm(im, cfg.TEST.SCALES)
        rois = O.pred_rois_for_blob(pb, sc)
        want_m, want_b, want_s = [], [], []
        for lvl in range(2):
            inds = np.where(rois[:, 0] == lvl)[0]
            if len(inds) == 0:
                continue
            r = rois[inds].copy()
            r[:, 0] -= r[:, 0].min()
            data, _ = O.prep_im_for_blob_cfm(im, cfg.TEST.SCALES[lvl:lvl + 1])
            ob = O.cfm_net_forward(w, data, r.astype(np.float32),
                                   (m14[inds].reshape(-1, 1, 14, 14).astype(np.float32) >= 0.4).astype(np.float32))
            want_m.append(ob["mask_prob"].reshape(-1, 1, 21, 21))
            want_s.append(ob["seg_cls_prob"])
            want_b.append(pb[inds])
        assert len(want_b) == 2                          # both pyramid levels are exercised
        assert np.array_equal(boxes, np.vstack(want_b).astype(np.float32))
        assert np.abs(masks - np.vstack(want_m)).max() < 3 * TOL
        assert np.abs(scores - np.vstack(want_s)).max() < 3 * TOL
        assert tw.get_result() == "seg-evaluated" and (tmp_path / "res_masks.pkl").exists()
        kind, all_boxes, all_masks = imdb.seen
        assert len(all_boxes) == 21 and all(len(all_boxes[j]) == 3 for j in range(21))
        n = sum(len(all_boxes[j][i]) for j in range(1, 21) for i in range(3))
        assert n > 0 and n == sum(len(all_masks[j][i]) for j in range(1, 21) for i in range(3))
    finally:
        cfg.TEST.SCALES, cfg.TEST.GROUP_SCALE, cfg.TEST.MAX_ROIS_GPU = saved
