"""The six device kernels that restate cv2.resize(INTER_LINEAR) -- prep_image_kernel,
paste_instances_kernel, binarize_masks_kernel, the mask targets of StageBridgeLayer and
ProposalTargetLayer (mask_target_row) and mask_layer_train_kernel -- equal the float32 model of
tests/cv_resize.py bit for bit, on masks with many samples at 0.4f or 1-2 ulps from it and on
seeded random inputs.  Every output buffer starts as a sentinel (0xFF bytes: NaN floats, -1 ints,
255 bytes), so an element a kernel leaves unwritten cannot pass for a 0."""
import numpy as np
import pytest
import torch

from tests import cv_resize as C

pytestmark = pytest.mark.gpu
F32 = np.float32


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _poison():
    """Leave the caching allocator's free blocks full of 0xFF bytes: the outputs the wrappers
    allocate next (torch.empty) start from the sentinel."""
    torch.cuda.synchronize()
    blocks = [torch.empty(64 << 20, dtype=torch.uint8, device="cuda")]
    blocks += [torch.empty(256 << 10, dtype=torch.uint8, device="cuda") for _ in range(48)]
    blocks += [torch.empty(4 << 10, dtype=torch.uint8, device="cuda") for _ in range(64)]
    for b in blocks:
        b.fill_(255)
    torch.cuda.synchronize()
    del blocks


@pytest.mark.parametrize("B,H,W,scale", [(2, 375, 500, 1.6), (1, 47, 61, 1.7), (1, 20, 30, 0.6),
                                         (1, 600, 1000, 1.0), (2, 33, 21, 21 / 33)])
def test_prep_blob_exact(B, H, W, scale):
    from mnc_b200 import ops
    rng = np.random.default_rng(H * W)
    im = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
    want = C.prep(im, scale, ops.PIXEL_MEANS)
    out = torch.full(want.shape, float("nan"), dtype=torch.float32, device="cuda")
    got = ops.prep_images(_cuda(im), scale, out=out).cpu().numpy()
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


def _paste_check(boxes, masks, cls, H, W):
    from mnc_b200 import ops
    _poison()
    n = len(boxes)
    inst, clsi, bgr = ops.paste_instances(_cuda(boxes[None]), _cuda(masks[None]), _cuda(cls[None]),
                                          _cuda(np.array([n], np.int32)), H, W, want_bgr=True)
    w_inst, w_cls, w_bgr, _ = C.paste(boxes, masks, cls, H, W)
    assert np.array_equal(inst[0].cpu().numpy(), w_inst)
    assert np.array_equal(clsi[0].cpu().numpy(), w_cls)
    assert np.array_equal(bgr[0].cpu().numpy(), w_bgr)


@pytest.mark.parametrize("seed", [1, 2])
def test_paste_instances_ties(seed):
    groups, H, W = C.paste_fixture(seed)
    for M, boxes, masks, cls in groups:
        _paste_check(boxes, masks, cls, H, W)


def test_paste_instances_random():
    from tests.util import random_boxes
    rng = np.random.default_rng(31)
    H, W, n = 375, 500, 60
    boxes = random_boxes(n, 31, width=W, height=H, smin=1, smax=300).astype(F32)
    boxes[:3] = [[W - 40, H - 30, W + 20, H + 9], [-10, -5, 30, 12], [7.5, 8.5, 7.5, 8.5]]
    masks = (1 / (1 + np.exp(-rng.normal(0, 2, (n, 21, 21))))).astype(F32)
    _paste_check(boxes, masks, rng.integers(1, 21, n).astype(np.int32), H, W)


def _binarize_check(rb, masks):
    from mnc_b200 import ops
    _poison()
    packed, off = ops.binarize_masks(_cuda(rb), _cuda(masks))
    want, w_off = C.binarize_masks(rb, masks)
    assert np.array_equal(off, w_off)
    assert np.array_equal(packed.cpu().numpy()[:w_off[-1]], want)


@pytest.mark.parametrize("seed", [2, 5])
def test_binarize_masks_ties(seed):
    for M, rb, masks in C.binarize_fixture(seed):
        _binarize_check(rb, masks)


def test_binarize_masks_random():
    from tests.util import random_boxes
    rng = np.random.default_rng(7)
    rb = np.round(random_boxes(64, 7, 500, 375, smin=1, smax=300)).astype(np.int32)
    masks = rng.uniform(0, 1, (64, 21, 21)).astype(F32)
    _binarize_check(rb, masks)


def _stage_bridge(case, gm, bbox_thresh=0.5):
    from mnc_b200 import ops
    _poison()
    out = ops.stage_bridge_train(
        _cuda(case["rois"]), _cuda(case["bbox_pred"]), _cuda(case["seg_cls_prob"]),
        _cuda(case["gt_boxes"]), _cuda(gm), _cuda(case["im_info"]), _cuda(case["mask_info"]),
        bbox_thresh=bbox_thresh)
    return ({k: out[k].cpu().numpy() for k in ("gt_mask_info", "mask_targets", "mask_weight")},
            int(out["state"][-1]))


def _with_ties(rng, info, nfg, gm):
    """Ties in the mask targets of the foreground rows, placed in (a copy of) the gt masks."""
    gm = gm.copy()
    lock = np.zeros(gm.shape, bool)
    for p in range(nfg):
        C.mask_target_ties(rng, info[p], gm, lock, max_ties=24)
    return gm


def _fixed_geometry_case():
    """The geometries of C.MT_EX as StageBridge rows: im_scale 1 and zero deltas decode RoI
    (x1, y1, x2, y2) to (x1, y1, x2 + 1, y2 + 1), clipped; bbox_thresh 0 makes every row
    foreground, so every geometry gets a target."""
    H, W = 160, 200
    ex = np.array([e for _, e in C.MT_EX], np.float64)
    rois = np.zeros((len(ex), 5), F32)
    rois[:, 1:] = ex - [0, 0, 1, 1]
    rois[:, 3] = np.maximum(rois[:, 3], rois[:, 1])
    rois[:, 4] = np.maximum(rois[:, 4], rois[:, 2])
    C_ = 21
    seg = np.full((len(ex), C_), F32(1.0 / C_))
    gt_boxes = np.array([list(g) + [3 + k] for k, g in enumerate(C.MT_GT)], F32)
    _, _, gm = C.mask_target_fixture(11)
    return dict(rois=rois, bbox_pred=np.zeros((len(ex), 4 * C_), F32), seg_cls_prob=seg,
                gt_boxes=gt_boxes, im_info=np.array([H, W, 1.0], F32),
                mask_info=np.array([[100, 100], [80, 75]], np.int32)), gm


def _bridge_cases():
    from oracle import oracle_train as T
    rng = np.random.default_rng(0)
    for seed in (40, 41, 42):
        case = T.make_case(seed, **(dict(H=480, W=640, im_scale=1.0, n=40, G=4) if seed % 2 else
                                    dict(n=48, G=5)))
        gm = case.pop("gt_masks").astype(F32) * rng.uniform(0.45, 1.0, case["mask_info"].shape[:1] +
                                                             (1, 1)).astype(F32)
        yield case, gm, 0.5
    case, gm = _fixed_geometry_case()
    yield case, gm, 0.0


def test_stage_bridge_mask_targets_and_mask_layer_ties():
    """Two passes: the first gives the rows' gt_mask_info (independent of the mask values), ties
    are then placed in the gt masks (targets) and in the predictions (MaskLayer) of those rows."""
    from mnc_b200 import ops
    from oracle import oracle_train as T
    rng = np.random.default_rng(1)
    total = 0
    for case, gm, bt in _bridge_cases():
        first, nfg = _stage_bridge(case, gm, bt)
        assert nfg > 0
        info = first["gt_mask_info"]
        gm_t = _with_ties(rng, info, nfg, gm)
        got, nfg2 = _stage_bridge(case, gm_t, bt)
        assert nfg2 == nfg and np.array_equal(got["gt_mask_info"], info)
        wt, ww = C.mask_targets(info, nfg, gm_t)
        assert np.array_equal(got["mask_targets"].reshape(wt.shape), wt)
        assert np.array_equal(got["mask_weight"].reshape(ww.shape), ww)
        total += int(wt.sum())
        # MaskLayer on these rows: predictions near the targets, ties in their ex-box resizes
        M = 21
        preds = T.mask_predictions(nfg, wt, info).reshape(len(info), M, M)
        for p in range(nfg):
            ex1, ey1, ex2, ey2 = (int(np.rint(v)) for v in info[p, 4:8])
            ew, eh = ex2 - ex1 + 1, ey2 - ey1 + 1
            C.place_ties(rng, preds[p], np.ones((M, M), bool), ew, eh, M / ew, M / eh, max_ties=24)
        preds = preds.reshape(len(info), M * M)
        for t in [0.5] + C.iou_thresholds(preds, gm_t, info)[:16]:
            _poison()
            lab = ops.mask_layer_train(_cuda(preds), _cuda(gm_t), _cuda(info), fg_seg_thresh=t)
            assert np.array_equal(lab.cpu().numpy(), C.mask_layer(preds, gm_t, info, t)), t
    assert total > 0


@pytest.mark.parametrize("seed", [4, 5])
def test_mask_layer_ties(seed):
    """The fixed-geometry MaskLayer rows (2x / 4x downscales, 1-wide boxes ...), with fg_seg_thresh
    at 0.5 and on each row's IoU edge."""
    from mnc_b200 import ops
    gm, groups = C.mask_layer_fixture(seed)
    for M, preds, info in groups:
        for t in [0.5] + C.iou_thresholds(preds, gm, info):
            _poison()
            lab = ops.mask_layer_train(_cuda(preds), _cuda(gm), _cuda(info), fg_seg_thresh=t)
            assert np.array_equal(lab.cpu().numpy(), C.mask_layer(preds, gm, info, t)), (M, t)


def test_proposal_target_mask_targets_ties():
    from mnc_b200 import ops
    from oracle import oracle_rpn_train as R
    rng = np.random.default_rng(2)
    for seed in (60, 61):
        H, W, info_ = ((38, 63, (600, 1000, 1.6)), (30, 50, (480, 800, 1.0)))[seed % 2]
        cs = R.make_case(seed, H, W, info_, 6, 200, scores=False)
        keys = rng.integers(0, 2 ** 32, (3, 206), dtype=np.uint64).astype(np.uint32)
        gm = cs["gt_masks"].astype(F32) * F32(0.8)

        def run(g):
            _poison()
            out = ops.proposal_target(_cuda(cs["rpn_rois"]), _cuda(cs["rois_index"]),
                                      _cuda(cs["gt_boxes"]), _cuda(g), _cuda(cs["mask_info"]),
                                      _cuda(cs["im_info"].ravel()),
                                      _cuda(keys.view(np.int32)))
            return ({k: out[k].cpu().numpy() for k in ("gt_masks_info", "mask_targets", "mask_weight")},
                    out["counts"].cpu().numpy())
        first, cnt = run(gm)
        K, nfg = int(cnt[0]), int(cnt[3])
        assert nfg > 0
        info = first["gt_masks_info"][:K]
        gm_t = _with_ties(rng, info, nfg, gm)
        got, cnt2 = run(gm_t)
        assert np.array_equal(cnt2, cnt) and np.array_equal(got["gt_masks_info"][:K], info)
        wt, ww = C.mask_targets(info, nfg, gm_t)
        assert np.array_equal(got["mask_targets"][:K].reshape(wt.shape), wt)
        assert np.array_equal(got["mask_weight"][:K].reshape(ww.shape), ww)
        assert np.all(got["mask_targets"][K:] == 0) and np.all(got["mask_weight"][K:] == 0)
