"""Row 3 of SURVEY.md section 8f -- result rendering and the AP^r evaluator boundary:
`_convert_pred_to_image` (lib/utils/vis_seg.py:101-131), `get_vis_dict` (tools/demo.py:103-120),
`voc_eval_sds` steps 3-7 (lib/utils/voc_eval.py:216-283) and `get_segmentation_result`
(lib/caffeWrapper/TesterWrapper.py:149-214), device path against the numpy/cv2 oracle.

The label images and binary masks equal the float32 model of the device's resize rule
(tests/cv_resize.py) exactly.  Against the oracle, which thresholds OpenCV's own resize (a
dependency of the reference, whose bits depend on IPP and the CPU), a pixel may differ only where
the model's resized value lies within cv_resize.CV2_ULPS of 0.4f."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _random_pred(seed, n, W, H, edge_cases=True):
    from tests.util import random_boxes
    rng = np.random.default_rng(seed)
    boxes = random_boxes(n, seed, width=W, height=H, smin=4, smax=400)
    if edge_cases and n >= 6:
        boxes[0] = [0, 0, 40.4, 30.6]                  # touches the top-left corner: empty [-1:1] slices
        boxes[1] = [W - 30, H - 20, W + 15, H + 9]     # sticks out of the image: clipped
        boxes[2] = [100.5, 50.5, 100.5, 50.5]          # one pixel (round-half-even both ways)
        boxes[3] = [0.4, 200, 1.6, 260]                # x1 rounds to 0, two pixels wide
        boxes[4] = [300, 0.5, 420, 1.5]                # y1 rounds to 0 (half-to-even), y2 to 2
        boxes[5] = [-20, -10, 5, 8]                    # negative corner
    scores = rng.uniform(0.5, 1.0, n).astype(np.float32)
    masks = 1.0 / (1.0 + np.exp(-rng.normal(0, 2, (n, 21, 21)))).astype(np.float32)
    cls = rng.integers(1, 21, n)
    return {"image_name": "x", "cls_name": [int(c) for c in cls],
            "boxes": [np.concatenate([b, [s]]).astype(np.float32) for b, s in zip(boxes, scores)],
            "masks": [m for m in masks]}


def _check_images(got, model, oracle, close):
    assert np.array_equal(got, model)
    assert np.all(close[model != oracle])


def _model(pred, W, H):
    from tests import cv_resize as C
    n = len(pred["boxes"])
    boxes = np.array(pred["boxes"], np.float32).reshape(n, 5)[:, :4]
    masks = np.array(pred["masks"], np.float32).reshape(n, 21, 21)
    return C.paste(boxes, masks, np.array(pred["cls_name"], np.int32), H, W)


@pytest.mark.parametrize("seed,n,W,H", [(1, 40, 500, 375), (2, 12, 1000, 600), (3, 300, 640, 480),
                                        (4, 0, 64, 48), (5, 1, 33, 21)])
def test_convert_pred_to_image_matches_oracle(seed, n, W, H):
    import mnc_b200.lib as L
    L.install()
    from utils.vis_seg import _convert_pred_to_image, _get_voc_color_map
    from oracle import oracle as O
    pred = _random_pred(seed, n, W, H)
    inst, cls, bgr = _convert_pred_to_image(W, H, pred, want_bgr=True)
    w_inst, w_cls = O.convert_pred_to_image(W, H, pred)
    assert inst.shape == (H, W) and inst.dtype == w_inst.dtype
    m_inst, m_cls, m_bgr, close = _model(pred, W, H)
    _check_images(inst, m_inst, w_inst, close)
    _check_images(cls, m_cls, w_cls, close)
    assert np.array_equal(bgr, m_bgr)
    cmap = _get_voc_color_map()
    assert np.array_equal(cmap, O.voc_color_map())
    assert np.array_equal(bgr, cmap[cls][:, :, ::-1].astype(np.uint8))
    if n:
        assert inst.max() <= n and set(np.unique(cls)) <= set(pred["cls_name"]) | {0, 150}


def test_later_instances_overwrite_earlier_ones():
    """Two identical boxes with all-ones masks: the second wins everywhere, outline = 150."""
    import mnc_b200.lib as L
    L.install()
    from utils.vis_seg import _convert_pred_to_image
    pred = {"cls_name": [3, 7], "boxes": [np.array([10, 10, 29, 24, 0.9], np.float32)] * 2,
            "masks": [np.ones((21, 21), np.float32)] * 2}
    inst, cls = _convert_pred_to_image(64, 48, pred)
    assert np.all(inst[10:25, 10:30] == 2) and inst.sum() == 2 * 15 * 20
    assert np.all(cls[12:23, 12:28] == 7)
    assert np.all(cls[10:25, 9:11] == 150) and np.all(cls[9:11, 10:30] == 150)
    assert cls[8, 10] == 0 and cls[10, 8] == 0


def test_binarize_masks_matches_cv2():
    import cv2
    from mnc_b200 import ops
    from tests.util import random_boxes
    from tests import cv_resize as C
    rng = np.random.default_rng(7)
    n = 64
    rb = np.round(random_boxes(n, 7, 500, 375, smin=1, smax=300)).astype(np.int32)
    masks = rng.uniform(0, 1, (n, 21, 21)).astype(np.float32)
    masks[:8] = (masks[:8] >= 0.4)        # binary inputs, as `_reformat_result` stores them
    packed, off = ops.binarize_masks(torch.from_numpy(rb).cuda(), torch.from_numpy(masks).cuda())
    packed = packed.cpu().numpy()
    m_packed, m_off = C.binarize_masks(rb, masks)
    assert np.array_equal(off, m_off) and np.array_equal(packed[:off[-1]], m_packed)
    for i in range(n):
        w, h = rb[i, 2] - rb[i, 0] + 1, rb[i, 3] - rb[i, 1] + 1
        want = cv2.resize(masks[i], (int(w), int(h))) >= 0.4
        got = packed[off[i]:off[i + 1]].reshape(h, w).astype(bool)
        close = C.in_cv2_band(C.box_resize(masks[i], *rb[i]))
        assert np.all(close[got != want]), i
    assert off[-1] == sum((rb[:, 2] - rb[:, 0] + 1) * (rb[:, 3] - rb[:, 1] + 1))


def _synthetic_gt_and_preds(seed, n_img=6, W=320, H=240):
    """Ground-truth instances (random rectangles-with-holes) and predictions, some of which are
    jittered copies of ground truth (true positives / duplicates), some noise."""
    rng = np.random.default_rng(seed)
    names = ["im%03d" % i for i in range(n_img)]
    gt, boxes_pkl, masks_pkl = {}, [], []
    for k, name in enumerate(names):
        g = []
        for _ in range(rng.integers(0, 4)):
            x1, y1 = rng.integers(0, W - 60), rng.integers(0, H - 60)
            w, h = rng.integers(20, 60), rng.integers(20, 60)
            m = rng.uniform(0, 1, (h, w)) > 0.15
            g.append({"mask_bound": np.array([x1, y1, x1 + w - 1, y1 + h - 1]), "mask": m})
        if g or k % 2 == 0:
            gt[name] = g          # some images are absent from the cache altogether
        dets, segs = [], []
        for gi in g:
            for _ in range(rng.integers(1, 3)):
                jit = rng.integers(-4, 5, 4)
                b = np.clip(gi["mask_bound"] + jit, 0, [W - 1, H - 1, W - 1, H - 1]).astype(np.float64)
                if b[2] < b[0] or b[3] < b[1]:
                    continue
                dets.append(np.concatenate([b + rng.uniform(-0.4, 0.4, 4), [rng.uniform(0.3, 1)]]))
                segs.append(rng.uniform(0.3, 1.0, (1, 21, 21)))
        for _ in range(rng.integers(0, 3)):
            x1, y1 = rng.integers(0, W - 50), rng.integers(0, H - 50)
            dets.append(np.array([x1, y1, x1 + rng.integers(5, 49), y1 + rng.integers(5, 49), rng.uniform(0, 1)], float))
            segs.append(rng.uniform(0, 1, (1, 21, 21)))
        boxes_pkl.append(np.array(dets, dtype=np.float32).reshape(-1, 5))
        masks_pkl.append(np.array(segs, dtype=np.float32).reshape(-1, 1, 21, 21))
    return names, gt, boxes_pkl, masks_pkl


@pytest.mark.parametrize("seed", [11, 12, 13])
def test_eval_sds_matches_oracle(seed):
    import mnc_b200.lib as L
    L.install()
    from utils.voc_eval import eval_sds_arrays
    from oracle import oracle as O
    names, gt, boxes_pkl, masks_pkl = _synthetic_gt_and_preds(seed)
    for thr in (0.5, 0.7):
        got = eval_sds_arrays(boxes_pkl, masks_pkl, names, gt, ov_thresh=thr)
        want = O.eval_sds(boxes_pkl, masks_pkl, names, gt, ov_thresh=thr)
        assert got == pytest.approx(want, abs=1e-12)
    assert 0.0 < O.eval_sds(boxes_pkl, masks_pkl, names, gt) <= 1.0


class _Imdb:
    """Duck-typed imdb over in-memory synthetic images (two sizes, so bucketing is exercised)."""
    def __init__(self, out_dir):
        from oracle import oracle as O
        self.images = [O.synthetic_image(0, 224, 320), O.synthetic_image(1, 200, 300),
                       O.synthetic_image(2, 224, 320)]
        self.image_index = ["a", "b", "c"]
        self.num_classes = 21
        self.output_dir = out_dir
        self.seen = None

    def image_at(self, i):
        return self.images[i]

    def evaluate_segmentation(self, all_boxes, all_masks, output_dir):
        self.seen = (all_boxes, all_masks, output_dir)
        return "evaluated"


def test_tester_wrapper_seg_task_equals_per_image_reference_flow(tmp_path):
    """Batched/bucketed `get_segmentation_result` == the reference's per-image flow
    (im_detect -> gpu_mask_voting) built from the same mirrored functions; pickles written."""
    import pickle
    import mnc_b200.lib as L
    L.install()
    from caffeWrapper.TesterWrapper import TesterWrapper
    from transform.mask_transform import gpu_mask_voting
    from mnc_b200 import weights as Wt
    w = Wt.make_weights(Wt.TINY_ARCH)
    imdb = _Imdb(str(tmp_path))
    tw = TesterWrapper(None, imdb, w, "seg", max_batch=2)
    assert tw.get_result() == "evaluated"
    all_boxes, all_masks, out_dir = imdb.seen
    assert len(all_boxes) == 21 and len(all_boxes[1]) == 3
    with open(tmp_path / "res_boxes.pkl", "rb") as f:
        assert len(pickle.load(f)) == 21
    assert (tmp_path / "res_masks.pkl").exists()
    total = 0
    for i, im in enumerate(imdb.images):
        boxes, masks, scores, valid, _ = tw.detector.im_detect_images(im[None])
        ok = valid[0].astype(bool)
        rm, rb = gpu_mask_voting(masks[0][ok], boxes[0][ok], scores[0][ok], 21, 100, im.shape[1], im.shape[0])
        for j in range(1, 21):
            assert np.array_equal(np.asarray(all_boxes[j][i], np.float32).reshape(-1, 5),
                                  np.asarray(rb[j - 1], np.float32).reshape(-1, 5))
            assert np.array_equal(np.asarray(all_masks[j][i]).reshape(-1, 1, 21, 21),
                                  np.asarray(rm[j - 1]).reshape(-1, 1, 21, 21))
            total += len(rb[j - 1])
    assert total > 0
    # second call reads the pickles back instead of recomputing (TesterWrapper.py:54-58)
    imdb.seen = None
    assert tw.get_result() == "evaluated" and imdb.seen is not None


def test_select_for_display_equals_get_vis_dict():
    import mnc_b200.lib as L
    L.install()
    from utils.vis_seg import get_vis_dict, _convert_pred_to_image
    from caffeWrapper.TesterWrapper import unpack_voting
    from mnc_b200 import ops
    from tests.util import random_boxes
    rng = np.random.default_rng(21)
    nb, H, W = 200, 375, 500
    boxes = torch.from_numpy(random_boxes(nb, 21, W, H)).cuda()[None]
    masks = torch.from_numpy(1 / (1 + np.exp(-rng.normal(0, 2, (1, nb, 1, 21, 21)))).astype(np.float32)).cuda()
    logits = rng.normal(0, 2.5, (1, nb, 21))
    scores = torch.from_numpy((np.exp(logits) / np.exp(logits).sum(-1, keepdims=True)).astype(np.float32)).cuda()
    hw = torch.tensor([[H, W]], dtype=torch.int32).cuda()
    vote = ops.mask_voting(boxes, masks, scores, hw, max_per_image=100)
    b, m, c, cnt = ops.select_for_display(vote, vis_thresh=0.5)
    inst, cls = ops.paste_instances(b, m, c, cnt, H, W)
    (list_mask, list_box), = unpack_voting(vote, 21)
    pred = get_vis_dict(list_box, list_mask, "x", ["c%d" % i for i in range(20)], vis_thresh=0.5)
    assert len(pred["boxes"]) == int(cnt[0]) and int(cnt[0]) > 0
    w_inst, w_cls = _convert_pred_to_image(W, H, pred)
    assert np.array_equal(inst[0].cpu().numpy(), w_inst) and np.array_equal(cls[0].cpu().numpy(), w_cls)
