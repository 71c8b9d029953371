"""numpy restatement of the TRAIN phase of the two cascade bridge layers, the checker of
mnc_b200/csrc/train_bridge.cu:
  StageBridgeLayer.forward_train   lib/pylayer/stage_bridge_layer.py:131-235
  StageBridgeLayer.backward        stage_bridge_layer.py:82-129
  MaskLayer.forward_train          lib/pylayer/mask_layer.py:56-93
  MaskLayer.backward               mask_layer.py:50-54
with the helpers they call (lib/transform/bbox_transform.py:39-203, mask_transform.py:16-80).
Every array keeps the dtype the reference gives it: the decoded boxes are float64 (the deltas are
copied into a float64 array, :153), the gt-side widths and centres of bbox_transform are float32,
and so are the gt boxes divided by im_scale (float32 array / Python float).  cv2 is the reference's
own dependency (INTER_LINEAR, as there).  The reference's Python 2 / numpy 1.x float indices are
taken as the integer they truncate to."""
import numpy as np

from oracle import oracle as O

# cfg.TRAIN defaults, lib/mnc_config.py:63-69,105
BBOX_NORMALIZE_MEANS = (0.0, 0.0, 0.0, 0.0)
BBOX_NORMALIZE_STDS = (0.1, 0.1, 0.2, 0.2)
BBOX_INSIDE_WEIGHTS = (1.0, 1.0, 1.0, 1.0)


def _bbox_transform(ex_rois, gt_rois):
    """bbox_transform.py:39-61: ex_rois float64, gt_rois float32."""
    ex_widths = ex_rois[:, 2] - ex_rois[:, 0] + 1.0
    ex_heights = ex_rois[:, 3] - ex_rois[:, 1] + 1.0
    ex_ctr_x = ex_rois[:, 0] + 0.5 * ex_widths
    ex_ctr_y = ex_rois[:, 1] + 0.5 * ex_heights
    gt_widths = gt_rois[:, 2] - gt_rois[:, 0] + 1.0
    gt_heights = gt_rois[:, 3] - gt_rois[:, 1] + 1.0
    gt_ctr_x = gt_rois[:, 0] + 0.5 * gt_widths
    gt_ctr_y = gt_rois[:, 1] + 0.5 * gt_heights
    dx = (gt_ctr_x - ex_ctr_x) / ex_widths
    dy = (gt_ctr_y - ex_ctr_y) / ex_heights
    dw = np.log(gt_widths / ex_widths)
    dh = np.log(gt_heights / ex_heights)
    return np.vstack((dx, dy, dw, dh)).transpose()


def _intersect_mask(ex_box, gt_box, gt_mask, mask_size, binarize_thresh):
    """mask_transform.py:49-80."""
    import cv2
    x1, y1 = max(ex_box[0], gt_box[0]), max(ex_box[1], gt_box[1])
    x2, y2 = min(ex_box[2], gt_box[2]), min(ex_box[3], gt_box[3])
    if x1 > x2 or y1 > y2:
        return np.zeros((mask_size, mask_size), dtype=bool)
    w, h = x2 - x1 + 1, y2 - y1 + 1
    ex_sy, ex_sx = y1 - ex_box[1], x1 - ex_box[0]
    gt_sy, gt_sx = y1 - gt_box[1], x1 - gt_box[0]
    inter = gt_mask[gt_sy:gt_sy + h, gt_sx:gt_sx + w]
    t = np.zeros((ex_box[3] - ex_box[1] + 1, ex_box[2] - ex_box[0] + 1))
    t[ex_sy:ex_sy + h, ex_sx:ex_sx + w] = inter
    t = cv2.resize(t.astype(np.float32), (mask_size, mask_size))
    return t >= binarize_thresh


def stage_bridge_forward(rois, bbox_pred, seg_cls_prob, gt_boxes, gt_masks, im_info, mask_info,
                         num_classes, normalize=True, means=BBOX_NORMALIZE_MEANS,
                         stds=BBOX_NORMALIZE_STDS, inside_weights=BBOX_INSIDE_WEIGHTS,
                         bbox_thresh=0.5, mask_size=21, binarize_thresh=0.4):
    """-> dict of the eight tops (float32: rois (K,5), labels (K,), mask_targets / mask_weight
    (K,1,M,M), gt_mask_info (K,12), bbox_targets / inside / outside weights (K,4C)) and the state
    the backward reads: keep_inds, reg_labels (n,), clip_keep (indices into the K rows), nfg.
    `normalize` is cfg.TRAIN.BBOX_NORMALIZE_TARGETS_PRECOMPUTED."""
    rois = np.asarray(rois, np.float32).reshape(-1, 5)
    bbox_pred = np.asarray(bbox_pred, np.float32)
    seg = np.asarray(seg_cls_prob, np.float32)
    gt_boxes = np.asarray(gt_boxes, np.float32)
    im_info = np.asarray(im_info, np.float32).reshape(-1)
    mask_info = np.asarray(mask_info).astype(np.int64)
    n = rois.shape[0]
    reg = seg[:, 1:].argmax(axis=1) + 1                                     # :145
    art = np.zeros((n, 4))                                                  # :153-156
    for i in range(n):
        art[i, :] = bbox_pred[i, 4 * reg[i]:4 * (reg[i] + 1)]
    all_rois = np.zeros((n, 5))                                             # :158-160
    if n:
        all_rois[:, 1:5] = O.bbox_transform_inv(rois[:, 1:5], art)
    zeros = np.zeros((gt_boxes.shape[0], 1), dtype=gt_boxes.dtype)
    all_rois = np.vstack((all_rois, np.hstack((zeros, gt_boxes[:, :-1]))))  # :161-164
    all_rois[:, 1:5], clip_keep = O.clip_boxes(all_rois[:, 1:5], im_info[:2])   # :165

    # _sample_output :187-235
    overlaps = O.bbox_overlaps(all_rois[:, 1:5], gt_boxes[:, :4])
    gt_assignment = overlaps.argmax(axis=1)
    max_overlaps = overlaps.max(axis=1)
    labels = gt_boxes[gt_assignment, 4]
    fg_inds = np.where(max_overlaps >= bbox_thresh)[0]
    bg_inds = np.where(max_overlaps < bbox_thresh)[0]
    keep_inds = np.append(fg_inds, bg_inds).astype(int)
    labels = labels[keep_inds]
    labels[len(fg_inds):] = 0
    rois_out = all_rois[keep_inds]
    targets = _bbox_transform(rois_out[:, 1:5], gt_boxes[gt_assignment[keep_inds], :4])
    if normalize:
        targets = (targets - np.array(means)) / np.array(stds)
    data = np.hstack((labels[:, np.newaxis], targets.astype(np.float32))).astype(np.float32)
    K = len(keep_inds)
    bbox_targets = np.zeros((K, 4 * num_classes), dtype=np.float32)      # :181-203
    bbox_inside = np.zeros(bbox_targets.shape, dtype=np.float32)
    for ind in np.where(data[:, 0] > 0)[0]:
        start = int(4 * data[ind, 0])
        bbox_targets[ind, start:start + 4] = data[ind, 1:]
        bbox_inside[ind, start:start + 4] = inside_weights
    bbox_outside = np.array(bbox_inside > 0).astype(np.float32)

    im_scale = float(im_info[2])
    scaled_rois = rois_out[:, 1:5] / im_scale
    scaled_gt = gt_boxes[:, :4] / im_scale
    masks = np.zeros((K, 1, mask_size, mask_size))
    info = np.zeros((K, 12))
    info[len(fg_inds):, :] = -1
    for i, val in enumerate(fg_inds):
        a = gt_assignment[val]
        gt_box = np.around(scaled_gt[a]).astype(int)
        ex_box = np.around(scaled_rois[i]).astype(int)
        gt_mask = np.asarray(gt_masks[a])[0:mask_info[a, 0], 0:mask_info[a, 1]]
        masks[i, ...] = _intersect_mask(ex_box, gt_box, gt_mask, mask_size, binarize_thresh)
        info[i, 0] = a
        info[i, 1:3] = mask_info[a]
        info[i, 3] = labels[i]
        info[i, 4:8] = ex_box
        info[i, 8:12] = gt_box
    mask_weight = np.zeros((K, 1, mask_size, mask_size))
    mask_weight[0:len(fg_inds)] = 1
    f = lambda x: x.astype(np.float32)
    return {"rois": f(rois_out), "labels": f(labels), "mask_targets": f(masks),
            "mask_weight": f(mask_weight), "gt_mask_info": f(info), "bbox_targets": f(bbox_targets),
            "bbox_inside_weights": bbox_inside, "bbox_outside_weights": bbox_outside,
            "keep_inds": keep_inds, "reg_labels": reg, "clip_keep": clip_keep,
            "nfg": len(fg_inds), "max_overlaps": max_overlaps}


def stage_bridge_backward(top_diff, state, rois, bbox_pred, clip_thresh=0.0, want_rois=True,
                          want_bbox=True):
    """stage_bridge_layer.py:82-129.  clip_thresh 0 means use_clip off.  -> (rois_diff (n,5),
    bbox_pred_diff (n,4C)); an output not wanted is None."""
    rois = np.asarray(rois, np.float32).reshape(-1, 5)
    deltas = np.asarray(bbox_pred, np.float32)
    top_diff = np.asarray(top_diff, np.float32)
    keep, reg, clip_keep = state["keep_inds"], state["reg_labels"], state["clip_keep"]
    d1, d2, d3, d4 = (top_diff[:, c] for c in (1, 2, 3, 4))
    W_old = rois[:, 2] - rois[:, 0]
    H_old = rois[:, 3] - rois[:, 1]
    rd = bd = None
    if want_rois:
        rd = np.zeros(rois.shape, np.float32)
        for ind, i in enumerate(keep):
            if i >= rd.shape[0] or reg[i] == 0:
                continue
            l4 = 4 * reg[i]
            rd[i, 1] = d1[ind]
            rd[i, 2] = d2[ind]
            rd[i, 3] = d3[ind] * (deltas[i, l4] + np.exp(deltas[i, l4 + 2]))
            rd[i, 4] = d4[ind] * (deltas[i, l4 + 1] + np.exp(deltas[i, l4 + 3]))
    if want_bbox:
        bd = np.zeros(deltas.shape, np.float32)
        for ind, i in enumerate(keep):
            if i >= bd.shape[0] or i not in clip_keep or reg[i] == 0:
                continue
            l4 = 4 * reg[i]
            bd[i, l4] = d1[ind] * W_old[i]
            bd[i, l4 + 1] = d2[ind] * H_old[i]
            bd[i, l4 + 2] = d3[ind] * np.exp(deltas[i, l4 + 2]) * W_old[i]
            bd[i, l4 + 3] = d4[ind] * np.exp(deltas[i, l4 + 3]) * H_old[i]
            if clip_thresh:
                bd[i, l4:l4 + 4] = np.minimum(np.maximum(bd[i, l4:l4 + 4], -clip_thresh),
                                              clip_thresh)
    return rd, bd


def mask_layer_forward(mask_pred, gt_masks, gt_masks_info, mask_size=21, binarize_thresh=0.4,
                       fg_seg_thresh=0.5):
    """mask_layer.py:56-93 -> labels (N,1) float32 (mask_proposal is a reshape of mask_pred)."""
    import cv2
    mask_pred = np.asarray(mask_pred, np.float32)
    info_all = np.asarray(gt_masks_info, np.float32).reshape(-1, 12)
    N = mask_pred.shape[0]
    top_label = np.zeros((info_all.shape[0], 1))
    for i in range(N):
        if info_all[i][0] == -1:
            continue
        info = info_all[i].astype(np.int64)                 # numpy 1.x float indices truncate
        gt_mask = np.asarray(gt_masks[info[0]])[0:info[1], 0:info[2]]
        ex_mask = mask_pred[i].reshape((mask_size, mask_size))
        ex_box = np.round(info_all[i][4:8]).astype(int)
        gt_box = np.round(info_all[i][8:12]).astype(int)
        ex_mask = cv2.resize(ex_mask.astype(np.float32),
                             (ex_box[2] - ex_box[0] + 1, ex_box[3] - ex_box[1] + 1))
        ex_mask = ex_mask >= binarize_thresh
        iou = O.mask_overlap(ex_box, gt_box, ex_mask, gt_mask)
        top_label[i][0] = 0 if iou < fg_seg_thresh else info_all[i][3]
    return top_label.astype(np.float32)


def mask_layer_backward(top_diff, labels):
    """mask_layer.py:50-54: rows with a positive label copy the top diff, the rest are 0."""
    top_diff = np.asarray(top_diff, np.float32)
    g = top_diff.reshape(top_diff.shape[0], -1)
    out = np.zeros(g.shape, np.float32)
    pos = np.where(np.asarray(labels).reshape(-1) > 0)[0]
    out[pos] = g[pos]
    return out


# --------------------------------------------------------------------------- synthetic inputs
def make_case(seed, H=600, W=1000, im_scale=1.6, n=64, G=3, C=21, n_ties=3):
    """One image's StageBridgeLayer bottoms, as the training net feeds them: gt boxes at integer
    positions of the original image scaled by im_scale, gt masks (G,Hm,Wm) bool of the original
    box size (mask_info (G,2) = their height, width; one mask zero over its lower right quarter),
    RoIs that are jittered gt boxes or random, small deltas with a few rows that decode out of the
    image, and seg_cls_prob rows of which `n_ties` tie between two classes at their maximum."""
    rng = np.random.default_rng(seed)
    Ho, Wo = int(H / im_scale), int(W / im_scale)
    gw = rng.integers(12, max(13, Wo // 3), G)
    gh = rng.integers(12, max(13, Ho // 3), G)
    gx = rng.integers(0, Wo - gw)
    gy = rng.integers(0, Ho - gh)
    if G:
        gx[0] = 0                                    # one gt box on the image edge
    orig = np.stack([gx, gy, gx + gw - 1, gy + gh - 1], 1)
    gt_boxes = np.zeros((G, 5), np.float32)
    gt_boxes[:, :4] = orig * np.float32(im_scale)
    gt_boxes[:, 4] = rng.integers(1, C, G)
    mask_info = np.stack([gh, gw], 1).astype(np.int32)
    Hm, Wm = int(gh.max()) if G else 1, int(gw.max()) if G else 1
    gt_masks = np.zeros((G, Hm, Wm), bool)
    for g in range(G):
        yy, xx = np.mgrid[0:gh[g], 0:gw[g]]
        r = ((yy - gh[g] / 2) / (gh[g] / 2)) ** 2 + ((xx - gw[g] / 2) / (gw[g] / 2)) ** 2
        gt_masks[g, :gh[g], :gw[g]] = (r < 0.8) ^ (rng.random((gh[g], gw[g])) < 0.05)
    if G > 1:
        gt_masks[1, gh[1] // 2:, gw[1] // 2:] = False
    rois = np.zeros((n, 5), np.float32)
    for i in range(n):
        if G and i < (3 * n) // 5:
            b = gt_boxes[i % G, :4].astype(np.float64)
            w, h = b[2] - b[0], b[3] - b[1]
            b = b + rng.normal(0, 0.12, 4) * np.array([w, h, w, h])
        else:
            cx, cy = rng.uniform(0, W), rng.uniform(0, H)
            w, h = np.exp(rng.uniform(np.log(16), np.log(400), 2))
            b = np.array([cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2])
        b[0::2] = np.clip(b[0::2], 0, W - 1)
        b[1::2] = np.clip(b[1::2], 0, H - 1)
        rois[i, 1:] = [min(b[0], b[2]), min(b[1], b[3]), max(b[0], b[2]), max(b[1], b[3])]
    bbox_pred = rng.normal(0, 0.1, (n, 4 * C)).astype(np.float32)
    bbox_pred[n - 4:, :] += np.float32(0.8)          # wider and shifted: these leave the image
    z = rng.normal(0, 1.0, (n, C))
    seg = np.exp(z - z.max(1, keepdims=True))
    seg = (seg / seg.sum(1, keepdims=True)).astype(np.float32)
    for i in range(min(n_ties, n)):
        a, b2 = sorted(rng.choice(np.arange(1, C), 2, replace=False))
        seg[i, a] = seg[i, b2] = seg[i].max() + np.float32(0.125)
    im_info = np.array([H, W, im_scale], np.float32)
    return dict(rois=rois, bbox_pred=bbox_pred, seg_cls_prob=seg, gt_boxes=gt_boxes,
                gt_masks=gt_masks, im_info=im_info, mask_info=mask_info)


def mask_predictions(seed, mask_targets, info):
    """MaskLayer bottoms derived from StageBridge's outputs: predictions close to the targets in
    rows of low noise (labels kept) and noisy in the others (labels zeroed by FG_SEG_THRESH)."""
    rng = np.random.default_rng(seed)
    K = mask_targets.shape[0]
    t = mask_targets.reshape(K, -1).astype(np.float32)
    sigma = np.where(np.arange(K) % 3 == 2, 0.9, 0.05)[:, None]
    z = 6.0 * (t - 0.5) + rng.normal(0, 1, t.shape) * 6.0 * sigma
    return (1.0 / (1.0 + np.exp(-z))).astype(np.float32)


def resize_values(mask_pred, info, mask_size=21):
    """The unthresholded cv2.resize values MaskLayer compares with BINARIZE_THRESH (for margins)."""
    import cv2
    out = []
    for i in range(mask_pred.shape[0]):
        if info[i][0] == -1:
            continue
        e = np.round(info[i][4:8]).astype(int)
        out.append(cv2.resize(mask_pred[i].reshape(mask_size, mask_size).astype(np.float32),
                              (e[2] - e[0] + 1, e[3] - e[1] + 1)).ravel())
    return np.concatenate(out) if out else np.zeros(0, np.float32)


def target_values(case, out, mask_size=21):
    """The unthresholded resized planes of StageBridge's foreground mask targets (for margins)."""
    import cv2
    vals = []
    gm, mi = case["gt_masks"], np.asarray(case["mask_info"]).astype(np.int64)
    for i in range(out["nfg"]):
        info = out["gt_mask_info"][i].astype(np.int64)
        ex, gt = info[4:8], info[8:12]
        x1, y1, x2, y2 = max(ex[0], gt[0]), max(ex[1], gt[1]), min(ex[2], gt[2]), min(ex[3], gt[3])
        if x1 > x2 or y1 > y2:
            continue
        crop = np.asarray(gm[info[0]])[0:mi[info[0], 0], 0:mi[info[0], 1]]
        t = np.zeros((ex[3] - ex[1] + 1, ex[2] - ex[0] + 1))
        t[y1 - ex[1]:y2 - ex[1] + 1, x1 - ex[0]:x2 - ex[0] + 1] = \
            crop[y1 - gt[1]:y2 - gt[1] + 1, x1 - gt[0]:x2 - gt[0] + 1]
        vals.append(cv2.resize(t.astype(np.float32), (mask_size, mask_size)).ravel())
    return np.concatenate(vals) if vals else np.zeros(0, np.float32)
