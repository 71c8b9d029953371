"""numpy restatement of the TRAIN phase of the three RPN-stage layers, the checker of
mnc_b200/csrc/rpn_train.cu:
  ProposalLayer.forward (TRAIN)    lib/pylayer/proposal_layer.py:52-175
  ProposalLayer.backward           proposal_layer.py:177-230
  ProposalTargetLayer.forward      lib/pylayer/proposal_target_layer.py:62-107, _sample_rois :118-216
  ProposalTargetLayer.backward     proposal_target_layer.py:109-115
  AnchorTargetLayer.forward        lib/pylayer/anchor_target_layer.py:51-209
Every array keeps the dtype the reference gives it.  The one change of semantics is the sampling:
npr.choice(cands, size, replace=False) becomes `choice` below, the `size` candidates with the
smallest (key, index) pairs for caller-supplied uint32 keys (DESIGN.md "RPN-stage training
layers").  The reference's Python 2 integer divisions and float indices are taken as the integers
they give there."""
import numpy as np

from oracle import oracle as O
from oracle import oracle_train as T

A = 9
# cfg.TRAIN defaults, lib/mnc_config.py:36-100 (RPN_POST_NMS_TOP_N: mnc_5stage.yml:4)
TRAIN = dict(BATCH_SIZE=64, FG_FRACTION=(0.3,), FG_THRESH_HI=(1.0,), FG_THRESH_LO=(0.5,),
             BG_FRACTION=(0.85, 0.15), BG_THRESH_HI=(0.5, 0.1), BG_THRESH_LO=(0.1, 0.0),
             RPN_POSITIVE_OVERLAP=0.7, RPN_NEGATIVE_OVERLAP=0.3, RPN_CLOBBER_POSITIVES=False,
             RPN_FG_FRACTION=0.5, RPN_BATCHSIZE=256, RPN_NMS_THRESH=0.7, RPN_PRE_NMS_TOP_N=12000,
             RPN_POST_NMS_TOP_N=300, RPN_MIN_SIZE=16, RPN_BBOX_INSIDE_WEIGHTS=(1.0, 1.0, 1.0, 1.0),
             RPN_POSITIVE_WEIGHT=-1.0)


def choice(cands, size, keys):
    """The `size` entries of `cands` with the smallest (keys[c], c); keys uint32 indexed by c.
    Returned in index order (the callers use the set only)."""
    cands = np.asarray(cands).astype(np.int64).ravel()
    size = int(size)
    if size <= 0:
        return cands[:0]
    k = np.asarray(keys).view(np.uint32).astype(np.uint64)[cands]
    order = np.lexsort((cands, k))
    return np.sort(cands[order[:size]])


# ------------------------------------------------------------------------------- ProposalLayer
def proposal_train_forward(prob, deltas, im_info, pre_nms_top_n=12000, post_nms_top_n=300,
                           nms_thresh=0.7, min_size=16, feat_stride=16):
    """-> (rois (R,5) float32, proposal_index (1,R) float32, state) with state the attributes the
    backward reads (_ind_after_filter, _ind_after_sort, _proposal_index, the two clip keeps)."""
    im_info = np.asarray(im_info, np.float32).reshape(-1)
    scores = prob[:, A:, :, :]
    H, W = scores.shape[-2:]
    anchors = O.shifted_anchors(H, W, feat_stride)
    _, anchor_keep = O.clip_boxes(anchors, im_info[:2])
    d = deltas.transpose((0, 2, 3, 1)).reshape((-1, 4))
    scores = scores.transpose((0, 2, 3, 1)).reshape((-1, 1))
    proposals = O.bbox_transform_inv(anchors, d)
    proposals, proposal_keep = O.clip_boxes(proposals, im_info[:2])
    keep = O.filter_small_boxes(proposals, min_size * im_info[2])
    proposals, scores = proposals[keep, :], scores[keep]
    ind_after_filter = keep
    order = O.order_desc(scores)
    if pre_nms_top_n > 0:
        order = order[:pre_nms_top_n]
    proposals, scores = proposals[order, :], scores[order]
    keep = O.nms(np.hstack((proposals, scores)), nms_thresh)
    if post_nms_top_n > 0:
        keep = keep[:post_nms_top_n]
    keep = np.asarray(keep, np.int64)
    rois = np.hstack((np.zeros((len(keep), 1), np.float32), proposals[keep, :].astype(np.float32)))
    index = ind_after_filter[order[keep]].reshape(1, len(keep)).astype(np.float32)
    state = dict(ind_after_filter=ind_after_filter, ind_after_sort=order, proposal_index=keep,
                 proposal_keep=proposal_keep, anchor_keep=anchor_keep, H=H, W=W)
    return rois, index, state


def proposal_backward(top_diff, state, deltas, clip_thresh=0.0):
    """proposal_layer.py:177-230 -> rpn_bbox_pred diff (1,4A,H,W) float32."""
    top_diff = np.asarray(top_diff, np.float32)
    diff = np.zeros(deltas.shape, np.float32)
    anchors = O.generate_anchors()
    nz = np.unique(np.where(abs(top_diff[:, :]) > 0)[0])
    pidx = np.asarray(state["proposal_index"])
    unmap_val = state["ind_after_filter"][state["ind_after_sort"][pidx[nz]]]
    wp = np.isin(unmap_val, state["proposal_keep"])
    wa = np.isin(unmap_val, state["anchor_keep"])
    c = unmap_val % A
    w = (unmap_val // A) % state["W"]
    h = (unmap_val // A // state["W"]) % state["H"]
    aw = anchors[c, 2] - anchors[c, 0]
    ah = anchors[c, 3] - anchors[c, 1]
    d1, d2, d3, d4 = (top_diff[nz, j] for j in (1, 2, 3, 4))
    dxc, dyc = d1 + d3, d2 + d4
    dw, dh = 0.5 * (d3 - d1), 0.5 * (d4 - d2)
    diff[0, 4 * c, h, w] = dxc * aw * wp * wa
    diff[0, 4 * c + 1, h, w] = dyc * ah * wp * wa
    diff[0, 4 * c + 2, h, w] = dw * np.exp(deltas[0, 4 * c + 2, h, w]) * aw * wp * wa
    diff[0, 4 * c + 3, h, w] = dh * np.exp(deltas[0, 4 * c + 3, h, w]) * ah * wp * wa
    if clip_thresh:
        for j in range(4):
            diff[0, 4 * c + j, h, w] = np.minimum(np.maximum(diff[0, 4 * c + j, h, w], -clip_thresh),
                                                  clip_thresh)
    return diff


# ------------------------------------------------------------------------- ProposalTargetLayer
def _bbox_transform32(ex, gt):
    """bbox_transform.py:39-61 on float32 ex and gt boxes (both float32 in _sample_rois)."""
    ew = ex[:, 2] - ex[:, 0] + 1.0
    eh = ex[:, 3] - ex[:, 1] + 1.0
    ecx = ex[:, 0] + 0.5 * ew
    ecy = ex[:, 1] + 0.5 * eh
    gw = gt[:, 2] - gt[:, 0] + 1.0
    gh = gt[:, 3] - gt[:, 1] + 1.0
    gcx = gt[:, 0] + 0.5 * gw
    gcy = gt[:, 1] + 0.5 * gh
    return np.vstack(((gcx - ecx) / ew, (gcy - ecy) / eh, np.log(gw / ew), np.log(gh / eh))).transpose()


def proposal_target_forward(rpn_rois, rois_index, gt_boxes, gt_masks, mask_info, im_info, keys,
                            num_classes=21, normalize=False, means=T.BBOX_NORMALIZE_MEANS,
                            stds=T.BBOX_NORMALIZE_STDS, inside_weights=T.BBOX_INSIDE_WEIGHTS,
                            mask_size=21, binarize_thresh=0.4, bp_all=True, **cfg):
    """-> dict of the ten tops at K rows (float32 as the blobs hold them) and keep_inds, fg_inds,
    bg_inds (the sampled rows), keep_ind (what the backward reads), max_overlaps.  keys uint32
    (#categories, n + G); cfg overrides TRAIN's BATCH_SIZE / FG_* / BG_* entries."""
    c = dict(TRAIN, **cfg)
    rpn_rois = np.asarray(rpn_rois, np.float32).reshape(-1, 5)
    gt_boxes = np.asarray(gt_boxes, np.float32)
    im_info = np.asarray(im_info, np.float32).reshape(-1)
    mask_info = np.asarray(mask_info).astype(np.int64)
    keys = np.asarray(keys).view(np.uint32)
    n, nf = rpn_rois.shape[0], len(c["FG_FRACTION"])
    zeros = np.zeros((gt_boxes.shape[0], 1), dtype=gt_boxes.dtype)
    all_rois = np.vstack((rpn_rois, np.hstack((zeros, gt_boxes[:, :-1]))))          # :76-80
    B = c["BATCH_SIZE"]
    overlaps = O.bbox_overlaps(all_rois[:, 1:5], gt_boxes[:, :4])                   # :127-132
    gt_assignment = overlaps.argmax(axis=1)
    max_overlaps = overlaps.max(axis=1)
    labels = gt_boxes[gt_assignment, 4]
    fg_inds = np.zeros(0)
    for i in range(nf):                                                              # :137-146
        cur = np.where((max_overlaps >= c["FG_THRESH_LO"][i]) & (max_overlaps <= c["FG_THRESH_HI"][i]))[0]
        cnt = min(cur.size, np.round(B * c["FG_FRACTION"][i]))
        if cur.size > 0:
            cur = choice(cur, cnt, keys[i])
        fg_inds = np.unique(np.hstack((fg_inds, cur)))
    nfg = fg_inds.size
    bg_inds = np.zeros(0)
    for i in range(len(c["BG_FRACTION"])):                                           # :148-159
        cur = np.where((max_overlaps >= c["BG_THRESH_LO"][i]) & (max_overlaps <= c["BG_THRESH_HI"][i]))[0]
        cnt = min(cur.size, np.round((B - nfg) * c["BG_FRACTION"][i]))
        if cur.size > 0:
            cur = choice(cur, cnt, keys[nf + i])
        bg_inds = np.unique(np.hstack((bg_inds, cur)))
    keep_inds = np.append(fg_inds, bg_inds).astype(int)                              # :162
    labels = labels[keep_inds]
    labels[nfg:] = 0
    rois = all_rois[keep_inds]
    t = _bbox_transform32(rois[:, 1:5], gt_boxes[gt_assignment[keep_inds], :4])
    if normalize:
        t = (t - np.array(means)) / np.array(stds)
    data = np.hstack((labels[:, np.newaxis], t.astype(np.float32))).astype(np.float32)
    K = len(keep_inds)
    bbox_targets = np.zeros((K, 4 * num_classes), np.float32)                        # :179-203
    bbox_inside = np.zeros(bbox_targets.shape, np.float32)
    for ind in np.where(data[:, 0] > 0)[0]:
        start = int(4 * data[ind, 0])
        bbox_targets[ind, start:start + 4] = data[ind, 1:]
        bbox_inside[ind, start:start + 4] = inside_weights
    bbox_outside = np.array(bbox_inside > 0).astype(np.float32)
    im_scale = im_info[2]
    scaled_rois = rois[:, 1:5] / float(im_scale)                                     # :186-214
    scaled_gt = gt_boxes[:, :4] / float(im_scale)
    masks = np.zeros((K, 1, mask_size, mask_size))
    info = np.zeros((K, 12))
    info[nfg:, :] = -1
    for i, val in enumerate(fg_inds):
        a = gt_assignment[int(val)]
        gt_box = np.around(scaled_gt[a]).astype(int)
        ex_box = np.around(scaled_rois[i]).astype(int)
        gt_mask = np.asarray(gt_masks[a])[0:mask_info[a, 0], 0:mask_info[a, 1]]
        masks[i, ...] = T._intersect_mask(ex_box, gt_box, gt_mask, mask_size, binarize_thresh)
        info[i, 0] = a
        info[i, 1:3] = mask_info[a]
        info[i, 3] = labels[i]
        info[i, 4:8] = ex_box
        info[i, 8:12] = gt_box
    mask_weight = np.zeros((K, 1, mask_size, mask_size))
    mask_weight[0:nfg] = 1
    idx = np.asarray(rois_index, np.float32).reshape(1, -1)
    mix_fg = idx[0, fg_inds[fg_inds < idx.shape[1]].astype(int)]                     # :96-105
    mix_bg = idx[0, bg_inds.astype(int)]
    f = lambda x: np.asarray(x).astype(np.float32)
    return {"rois": f(rois), "labels": f(labels), "bbox_targets": bbox_targets,
            "bbox_inside_weights": bbox_inside, "bbox_outside_weights": bbox_outside,
            "mask_targets": f(masks), "mask_weight": f(mask_weight), "gt_masks_info": f(info),
            "fg_inds": f(mix_fg), "bg_inds": f(mix_bg), "keep_inds": keep_inds,
            "sampled_fg": fg_inds.astype(np.int64), "sampled_bg": bg_inds.astype(np.int64),
            "keep_ind": keep_inds if bp_all else fg_inds.astype(np.int64),
            "max_overlaps": max_overlaps}


def proposal_target_backward(top_diff, keep_ind, n):
    """proposal_target_layer.py:109-115: rows of keep_ind < n take the top rows (the last wins)."""
    diff = np.zeros((n, 5), np.float32)
    keep_ind = np.asarray(keep_ind)
    valid = np.where(keep_ind < n)[0]
    diff[keep_ind[valid].astype(int), :] = np.asarray(top_diff, np.float32)[valid, :]
    return diff


# --------------------------------------------------------------------------- AnchorTargetLayer
def anchor_target_forward(H, W, gt_boxes, im_info, keys, fg_inds=None, bg_inds=None,
                          feat_stride=16, allowed_border=0, **cfg):
    """-> (labels (1,1,A*H,W), bbox_targets, bbox_inside_weights, bbox_outside_weights
    (1,4A,H,W)) float32; fg_inds / bg_inds None: MIX_INDEX off."""
    c = dict(TRAIN, **cfg)
    gt_boxes = np.asarray(gt_boxes, np.float32)
    im_info = np.asarray(im_info, np.float32).reshape(-1)
    keys = np.asarray(keys).view(np.uint32).ravel()
    all_anchors = O.shifted_anchors(H, W, feat_stride)
    total = all_anchors.shape[0]
    inds_inside = np.where((all_anchors[:, 0] >= -allowed_border) &                  # :80-85
                           (all_anchors[:, 1] >= -allowed_border) &
                           (all_anchors[:, 2] < im_info[1] + allowed_border) &
                           (all_anchors[:, 3] < im_info[0] + allowed_border))[0]
    anchors = all_anchors[inds_inside, :]
    labels = np.empty((len(inds_inside),), np.float32)
    labels.fill(-1)
    overlaps = O.bbox_overlaps(anchors, gt_boxes[:, :4])                               # :93-98
    argmax = overlaps.argmax(axis=1)
    max_ov = overlaps[np.arange(len(inds_inside)), argmax]
    gt_argmax = overlaps.argmax(axis=0)
    gt_max = overlaps[gt_argmax, np.arange(overlaps.shape[1])]
    gt_argmax = np.where(overlaps == gt_max)[0]
    if not c["RPN_CLOBBER_POSITIVES"]:
        labels[max_ov < c["RPN_NEGATIVE_OVERLAP"]] = 0
    labels[gt_argmax] = 1
    labels[max_ov >= c["RPN_POSITIVE_OVERLAP"]] = 1
    if c["RPN_CLOBBER_POSITIVES"]:
        labels[max_ov < c["RPN_NEGATIVE_OVERLAP"]] = 0
    num_fg = int(c["RPN_FG_FRACTION"] * c["RPN_BATCHSIZE"])                           # :115-134
    fg = np.where(labels == 1)[0]
    if len(fg) > num_fg:
        labels[_choice_mapped(fg, len(fg) - num_fg, keys, inds_inside)] = -1
    num_bg = c["RPN_BATCHSIZE"] - np.sum(labels == 1)
    bg = np.where(labels == 0)[0]
    if len(bg) > num_bg:
        labels[_choice_mapped(bg, len(bg) - num_bg, keys, inds_inside)] = -1
    if fg_inds is not None:                                                            # :136-150
        ufg = [np.where(i == inds_inside)[0] for i in list(np.asarray(fg_inds).ravel())]
        ubg = [np.where(i == inds_inside)[0] for i in list(np.asarray(bg_inds).ravel())]
        labels[[z[0] for z in ubg if len(z)]] = 0
        labels[[z[0] for z in ufg if len(z)]] = 1
    targets = T._bbox_transform(anchors, gt_boxes[argmax, :4]).astype(np.float32)     # :152
    inside_w = np.zeros((len(inds_inside), 4), np.float32)
    inside_w[labels == 1, :] = np.array(c["RPN_BBOX_INSIDE_WEIGHTS"])
    outside_w = np.zeros((len(inds_inside), 4), np.float32)
    if c["RPN_POSITIVE_WEIGHT"] < 0:
        num_examples = np.sum(labels >= 0)
        pw = nw = np.ones((1, 4)) * 1.0 / num_examples
    else:
        pw = c["RPN_POSITIVE_WEIGHT"] / np.sum(labels == 1)
        nw = (1.0 - c["RPN_POSITIVE_WEIGHT"]) / np.sum(labels == 0)
    outside_w[labels == 1, :] = pw
    outside_w[labels == 0, :] = nw

    def unmap(data, fill):
        ret = np.empty((total,) + data.shape[1:], np.float32)
        ret.fill(fill)
        ret[inds_inside] = data
        return ret
    labels = unmap(labels, -1).reshape((1, H, W, A)).transpose(0, 3, 1, 2).reshape((1, 1, A * H, W))
    tops = [unmap(x, 0).reshape((1, H, W, A * 4)).transpose(0, 3, 1, 2)
            for x in (targets, inside_w, outside_w)]
    return (np.ascontiguousarray(labels),) + tuple(np.ascontiguousarray(t) for t in tops)


def _choice_mapped(cands, size, keys, inds_inside):
    """choice over positions in inds_inside, keyed and tie-broken by their anchor index."""
    return np.searchsorted(inds_inside, choice(inds_inside[cands], size, keys))


# --------------------------------------------------------------------------- synthetic inputs
def make_case(seed, H=38, W=63, im_info=(600, 1000, 1.6), G=3, n=300, scores=True):
    """One image's RPN-stage bottoms: tie-free RPN scores and small deltas (1,2A,H,W) /
    (1,4A,H,W), gt boxes at integer positions of the original image scaled by im_scale with
    elliptic gt masks (mask_info = their height, width), and n RPN RoIs -- jittered gt boxes and
    random boxes -- with distinct anchor indices as rpn_rois_index (1,n)."""
    rng = np.random.default_rng(seed)
    im_h, im_w, s = im_info
    prob = None
    if scores:
        fg = rng.permutation(np.linspace(0.001, 0.999, A * H * W)).astype(np.float32).reshape(1, A, H, W)
        prob = np.concatenate([1 - fg, fg], axis=1).astype(np.float32)
    deltas = rng.normal(0, 0.2, size=(1, 4 * A, H, W)).astype(np.float32)
    Ho, Wo = int(im_h / s), int(im_w / s)
    gw = rng.integers(20, max(21, Wo // 3), G)
    gh = rng.integers(20, max(21, Ho // 3), G)
    gx = rng.integers(0, Wo - gw)
    gy = rng.integers(0, Ho - gh)
    gt = np.zeros((G, 5), np.float32)
    gt[:, :4] = np.stack([gx, gy, gx + gw - 1, gy + gh - 1], 1) * np.float32(s)
    gt[:, 4] = rng.integers(1, 21, G)
    mask_info = np.stack([gh, gw], 1).astype(np.int32)
    gm = np.zeros((G, int(gh.max()), int(gw.max())), bool)
    for g in range(G):
        yy, xx = np.mgrid[0:gh[g], 0:gw[g]]
        r = ((yy - gh[g] / 2) / (gh[g] / 2)) ** 2 + ((xx - gw[g] / 2) / (gw[g] / 2)) ** 2
        gm[g, :gh[g], :gw[g]] = (r < 0.8) ^ (rng.random((gh[g], gw[g])) < 0.05)
    rois = np.zeros((n, 5), np.float32)
    for i in range(n):
        if i < n // 3:
            b = gt[i % G, :4].astype(np.float64)
            w, h = b[2] - b[0], b[3] - b[1]
            b = b + rng.normal(0, 0.15, 4) * np.array([w, h, w, h])
        else:
            cx, cy = rng.uniform(0, im_w), rng.uniform(0, im_h)
            w, h = np.exp(rng.uniform(np.log(16), np.log(400), 2))
            b = np.array([cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2])
        b[0::2] = np.clip(b[0::2], 0, im_w - 1)
        b[1::2] = np.clip(b[1::2], 0, im_h - 1)
        rois[i, 1:] = [min(b[0], b[2]), min(b[1], b[3]), max(b[0], b[2]), max(b[1], b[3])]
    index = rng.choice(A * H * W, n, replace=False).astype(np.float32).reshape(1, n)
    return dict(prob=prob, deltas=deltas, gt_boxes=gt, gt_masks=gm, mask_info=mask_info,
                im_info=np.array([im_info], np.float32), rpn_rois=rois, rois_index=index)
