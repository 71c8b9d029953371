"""Device-tensor wrappers over the non-dense C-ABI entry points (include/mnc_b200.h).

All arguments are CUDA torch tensors; everything is launched on torch's current stream.  PyTorch is
only the allocator / stream provider here: every computation happens in libmnc_b200.so.
"""
import ctypes

import torch

from ._lib import lib, ptr, cur_stream, check


def _i32(*shape, device):
    return torch.empty(shape, dtype=torch.int32, device=device)


# ----------------------------------------------------------------------------- sort / NMS
def rank_sort_desc(keys, n, problems, outer_stride, inner_stride=0, inner=1, key_stride=1,
                   valid=None):
    """-> (order int32 [problems, n], n_valid int32 [problems])."""
    dev = keys.device
    order = _i32(problems, n, device=dev)
    n_valid = _i32(problems, device=dev)
    check(lib.mnc_rank_sort_desc(ptr(keys), outer_stride, inner_stride, inner, key_stride,
                                 ptr(valid), n, problems, ptr(order), ptr(n_valid),
                                 cur_stream()), "mnc_rank_sort_desc")
    return order, n_valid


def topk_sort_desc(keys, n, problems, k, outer_stride, inner_stride=0, inner=1, key_stride=1,
                   valid=None):
    """The k best entries in (key desc, index asc) order.
    -> (order int32 [problems, min(k, n)], n_out int32 [problems])."""
    dev = keys.device
    kk = min(k, n)
    order = _i32(problems, kk, device=dev)
    n_out = _i32(problems, device=dev)
    check(lib.mnc_topk_sort_desc(ptr(keys), outer_stride, inner_stride, inner, key_stride,
                                 ptr(valid), n, problems, kk, ptr(order), kk, ptr(n_out),
                                 cur_stream()), "mnc_topk_sort_desc")
    return order, n_out


def gather_boxes(src, src_stride, src_outer_stride, inner, order, counts, n_out, problems):
    """-> (sorted boxes fp32 [problems, n_out, 4], counts int32 [problems])."""
    dev = src.device
    dst = torch.zeros((problems, n_out, 4), dtype=torch.float32, device=dev)
    out_counts = _i32(problems, device=dev)
    check(lib.mnc_gather_boxes(ptr(src), src_stride, src_outer_stride, inner, ptr(order),
                               order.shape[1], ptr(counts), n_out, problems, ptr(dst),
                               ptr(out_counts), cur_stream()), "mnc_gather_boxes")
    return dst, out_counts


_nms_ws = {}


def nms_sorted(boxes, counts, thresh, max_keep):
    """boxes fp32 [problems, n_max, 4] score-sorted; counts int32 [problems] or None.
    -> (keep int32 [problems, max_keep], num int32 [problems])."""
    problems, n_max, stride = boxes.shape
    dev = boxes.device
    nbytes = lib.mnc_nms_workspace_bytes(n_max, problems)
    key = (dev, nbytes)
    ws = _nms_ws.get(key)
    if ws is None:
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _nms_ws.clear()
        _nms_ws[key] = ws
    mk = max_keep if max_keep > 0 else n_max
    keep = _i32(problems, mk, device=dev)
    num = _i32(problems, device=dev)
    check(lib.mnc_nms_sorted(ptr(boxes), stride, n_max * stride, ptr(counts), n_max, problems,
                             thresh, mk, ptr(ws), ptr(keep), mk, ptr(num),
                             cur_stream()), "mnc_nms_sorted",
          launches=lib.mnc_nms_sorted_launches(n_max, mk))
    return keep, num


DEFAULT_NMS_MODE = 2


def nms_set_lazy(mode):
    """A/B and cross-check switch of the capped NMS mnc_nms_sorted picks when max_keep << n:
    3 = thread-block cluster, 256-candidate rounds; 2 = cluster, 64-candidate rounds; 1 = one CTA
    per problem; 0 / False = always the suppression-matrix pair (nms_mask + nms_scan); True = the
    library default.  Returns the previous mode (int)."""
    mode = DEFAULT_NMS_MODE if mode is True else (0 if mode is False else int(mode))
    return int(lib.mnc_nms_set_lazy(mode))


# ----------------------------------------------------------------------------- proposal pieces
def generate_anchors():
    import numpy as np
    out = np.zeros((9, 4), dtype=np.float32)
    check(lib.mnc_generate_anchors(ptr(out)), "mnc_generate_anchors")
    return out


def rpn_decode(cls, bbox, im_info, batch, H, W, layout, apply_softmax, feat_stride=16,
               min_size=16.0):
    """layout 'nchw': cls (B,18,H,W), bbox (B,36,H,W); 'nhwc': one buffer (B,H,W,Cpad) where
    channels [0,18) are cls and [18,54) bbox (then `bbox` is ignored)."""
    dev = cls.device
    total = H * W * 9
    proposals = torch.empty((batch, total, 4), dtype=torch.float32, device=dev)
    scores = torch.empty((batch, total), dtype=torch.float32, device=dev)
    valid = torch.empty((batch, total), dtype=torch.uint8, device=dev)
    if layout == "nchw":
        ci, cc, cp = 18 * H * W, H * W, 1
        bi, bc, bp = 36 * H * W, H * W, 1
        bptr = ptr(bbox)
    else:
        cpad = cls.shape[-1]
        ci, cc, cp = H * W * cpad, 1, cpad
        bi, bc, bp = ci, cc, cp
        bptr = cls.data_ptr() + 18 * 4
    check(lib.mnc_rpn_decode(ptr(cls), ci, cc, cp, bptr, bi, bc, bp, ptr(im_info), batch, H, W,
                             feat_stride, min_size, int(apply_softmax), ptr(proposals), ptr(scores),
                             ptr(valid), cur_stream()), "mnc_rpn_decode")
    return proposals, scores, valid


def write_rois(sorted_boxes, keep, num_keep, max_rois, batch_index_mode):
    batch, n_sorted, _ = sorted_boxes.shape
    dev = sorted_boxes.device
    rois = torch.empty((batch, max_rois, 5), dtype=torch.float32, device=dev)
    counts = _i32(batch, device=dev)
    check(lib.mnc_write_rois(ptr(sorted_boxes), n_sorted, ptr(keep), keep.shape[1], ptr(num_keep),
                             max_rois, batch, int(batch_index_mode), ptr(rois), ptr(counts),
                             cur_stream()), "mnc_write_rois")
    return rois, counts


def proposals_from_rpn(cls, bbox, im_info, batch, H, W, layout, apply_softmax, pre_nms_top_n=6000,
                       post_nms_top_n=300, nms_thresh=0.7, min_size=16.0, batch_index_mode=True,
                       return_intermediate=False):
    """Whole ProposalLayer.forward on device (lib/pylayer/proposal_layer.py:52-175)."""
    proposals, scores, valid = rpn_decode(cls, bbox, im_info, batch, H, W, layout, apply_softmax,
                                          min_size=min_size)
    total = H * W * 9
    n_sorted = min(pre_nms_top_n, total) if pre_nms_top_n > 0 else total
    if 8 * (1 << max(n_sorted - 1, 1).bit_length()) + 4 * total <= 200 * 1024:
        order, n_valid = topk_sort_desc(scores, total, batch, n_sorted, outer_stride=total, valid=valid)
    else:   # beyond the select kernel's shared-memory budget: sort everything
        order, n_valid = rank_sort_desc(scores, total, batch, outer_stride=total, valid=valid)
    sorted_boxes, counts = gather_boxes(proposals, 4, total * 4, 1, order, n_valid, n_sorted, batch)
    keep, num = nms_sorted(sorted_boxes, counts, nms_thresh, post_nms_top_n)
    rois, roi_counts = write_rois(sorted_boxes, keep, num, post_nms_top_n, batch_index_mode)
    if return_intermediate:
        return rois, roi_counts, dict(proposals=proposals, scores=scores, valid=valid, order=order,
                                      n_valid=n_valid, sorted_boxes=sorted_boxes, counts=counts,
                                      keep=keep, num=num)
    return rois, roi_counts


def stage_bridge(rois, bbox_pred, seg_cls_prob, im_info, rois_per_img):
    """rois [T,5], bbox_pred [T,>=84] (row stride = bbox_pred.stride(0)), seg_cls_prob [T,21]."""
    total = rois.shape[0]
    out = torch.empty_like(rois)
    check(lib.mnc_stage_bridge(ptr(rois), ptr(bbox_pred), bbox_pred.stride(0), ptr(seg_cls_prob),
                               seg_cls_prob.stride(0), seg_cls_prob.shape[1], ptr(im_info),
                               rois_per_img, total, ptr(out), cur_stream()), "mnc_stage_bridge")
    return out


def softmax_rows(x, cols=None, out=None):
    rows = x.shape[0]
    cols = cols or x.shape[1]
    if out is None:
        out = torch.empty((rows, cols), dtype=torch.float32, device=x.device)
    check(lib.mnc_softmax_rows(ptr(x), x.stride(0), rows, cols, ptr(out), out.stride(0),
                               cur_stream()), "mnc_softmax_rows")
    return out


def unscale_clip(rois, rois_per_img, im_scale, im_hw):
    total = rois.shape[0]
    boxes = torch.empty((total, 4), dtype=torch.float32, device=rois.device)
    check(lib.mnc_unscale_clip(ptr(rois), total, rois_per_img, ptr(im_scale), ptr(im_hw),
                               ptr(boxes), cur_stream()), "mnc_unscale_clip")
    return boxes


def record_layout(B, n, msz=441, ncls=21):
    """Offsets (in floats) of the sections of the per-step output record and its length."""
    o_boxes = (B + 3) // 4 * 4
    o_scores = o_boxes + B * 2 * n * 4
    o_masks = o_scores + B * 2 * n * ncls
    return o_boxes, o_scores, o_masks, o_masks + B * 2 * n * msz


def record_views(rec, B, n, msz=441, ncls=21):
    ob, os_, om, end = record_layout(B, n, msz, ncls)
    side = int(round(msz ** 0.5))
    return (rec[:B], rec[ob:os_].view(B, 2 * n, 4), rec[os_:om].view(B, 2 * n, ncls),
            rec[om:end].view(B, 2 * n, 1, side, side))


def detect_tail(o, B, n, im_scale, im_hw, rec, valid):
    """im_detect tail into the record buffer `rec` (fp32, record_layout(B, n)[3] floats) and
    `valid` (uint8 [B, 2n]).  Returns (counts, boxes, scores, masks) views of rec."""
    msz = o["mask_proposal"].shape[-1] * o["mask_proposal"].shape[-2]
    ncls = o["seg_cls_prob"].shape[-1]
    counts, boxes, scores, masks = record_views(rec, B, n, msz, ncls)
    check(lib.mnc_detect_tail(ptr(o["rois"]), ptr(o["rois_ext"]), ptr(o["mask_proposal"]),
                              ptr(o["mask_proposal_ext"]), ptr(o["seg_cls_prob"]),
                              ptr(o["seg_cls_prob_ext"]), ptr(o["roi_counts"]), ptr(im_scale),
                              ptr(im_hw), B, n, msz, ncls, ptr(counts), ptr(boxes), ptr(scores),
                              ptr(masks), ptr(valid), cur_stream()), "mnc_detect_tail")
    return counts, boxes, scores, masks


def decode_class_boxes(rois, bbox_pred, rois_per_img, im_scale, im_hw, ncls=21):
    """-> (R, ncls*4) fp32: per-class decoded boxes in original-image coordinates, clipped."""
    R = rois.shape[0]
    out = torch.empty((R, ncls * 4), dtype=torch.float32, device=rois.device)
    check(lib.mnc_decode_class_boxes(ptr(rois), R, rois_per_img, ptr(bbox_pred),
                                     bbox_pred.stride(0), ncls, ptr(im_scale), ptr(im_hw), ptr(out),
                                     cur_stream()), "mnc_decode_class_boxes")
    return out


# ----------------------------------------------------------------------------- RoI / mask layers
def roi_warp_nchw(feat, rois, pooled_h, pooled_w, spatial_scale=0.0625, out=None):
    B, C, H, W = feat.shape
    R = rois.shape[0]
    if out is None:
        out = torch.empty((R, C, pooled_h, pooled_w), dtype=torch.float32, device=feat.device)
    check(lib.mnc_roi_warp_nchw(ptr(feat), C, H, W, ptr(rois), R, pooled_h, pooled_w, spatial_scale,
                                ptr(out), cur_stream()), "mnc_roi_warp_nchw")
    return out


def mask_resize_nchw(x, out_h, out_w):
    N, C, ih, iw = x.shape
    out = torch.empty((N, C, out_h, out_w), dtype=torch.float32, device=x.device)
    check(lib.mnc_mask_resize_nchw(ptr(x), N, C, ih, iw, out_h, out_w, ptr(out),
                                   cur_stream()), "mnc_mask_resize_nchw")
    return out


def mask_pool_nchw(feat, mask, out=None):
    N, C, H, W = feat.shape
    if mask.shape != (N, 1, H, W):
        raise ValueError("MaskPooling: mask must be (N,1,H,W) matching feat "
                         "(mask_pooling_layer.cpp:20-29)")
    if out is None:
        out = torch.empty_like(feat)
    check(lib.mnc_mask_pool_nchw(ptr(feat), ptr(mask), N, C, H, W, ptr(out),
                                 cur_stream()), "mnc_mask_pool_nchw")
    return out


def roi_warp_split(feat, C, H, W, rois, sub, out14, out7, spatial_scale=0.0625):
    """feat fp32 NHWC [B,H,W,C]; rois [R,5]; out14 split [2,R,14,14,C]; out7 split [2,R,7,7,C]."""
    R = rois.shape[0]
    assert feat.dtype == torch.float32
    check(lib.mnc_roi_warp_split(ptr(feat), C, H, W, ptr(rois), R, sub, spatial_scale,
                                 ptr(out14[0]), ptr(out14[1]), ptr(out7[0]), ptr(out7[1]),
                                 cur_stream()), "mnc_roi_warp_split")


def roi_warp_tri(feat, C, H, W, rois, sub, out14, out7, exp, spatial_scale=0.0625):
    """roi_warp_split with tri-plane outputs (mnc_b200.dense.Tri) written with exponent `exp`."""
    R = rois.shape[0]
    assert feat.dtype == torch.float32
    out14.exp = out7.exp = int(exp)
    check(lib.mnc_roi_warp_tri(ptr(feat), C, H, W, ptr(rois), R, sub, spatial_scale, 2.0 ** exp,
                               ptr(out14.h), ptr(out14.l), ptr(out14.c), ptr(out7.h), ptr(out7.l),
                               ptr(out7.c), cur_stream()), "mnc_roi_warp_tri")


def mask_pool_tri(feat14, mask14, R, C, out7):
    """MaskPooling + 2x2 max pool on tri-plane features; the output takes the input's exponent."""
    out7.exp = feat14.exp
    check(lib.mnc_mask_pool_tri(ptr(feat14.h), ptr(feat14.l), ptr(mask14), R, C, ptr(out7.h),
                                ptr(out7.l), ptr(out7.c), cur_stream()), "mnc_mask_pool_tri")


def sigmoid_mask_resize(logits, R, mask_size=21, out_size=14):
    dev = logits.device
    mp = torch.empty((R, 1, mask_size, mask_size), dtype=torch.float32, device=dev)
    mr = torch.empty((R, 1, out_size, out_size), dtype=torch.float32, device=dev)
    check(lib.mnc_sigmoid_mask_resize(ptr(logits), logits.stride(0), R, mask_size, out_size,
                                      ptr(mp), ptr(mr), cur_stream()), "mnc_sigmoid_mask_resize")
    return mp, mr


def mask_pool_split(feat14, mask14, R, C, out7):
    check(lib.mnc_mask_pool_split(ptr(feat14[0]), ptr(feat14[1]), ptr(mask14), R, C, ptr(out7[0]),
                                  ptr(out7[1]), cur_stream()), "mnc_mask_pool_split")


def roi_pool_nchw(feat, rois, pooled_h, pooled_w, spatial_scale=0.0625, out=None, argmax=None):
    """ROIPoolingLayer forward (roi_pooling_layer.cu:17-105) on fp32 NCHW device tensors."""
    B, C, H, W = feat.shape
    R = rois.shape[0]
    if out is None:
        out = torch.empty((R, C, pooled_h, pooled_w), dtype=torch.float32, device=feat.device)
    check(lib.mnc_roi_pool_nchw(ptr(feat), C, H, W, ptr(rois), R, pooled_h, pooled_w, spatial_scale,
                                ptr(out), ptr(argmax), cur_stream()), "mnc_roi_pool_nchw")
    return out


def roi_pool_split(feat, C, H, W, rois, pooled, out, spatial_scale=0.0625):
    """feat fp32 NHWC [B,H,W,C]; rois [R,5]; out split [2,R,P,P,C] (ROIPooling)."""
    check(lib.mnc_roi_pool_split(ptr(feat), C, H, W, ptr(rois), rois.shape[0], pooled,
                                 spatial_scale, ptr(out[0]), ptr(out[1]),
                                 cur_stream()), "mnc_roi_pool_split")


def roi_sample_split(feat, C, H, W, rois, pooled, out, spatial_scale=0.0625):
    """feat fp32 NHWC [B,H,W,C]; rois [R,5]; out split [2,R,P,P,C] (ROIWarping, no pool after)."""
    check(lib.mnc_roi_sample_split(ptr(feat), C, H, W, ptr(rois), rois.shape[0], pooled,
                                   spatial_scale, ptr(out[0]), ptr(out[1]),
                                   cur_stream()), "mnc_roi_sample_split")


# ----------------------------------------------------------------------------- layer backward passes
def roi_warp_backward_nchw(feat, rois, top_diff, pooled_h, pooled_w, spatial_scale=0.0625,
                           want_feat=True, want_rois=True):
    """ROIWarpingLayer backward (roi_warping_layer.cu:175-436).  feat (B,C,H,W), rois (R,5),
    top_diff (R,C,ph,pw) -> (feat_diff (B,C,H,W) or None, rois_diff (R,5) or None)."""
    B, C, H, W = feat.shape
    R = rois.shape[0]
    new = torch.zeros if R == 0 else torch.empty       # R = 0: the library writes nothing
    fd = new(feat.shape, dtype=torch.float32, device=feat.device) if want_feat else None
    rd = new((R, 5), dtype=torch.float32, device=feat.device) if want_rois else None
    check(lib.mnc_roi_warp_backward_nchw(ptr(feat), B, C, H, W, ptr(rois), R, pooled_h, pooled_w,
                                         spatial_scale, ptr(top_diff), ptr(fd), ptr(rd),
                                         cur_stream()), "mnc_roi_warp_backward_nchw",
          launches=int(want_feat) + 2 * int(want_rois))
    return fd, rd


def mask_resize_backward_nchw(top_diff, in_h, in_w):
    """MaskResizeLayer backward (mask_resize_layer.cu:135-183): top_diff (N,C,oh,ow) -> (N,C,in_h,in_w)."""
    N, C, oh, ow = top_diff.shape
    out = torch.empty((N, C, in_h, in_w), dtype=torch.float32, device=top_diff.device)
    check(lib.mnc_mask_resize_backward_nchw(ptr(top_diff), N, C, in_h, in_w, oh, ow, ptr(out),
                                            cur_stream()), "mnc_mask_resize_backward_nchw")
    return out


def mask_pool_backward_nchw(feat, mask, top_diff, want_feat=True, want_mask=True):
    """MaskPoolingLayer backward (mask_pooling_layer.cu:43-99) -> (feat_diff or None, mask_diff or None)."""
    N, C, H, W = feat.shape
    if mask.shape != (N, 1, H, W):
        raise ValueError("MaskPooling: mask must be (N,1,H,W) matching feat "
                         "(mask_pooling_layer.cpp:20-29)")
    fd = torch.empty_like(feat) if want_feat else None
    md = torch.empty_like(mask) if want_mask else None
    check(lib.mnc_mask_pool_backward_nchw(ptr(feat), ptr(mask), ptr(top_diff), N, C, H, W, ptr(fd),
                                          ptr(md), cur_stream()),
          "mnc_mask_pool_backward_nchw", launches=int(want_feat) + int(want_mask))
    return fd, md


def roi_pool_backward_nchw(top_diff, argmax, feat_shape, rois, pooled_h, pooled_w,
                           spatial_scale=0.0625):
    """ROIPoolingLayer backward (roi_pooling_layer.cu:94-184): top_diff and the int32 argmax of
    roi_pool_nchw, both (R,C,ph,pw) -> feat_diff of feat_shape (B,C,H,W)."""
    B, C, H, W = feat_shape
    R = rois.shape[0]
    new = torch.zeros if R == 0 else torch.empty
    out = new((B, C, H, W), dtype=torch.float32, device=top_diff.device)
    check(lib.mnc_roi_pool_backward_nchw(ptr(top_diff), ptr(argmax), B, C, H, W, ptr(rois), R,
                                         pooled_h, pooled_w, spatial_scale, ptr(out),
                                         cur_stream()), "mnc_roi_pool_backward_nchw")
    return out


# ----------------------------------------------------------------------------- mask voting
class VotingOverflow(RuntimeError):
    pass


def mask_voting(boxes, masks, scores, im_hw, max_per_image=100, nms_thresh=0.3, iou_thresh=0.5,
                max_results=128, box_valid=None):
    """Batched device pipeline of gpu_mask_voting (lib/transform/mask_transform.py:213-286).
    boxes [B,nb,4] fp32, masks [B,nb,1,M,M] fp32, scores [B,nb,ncls] fp32, im_hw [B,2] int32.
    box_valid: optional uint8 [B,nb]; rows with 0 are padding and take no part.
    Returns dict of device tensors: n_res [B], class_bar [B,ncls-1], res_score [B,max_results],
    res_class, result_mask [B,max_results,1,M,M], result_box [B,max_results,4] int32, plus the
    candidate lists."""
    B, nb, ncls = scores.shape
    M = masks.shape[-1]
    dev = boxes.device
    nprob = B * (ncls - 1)
    # per-class score sort: problem p = (img, c-1); keys at scores[img, :, c]
    valid_p = None
    if box_valid is not None:
        valid_p = box_valid.view(B, 1, nb).expand(B, ncls - 1, nb).contiguous()
    order, n_valid = rank_sort_desc(scores[:, :, 1:], nb, nprob, outer_stride=nb * ncls,
                                    inner_stride=1, inner=ncls - 1, key_stride=ncls, valid=valid_p)
    sorted_boxes, counts = gather_boxes(boxes, 4, nb * 4, ncls - 1, order, n_valid, nb, nprob)
    keep, num = nms_sorted(sorted_boxes, counts, nms_thresh, min(max_per_image, nb))
    res_idx = _i32(B, max_results, device=dev)
    res_cls = _i32(B, max_results, device=dev)
    res_score = torch.zeros((B, max_results), dtype=torch.float32, device=dev)
    n_res = _i32(B, device=dev)
    class_bar = _i32(B, ncls - 1, device=dev)
    overflow = torch.zeros(1, dtype=torch.int32, device=dev)
    check(lib.mnc_vote_select(ptr(scores), nb, ncls, ptr(order), ptr(keep), keep.shape[1], ptr(num),
                              max_per_image, max_results, B, ptr(res_idx), ptr(res_cls),
                              ptr(res_score), ptr(n_res), ptr(class_bar), ptr(overflow),
                              cur_stream()), "mnc_vote_select")
    cand_inds = _i32(B, max_results, nb, device=dev)
    cand_w = torch.empty((B, max_results, nb), dtype=torch.float32, device=dev)   # lists only; gaps unread
    cand_begin = _i32(B, max_results, device=dev)
    cand_end = _i32(B, max_results, device=dev)
    check(lib.mnc_vote_candidates(ptr(boxes), ptr(scores), ptr(box_valid), nb, ncls, ptr(res_idx),
                                  ptr(res_cls), ptr(n_res), max_results, B, iou_thresh,
                                  ptr(cand_inds), ptr(cand_w), ptr(cand_begin), ptr(cand_end),
                                  cur_stream()), "mnc_vote_candidates")
    bbox_ws = _i32(B * max_results * 4 + B, device=dev)   # tight boxes + per-image range flag
    out_mask = torch.zeros((B, max_results, 1, M, M), dtype=torch.float32, device=dev)
    out_box = torch.zeros((B, max_results, 4), dtype=torch.int32, device=dev)
    check(lib.mnc_mv_device(ptr(boxes), ptr(masks), nb, 4, M, ptr(cand_inds), ptr(cand_w),
                            max_results * nb, ptr(cand_begin), ptr(cand_end), ptr(n_res),
                            max_results, B, ptr(im_hw), ptr(bbox_ws), ptr(out_mask), ptr(out_box),
                            cur_stream()), "mnc_mv_device",
          launches=lib.mnc_mv_device_launches())
    return dict(n_res=n_res, class_bar=class_bar, res_score=res_score, res_class=res_cls,
                res_box_idx=res_idx, result_mask=out_mask, result_box=out_box,
                cand_inds=cand_inds, cand_weights=cand_w, cand_begin=cand_begin, cand_end=cand_end,
                overflow=overflow, order=order, keep=keep, num_keep=num)


def mv_set_two_pass(on):
    """A/B and cross-check switch of mnc_mv_device: False = one full sweep of each result's region
    instead of the coarse pass + exact border pass.  Returns the previous setting."""
    return bool(lib.mnc_mv_set_two_pass(1 if on else 0))


def mask_voting_checked(boxes, masks, scores, im_hw, max_per_image=100, box_valid=None, **kw):
    """mask_voting that never truncates: the reference keeps EVERY kept row whose score ties the
    global threshold (mask_transform.py:258), so when more rows tie than `max_results` has slots
    the device reports it and the call is repeated with room (one host read of a 4-byte flag)."""
    cap = kw.pop("max_results", max(128, max_per_image + 28))
    nb = boxes.shape[1]
    while True:
        r = mask_voting(boxes, masks, scores, im_hw, max_per_image=max_per_image, max_results=cap,
                        box_valid=box_valid, **kw)
        if int(r["overflow"].item()) == 0:
            return r
        if cap >= nb * (scores.shape[2] - 1):
            raise VotingOverflow("mask voting overflow at max_results = %d" % cap)
        cap = min(2 * cap, nb * (scores.shape[2] - 1))


# ----------------------------------------------------------------------------- input preparation
PIXEL_MEANS = (102.9801, 115.9465, 122.7717)   # cfg.PIXEL_MEANS, lib/mnc_config.py:20


def im_scale_for(shape, target_size=600, max_size=1000):
    """Scale rule of prep_im_for_blob (lib/utils/blob.py:41-46)."""
    import numpy as np
    im_size_min = min(shape[0], shape[1])
    im_size_max = max(shape[0], shape[1])
    im_scale = float(target_size) / float(im_size_min)
    if np.round(im_scale * im_size_max) > max_size:
        im_scale = float(max_size) / float(im_size_max)
    return im_scale


def prep_images(images_u8, scale, out=None, pixel_means=PIXEL_MEANS):
    """images_u8: uint8 CUDA tensor [B,H,W,3] (BGR).  -> fp32 [B,3,round(H*s),round(W*s)]."""
    import numpy as np
    B, H, W, _ = images_u8.shape
    out_h, out_w = int(np.rint(H * scale)), int(np.rint(W * scale))
    if out is None:
        out = torch.empty((B, 3, out_h, out_w), dtype=torch.float32, device=images_u8.device)
    means = (ctypes.c_double * 3)(*pixel_means)
    check(lib.mnc_prep_images(ptr(images_u8), B, H, W, means, scale, out_h, out_w, ptr(out),
                              cur_stream()), "mnc_prep_images")
    return out


# ----------------------------------------------------------------------------- result rendering
def paste_instances(boxes, masks, cls, counts, H, W, thresh=0.4, want_bgr=False):
    """Batched `_convert_pred_to_image` (lib/utils/vis_seg.py:101-131).  boxes [B,n,>=4] fp32,
    masks [B,n,(1,)M,M] fp32, cls [B,n] int32, counts [B] int32 -- device tensors, instances in
    painting order.  -> inst_img, cls_img int32 [B,H,W] (+ uint8 BGR [B,H,W,3] colour image)."""
    B, n, box_dim = boxes.shape
    M = masks.shape[-1]
    dev = boxes.device
    boxes = boxes.contiguous().float()
    masks = masks.contiguous().float()
    cls = cls.contiguous().to(torch.int32)
    counts = counts.contiguous().to(torch.int32)
    inst = torch.empty((B, H, W), dtype=torch.int32, device=dev)
    clsi = torch.empty((B, H, W), dtype=torch.int32, device=dev)
    bgr = torch.empty((B, H, W, 3), dtype=torch.uint8, device=dev) if want_bgr else None
    check(lib.mnc_paste_instances(ptr(boxes), box_dim, ptr(masks), ptr(cls), ptr(counts), B, n, M,
                                  H, W, thresh, ptr(inst), ptr(clsi), ptr(bgr), cur_stream()),
          "mnc_paste_instances")
    return (inst, clsi, bgr) if want_bgr else (inst, clsi)


def select_for_display(vote, vis_thresh=0.5):
    """`get_vis_dict` (tools/demo.py:103-120) on the device: keep voted results with
    score >= vis_thresh, order preserved (results are class-major, as the reference's loops
    visit them).  vote: the dict `mask_voting` returns.  -> boxes [B,R,4] fp32, masks, cls, counts."""
    n_res, score = vote["n_res"], vote["res_score"]
    B, R = score.shape
    live = (torch.arange(R, device=score.device)[None, :] < n_res[:, None]) & (score >= vis_thresh)
    perm = torch.sort((~live).to(torch.int8), dim=1, stable=True).indices
    boxes = torch.gather(vote["result_box"].float(), 1, perm[:, :, None].expand(B, R, 4))
    M = vote["result_mask"].shape[-1]
    masks = torch.gather(vote["result_mask"].view(B, R, M * M), 1, perm[:, :, None].expand(B, R, M * M))
    cls = torch.gather(vote["res_class"], 1, perm)
    return boxes, masks.view(B, R, M, M), cls, live.sum(dim=1).to(torch.int32)


def binarize_masks(rboxes, masks, thresh=0.4):
    """cv2.resize(mask, box size) >= thresh for every prediction (lib/utils/voc_eval.py:249-251).
    rboxes int32 [n,4] (rounded boxes), masks fp32 [n,M,M], both on the device.
    -> (packed uint8 device tensor, offsets int64 host array of n+1 entries)."""
    import numpy as np
    n = rboxes.shape[0]
    M = masks.shape[-1]
    rb = rboxes.contiguous().to(torch.int32)
    hb = rb.cpu().numpy().astype(np.int64)
    areas = np.maximum(hb[:, 2] - hb[:, 0] + 1, 0) * np.maximum(hb[:, 3] - hb[:, 1] + 1, 0)
    offsets = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(areas, out=offsets[1:])
    out = torch.empty((max(int(offsets[-1]), 1),), dtype=torch.uint8, device=rboxes.device)
    d_off = torch.from_numpy(offsets[:-1].copy()).to(rboxes.device)
    check(lib.mnc_binarize_masks(ptr(rb), ptr(masks.contiguous().float()), n, M, thresh, ptr(d_off),
                                 int(areas.max()) if n else 0, ptr(out),
                                 cur_stream()), "mnc_binarize_masks")
    return out, offsets


# ------------------------------------------------------------ training-phase cascade bridge layers
def _f32(t):
    return t.contiguous().to(torch.float32)


def stage_bridge_train(rois, bbox_pred, seg_cls_prob, gt_boxes, gt_masks, im_info, mask_info,
                       means=None, stds=None, inside_weights=(1.0, 1.0, 1.0, 1.0), bbox_thresh=0.5,
                       mask_size=21, binarize_thresh=0.4):
    """StageBridgeLayer.forward_train (lib/pylayer/stage_bridge_layer.py:131-235), one image.
    Device tensors rois (n,5), bbox_pred (n,4C), seg_cls_prob (n,C), gt_boxes (G,5), gt_masks
    (G,Hm,Wm) 0/1, im_info (3,), mask_info (G,2).  means / stds (4 floats each, or None: targets
    not normalised) are cfg.TRAIN.BBOX_NORMALIZE_MEANS / STDS when
    BBOX_NORMALIZE_TARGETS_PRECOMPUTED.  -> dict of the eight tops (K = n + G rows, foreground
    first) and `state`, the int32 buffer mnc_stage_bridge_train_backward reads."""
    n, G = rois.shape[0], gt_boxes.shape[0]
    C = seg_cls_prob.shape[1]
    if bbox_pred.shape != (n, 4 * C) or gt_masks.dim() != 3 or mask_info.shape != (G, 2):
        raise ValueError("stage_bridge_train: inconsistent shapes")
    if (means is None) != (stds is None):
        raise ValueError("stage_bridge_train: give both means and stds, or neither")
    K, M, dev = n + G, mask_size, rois.device
    e = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
    out = {"rois": e(K, 5), "labels": e(K), "mask_targets": e(K, 1, M, M),
           "mask_weight": e(K, 1, M, M), "gt_mask_info": e(K, 12), "bbox_targets": e(K, 4 * C),
           "bbox_inside_weights": e(K, 4 * C), "bbox_outside_weights": e(K, 4 * C),
           "state": torch.empty(2 * K + 2 * n + 1, dtype=torch.int32, device=dev)}
    dbl4 = lambda v: None if v is None else (ctypes.c_double * 4)(*[float(x) for x in v])
    gm = _f32(gt_masks)
    check(lib.mnc_stage_bridge_train(
        ptr(_f32(rois)), n, ptr(_f32(bbox_pred)), ptr(_f32(seg_cls_prob)), C, ptr(_f32(gt_boxes)),
        G, ptr(gm), gm.shape[1], gm.shape[2], ptr(_f32(im_info)),
        ptr(mask_info.contiguous().to(torch.int32)), dbl4(means), dbl4(stds),
        (ctypes.c_float * 4)(*[float(x) for x in inside_weights]), bbox_thresh, M, binarize_thresh,
        *[ptr(out[k]) for k in (
            "rois", "labels", "mask_targets", "mask_weight", "gt_mask_info", "bbox_targets",
            "bbox_inside_weights", "bbox_outside_weights", "state")], cur_stream()),
        "mnc_stage_bridge_train", launches=2)
    return out


def stage_bridge_train_backward(top_diff, state, rois, bbox_pred, G, clip_thresh=0.0,
                                want_rois=True, want_bbox=True):
    """StageBridgeLayer.backward (stage_bridge_layer.py:82-129).  top_diff (K,5) is the diff of the
    `rois` top; clip_thresh = 1 / clip_base with use_clip, else 0.
    -> (rois_diff (n,5) or None, bbox_pred_diff (n,4C) or None)."""
    n = rois.shape[0]
    C4 = bbox_pred.shape[1]
    dev = rois.device
    new = torch.zeros if n == 0 else torch.empty
    rd = new((n, 5), dtype=torch.float32, device=dev) if want_rois else None
    bd = new((n, C4), dtype=torch.float32, device=dev) if want_bbox else None
    check(lib.mnc_stage_bridge_train_backward(
        ptr(_f32(top_diff)), ptr(state), ptr(_f32(rois)), ptr(_f32(bbox_pred)), n, G, C4 // 4,
        clip_thresh, ptr(rd), ptr(bd), cur_stream()),
        "mnc_stage_bridge_train_backward", launches=int(n > 0 and (want_rois or want_bbox)))
    return rd, bd


def mask_layer_train(mask_pred, gt_masks, gt_masks_info, binarize_thresh=0.4, fg_seg_thresh=0.5):
    """MaskLayer.forward_train (lib/pylayer/mask_layer.py:56-93): mask_pred (N,M*M) or
    (N,1,M,M), gt_masks (G,Hm,Wm) 0/1, gt_masks_info (N,12) as stage_bridge_train writes it
    -> labels (N,) float32."""
    N = mask_pred.shape[0]
    M = int(round((mask_pred.numel() // max(N, 1)) ** 0.5)) if N else 21
    gm = _f32(gt_masks)
    labels = torch.empty((N,), dtype=torch.float32, device=mask_pred.device)
    check(lib.mnc_mask_layer_train(ptr(_f32(mask_pred)), N, M, ptr(gm), gm.shape[0], gm.shape[1],
                                   gm.shape[2], ptr(_f32(gt_masks_info)), binarize_thresh,
                                   fg_seg_thresh, ptr(labels),
                                   cur_stream()), "mnc_mask_layer_train")
    return labels


def mask_layer_train_backward(top_diff, labels):
    """MaskLayer.backward (mask_layer.py:50-54): rows with label > 0 copy top_diff, others 0.
    top_diff (N,1,M,M) -> (N,M*M)."""
    N = top_diff.shape[0]
    M = top_diff.shape[-1]
    out = torch.empty((N, M * M), dtype=torch.float32, device=top_diff.device)
    check(lib.mnc_mask_layer_train_backward(ptr(_f32(top_diff)), ptr(_f32(labels)), N, M, ptr(out),
                                            cur_stream()), "mnc_mask_layer_train_backward")
    return out


# ------------------------------------------------------------------ training-phase RPN-stage layers
def sample_keys(*shape, device):
    """Random uint32 sampling keys (as int32) from torch's generator on `device`: the chosen subset
    of a category is its candidates with the smallest (key, index) pairs (include/mnc_b200.h)."""
    return torch.randint(-2 ** 31, 2 ** 31, shape, dtype=torch.int32, device=device)


def proposal_train(cls, bbox, im_info, H, W, pre_nms_top_n=12000, post_nms_top_n=300,
                   nms_thresh=0.7, min_size=16.0, feat_stride=16):
    """ProposalLayer.forward, TRAIN phase (lib/pylayer/proposal_layer.py:52-175), one image: the
    TEST chain, then the proposal_index top and the backward's state.  cls (1,2A,H,W) scores,
    bbox (1,4A,H,W).  -> (rois (R,5), proposal_index (R,), count int32 (1,), state int32 (R,2));
    rows past count are zero RoIs with index -1."""
    cls, bbox, im_info = _f32(cls), _f32(bbox), _f32(im_info).view(1, 3)
    rois, counts, mid = proposals_from_rpn(cls, bbox, im_info, 1, H, W, "nchw", apply_softmax=False,
                                           pre_nms_top_n=pre_nms_top_n, post_nms_top_n=post_nms_top_n,
                                           nms_thresh=nms_thresh, min_size=min_size,
                                           batch_index_mode=False, return_intermediate=True)
    R = rois.shape[1]
    index = torch.empty((R,), dtype=torch.float32, device=cls.device)
    state = _i32(R, 2, device=cls.device)
    check(lib.mnc_proposal_train_state(ptr(mid["order"]), ptr(mid["keep"]), ptr(mid["num"]), R,
                                       ptr(bbox), H, W, feat_stride, ptr(im_info), ptr(index),
                                       ptr(state), cur_stream()),
          "mnc_proposal_train_state", launches=int(R > 0))
    return rois[0], index, counts, state


def proposal_backward(top_diff, state, bbox, clip_thresh=0.0):
    """ProposalLayer.backward (proposal_layer.py:177-230): top_diff (R,5) of the rois top, bbox
    (1,4A,H,W) the rpn_bbox_pred data -> its diff (1,4A,H,W)."""
    bbox = _f32(bbox)
    H, W = bbox.shape[-2:]
    out = torch.empty_like(bbox)
    R = state.shape[0]
    check(lib.mnc_proposal_backward(ptr(_f32(top_diff)), R, ptr(state), ptr(bbox), H, W,
                                    clip_thresh, ptr(out), cur_stream()),
          "mnc_proposal_backward", launches=1 + int(R > 0))
    return out


def proposal_target_capacity(batch_size, fg_fraction, bg_fraction):
    return int(lib.mnc_proposal_target_capacity(batch_size, len(fg_fraction), len(bg_fraction)))


def proposal_target(rpn_rois, rpn_rois_index, gt_boxes, gt_masks, mask_info, im_info, keys,
                    batch_size=64, fg_fraction=(0.3,), fg_thresh_lo=(0.5,), fg_thresh_hi=(1.0,),
                    bg_fraction=(0.85, 0.15), bg_thresh_lo=(0.1, 0.0), bg_thresh_hi=(0.5, 0.1),
                    means=None, stds=None, inside_weights=(1.0, 1.0, 1.0, 1.0), mask_size=21,
                    binarize_thresh=0.4, num_classes=21, n_valid=None):
    """ProposalTargetLayer.forward (lib/pylayer/proposal_target_layer.py:62-107,118-216), one image.
    rpn_rois (n,5), rpn_rois_index (n,) or (1,n) (MIX_INDEX), gt_boxes (G,5), gt_masks (G,Hm,Wm)
    0/1, mask_info (G,2), im_info (3,), keys int32 (len(fg_fraction) + len(bg_fraction), n + G).
    Config defaults are cfg.TRAIN's (lib/mnc_config.py:36-69); means / stds None: targets not
    normalised.  n_valid: int32 device count (proposal_train's `count`) -- rows of rpn_rois past it
    are padding and take no part -- or None: all n rows are RoIs.  -> dict of the tops at Kmax = proposal_target_capacity(...) rows, `counts` int32
    (4,) = K, #fg_inds, #bg_inds, #fg rows, and `state` for proposal_target_backward."""
    n, G = rpn_rois.shape[0], gt_boxes.shape[0]
    ncat = len(fg_fraction) + len(bg_fraction)
    if keys.shape != (ncat, n + G) or mask_info.shape != (G, 2) or gt_masks.dim() != 3:
        raise ValueError("proposal_target: inconsistent shapes")
    if (means is None) != (stds is None):
        raise ValueError("proposal_target: give both means and stds, or neither")
    dev = rpn_rois.device
    Kmax = proposal_target_capacity(batch_size, fg_fraction, bg_fraction)
    M, C = mask_size, num_classes
    e = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
    out = {"rois": e(Kmax, 5), "labels": e(Kmax), "bbox_targets": e(Kmax, 4 * C),
           "bbox_inside_weights": e(Kmax, 4 * C), "bbox_outside_weights": e(Kmax, 4 * C),
           "mask_targets": e(Kmax, 1, M, M), "mask_weight": e(Kmax, 1, M, M),
           "gt_masks_info": e(Kmax, 12), "fg_inds": e(Kmax), "bg_inds": e(Kmax),
           "counts": _i32(4, device=dev),
           "state": _i32(int(lib.mnc_proposal_target_state_ints(n, G, Kmax)), device=dev)}
    dbl = lambda v: None if v is None else (ctypes.c_double * len(v))(*[float(x) for x in v])
    gm = _f32(gt_masks)
    idx = _f32(rpn_rois_index).reshape(-1) if n else None
    check(lib.mnc_proposal_target(
        ptr(_f32(rpn_rois)), n, ptr(idx),
        ptr(None if n_valid is None else n_valid.contiguous().to(torch.int32)), ptr(_f32(gt_boxes)),
        G, ptr(gm), gm.shape[1], gm.shape[2], ptr(mask_info.contiguous().to(torch.int32)),
        ptr(_f32(im_info)), ptr(keys.contiguous().to(torch.int32)), batch_size,
        len(fg_fraction), dbl(fg_fraction), dbl(fg_thresh_lo), dbl(fg_thresh_hi),
        len(bg_fraction), dbl(bg_fraction), dbl(bg_thresh_lo), dbl(bg_thresh_hi),
        dbl(means), dbl(stds), (ctypes.c_float * 4)(*[float(x) for x in inside_weights]), M,
        binarize_thresh, C, Kmax, *[ptr(out[k]) for k in (
            "rois", "labels", "bbox_targets", "bbox_inside_weights", "bbox_outside_weights",
            "mask_targets", "mask_weight", "gt_masks_info", "fg_inds", "bg_inds", "counts",
            "state")], cur_stream()), "mnc_proposal_target", launches=2)
    return out


def proposal_target_backward(top_diff, state, n, G, bp_all=True):
    """ProposalTargetLayer.backward (proposal_target_layer.py:109-115): top_diff (Kmax,5) of the
    rois top -> rpn_rois diff (n,5); rows >= K of top_diff are never read."""
    dev = state.device
    out = (torch.zeros if n == 0 else torch.empty)((n, 5), dtype=torch.float32, device=dev)
    check(lib.mnc_proposal_target_backward(ptr(_f32(top_diff)), ptr(state), n, G, int(bool(bp_all)),
                                           ptr(out), cur_stream()),
          "mnc_proposal_target_backward", launches=int(n > 0))
    return out


def anchor_target(H, W, gt_boxes, im_info, keys, fg_inds=None, bg_inds=None, counts=None,
                  feat_stride=16, allowed_border=0, negative_overlap=0.3, positive_overlap=0.7,
                  clobber_positives=False, fg_fraction=0.5, batch_size=256, positive_weight=-1.0,
                  inside_weights=(1.0, 1.0, 1.0, 1.0)):
    """AnchorTargetLayer.forward (lib/pylayer/anchor_target_layer.py:51-209), one image.  gt_boxes
    (G,5), im_info (3,), keys int32 (H*W*A,) in (h, w, a) order; fg_inds / bg_inds / counts as
    proposal_target returns them (MIX_INDEX) or None.  Config defaults are cfg.TRAIN's
    (lib/mnc_config.py:75-98).  -> (labels (1,1,A*H,W), bbox_targets, bbox_inside_weights,
    bbox_outside_weights (1,4A,H,W))."""
    dev = gt_boxes.device
    A = 9
    if keys.numel() != H * W * A:
        raise ValueError("anchor_target: keys must hold one key per anchor")
    if (fg_inds is None) != (counts is None) or (bg_inds is None) != (counts is None):
        raise ValueError("anchor_target: give fg_inds, bg_inds and counts together")
    G = gt_boxes.shape[0]
    ws = torch.empty(int(lib.mnc_anchor_target_workspace_bytes(H, W, G)), dtype=torch.uint8,
                     device=dev)
    labels = torch.empty((1, 1, A * H, W), dtype=torch.float32, device=dev)
    t = [torch.empty((1, 4 * A, H, W), dtype=torch.float32, device=dev) for _ in range(3)]
    cap = fg_inds.numel() if fg_inds is not None else 0
    check(lib.mnc_anchor_target(
        H, W, feat_stride, allowed_border, ptr(_f32(gt_boxes)), G, ptr(_f32(im_info)),
        ptr(keys.contiguous().to(torch.int32)), ptr(None if fg_inds is None else _f32(fg_inds)),
        ptr(None if bg_inds is None else _f32(bg_inds)), ptr(counts), cap, negative_overlap,
        positive_overlap, int(bool(clobber_positives)), fg_fraction, batch_size, positive_weight,
        (ctypes.c_float * 4)(*[float(x) for x in inside_weights]), ptr(ws), ptr(labels),
        ptr(t[0]), ptr(t[1]), ptr(t[2]), cur_stream()), "mnc_anchor_target", launches=5)
    return (labels, *t)
