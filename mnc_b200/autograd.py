"""The four Caffe layers as torch.autograd.Functions: the forward is the layer's *_nchw entry
point, the backward the matching *_backward_nchw one (include/mnc_b200.h), so ``loss.backward()``
reaches the feature map, the RoI coordinates and the mask with the reference's gradients
(DESIGN.md "Backward semantics").  fp32 contiguous CUDA tensors; no PyTorch arithmetic on the hot
path.

    feat.requires_grad_(); rois.requires_grad_()
    out = autograd.roi_warp(feat, rois, 28, 28, 0.0625)
    out.sum().backward()        # feat.grad (B,C,H,W), rois.grad (R,5)

The TRAIN phase of the cascade bridges (StageBridgeLayer, MaskLayer) and of the RPN-stage layers
(ProposalLayer, ProposalTargetLayer, AnchorTargetLayer) is here too: their outputs that feed the
next stage are differentiable, the targets they compute are not, so

    rois_ext, *targets = autograd.stage_bridge_train(rois, bbox_pred, seg_cls_prob, ...)
    autograd.roi_warp(conv5_3, rois_ext, 28, 28)

carries the RoI coordinate gradient on into bbox_pred, as the 5-stage training net does.
"""
import torch

from . import ops


def _c(t):
    return t.detach().contiguous()


class _RoiWarp(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feat, rois, pooled_h, pooled_w, spatial_scale):
        feat, rois = _c(feat), _c(rois)
        ctx.save_for_backward(feat, rois)
        ctx.geom = (pooled_h, pooled_w, spatial_scale)
        return ops.roi_warp_nchw(feat, rois, pooled_h, pooled_w, spatial_scale)

    @staticmethod
    def backward(ctx, grad):
        feat, rois = ctx.saved_tensors
        fd, rd = ops.roi_warp_backward_nchw(feat, rois, _c(grad), *ctx.geom,
                                            want_feat=ctx.needs_input_grad[0],
                                            want_rois=ctx.needs_input_grad[1])
        return fd, rd, None, None, None


class _MaskResize(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, out_h, out_w):
        ctx.in_hw = x.shape[2:]
        return ops.mask_resize_nchw(_c(x), out_h, out_w)

    @staticmethod
    def backward(ctx, grad):
        return ops.mask_resize_backward_nchw(_c(grad), *ctx.in_hw), None, None


class _MaskPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feat, mask):
        feat, mask = _c(feat), _c(mask)
        ctx.save_for_backward(feat, mask)
        return ops.mask_pool_nchw(feat, mask)

    @staticmethod
    def backward(ctx, grad):
        feat, mask = ctx.saved_tensors
        return ops.mask_pool_backward_nchw(feat, mask, _c(grad), want_feat=ctx.needs_input_grad[0],
                                           want_mask=ctx.needs_input_grad[1])


class _RoiPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feat, rois, pooled_h, pooled_w, spatial_scale):
        feat, rois = _c(feat), _c(rois)
        argmax = torch.empty((rois.shape[0], feat.shape[1], pooled_h, pooled_w), dtype=torch.int32,
                             device=feat.device)
        out = ops.roi_pool_nchw(feat, rois, pooled_h, pooled_w, spatial_scale, argmax=argmax)
        ctx.save_for_backward(rois, argmax)
        ctx.geom = (feat.shape, pooled_h, pooled_w, spatial_scale)
        return out

    @staticmethod
    def backward(ctx, grad):
        rois, argmax = ctx.saved_tensors
        shape, ph, pw, ss = ctx.geom
        # ROIPooling has no gradient for the RoI coordinates (roi_pooling_layer.cu:167-184)
        return ops.roi_pool_backward_nchw(_c(grad), argmax, shape, rois, ph, pw, ss), None, None, None, None


def roi_warp(feat, rois, pooled_h, pooled_w, spatial_scale=0.0625):
    """ROIWarping: feat (B,C,H,W), rois (R,5) -> (R,C,pooled_h,pooled_w); differentiable in both."""
    return _RoiWarp.apply(feat, rois, pooled_h, pooled_w, spatial_scale)


def mask_resize(x, out_h, out_w):
    """MaskResize: (N,C,ih,iw) -> (N,C,out_h,out_w)."""
    return _MaskResize.apply(x, out_h, out_w)


def mask_pool(feat, mask):
    """MaskPooling: feat (N,C,H,W) * mask (N,1,H,W); differentiable in both."""
    return _MaskPool.apply(feat, mask)


def roi_pool(feat, rois, pooled_h, pooled_w, spatial_scale=0.0625):
    """ROIPooling: feat (B,C,H,W), rois (R,5) -> (R,C,pooled_h,pooled_w); differentiable in feat."""
    return _RoiPool.apply(feat, rois, pooled_h, pooled_w, spatial_scale)


class _StageBridgeTrain(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rois, bbox_pred, seg_cls_prob, gt_boxes, gt_masks, im_info, mask_info, kw,
                clip_thresh):
        rois, bbox_pred = _c(rois), _c(bbox_pred)
        out = ops.stage_bridge_train(rois, bbox_pred, _c(seg_cls_prob), _c(gt_boxes), _c(gt_masks),
                                     _c(im_info), _c(mask_info), **kw)
        ctx.save_for_backward(rois, bbox_pred, out["state"])
        ctx.G, ctx.clip_thresh = gt_boxes.shape[0], clip_thresh
        targets = [out[k] for k in _BRIDGE_TARGETS]
        ctx.mark_non_differentiable(*targets)
        return (out["rois"], *targets)

    @staticmethod
    def backward(ctx, grad, *unused):
        rois, bbox_pred, state = ctx.saved_tensors
        rd, bd = ops.stage_bridge_train_backward(_c(grad), state, rois, bbox_pred, ctx.G,
                                                 ctx.clip_thresh, want_rois=ctx.needs_input_grad[0],
                                                 want_bbox=ctx.needs_input_grad[1])
        return (rd, bd) + (None,) * 7


_BRIDGE_TARGETS = ("labels", "mask_targets", "mask_weight", "gt_mask_info", "bbox_targets",
                   "bbox_inside_weights", "bbox_outside_weights")


class _MaskLayerTrain(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mask_pred, gt_masks, gt_masks_info, kw):
        N = mask_pred.shape[0]
        labels = ops.mask_layer_train(_c(mask_pred), _c(gt_masks), _c(gt_masks_info), **kw)
        ctx.save_for_backward(labels)
        ctx.shape = mask_pred.shape
        ctx.mark_non_differentiable(labels)
        M = int(round((mask_pred.numel() // max(N, 1)) ** 0.5)) if N else 21
        return _c(mask_pred).view(N, 1, M, M), labels.view(N, 1)

    @staticmethod
    def backward(ctx, grad, unused):
        labels, = ctx.saved_tensors
        return ops.mask_layer_train_backward(_c(grad), labels).view(ctx.shape), None, None, None


def stage_bridge_train(rois, bbox_pred, seg_cls_prob, gt_boxes, gt_masks, im_info, mask_info,
                       means=None, stds=None, inside_weights=(1.0, 1.0, 1.0, 1.0), bbox_thresh=0.5,
                       mask_size=21, binarize_thresh=0.4, clip_thresh=0.0):
    """StageBridgeLayer, TRAIN phase (ops.stage_bridge_train).  -> (rois_ext (K,5), labels,
    mask_targets, mask_weight, gt_mask_info, bbox_targets, bbox_inside_weights,
    bbox_outside_weights); rois_ext is differentiable in rois and bbox_pred (the reference's
    backward, clip_thresh = 1 / clip_base with use_clip, else 0), the targets are not."""
    kw = dict(means=means, stds=stds, inside_weights=inside_weights, bbox_thresh=bbox_thresh,
              mask_size=mask_size, binarize_thresh=binarize_thresh)
    return _StageBridgeTrain.apply(rois, bbox_pred, seg_cls_prob, gt_boxes, gt_masks, im_info,
                                   mask_info, kw, clip_thresh)


def mask_layer_train(mask_pred, gt_masks, gt_masks_info, binarize_thresh=0.4, fg_seg_thresh=0.5):
    """MaskLayer, TRAIN phase (ops.mask_layer_train).  -> (mask_proposal (N,1,M,M), a reshape of
    mask_pred differentiable in it, labels (N,1)); the gradient reaches the rows with label > 0."""
    return _MaskLayerTrain.apply(mask_pred, gt_masks, gt_masks_info,
                                 dict(binarize_thresh=binarize_thresh, fg_seg_thresh=fg_seg_thresh))


# --------------------------------------------------------------------- RPN-stage training layers
class _ProposalTrain(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rpn_cls_prob, rpn_bbox_pred, im_info, H, W, kw, clip_thresh):
        bbox = _c(rpn_bbox_pred)
        rois, index, count, state = ops.proposal_train(_c(rpn_cls_prob), bbox, _c(im_info), H, W, **kw)
        ctx.save_for_backward(bbox, state)
        ctx.clip_thresh = clip_thresh
        ctx.mark_non_differentiable(index, count)
        return rois, index, count

    @staticmethod
    def backward(ctx, grad, *unused):
        bbox, state = ctx.saved_tensors
        if not ctx.needs_input_grad[1]:
            return (None,) * 7
        return None, ops.proposal_backward(_c(grad), state, bbox, ctx.clip_thresh), None, None, None, None, None


class _ProposalTarget(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rpn_rois, rpn_rois_index, gt_boxes, gt_masks, mask_info, im_info, keys, kw,
                bp_all):
        out = ops.proposal_target(_c(rpn_rois), _c(rpn_rois_index), _c(gt_boxes), _c(gt_masks),
                                  _c(mask_info), _c(im_info), _c(keys), **kw)
        ctx.save_for_backward(out["state"])
        ctx.nG = (rpn_rois.shape[0], gt_boxes.shape[0])
        ctx.bp_all = bp_all
        targets = [out[k] for k in PROPOSAL_TARGET_TOPS[1:]] + [out["counts"]]
        ctx.mark_non_differentiable(*targets)
        return (out["rois"], *targets)

    @staticmethod
    def backward(ctx, grad, *unused):
        state, = ctx.saved_tensors
        rd = ops.proposal_target_backward(_c(grad), state, *ctx.nG, ctx.bp_all) \
            if ctx.needs_input_grad[0] else None
        return (rd,) + (None,) * 8


PROPOSAL_TARGET_TOPS = ("rois", "labels", "bbox_targets", "bbox_inside_weights",
                        "bbox_outside_weights", "mask_targets", "mask_weight", "gt_masks_info",
                        "fg_inds", "bg_inds")


def proposal_train(rpn_cls_prob, rpn_bbox_pred, im_info, pre_nms_top_n=12000, post_nms_top_n=300,
                   nms_thresh=0.7, min_size=16.0, clip_thresh=0.0):
    """ProposalLayer, TRAIN phase (ops.proposal_train).  rpn_cls_prob (1,2A,H,W), rpn_bbox_pred
    (1,4A,H,W).  -> (rois (R,5), proposal_index (R,), count (1,)); rois is differentiable in
    rpn_bbox_pred with the reference's backward (clip_thresh = 1 / clip_base with use_clip, else
    0).  R = post_nms_top_n; rows past count are zero RoIs with index -1: pass count on to
    proposal_target, which then ignores them (no synchronisation).  Defaults: cfg.TRAIN with mnc_5stage.yml's RPN_POST_NMS_TOP_N."""
    H, W = rpn_bbox_pred.shape[-2:]
    kw = dict(pre_nms_top_n=pre_nms_top_n, post_nms_top_n=post_nms_top_n, nms_thresh=nms_thresh,
              min_size=min_size)
    return _ProposalTrain.apply(rpn_cls_prob, rpn_bbox_pred, im_info, H, W, kw, clip_thresh)


def proposal_target(rpn_rois, rpn_rois_index, gt_boxes, gt_masks, mask_info, im_info, keys=None,
                    bp_all=True, count=None, **kw):
    """ProposalTargetLayer (ops.proposal_target; keyword config as there).  keys None: drawn with
    ops.sample_keys (torch's generator on the device).  count: proposal_train's device count, the
    rows of rpn_rois that are RoIs (None: all).  -> (rois, labels, bbox_targets,
    bbox_inside_weights, bbox_outside_weights, mask_targets, mask_weight, gt_masks_info, fg_inds,
    bg_inds, counts), padded to the capacity; rois is differentiable in rpn_rois (the rows of
    keep_inds, or of the fg rows with bp_all off), the rest is not."""
    if keys is None:
        ncat = len(kw.get("fg_fraction", (0.3,))) + len(kw.get("bg_fraction", (0.85, 0.15)))
        keys = ops.sample_keys(ncat, rpn_rois.shape[0] + gt_boxes.shape[0], device=rpn_rois.device)
    return _ProposalTarget.apply(rpn_rois, rpn_rois_index, gt_boxes, gt_masks, mask_info, im_info,
                                 keys, dict(kw, n_valid=count), bp_all)


def anchor_target(H, W, gt_boxes, im_info, fg_inds=None, bg_inds=None, counts=None, keys=None,
                  **kw):
    """AnchorTargetLayer (ops.anchor_target; not differentiable).  keys None: drawn with
    ops.sample_keys."""
    if keys is None:
        keys = ops.sample_keys(H * W * 9, device=gt_boxes.device)
    with torch.no_grad():
        return ops.anchor_target(H, W, gt_boxes.detach(), im_info.detach(), keys, fg_inds, bg_inds,
                                 counts, **kw)
