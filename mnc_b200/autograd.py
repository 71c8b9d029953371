"""The four Caffe layers as torch.autograd.Functions: the forward is the layer's *_nchw entry
point, the backward the matching *_backward_nchw one (include/mnc_b200.h), so ``loss.backward()``
reaches the feature map, the RoI coordinates and the mask with the reference's gradients
(DESIGN.md "Backward semantics").  fp32 contiguous CUDA tensors; no PyTorch arithmetic on the hot
path.

    feat.requires_grad_(); rois.requires_grad_()
    out = autograd.roi_warp(feat, rois, 28, 28, 0.0625)
    out.sum().backward()        # feat.grad (B,C,H,W), rois.grad (R,5)
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
