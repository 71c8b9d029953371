"""Host mirrors of the native MNC Caffe layers, keeping the C++ layer contract
(LayerSetUp once, Reshape before every forward, Forward_gpu, Backward_gpu;
caffe-mnc/include/caffe/layer.hpp:131,336-346,452-487).  bottom/top are lists of caffe.Blob; layer
params are the prototxt message as a dict.  Backward reads top[0].diff and writes bottom[i].diff
with the zeroing rules of each reference Backward_gpu.  CPU mode is LOG(FATAL) in the reference
(roi_warping_layer.cpp:47) and absent here."""
import numpy as np
import torch

from mnc_b200 import ops


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda()


def _diff(blob):
    """blob.diff, (re)allocated as zeros when missing or not of the data's shape."""
    if blob.diff is None or blob.diff.shape != blob.data.shape:
        blob.diff = np.zeros(blob.data.shape, dtype=np.float32)
    return blob.diff


class _NativeLayer(object):
    def __init__(self, layer_param=None):
        self.layer_param_ = layer_param or {}

    def LayerSetUp(self, bottom, top):
        pass

    def Reshape(self, bottom, top):
        pass

    def Forward_cpu(self, bottom, top):
        raise NotImplementedError("NOT_IMPLEMENTED (as in the reference)")

    def Forward(self, bottom, top):
        self.Reshape(bottom, top)
        self.Forward_gpu(bottom, top)

    def Backward_cpu(self, top, propagate_down, bottom):
        raise NotImplementedError("NOT_IMPLEMENTED (as in the reference)")

    def Backward(self, top, propagate_down, bottom):
        self.Backward_gpu(top, propagate_down, bottom)


class ROIWarpingLayer(_NativeLayer):
    """roi_warping_layer.cpp:20-42 (setup/reshape), roi_warping_layer.cu:110-122 (forward)."""

    def LayerSetUp(self, bottom, top):
        p = self.layer_param_.get("roi_warping_param", {})
        if p.get("pooled_h", 0) <= 0:
            raise ValueError("pooled_h must be > 0")
        if p.get("pooled_w", 0) <= 0:
            raise ValueError("pooled_w must be > 0")
        self.pooled_height_ = int(p["pooled_h"])
        self.pooled_width_ = int(p["pooled_w"])
        self.spatial_scale_ = float(p.get("spatial_scale", 1.0))

    def Reshape(self, bottom, top):
        if len(bottom) != 2 or len(top) != 1:
            raise ValueError("ROIWarping takes exactly 2 bottoms and 1 top")
        self.channels_ = bottom[0].channels
        self.height_ = bottom[0].height
        self.width_ = bottom[0].width
        top[0].reshape(bottom[1].num, self.channels_, self.pooled_height_, self.pooled_width_)

    def Forward_gpu(self, bottom, top):
        out = ops.roi_warp_nchw(_dev(bottom[0].data), _dev(bottom[1].data).view(-1, 5),
                                self.pooled_height_, self.pooled_width_, self.spatial_scale_)
        top[0].data[...] = out.cpu().numpy()

    def Backward_gpu(self, top, propagate_down, bottom):
        """roi_warping_layer.cu:379-436: both diffs are zeroed, then filled where propagated."""
        fd, rd = _diff(bottom[0]), _diff(bottom[1])
        want_f, want_r = bool(propagate_down[0]), bool(propagate_down[1])
        gf, gr = None, None
        if want_f or want_r:
            gf, gr = ops.roi_warp_backward_nchw(
                _dev(bottom[0].data), _dev(bottom[1].data).view(-1, 5), _dev(top[0].diff),
                self.pooled_height_, self.pooled_width_, self.spatial_scale_,
                want_feat=want_f, want_rois=want_r)
        fd[...] = gf.cpu().numpy() if want_f else 0
        rd[...] = gr.cpu().numpy().reshape(rd.shape) if want_r else 0


class MaskResizeLayer(_NativeLayer):
    """mask_resize_layer.cpp:13-30, mask_resize_layer.cu:76-84."""

    def LayerSetUp(self, bottom, top):
        p = self.layer_param_.get("mask_resize_param", {})
        self.output_height_ = int(p["output_height"])
        self.output_width_ = int(p["output_width"])

    def Reshape(self, bottom, top):
        b = bottom[0]
        top[0].reshape(b.num, b.channels, self.output_height_, self.output_width_)

    def Forward_gpu(self, bottom, top):
        out = ops.mask_resize_nchw(_dev(bottom[0].data), self.output_height_, self.output_width_)
        top[0].data[...] = out.cpu().numpy()

    def Backward_gpu(self, top, propagate_down, bottom):
        """mask_resize_layer.cu:175-183: always writes the bottom diff."""
        b = bottom[0]
        _diff(b)[...] = ops.mask_resize_backward_nchw(_dev(top[0].diff), b.height, b.width).cpu().numpy()


class MaskPoolingLayer(_NativeLayer):
    """mask_pooling_layer.cpp:20-29 (shape CHECKs), mask_pooling_layer.cu:29-41."""

    def Reshape(self, bottom, top):
        f, m = bottom[0], bottom[1]
        if f.num != m.num or f.height != m.height or f.width != m.width or m.channels != 1:
            raise ValueError("MaskPooling: feature (N,C,H,W) and mask (N,1,H,W) must agree")
        top[0].reshape(*f.shape)

    def Forward_gpu(self, bottom, top):
        out = ops.mask_pool_nchw(_dev(bottom[0].data), _dev(bottom[1].data))
        top[0].data[...] = out.cpu().numpy()

    def Backward_gpu(self, top, propagate_down, bottom):
        """mask_pooling_layer.cu:78-99: the feature diff is always zeroed, then filled if
        propagated; the mask diff is written only when propagated."""
        want_f, want_m = bool(propagate_down[0]), bool(propagate_down[1])
        fd = _diff(bottom[0])
        gf, gm = None, None
        if want_f or want_m:
            gf, gm = ops.mask_pool_backward_nchw(_dev(bottom[0].data), _dev(bottom[1].data),
                                                 _dev(top[0].diff), want_feat=want_f, want_mask=want_m)
        fd[...] = gf.cpu().numpy() if want_f else 0
        if want_m:
            _diff(bottom[1])[...] = gm.cpu().numpy()


LAYER_TYPES = {"ROIWarping": ROIWarpingLayer, "MaskResize": MaskResizeLayer,
               "MaskPooling": MaskPoolingLayer}


class ROIPoolingLayer(_NativeLayer):
    """roi_pooling_layer.cpp:20-44 (setup/reshape), roi_pooling_layer.cu:80-105 (forward); the
    layer type of the CFM test net (models/VGG16/cfm/test.prototxt:399-465)."""

    def LayerSetUp(self, bottom, top):
        p = self.layer_param_.get("roi_pooling_param", {})
        if p.get("pooled_h", 0) <= 0:
            raise ValueError("pooled_h must be > 0")
        if p.get("pooled_w", 0) <= 0:
            raise ValueError("pooled_w must be > 0")
        self.pooled_height_ = int(p["pooled_h"])
        self.pooled_width_ = int(p["pooled_w"])
        self.spatial_scale_ = float(p.get("spatial_scale", 1.0))

    def Reshape(self, bottom, top):
        self.channels_ = bottom[0].channels
        self.height_ = bottom[0].height
        self.width_ = bottom[0].width
        top[0].reshape(bottom[1].num, self.channels_, self.pooled_height_, self.pooled_width_)
        self.max_idx_ = np.zeros((bottom[1].num, self.channels_, self.pooled_height_,
                                  self.pooled_width_), dtype=np.int32)

    def Forward_gpu(self, bottom, top):
        arg = torch.empty(self.max_idx_.shape, dtype=torch.int32, device="cuda")
        out = ops.roi_pool_nchw(_dev(bottom[0].data), _dev(bottom[1].data).view(-1, 5),
                                self.pooled_height_, self.pooled_width_, self.spatial_scale_,
                                argmax=arg)
        top[0].data[...] = out.cpu().numpy()
        self.max_idx_[...] = arg.cpu().numpy()

    def Backward_gpu(self, top, propagate_down, bottom):
        """roi_pooling_layer.cu:167-184: nothing is touched unless the feature is propagated; the
        gradient is routed through the argmax of the last forward."""
        if not propagate_down[0]:
            return
        g = ops.roi_pool_backward_nchw(_dev(top[0].diff), torch.from_numpy(self.max_idx_).cuda(),
                                       bottom[0].shape, _dev(bottom[1].data).view(-1, 5),
                                       self.pooled_height_, self.pooled_width_, self.spatial_scale_)
        _diff(bottom[0])[...] = g.cpu().numpy()
