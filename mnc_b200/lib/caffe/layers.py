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


# ------------------------------------------------------------------ training-net loss layers
class _LossLayer(_NativeLayer):
    """LossLayer (loss_layer.cpp:8-27): loss_weight 1 unless given, which Layer::SetUp copies to
    top[0]'s diff (layer.hpp:417-433); bottoms 0 and 1 agree in num; the top is a scalar."""

    def LayerSetUp(self, bottom, top):
        w = self.layer_param_.get("loss_weight", 1.0)
        w = w[0] if isinstance(w, (list, tuple)) else w
        top[0].diff = np.full((), w, dtype=np.float32)

    def Reshape(self, bottom, top):
        if bottom[0].num != bottom[1].num:
            raise ValueError("The data and label should have the same number.")
        top[0].reshape()

    def _top_diff(self, top):
        return _dev(top[0].diff)

    def _no_label_backward(self, propagate_down):
        if len(propagate_down) > 1 and any(propagate_down[1:]):
            raise ValueError("%s Layer cannot backpropagate to label inputs." % self.TYPE)


class SoftmaxWithLossLayer(_LossLayer):
    """softmax_loss_layer.cpp:10-56 (setup / reshape), softmax_loss_layer.cu:32-124."""
    TYPE = "SoftmaxWithLoss"

    def LayerSetUp(self, bottom, top):
        _LossLayer.LayerSetUp(self, bottom, top)
        if self.layer_param_.get("softmax_param", {}).get("axis", 1) != 1:
            raise ValueError("SoftmaxWithLoss: only the channel axis (1) is supported")
        p = self.layer_param_.get("loss_param", {})
        self.ignore_label_ = int(p["ignore_label"]) if "ignore_label" in p else None
        if "normalization" not in p and "normalize" in p:
            self.normalization_ = "VALID" if p["normalize"] else "BATCH_SIZE"
        else:
            self.normalization_ = p.get("normalization", "VALID")
        if self.normalization_ not in ops.NORMALIZATION:
            raise ValueError("Unknown normalization mode: %s" % self.normalization_)

    def Reshape(self, bottom, top):
        _LossLayer.Reshape(self, bottom, top)
        b = bottom[0]
        if b.num * (b.count // max(b.num * b.channels, 1)) != bottom[1].count:
            raise ValueError("Number of labels must match number of predictions")
        if len(top) >= 2:
            top[1].reshape(*b.shape)

    def Forward_gpu(self, bottom, top):
        loss, self.prob_ = ops.softmax_loss(_dev(bottom[0].data), _dev(bottom[1].data),
                                            self.ignore_label_, self.normalization_)
        top[0].data[...] = loss.cpu().numpy()
        if len(top) == 2:
            top[1].data[...] = self.prob_.cpu().numpy()

    def Backward_gpu(self, top, propagate_down, bottom):
        self._no_label_backward(propagate_down)
        if propagate_down[0]:
            g = ops.softmax_loss_backward(self.prob_, _dev(bottom[1].data), self._top_diff(top),
                                          self.ignore_label_, self.normalization_)
            _diff(bottom[0])[...] = g.cpu().numpy()


class SmoothL1LossLayer(_LossLayer):
    """smooth_L1_loss_layer.cpp:13-44 (setup / reshape), smooth_L1_loss_layer.cu:31-106.  The
    backward to bottom 1 (the targets) is not reachable in the training net and not provided."""
    TYPE = "SmoothL1Loss"

    def LayerSetUp(self, bottom, top):
        _LossLayer.LayerSetUp(self, bottom, top)
        self.sigma_ = float(self.layer_param_.get("smooth_l1_loss_param", {}).get("sigma", 1.0))
        self.has_weights_ = len(bottom) >= 3
        if self.has_weights_ and len(bottom) != 4:
            raise ValueError("If weights are used, must specify both inside and outside weights")

    def Reshape(self, bottom, top):
        _LossLayer.Reshape(self, bottom, top)
        b = bottom[0]
        for o in bottom[1:]:
            if (o.channels, o.height, o.width) != (b.channels, b.height, b.width):
                raise ValueError("SmoothL1Loss: bottoms must agree in channels, height and width")

    def _args(self, bottom):
        t = [_dev(x.data) for x in bottom]
        return t + [None] * (4 - len(t))

    def Forward_gpu(self, bottom, top):
        top[0].data[...] = ops.smooth_l1_loss(*self._args(bottom), sigma=self.sigma_).cpu().numpy()

    def Backward_gpu(self, top, propagate_down, bottom):
        if len(propagate_down) > 1 and propagate_down[1]:
            raise ValueError("SmoothL1Loss: the backward to the targets is not provided")
        if propagate_down[0]:
            g = ops.smooth_l1_loss_backward(*self._args(bottom), sigma=self.sigma_,
                                            top_diff=self._top_diff(top))
            _diff(bottom[0])[...] = g.cpu().numpy()


class SigmoidCrossEntropyLossLayer(_LossLayer):
    """sigmoid_cross_entropy_loss_layer.cpp:8-97, MNC's form: a third bottom weighs each element
    and normalises by the weights' sum; with that sum 0 the top is left as it was."""
    TYPE = "SigmoidCrossEntropyLoss"

    def Reshape(self, bottom, top):
        _LossLayer.Reshape(self, bottom, top)
        if bottom[0].count != bottom[1].count:
            raise ValueError("SIGMOID_CROSS_ENTROPY_LOSS layer inputs must have the same count.")
        if len(bottom) == 3 and bottom[0].count != bottom[2].count:
            raise ValueError("SIGMOID_CROSS_ENTROPY_LOSS layer weight must be the same count")

    def _args(self, bottom):
        return [_dev(x.data) for x in bottom[:3]] + [None] * (3 - min(len(bottom), 3))

    def Forward_gpu(self, bottom, top):
        out = _dev(top[0].data if top[0].data.shape == () else 0.0).reshape(())
        top[0].data[...] = ops.sigmoid_ce_loss(*self._args(bottom), out=out).cpu().numpy()

    def Backward_gpu(self, top, propagate_down, bottom):
        self._no_label_backward(propagate_down)
        if propagate_down[0]:
            g = ops.sigmoid_ce_loss_backward(*self._args(bottom), top_diff=self._top_diff(top))
            _diff(bottom[0])[...] = g.cpu().numpy()


class AccuracyLayer(_NativeLayer):
    """accuracy_layer.cpp:10-103, top 0 only (the per-class top is not provided)."""

    def LayerSetUp(self, bottom, top):
        p = self.layer_param_.get("accuracy_param", {})
        self.top_k_ = int(p.get("top_k", 1))
        self.ignore_label_ = int(p["ignore_label"]) if "ignore_label" in p else None
        if p.get("axis", 1) != 1:
            raise ValueError("Accuracy: only the channel axis (1) is supported")
        if len(top) > 1:
            raise ValueError("Accuracy: the per-class top is not provided")

    def Reshape(self, bottom, top):
        b = bottom[0]
        if self.top_k_ > b.count // max(bottom[1].count, 1):
            raise ValueError("top_k must be less than or equal to the number of classes.")
        if b.num * (b.count // max(b.num * b.channels, 1)) != bottom[1].count:
            raise ValueError("Number of labels must match number of predictions")
        top[0].reshape()

    def Forward_gpu(self, bottom, top):
        top[0].data[...] = ops.accuracy(_dev(bottom[0].data), _dev(bottom[1].data), self.top_k_,
                                        self.ignore_label_).cpu().numpy()

    def Backward_gpu(self, top, propagate_down, bottom):
        if any(propagate_down):
            raise NotImplementedError("NOT_IMPLEMENTED (as in the reference)")



# ------------------------------------------------------------------ head layers of the training net
class InnerProductLayer(_NativeLayer):
    """inner_product_layer.cpp:10-87 (setup / reshape, axis 1), inner_product_layer.cu:9-55.
    blobs_ = [W (N, K), b (N)]; set their data before the first Forward.  Backward ADDS to the
    blobs' diffs (beta 1), so a layer given another layer's blobs_ (fc6_ext sharing fc6's) sums the
    two uses' gradients, as Caffe's shared parameters do; the solver zeroes them per step."""

    def LayerSetUp(self, bottom, top):
        from mnc_b200.lib.caffe import Blob
        p = self.layer_param_.get("inner_product_param", {})
        if int(p.get("axis", 1)) != 1:
            raise ValueError("InnerProduct: only axis 1 is supported")
        if p.get("transpose", False):
            raise ValueError("InnerProduct: transpose is not supported")
        self.N_ = int(p["num_output"])
        self.bias_term_ = bool(p.get("bias_term", True))
        self.K_ = bottom[0].count // bottom[0].num
        self.blobs_ = [Blob(self.N_, self.K_)] + ([Blob(self.N_)] if self.bias_term_ else [])
        self.param_propagate_down_ = [True] * len(self.blobs_)

    def Reshape(self, bottom, top):
        if bottom[0].count // bottom[0].num != self.K_:
            raise ValueError("Input size incompatible with inner product parameters.")
        top[0].reshape(bottom[0].num, self.N_)

    def _params(self):
        w = _dev(self.blobs_[0].data)
        b = _dev(self.blobs_[1].data) if self.bias_term_ else None
        return w, b

    def Forward_gpu(self, bottom, top):
        w, b = self._params()
        top[0].data[...] = ops.fc_forward(_dev(bottom[0].data), w, b).cpu().numpy()

    def Backward_gpu(self, top, propagate_down, bottom):
        w, _ = self._params()
        want_w = self.param_propagate_down_[0]
        want_b = self.bias_term_ and self.param_propagate_down_[1]
        want_x = bool(propagate_down[0])
        dw = _dev(_diff(self.blobs_[0])) if want_w else None
        db = _dev(_diff(self.blobs_[1])) if want_b else None
        if not (want_w or want_b or want_x):
            return
        dx = ops.fc_backward(_dev(bottom[0].data), w, _dev(top[0].diff), dw=dw, db=db,
                             want_dx=want_x)
        if want_w:
            self.blobs_[0].diff[...] = dw.cpu().numpy()
        if want_b:
            self.blobs_[1].diff[...] = db.cpu().numpy()
        if want_x:
            _diff(bottom[0])[...] = dx.cpu().numpy().reshape(bottom[0].shape)


class PoolingLayer(_NativeLayer):
    """pooling_layer.cpp:12-100 (setup / reshape), pooling_layer.cu MaxPoolForward /
    MaxPoolBackward; MAX only, kernel 2, stride 2, pad 0 (the head pools of the nets)."""

    def LayerSetUp(self, bottom, top):
        p = self.layer_param_.get("pooling_param", {})
        ok = (p.get("pool", "MAX") in ("MAX", 0) and int(p.get("kernel_size", 0)) == 2 and
              int(p.get("stride", 1)) == 2 and int(p.get("pad", 0)) == 0 and
              not p.get("global_pooling", False))
        if not ok:
            raise ValueError("Pooling: only MAX with kernel_size 2, stride 2, pad 0 is supported")

    def Reshape(self, bottom, top):
        b = bottom[0]
        top[0].reshape(b.num, b.channels, ops._pool_out(b.height), ops._pool_out(b.width))

    def Forward_gpu(self, bottom, top):
        y, self.max_idx_ = ops.max_pool_nchw(_dev(bottom[0].data))
        top[0].data[...] = y.cpu().numpy()

    def Backward_gpu(self, top, propagate_down, bottom):
        """pooling_layer.cu: nothing is written unless propagated."""
        if not propagate_down[0]:
            return
        _diff(bottom[0])[...] = ops.max_pool_backward_nchw(
            _dev(top[0].diff), self.max_idx_, bottom[0].shape).cpu().numpy()


class ReLULayer(_NativeLayer):
    """relu_layer.cu:9-41, negative_slope 0 (the nets' ReLUs)."""

    def LayerSetUp(self, bottom, top):
        if float(self.layer_param_.get("relu_param", {}).get("negative_slope", 0.0)) != 0.0:
            raise ValueError("ReLU: only negative_slope 0 is supported")

    def Reshape(self, bottom, top):
        top[0].reshape(*bottom[0].shape)

    def Forward_gpu(self, bottom, top):
        top[0].data[...] = ops.relu(_dev(bottom[0].data)).cpu().numpy()

    def Backward_gpu(self, top, propagate_down, bottom):
        if propagate_down[0]:
            _diff(bottom[0])[...] = ops.relu_backward(_dev(bottom[0].data),
                                                      _dev(top[0].diff)).cpu().numpy()


class SigmoidLayer(_NativeLayer):
    """sigmoid_layer.cu:10-40; the backward reads the top's data."""

    def Reshape(self, bottom, top):
        top[0].reshape(*bottom[0].shape)

    def Forward_gpu(self, bottom, top):
        top[0].data[...] = ops.sigmoid(_dev(bottom[0].data)).cpu().numpy()

    def Backward_gpu(self, top, propagate_down, bottom):
        if propagate_down[0]:
            _diff(bottom[0])[...] = ops.sigmoid_backward(_dev(top[0].data),
                                                         _dev(top[0].diff)).cpu().numpy()


def _conv_field(p, name, default):
    """A repeated uint field of convolution_param (kernel_size, pad, stride, dilation) as one value:
    a single entry, or several equal ones; unequal entries (a non-square form) raise."""
    v = p.get(name, default)
    vals = [int(u) for u in v] if isinstance(v, (list, tuple)) else [int(v)]
    if not vals:
        vals = [default]
    if len(set(vals)) != 1:
        raise ValueError("Convolution: only square %s is supported" % name)
    return vals[0]


class ConvolutionLayer(_NativeLayer):
    """base_conv_layer.cpp:12-186 (setup / reshape), conv_layer.cu:10-62; stride 1 with kernel 3 /
    pad 1 or kernel 1 / pad 0, dilation 1, group 1 (the trunk and RPN convolutions of the nets).
    blobs_ = [W (Cout, Cin, k, k), b (Cout)]; set their data before the first Forward.  Backward
    ADDS to the blobs' diffs (beta 1) and honours param_propagate_down_ (False for a frozen,
    lr_mult 0, layer: its diffs are neither computed nor touched) and propagate_down."""

    def LayerSetUp(self, bottom, top):
        from mnc_b200.lib.caffe import Blob
        p = self.layer_param_.get("convolution_param", {})
        for hw in ("kernel_h", "kernel_w", "pad_h", "pad_w", "stride_h", "stride_w"):
            if hw in p:
                raise ValueError("Convolution: %s is not supported" % hw)
        k = _conv_field(p, "kernel_size", 0)
        pad = _conv_field(p, "pad", 0)
        stride = _conv_field(p, "stride", 1)
        dilation = _conv_field(p, "dilation", 1)
        if not (stride == 1 and dilation == 1 and int(p.get("group", 1)) == 1 and
                int(p.get("axis", 1)) == 1 and (k, pad) in ((3, 1), (1, 0))):
            raise ValueError("Convolution: only kernel 3 / pad 1 or kernel 1 / pad 0 at stride 1, "
                             "dilation 1, group 1 is supported")
        self.k_, self.pad_ = k, pad
        self.num_output_ = int(p["num_output"])
        self.bias_term_ = bool(p.get("bias_term", True))
        self.channels_ = bottom[0].channels
        self.blobs_ = [Blob(self.num_output_, self.channels_, k, k)] + \
            ([Blob(self.num_output_)] if self.bias_term_ else [])
        self.param_propagate_down_ = [True] * len(self.blobs_)

    def Reshape(self, bottom, top):
        b = bottom[0]
        if b.channels != self.channels_:
            raise ValueError("Input size incompatible with convolution kernel.")
        top[0].reshape(b.num, self.num_output_, b.height, b.width)

    def _params(self):
        w = _dev(self.blobs_[0].data)
        b = _dev(self.blobs_[1].data) if self.bias_term_ else None
        return w, b

    def Forward_gpu(self, bottom, top):
        w, b = self._params()
        top[0].data[...] = ops.conv_forward(_dev(bottom[0].data), w, b, pad=self.pad_).cpu().numpy()

    def Backward_gpu(self, top, propagate_down, bottom):
        w, _ = self._params()
        want_w = self.param_propagate_down_[0]
        want_b = self.bias_term_ and self.param_propagate_down_[1]
        want_x = bool(propagate_down[0])
        if not (want_w or want_b or want_x):
            return
        dw = _dev(_diff(self.blobs_[0])) if want_w else None
        db = _dev(_diff(self.blobs_[1])) if want_b else None
        dx = ops.conv_backward(_dev(bottom[0].data), w, _dev(top[0].diff), dw=dw, db=db,
                               want_dx=want_x)
        if want_w:
            self.blobs_[0].diff[...] = dw.cpu().numpy()
        if want_b:
            self.blobs_[1].diff[...] = db.cpu().numpy()
        if want_x:
            _diff(bottom[0])[...] = dx.cpu().numpy()
