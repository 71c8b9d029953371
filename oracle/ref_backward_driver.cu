// oracle/ref_backward_driver.cu -- TEST INFRASTRUCTURE.  C entry points that run the reference's
// own layer objects (compiled unmodified from the reference checkout, see oracle/Makefile) the
// way Caffe's Net does for a training step: construct from a LayerParameter, SetUp (LayerSetUp +
// Reshape), Forward (Reshape + Forward_gpu), fill the top diff, then Backward (Backward_gpu) on the
// same layer object, so the argmax / buffer blobs it reads are the layer's own.  Plain host
// pointers in and out; ctypes binds these in tests/test_ref_pin_backward.py and
// scripts/bench_roi_backward.py.
#include <cstring>

#include "caffe/fast_rcnn_layers.hpp"
#include "caffe/layers/mask_resize_layer.hpp"

using namespace caffe;

namespace {
// Layer::Backward in GPU mode (caffe-mnc/include/caffe/layer.hpp:472-487) is Backward_gpu, which
// the layer classes keep protected: reach it from a subclass.
template <typename L>
struct Open : L {
  explicit Open(const LayerParameter& p) : L(p) {}
  void Backward(const vector<Blob<float>*>& top, const vector<bool>& propagate_down,
                const vector<Blob<float>*>& bottom) {
    this->Backward_gpu(top, propagate_down, bottom);
  }
};

void fill(Blob<float>* b, const float* src) {
  std::memcpy(b->mutable_cpu_data(), src, sizeof(float) * b->count());
}
void fill_diff(Blob<float>* b, const float* src) {
  std::memcpy(b->mutable_cpu_diff(), src, sizeof(float) * b->count());
}
void fetch_diff(Blob<float>* b, float* dst) {
  if (dst) std::memcpy(dst, b->cpu_diff(), sizeof(float) * b->count());
}
// Backward, then (iters > 0) `iters` more Backward calls on the same layer, each between a pair
// of CUDA events; times[i] receives the i-th call's milliseconds.
template <typename L>
int backward(Open<L>* layer, const vector<Blob<float>*>& top, const vector<bool>& pd,
             const vector<Blob<float>*>& bottom, int iters, float* times) {
  layer->Backward(top, pd, bottom);
  if (cudaDeviceSynchronize() != cudaSuccess) return 1;
  if (iters > 0) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    for (int i = 0; i < iters; ++i) {
      cudaEventRecord(e0);
      layer->Backward(top, pd, bottom);
      cudaEventRecord(e1);
      cudaEventSynchronize(e1);
      cudaEventElapsedTime(times + i, e0, e1);
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    // the timed calls recompute what the first one wrote
    if (cudaDeviceSynchronize() != cudaSuccess) return 1;
  }
  return 0;
}
}  // namespace

extern "C" {

// ---------------------------------------------------------------------------------------------
// Backward entry points: SetUp, Forward, top diff filled, then Backward_gpu on the same layer.
// Output diffs may be NULL (not fetched).  iters / times: see backward() above.

// ROIWarpingLayer::Backward_gpu (roi_warping_layer.cu:379-436).  Callers must not set pd1 for RoIs
// with a sample outside the map (the coordinate kernel then reads outside the sampled plane) or
// with end < start (it asserts).
int ref_roi_warp_backward(const float* feat, int B, int C, int H, int W, const float* rois, int R,
                          int ph, int pw, float spatial_scale, const float* top_diff, int pd0,
                          int pd1, float* feat_diff, float* rois_diff, int iters, float* times) {
  LayerParameter p;
  p.roi_warping_param_.pooled_h_ = ph;
  p.roi_warping_param_.pooled_w_ = pw;
  p.roi_warping_param_.spatial_scale_ = spatial_scale;
  Open<ROIWarpingLayer<float> > layer(p);
  Blob<float> b0, b1, t0;
  b0.Reshape(B, C, H, W);
  b1.Reshape(R, 5, 1, 1);
  fill(&b0, feat);
  fill(&b1, rois);
  vector<Blob<float>*> bottom(2), top(1);
  bottom[0] = &b0; bottom[1] = &b1; top[0] = &t0;
  layer.SetUp(bottom, top);
  layer.Forward(bottom, top, true);
  if (cudaDeviceSynchronize() != cudaSuccess) return 1;
  fill_diff(&t0, top_diff);
  vector<bool> pd(2);
  pd[0] = pd0 != 0; pd[1] = pd1 != 0;
  if (backward(&layer, top, pd, bottom, iters, times)) return 1;
  fetch_diff(&b0, feat_diff);
  fetch_diff(&b1, rois_diff);
  return 0;
}

// MaskResizeLayer::Backward_gpu (mask_resize_layer.cu:175-183).  The caller keeps every
// reference read of top_diff inside the blob (see tests/test_ref_pin_backward.py).
int ref_mask_resize_backward(const float* in, int N, int C, int ih, int iw, int oh, int ow,
                             const float* top_diff, float* in_diff, int iters, float* times) {
  LayerParameter p;
  p.mask_resize_param_.output_height_ = oh;
  p.mask_resize_param_.output_width_ = ow;
  Open<MaskResizeLayer<float> > layer(p);
  Blob<float> b0, t0;
  b0.Reshape(N, C, ih, iw);
  fill(&b0, in);
  vector<Blob<float>*> bottom(1), top(1);
  bottom[0] = &b0; top[0] = &t0;
  layer.SetUp(bottom, top);
  layer.Forward(bottom, top, true);
  if (cudaDeviceSynchronize() != cudaSuccess) return 1;
  fill_diff(&t0, top_diff);
  vector<bool> pd(1, true);
  if (backward(&layer, top, pd, bottom, iters, times)) return 1;
  fetch_diff(&b0, in_diff);
  return 0;
}

// MaskPoolingLayer::Backward_gpu (mask_pooling_layer.cu:78-99)
int ref_mask_pool_backward(const float* feat, const float* mask, int N, int C, int H, int W,
                           const float* top_diff, int pd0, int pd1, float* feat_diff,
                           float* mask_diff, int iters, float* times) {
  LayerParameter p;
  Open<MaskPoolingLayer<float> > layer(p);
  Blob<float> b0, b1, t0;
  b0.Reshape(N, C, H, W);
  b1.Reshape(N, 1, H, W);
  fill(&b0, feat);
  fill(&b1, mask);
  vector<Blob<float>*> bottom(2), top(1);
  bottom[0] = &b0; bottom[1] = &b1; top[0] = &t0;
  layer.SetUp(bottom, top);
  layer.Forward(bottom, top, true);
  if (cudaDeviceSynchronize() != cudaSuccess) return 1;
  fill_diff(&t0, top_diff);
  vector<bool> pd(2);
  pd[0] = pd0 != 0; pd[1] = pd1 != 0;
  if (backward(&layer, top, pd, bottom, iters, times)) return 1;
  fetch_diff(&b0, feat_diff);
  fetch_diff(&b1, mask_diff);
  return 0;
}

// ROIPoolingLayer::Backward_gpu (roi_pooling_layer.cu:167-184)
int ref_roi_pool_backward(const float* feat, int B, int C, int H, int W, const float* rois, int R,
                          int ph, int pw, float spatial_scale, const float* top_diff, int pd0,
                          float* feat_diff, int iters, float* times) {
  LayerParameter p;
  p.roi_pooling_param_.pooled_h_ = ph;
  p.roi_pooling_param_.pooled_w_ = pw;
  p.roi_pooling_param_.spatial_scale_ = spatial_scale;
  Open<ROIPoolingLayer<float> > layer(p);
  Blob<float> b0, b1, t0;
  b0.Reshape(B, C, H, W);
  b1.Reshape(R, 5, 1, 1);
  fill(&b0, feat);
  fill(&b1, rois);
  vector<Blob<float>*> bottom(2), top(1);
  bottom[0] = &b0; bottom[1] = &b1; top[0] = &t0;
  layer.SetUp(bottom, top);
  layer.Forward(bottom, top, true);
  if (cudaDeviceSynchronize() != cudaSuccess) return 1;
  fill_diff(&t0, top_diff);
  vector<bool> pd(2);
  pd[0] = pd0 != 0; pd[1] = false;
  if (backward(&layer, top, pd, bottom, iters, times)) return 1;
  fetch_diff(&b0, feat_diff);
  return 0;
}

}  // extern "C"
