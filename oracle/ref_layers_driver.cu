// oracle/ref_layers_driver.cu -- TEST INFRASTRUCTURE.  C entry points that run the reference's own
// layer objects (compiled unmodified from a reference checkout, see oracle/Makefile) the way
// Caffe's Net does: construct from a LayerParameter, SetUp (LayerSetUp + Reshape), Forward
// (Reshape + Forward_gpu / Forward_cpu).  Plain host pointers in and out; ctypes binds these in
// tests/test_ref_pin.py.
#include <cstring>

#include "caffe/fast_rcnn_layers.hpp"
#include "caffe/layers/mask_resize_layer.hpp"

using namespace caffe;

namespace {
void fill(Blob<float>* b, const float* src) {
  std::memcpy(b->mutable_cpu_data(), src, sizeof(float) * b->count());
}
void fetch(Blob<float>* b, float* dst) {
  std::memcpy(dst, b->cpu_data(), sizeof(float) * b->count());
}
}  // namespace

extern "C" {

// ROIWarpingLayer (roi_warping_layer.cpp:20-42 setup, roi_warping_layer.cu:110-122 forward)
int ref_roi_warp(const float* feat, int B, int C, int H, int W, const float* rois, int R, int ph,
                 int pw, float spatial_scale, float* out) {
  LayerParameter p;
  p.roi_warping_param_.pooled_h_ = ph;
  p.roi_warping_param_.pooled_w_ = pw;
  p.roi_warping_param_.spatial_scale_ = spatial_scale;
  ROIWarpingLayer<float> layer(p);
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
  fetch(&t0, out);
  return 0;
}

// MaskResizeLayer (mask_resize_layer.cpp:13-30, mask_resize_layer.cu:76-84)
int ref_mask_resize(const float* in, int N, int C, int ih, int iw, int oh, int ow, float* out) {
  LayerParameter p;
  p.mask_resize_param_.output_height_ = oh;
  p.mask_resize_param_.output_width_ = ow;
  MaskResizeLayer<float> layer(p);
  Blob<float> b0, t0;
  b0.Reshape(N, C, ih, iw);
  fill(&b0, in);
  vector<Blob<float>*> bottom(1), top(1);
  bottom[0] = &b0; top[0] = &t0;
  layer.SetUp(bottom, top);
  layer.Forward(bottom, top, true);
  if (cudaDeviceSynchronize() != cudaSuccess) return 1;
  fetch(&t0, out);
  return 0;
}

// MaskPoolingLayer (mask_pooling_layer.cpp:20-29, mask_pooling_layer.cu:29-41)
int ref_mask_pool(const float* feat, const float* mask, int N, int C, int H, int W, float* out) {
  LayerParameter p;
  MaskPoolingLayer<float> layer(p);
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
  fetch(&t0, out);
  return 0;
}

// ROIPoolingLayer (roi_pooling_layer.cpp:19-44 setup, :46-132 Forward_cpu,
// roi_pooling_layer.cu:79-92 Forward_gpu); use_gpu = 0 runs the reference's CPU forward, which
// needs no device.  The argmax blob is protected in the class, so only `top` is returned.
int ref_roi_pool(const float* feat, int B, int C, int H, int W, const float* rois, int R, int ph,
                 int pw, float spatial_scale, int use_gpu, float* out) {
  LayerParameter p;
  p.roi_pooling_param_.pooled_h_ = ph;
  p.roi_pooling_param_.pooled_w_ = pw;
  p.roi_pooling_param_.spatial_scale_ = spatial_scale;
  ROIPoolingLayer<float> layer(p);
  Blob<float> b0, b1, t0;
  b0.Reshape(B, C, H, W);
  b1.Reshape(R, 5, 1, 1);
  fill(&b0, feat);
  fill(&b1, rois);
  vector<Blob<float>*> bottom(2), top(1);
  bottom[0] = &b0; bottom[1] = &b1; top[0] = &t0;
  layer.SetUp(bottom, top);
  layer.Forward(bottom, top, use_gpu != 0);
  if (use_gpu && cudaDeviceSynchronize() != cudaSuccess) return 1;
  fetch(&t0, out);
  return 0;
}

}  // extern "C"
