// oracle/ref_heads_driver.cu -- TEST INFRASTRUCTURE.  C entry points that run the reference's head
// layers (InnerProduct, Pooling MAX, ReLU, Sigmoid), compiled UNMODIFIED from a reference checkout
// (oracle/Makefile), as Caffe runs them in GPU mode: SetUp, the parameters written, Forward, the
// top diff written, Backward on the same object.  Host arrays in and out.  No layer arithmetic
// here.
#include <vector>

#include "caffe/layers/inner_product_layer.hpp"
#include "caffe/layers/pooling_layer.hpp"
#include "caffe/layers/relu_layer.hpp"
#include "caffe/layers/sigmoid_layer.hpp"

using caffe::Blob;
using caffe::LayerParameter;
using std::vector;

namespace {
void copy_in(const float* src, int n, float* dst) {
  for (int i = 0; i < n; ++i) dst[i] = src[i];
}
template <typename T>
void copy_out(const T* src, int n, T* dst) {
  if (dst)
    for (int i = 0; i < n; ++i) dst[i] = src[i];
}
template <typename L>
void run(L& layer, Blob<float>& bottom, Blob<float>& top, const float* dy, float* y) {
  vector<Blob<float>*> bv(1, &bottom), tv(1, &top);
  layer.Forward(bv, tv);
  copy_out(top.cpu_data(), top.count(), y);
  copy_in(dy, top.count(), top.mutable_cpu_diff());
  layer.Backward(tv, vector<bool>(1, true), bv);
}
struct Pool : caffe::PoolingLayer<float> {
  explicit Pool(const LayerParameter& p) : caffe::PoolingLayer<float>(p) {}
  const Blob<int>& mask() const { return this->max_idx_; }
};
}  // namespace

// x (M, K), w (N, K), b (N) or NULL; dy (M, N); dw / db hold the diffs' initial contents and
// receive them after Backward (beta 1); y (M, N), dx (M, K).
extern "C" void ref_inner_product(const float* x, const float* w, const float* b, const float* dy,
                                  int M, int N, int K, float* y, float* dx, float* dw, float* db) {
  LayerParameter p;
  p.inner_product_param_.num_output_ = N;
  p.inner_product_param_.bias_term_ = b != 0;
  vector<int> xs(2), ys(2);
  xs[0] = M; xs[1] = K;
  Blob<float> bottom(xs), top;
  copy_in(x, M * K, bottom.mutable_cpu_data());
  caffe::InnerProductLayer<float> layer(p);
  vector<Blob<float>*> bv(1, &bottom), tv(1, &top);
  layer.SetUp(bv, tv);
  copy_in(w, N * K, layer.blobs()[0]->mutable_cpu_data());
  copy_in(dw, N * K, layer.blobs()[0]->mutable_cpu_diff());
  if (b) {
    copy_in(b, N, layer.blobs()[1]->mutable_cpu_data());
    copy_in(db, N, layer.blobs()[1]->mutable_cpu_diff());
  }
  run(layer, bottom, top, dy, y);
  copy_out(bottom.cpu_diff(), M * K, dx);
  copy_out(layer.blobs()[0]->cpu_diff(), N * K, dw);
  if (b) copy_out(layer.blobs()[1]->cpu_diff(), N, db);
}

// Pooling MAX, kernel 2, stride 2, pad 0: x (N, C, H, W) -> y, mask (N, C, PH, PW); dy -> dx.
extern "C" void ref_max_pool(const float* x, int N, int C, int H, int W, const float* dy, float* y,
                             int* mask, float* dx) {
  LayerParameter p;
  p.pooling_param_.has_kernel_size_ = true;
  p.pooling_param_.kernel_size_ = 2;
  p.pooling_param_.has_stride_ = true;
  p.pooling_param_.stride_ = 2;
  Blob<float> bottom, top;
  bottom.Reshape(N, C, H, W);
  copy_in(x, bottom.count(), bottom.mutable_cpu_data());
  Pool layer(p);
  vector<Blob<float>*> bv(1, &bottom), tv(1, &top);
  layer.SetUp(bv, tv);
  run(layer, bottom, top, dy, y);
  copy_out(layer.mask().cpu_data(), top.count(), mask);
  copy_out(bottom.cpu_diff(), bottom.count(), dx);
}

// kind 0: ReLU (negative_slope 0), 1: Sigmoid; n elements.
extern "C" void ref_neuron(int kind, const float* x, int n, const float* dy, float* y, float* dx) {
  LayerParameter p;
  vector<int> s(1, n);
  Blob<float> bottom(s), top;
  copy_in(x, n, bottom.mutable_cpu_data());
  vector<Blob<float>*> bv(1, &bottom), tv(1, &top);
  if (kind == 0) {
    caffe::ReLULayer<float> layer(p);
    layer.SetUp(bv, tv);
    run(layer, bottom, top, dy, y);
  } else {
    caffe::SigmoidLayer<float> layer(p);
    layer.SetUp(bv, tv);
    run(layer, bottom, top, dy, y);
  }
  copy_out(bottom.cpu_diff(), n, dx);
}
