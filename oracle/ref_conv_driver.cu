// oracle/ref_conv_driver.cu -- TEST INFRASTRUCTURE.  A C entry point that runs the reference's
// ConvolutionLayer, compiled UNMODIFIED from a reference checkout with its im2col
// (oracle/Makefile), as Caffe runs it in GPU mode: SetUp, the parameters written, Forward, the top
// diff written, Backward on the same object.  Host arrays in and out.  No layer arithmetic here.
#include <vector>

#include "caffe/layers/conv_layer.hpp"

using caffe::Blob;
using caffe::LayerParameter;
using std::vector;

namespace {
void copy_in(const float* src, long long n, float* dst) {
  for (long long i = 0; i < n; ++i) dst[i] = src[i];
}
void copy_out(const float* src, long long n, float* dst) {
  if (dst)
    for (long long i = 0; i < n; ++i) dst[i] = src[i];
}
}  // namespace

// x (N, Cin, H, W), w (Cout, Cin, k, k), b (Cout) or NULL, stride 1, dilation 1, group 1;
// dy (N, Cout, H', W').  dw / db hold the diffs' initial contents and receive them after Backward
// (beta 1); y (N, Cout, H', W'), dx (N, Cin, H, W).
extern "C" void ref_convolution(const float* x, const float* w, const float* b, const float* dy,
                                int N, int Cin, int H, int W, int Cout, int k, int pad, float* y,
                                float* dx, float* dw, float* db) {
  LayerParameter p;
  p.convolution_param_.num_output_ = Cout;
  p.convolution_param_.bias_term_ = b != 0;
  p.convolution_param_.kernel_size_.push_back(k);
  p.convolution_param_.pad_.push_back(pad);
  Blob<float> bottom, top;
  bottom.Reshape(N, Cin, H, W);
  copy_in(x, bottom.count(), bottom.mutable_cpu_data());
  caffe::ConvolutionLayer<float> layer(p);
  vector<Blob<float>*> bv(1, &bottom), tv(1, &top);
  layer.SetUp(bv, tv);
  const long long nw = static_cast<long long>(Cout) * Cin * k * k;
  copy_in(w, nw, layer.blobs()[0]->mutable_cpu_data());
  copy_in(dw, nw, layer.blobs()[0]->mutable_cpu_diff());
  if (b) {
    copy_in(b, Cout, layer.blobs()[1]->mutable_cpu_data());
    copy_in(db, Cout, layer.blobs()[1]->mutable_cpu_diff());
  }
  layer.Forward(bv, tv);
  copy_out(top.cpu_data(), top.count(), y);
  copy_in(dy, top.count(), top.mutable_cpu_diff());
  layer.Backward(tv, vector<bool>(1, true), bv);
  copy_out(bottom.cpu_diff(), bottom.count(), dx);
  copy_out(layer.blobs()[0]->cpu_diff(), nw, dw);
  if (b) copy_out(layer.blobs()[1]->cpu_diff(), Cout, db);
}
