// oracle/ref_loss_driver.cu -- TEST INFRASTRUCTURE.  C entry points that run the reference's loss
// layers, compiled UNMODIFIED from a reference checkout (oracle/Makefile), as Caffe runs them in
// GPU mode: SetUp, Forward, the top diff filled with the loss weight (what Net::Backward finds
// there), Backward on the same object.  Host arrays in and out; `ms` (may be NULL) receives the
// event time of Forward + Backward, the reference's host round trips included.  No layer
// arithmetic here.
#include <vector>

#include "caffe/fast_rcnn_layers.hpp"
#include "caffe/layers/accuracy_layer.hpp"
#include "caffe/layers/sigmoid_cross_entropy_loss_layer.hpp"
#include "caffe/layers/softmax_layer.hpp"
#include "caffe/layers/softmax_loss_layer.hpp"

namespace caffe {
template <typename Dtype>
shared_ptr<Layer<Dtype> > LayerRegistry<Dtype>::CreateLayer(const LayerParameter& param) {
  CHECK(param.type() == "Softmax") << "the stub registry creates Softmax only";
  return shared_ptr<Layer<Dtype> >(new SoftmaxLayer<Dtype>(param));
}
template struct LayerRegistry<float>;
template struct LayerRegistry<double>;
}  // namespace caffe

using caffe::Blob;
using caffe::LayerParameter;
using std::vector;

namespace {
Blob<float>* blob(const vector<int>& shape, const float* src) {
  Blob<float>* b = new Blob<float>(shape);
  if (src) {
    float* d = b->mutable_cpu_data();
    for (int i = 0; i < b->count(); ++i) d[i] = src[i];
  }
  return b;
}
void copy_out(const float* src, int n, float* dst) {
  if (dst)
    for (int i = 0; i < n; ++i) dst[i] = src[i];
}
struct Timer {
  cudaEvent_t a, b;
  Timer() { cudaEventCreate(&a); cudaEventCreate(&b); cudaEventRecord(a); }
  void stop(float* ms) {
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    if (ms) cudaEventElapsedTime(ms, a, b);
    cudaEventDestroy(a);
    cudaEventDestroy(b);
  }
};
template <typename L>
void run(L& layer, const vector<Blob<float>*>& bottom, Blob<float>& top, float loss_weight,
         const vector<bool>& pd, float* ms) {
  vector<Blob<float>*> tv(1, &top);
  layer.SetUp(bottom, tv);
  Timer t;
  layer.Forward(bottom, tv);
  top.mutable_cpu_diff()[0] = loss_weight;
  layer.Backward(tv, pd, bottom);
  t.stop(ms);
}
struct SoftmaxWithLoss : caffe::SoftmaxWithLossLayer<float> {
  explicit SoftmaxWithLoss(const LayerParameter& p) : caffe::SoftmaxWithLossLayer<float>(p) {}
  const Blob<float>& prob() const { return this->prob_; }
};
}  // namespace

// normalization: 0..3 (LossParameter.NormalizationMode), or -1 for the prototxt's `normalize`
// with value `normalize`.
extern "C" void ref_softmax_loss(const float* x, const float* labels, int outer, int C, int inner,
                                 int has_ignore, int ignore_label, int normalization,
                                 int normalize, float loss_weight, float* loss, float* prob,
                                 float* diff, float* ms) {
  LayerParameter p;
  p.loss_param_.has_ignore_label_ = has_ignore != 0;
  p.loss_param_.ignore_label_ = ignore_label;
  if (normalization >= 0) {
    p.loss_param_.has_normalization_ = true;
    p.loss_param_.normalization_ = static_cast<caffe::LossParameter_NormalizationMode>(normalization);
  } else {
    p.loss_param_.has_normalize_ = true;
    p.loss_param_.normalize_ = normalize != 0;
  }
  p.add_loss_weight(loss_weight);
  vector<int> xs(3), ls(2);
  xs[0] = outer; xs[1] = C; xs[2] = inner;
  ls[0] = outer; ls[1] = inner;
  vector<Blob<float>*> bottom;
  bottom.push_back(blob(xs, x));
  bottom.push_back(blob(ls, labels));
  Blob<float> top;
  SoftmaxWithLoss layer(p);
  vector<bool> pd(2, false);
  pd[0] = true;
  run(layer, bottom, top, loss_weight, pd, ms);
  copy_out(top.cpu_data(), 1, loss);
  copy_out(layer.prob().cpu_data(), bottom[0]->count(), prob);
  copy_out(bottom[0]->cpu_diff(), bottom[0]->count(), diff);
  for (size_t i = 0; i < bottom.size(); ++i) delete bottom[i];
}

// inside_weights / outside_weights both NULL: the two-bottom form.
extern "C" void ref_smooth_l1_loss(const float* pred, const float* target,
                                   const float* inside_weights, const float* outside_weights,
                                   int num, int channels, int height, int width, float sigma,
                                   float loss_weight, float* loss, float* diff, float* ms) {
  LayerParameter p;
  p.smooth_l1_loss_param_.sigma_ = sigma;
  p.add_loss_weight(loss_weight);
  vector<int> s(4);
  s[0] = num; s[1] = channels; s[2] = height; s[3] = width;
  vector<Blob<float>*> bottom;
  bottom.push_back(blob(s, pred));
  bottom.push_back(blob(s, target));
  if (inside_weights) {
    bottom.push_back(blob(s, inside_weights));
    bottom.push_back(blob(s, outside_weights));
  }
  Blob<float> top;
  caffe::SmoothL1LossLayer<float> layer(p);
  vector<bool> pd(bottom.size(), false);
  pd[0] = true;
  run(layer, bottom, top, loss_weight, pd, ms);
  copy_out(top.cpu_data(), 1, loss);
  copy_out(bottom[0]->cpu_diff(), bottom[0]->count(), diff);
  for (size_t i = 0; i < bottom.size(); ++i) delete bottom[i];
}

// weights NULL: the two-bottom form.  loss holds the top's value before the call (the layer leaves
// it untouched when the weights sum to 0).
extern "C" void ref_sigmoid_ce_loss(const float* x, const float* targets, const float* weights,
                                    int num, int dim, float loss_weight, float* loss, float* diff,
                                    float* ms) {
  LayerParameter p;
  p.add_loss_weight(loss_weight);
  vector<int> s(2);
  s[0] = num; s[1] = dim;
  vector<Blob<float>*> bottom;
  bottom.push_back(blob(s, x));
  bottom.push_back(blob(s, targets));
  if (weights) bottom.push_back(blob(s, weights));
  Blob<float> top;
  caffe::SigmoidCrossEntropyLossLayer<float> layer(p);
  vector<Blob<float>*> tv(1, &top);
  layer.SetUp(bottom, tv);
  top.mutable_cpu_data()[0] = *loss;
  vector<bool> pd(bottom.size(), false);
  pd[0] = true;
  Timer t;
  layer.Forward(bottom, tv);
  top.mutable_cpu_diff()[0] = loss_weight;
  layer.Backward(tv, pd, bottom);
  t.stop(ms);
  copy_out(top.cpu_data(), 1, loss);
  copy_out(bottom[0]->cpu_diff(), bottom[0]->count(), diff);
  for (size_t i = 0; i < bottom.size(); ++i) delete bottom[i];
}

extern "C" void ref_accuracy(const float* x, const float* labels, int outer, int C, int inner,
                             int top_k, int has_ignore, int ignore_label, float* accuracy) {
  LayerParameter p;
  p.accuracy_param_.top_k_ = top_k;
  p.accuracy_param_.has_ignore_label_ = has_ignore != 0;
  p.accuracy_param_.ignore_label_ = ignore_label;
  vector<int> xs(3), ls(2);
  xs[0] = outer; xs[1] = C; xs[2] = inner;
  ls[0] = outer; ls[1] = inner;
  vector<Blob<float>*> bottom;
  bottom.push_back(blob(xs, x));
  bottom.push_back(blob(ls, labels));
  Blob<float> top;
  caffe::AccuracyLayer<float> layer(p);
  vector<Blob<float>*> tv(1, &top);
  layer.SetUp(bottom, tv);
  layer.Forward(bottom, tv);
  copy_out(top.cpu_data(), 1, accuracy);
  for (size_t i = 0; i < bottom.size(); ++i) delete bottom[i];
}
