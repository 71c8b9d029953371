// oracle/ref_stub_heads -- TEST INFRASTRUCTURE.  Stand-in for caffe/layer.hpp as Caffe runs in GPU
// mode, with the learnable parameters the head layers own (blobs_, param_propagate_down_):
// SetUp = LayerSetUp, Reshape (layer.hpp:67-77); Forward = Reshape, Forward_gpu (:446-470);
// Backward = Backward_gpu (:472-487).  A layer without a _gpu form falls back to its _cpu form.
#ifndef MNC_REF_STUB_HEADS_LAYER_HPP_
#define MNC_REF_STUB_HEADS_LAYER_HPP_
#include "caffe/blob.hpp"
#include "caffe/common.hpp"
#include "caffe/proto/caffe.pb.h"
#include "caffe/util/math_functions.hpp"

namespace caffe {
template <typename Dtype>
class Layer {
 public:
  explicit Layer(const LayerParameter& param) : layer_param_(param), phase_(param.phase()) {}
  virtual ~Layer() {}
  void SetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
    LayerSetUp(bottom, top);
    Reshape(bottom, top);
  }
  virtual void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {}
  virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) = 0;
  Dtype Forward(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
    Reshape(bottom, top);
    Forward_gpu(bottom, top);
    return Dtype(0);
  }
  void Backward(const vector<Blob<Dtype>*>& top, const vector<bool>& propagate_down,
                const vector<Blob<Dtype>*>& bottom) {
    Backward_gpu(top, propagate_down, bottom);
  }
  vector<shared_ptr<Blob<Dtype> > >& blobs() { return blobs_; }
  const LayerParameter& layer_param() const { return layer_param_; }
  virtual inline const char* type() const { return ""; }
  virtual inline int ExactNumBottomBlobs() const { return -1; }
  virtual inline int MinBottomBlobs() const { return -1; }
  virtual inline int MaxBottomBlobs() const { return -1; }
  virtual inline int ExactNumTopBlobs() const { return -1; }
  virtual inline int MinTopBlobs() const { return -1; }
  virtual inline int MaxTopBlobs() const { return -1; }
  virtual inline bool EqualNumBottomTopBlobs() const { return false; }
  virtual inline bool AutoTopBlobs() const { return false; }
  virtual inline bool AllowForceBackward(const int bottom_index) const { return true; }

 protected:
  LayerParameter layer_param_;
  Phase phase_;
  vector<shared_ptr<Blob<Dtype> > > blobs_;
  vector<bool> param_propagate_down_;
  virtual void Forward_cpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) = 0;
  virtual void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
    Forward_cpu(bottom, top);
  }
  virtual void Backward_cpu(const vector<Blob<Dtype>*>& top, const vector<bool>& propagate_down,
                            const vector<Blob<Dtype>*>& bottom) = 0;
  virtual void Backward_gpu(const vector<Blob<Dtype>*>& top, const vector<bool>& propagate_down,
                            const vector<Blob<Dtype>*>& bottom) {
    Backward_cpu(top, propagate_down, bottom);
  }
};
}  // namespace caffe
#endif
