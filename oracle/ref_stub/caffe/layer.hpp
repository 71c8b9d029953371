// oracle/ref_stub -- TEST INFRASTRUCTURE.  Stand-in for caffe/layer.hpp (+ the LayerRegistry of
// layer_factory.hpp) as Caffe runs in GPU mode, with the learnable parameters a layer owns
// (blobs_, param_propagate_down_): SetUp = LayerSetUp, Reshape, SetLossWeights (layer.hpp:67-77,
// 417-433); Forward = Reshape, Forward_gpu (:446-470), or Forward_cpu when the driver asks for the
// CPU path; Backward = Backward_gpu (:472-487).  A layer without Forward_gpu / Backward_gpu falls
// back to its _cpu form, as in Caffe.  LayerRegistry<Dtype>::CreateLayer is defined by the driver
// that needs it (oracle/ref_loss_driver.cu).
#ifndef MNC_REF_STUB_LAYER_HPP_
#define MNC_REF_STUB_LAYER_HPP_
#include "caffe/blob.hpp"
#include "caffe/common.hpp"
#include "caffe/proto/caffe.pb.h"
#include "caffe/util/math_functions.hpp"

namespace caffe {
template <typename Dtype> class Layer;

template <typename Dtype>
struct LayerRegistry {
  static shared_ptr<Layer<Dtype> > CreateLayer(const LayerParameter& param);
};

template <typename Dtype>
class Layer {
 public:
  explicit Layer(const LayerParameter& param) : layer_param_(param), phase_(param.phase()) {}
  virtual ~Layer() {}
  void SetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
    LayerSetUp(bottom, top);
    Reshape(bottom, top);
    SetLossWeights(top);
  }
  virtual void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {}
  virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) = 0;
  Dtype Forward(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top,
                bool gpu = true) {
    Reshape(bottom, top);
    if (gpu) Forward_gpu(bottom, top); else Forward_cpu(bottom, top);
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
  void SetLossWeights(const vector<Blob<Dtype>*>& top) {
    for (int i = 0; i < layer_param_.loss_weight_size() && i < static_cast<int>(top.size()); ++i)
      caffe_set(top[i]->count(), Dtype(layer_param_.loss_weight(i)), top[i]->mutable_cpu_diff());
  }
};
}  // namespace caffe
#endif
