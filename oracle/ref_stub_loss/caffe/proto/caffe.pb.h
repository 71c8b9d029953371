// oracle/ref_stub_loss -- TEST INFRASTRUCTURE.  Stand-in for the protoc-generated caffe.pb.h: the
// messages the loss layers read (caffe-mnc/src/caffe/proto/caffe.proto: LossParameter :427-451,
// AccuracyParameter :456-471, SmoothL1LossParameter :1087, SoftmaxParameter), with the proto
// defaults and has_ flags.
#ifndef MNC_REF_STUB_LOSS_CAFFE_PB_H_
#define MNC_REF_STUB_LOSS_CAFFE_PB_H_
#include <string>
#include <vector>
namespace caffe {
enum Phase { TRAIN = 0, TEST = 1 };
enum LossParameter_NormalizationMode {
  LossParameter_NormalizationMode_FULL = 0,
  LossParameter_NormalizationMode_VALID = 1,
  LossParameter_NormalizationMode_BATCH_SIZE = 2,
  LossParameter_NormalizationMode_NONE = 3
};
inline const std::string& LossParameter_NormalizationMode_Name(LossParameter_NormalizationMode) {
  static const std::string s("UNKNOWN");
  return s;
}
struct LossParameter {
  bool has_ignore_label_ = false, has_normalization_ = false, has_normalize_ = false;
  int ignore_label_ = 0;
  LossParameter_NormalizationMode normalization_ = LossParameter_NormalizationMode_VALID;
  bool normalize_ = false;
  bool has_ignore_label() const { return has_ignore_label_; }
  int ignore_label() const { return ignore_label_; }
  bool has_normalization() const { return has_normalization_; }
  LossParameter_NormalizationMode normalization() const { return normalization_; }
  bool has_normalize() const { return has_normalize_; }
  bool normalize() const { return normalize_; }
};
struct SoftmaxParameter {
  int axis_ = 1;
  int axis() const { return axis_; }
};
struct SmoothL1LossParameter {
  float sigma_ = 1.f;
  float sigma() const { return sigma_; }
};
struct AccuracyParameter {
  unsigned top_k_ = 1;
  int axis_ = 1;
  bool has_ignore_label_ = false;
  int ignore_label_ = 0;
  unsigned top_k() const { return top_k_; }
  int axis() const { return axis_; }
  bool has_ignore_label() const { return has_ignore_label_; }
  int ignore_label() const { return ignore_label_; }
};
struct LayerParameter {
  Phase phase_ = TRAIN;
  std::string type_;
  std::vector<float> loss_weight_;
  LossParameter loss_param_;
  SoftmaxParameter softmax_param_;
  SmoothL1LossParameter smooth_l1_loss_param_;
  AccuracyParameter accuracy_param_;
  Phase phase() const { return phase_; }
  const std::string& type() const { return type_; }
  void set_type(const std::string& t) { type_ = t; }
  int loss_weight_size() const { return static_cast<int>(loss_weight_.size()); }
  float loss_weight(int i) const { return loss_weight_[i]; }
  void add_loss_weight(float w) { loss_weight_.push_back(w); }
  const LossParameter& loss_param() const { return loss_param_; }
  const SoftmaxParameter& softmax_param() const { return softmax_param_; }
  const SmoothL1LossParameter& smooth_l1_loss_param() const { return smooth_l1_loss_param_; }
  const AccuracyParameter& accuracy_param() const { return accuracy_param_; }
};
}  // namespace caffe
#endif
