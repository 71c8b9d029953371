// oracle/ref_stub_heads -- TEST INFRASTRUCTURE.  Stand-in for the protoc-generated caffe.pb.h with
// the messages the head layers read (caffe-mnc/src/caffe/proto/caffe.proto: InnerProductParameter,
// PoolingParameter, ReLUParameter, FillerParameter), the proto defaults and has_ flags.  Shadows
// ref_stub_loss's version on the include path of oracle/heads.mk.
#ifndef MNC_REF_STUB_HEADS_CAFFE_PB_H_
#define MNC_REF_STUB_HEADS_CAFFE_PB_H_
#include <string>
#include <vector>
namespace caffe {
enum Phase { TRAIN = 0, TEST = 1 };
struct FillerParameter {};
struct InnerProductParameter {
  unsigned num_output_ = 0;
  bool bias_term_ = true;
  int axis_ = 1;
  FillerParameter weight_filler_, bias_filler_;
  unsigned num_output() const { return num_output_; }
  bool bias_term() const { return bias_term_; }
  int axis() const { return axis_; }
  const FillerParameter& weight_filler() const { return weight_filler_; }
  const FillerParameter& bias_filler() const { return bias_filler_; }
};
enum PoolingParameter_PoolMethod {
  PoolingParameter_PoolMethod_MAX = 0,
  PoolingParameter_PoolMethod_AVE = 1,
  PoolingParameter_PoolMethod_STOCHASTIC = 2
};
struct PoolingParameter {
  PoolingParameter_PoolMethod pool_ = PoolingParameter_PoolMethod_MAX;
  bool has_kernel_size_ = false, has_pad_ = false, has_stride_ = false, global_pooling_ = false;
  unsigned kernel_size_ = 0, pad_ = 0, stride_ = 1;
  PoolingParameter_PoolMethod pool() const { return pool_; }
  bool global_pooling() const { return global_pooling_; }
  bool has_kernel_size() const { return has_kernel_size_; }
  unsigned kernel_size() const { return kernel_size_; }
  bool has_kernel_h() const { return false; }
  bool has_kernel_w() const { return false; }
  unsigned kernel_h() const { return 0; }
  unsigned kernel_w() const { return 0; }
  bool has_pad() const { return has_pad_; }
  unsigned pad() const { return pad_; }
  bool has_pad_h() const { return false; }
  bool has_pad_w() const { return false; }
  unsigned pad_h() const { return 0; }
  unsigned pad_w() const { return 0; }
  bool has_stride() const { return has_stride_; }
  unsigned stride() const { return stride_; }
  bool has_stride_h() const { return false; }
  bool has_stride_w() const { return false; }
  unsigned stride_h() const { return 0; }
  unsigned stride_w() const { return 0; }
};
struct ReLUParameter {
  float negative_slope_ = 0.f;
  float negative_slope() const { return negative_slope_; }
};
struct LayerParameter {
  Phase phase_ = TRAIN;
  std::string type_;
  std::vector<float> loss_weight_;
  InnerProductParameter inner_product_param_;
  PoolingParameter pooling_param_;
  ReLUParameter relu_param_;
  Phase phase() const { return phase_; }
  const std::string& type() const { return type_; }
  int loss_weight_size() const { return static_cast<int>(loss_weight_.size()); }
  float loss_weight(int i) const { return loss_weight_[i]; }
  const InnerProductParameter& inner_product_param() const { return inner_product_param_; }
  const PoolingParameter& pooling_param() const { return pooling_param_; }
  const ReLUParameter& relu_param() const { return relu_param_; }
};
}  // namespace caffe
#endif
