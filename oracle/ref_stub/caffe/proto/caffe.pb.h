// oracle/ref_stub -- TEST INFRASTRUCTURE.  Stand-in for the protoc-generated caffe.pb.h: only the
// messages the drivers set and the layers read (caffe-mnc/src/caffe/proto/caffe.proto:
// ROIPoolingParameter, ROIWarpingParameter :1022-1030, MaskResizeParameter :1032-1035,
// LossParameter :427-451, AccuracyParameter :456-471, SmoothL1LossParameter :1087,
// SoftmaxParameter, InnerProductParameter, PoolingParameter, ReLUParameter, ConvolutionParameter,
// FillerParameter), with the proto defaults and has_ flags; repeated fields are vectors.
#ifndef MNC_REF_STUB_CAFFE_PB_H_
#define MNC_REF_STUB_CAFFE_PB_H_
#include <string>
#include <vector>
namespace caffe {
enum Phase { TRAIN = 0, TEST = 1 };
struct FillerParameter {};

struct ROIPoolingParameter {
  unsigned pooled_h_ = 0, pooled_w_ = 0;
  float spatial_scale_ = 1.f;
  unsigned pooled_h() const { return pooled_h_; }
  unsigned pooled_w() const { return pooled_w_; }
  float spatial_scale() const { return spatial_scale_; }
};
struct ROIWarpingParameter {
  unsigned pooled_h_ = 0, pooled_w_ = 0;
  float spatial_scale_ = 1.f;
  unsigned pooled_h() const { return pooled_h_; }
  unsigned pooled_w() const { return pooled_w_; }
  float spatial_scale() const { return spatial_scale_; }
};
struct MaskResizeParameter {
  unsigned output_height_ = 1, output_width_ = 1;
  unsigned output_height() const { return output_height_; }
  unsigned output_width() const { return output_width_; }
};

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
struct ConvolutionParameter {
  unsigned num_output_ = 0;
  bool bias_term_ = true;
  std::vector<unsigned> pad_, kernel_size_, stride_, dilation_;
  unsigned group_ = 1;
  int axis_ = 1;
  bool force_nd_im2col_ = false;
  FillerParameter weight_filler_, bias_filler_;
  unsigned num_output() const { return num_output_; }
  bool bias_term() const { return bias_term_; }
  int pad_size() const { return static_cast<int>(pad_.size()); }
  unsigned pad(int i) const { return pad_[i]; }
  int kernel_size_size() const { return static_cast<int>(kernel_size_.size()); }
  unsigned kernel_size(int i) const { return kernel_size_[i]; }
  int stride_size() const { return static_cast<int>(stride_.size()); }
  unsigned stride(int i) const { return stride_[i]; }
  int dilation_size() const { return static_cast<int>(dilation_.size()); }
  unsigned dilation(int i) const { return dilation_[i]; }
  bool has_pad_h() const { return false; }
  bool has_pad_w() const { return false; }
  unsigned pad_h() const { return 0; }
  unsigned pad_w() const { return 0; }
  bool has_kernel_h() const { return false; }
  bool has_kernel_w() const { return false; }
  unsigned kernel_h() const { return 0; }
  unsigned kernel_w() const { return 0; }
  bool has_stride_h() const { return false; }
  bool has_stride_w() const { return false; }
  unsigned stride_h() const { return 0; }
  unsigned stride_w() const { return 0; }
  unsigned group() const { return group_; }
  int axis() const { return axis_; }
  bool force_nd_im2col() const { return force_nd_im2col_; }
  const FillerParameter& weight_filler() const { return weight_filler_; }
  const FillerParameter& bias_filler() const { return bias_filler_; }
};

struct LayerParameter {
  Phase phase_ = TRAIN;
  std::string type_;
  std::vector<float> loss_weight_;
  ROIPoolingParameter roi_pooling_param_;
  ROIWarpingParameter roi_warping_param_;
  MaskResizeParameter mask_resize_param_;
  LossParameter loss_param_;
  SoftmaxParameter softmax_param_;
  SmoothL1LossParameter smooth_l1_loss_param_;
  AccuracyParameter accuracy_param_;
  InnerProductParameter inner_product_param_;
  PoolingParameter pooling_param_;
  ReLUParameter relu_param_;
  ConvolutionParameter convolution_param_;
  Phase phase() const { return phase_; }
  const std::string& type() const { return type_; }
  void set_type(const std::string& t) { type_ = t; }
  int loss_weight_size() const { return static_cast<int>(loss_weight_.size()); }
  float loss_weight(int i) const { return loss_weight_[i]; }
  void add_loss_weight(float w) { loss_weight_.push_back(w); }
  const ROIPoolingParameter& roi_pooling_param() const { return roi_pooling_param_; }
  const ROIWarpingParameter& roi_warping_param() const { return roi_warping_param_; }
  const MaskResizeParameter& mask_resize_param() const { return mask_resize_param_; }
  const LossParameter& loss_param() const { return loss_param_; }
  const SoftmaxParameter& softmax_param() const { return softmax_param_; }
  const SmoothL1LossParameter& smooth_l1_loss_param() const { return smooth_l1_loss_param_; }
  const AccuracyParameter& accuracy_param() const { return accuracy_param_; }
  const InnerProductParameter& inner_product_param() const { return inner_product_param_; }
  const PoolingParameter& pooling_param() const { return pooling_param_; }
  const ReLUParameter& relu_param() const { return relu_param_; }
  const ConvolutionParameter& convolution_param() const { return convolution_param_; }
};
}  // namespace caffe
#endif
