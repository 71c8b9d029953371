// oracle/ref_stub_conv -- TEST INFRASTRUCTURE.  Stand-in for the protoc-generated caffe.pb.h with
// the messages the Convolution layer reads (caffe-mnc/src/caffe/proto/caffe.proto:
// ConvolutionParameter, FillerParameter), the proto defaults and has_ flags; the repeated
// kernel_size / pad / stride / dilation fields are vectors.  Shadows ref_stub_heads's and
// ref_stub_loss's versions on the include path of oracle/conv.mk.
#ifndef MNC_REF_STUB_CONV_CAFFE_PB_H_
#define MNC_REF_STUB_CONV_CAFFE_PB_H_
#include <string>
#include <vector>
namespace caffe {
enum Phase { TRAIN = 0, TEST = 1 };
struct FillerParameter {};
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
  ConvolutionParameter convolution_param_;
  Phase phase() const { return phase_; }
  const std::string& type() const { return type_; }
  const ConvolutionParameter& convolution_param() const { return convolution_param_; }
};
}  // namespace caffe
#endif
