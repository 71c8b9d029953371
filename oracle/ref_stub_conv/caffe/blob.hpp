// oracle/ref_stub_conv -- TEST INFRASTRUCTURE.  Stand-in for caffe/blob.hpp: ref_stub_heads's blob
// with the two members base_conv_layer.{hpp,cpp} also compile against, shape_string() (its LOG
// messages) and gpu_shape() (the N-d im2col path, which a 2-d convolution never takes).  Data and
// diff live in managed memory, so the host and device views are one buffer; every host access
// synchronises the device first, which gives SyncedMemory's head moves in both directions.
#ifndef MNC_REF_STUB_CONV_BLOB_HPP_
#define MNC_REF_STUB_CONV_BLOB_HPP_
#include <cstring>

#include "caffe/common.hpp"

namespace caffe {
template <typename Dtype>
class Blob {
 public:
  Blob() : data_(0), diff_(0), count_(0), capacity_(0) {}
  explicit Blob(const vector<int>& shape) : data_(0), diff_(0), count_(0), capacity_(0) {
    Reshape(shape);
  }
  ~Blob() { release(); }
  void Reshape(const int num, const int channels, const int height, const int width) {
    vector<int> s(4);
    s[0] = num; s[1] = channels; s[2] = height; s[3] = width;
    Reshape(s);
  }
  void Reshape(const vector<int>& shape) {
    shape_ = shape;
    count_ = 1;
    for (size_t i = 0; i < shape.size(); ++i) count_ *= shape[i];
    if (count_ > capacity_) {
      release();
      capacity_ = count_;
    }
  }
  void ReshapeLike(const Blob& other) { Reshape(other.shape()); }
  // the driver gives SoftmaxWithLoss one top, so the prob top that would share data is never made
  void ShareData(const Blob&) { LOG(FATAL) << "ShareData: not provided by the stub"; }
  const vector<int>& shape() const { return shape_; }
  string shape_string() const {
    std::ostringstream os;
    for (size_t i = 0; i < shape_.size(); ++i) os << shape_[i] << " ";
    os << "(" << count_ << ")";
    return os.str();
  }
  const int* gpu_shape() const {
    LOG(FATAL) << "gpu_shape: the N-d im2col path is not run";
    return 0;
  }
  int shape(int i) const { return shape_[CanonicalAxisIndex(i)]; }
  int num_axes() const { return static_cast<int>(shape_.size()); }
  int count() const { return count_; }
  int count(int start, int end) const {
    int c = 1;
    for (int i = start; i < end; ++i) c *= shape_[i];
    return c;
  }
  int count(int start) const { return count(start, num_axes()); }
  int CanonicalAxisIndex(int axis) const { return axis < 0 ? axis + num_axes() : axis; }
  int offset(const int n, const int c = 0, const int h = 0, const int w = 0) const {
    return ((n * channels() + c) * height() + h) * width() + w;
  }
  int num() const { return dim(0); }
  int channels() const { return dim(1); }
  int height() const { return dim(2); }
  int width() const { return dim(3); }
  const Dtype* cpu_data() const { return host(&data_); }
  const Dtype* gpu_data() const { return buf(&data_); }
  const Dtype* cpu_diff() const { return host(&diff_); }
  const Dtype* gpu_diff() const { return buf(&diff_); }
  Dtype* mutable_cpu_data() { return host(&data_); }
  Dtype* mutable_gpu_data() { return buf(&data_); }
  Dtype* mutable_cpu_diff() { return host(&diff_); }
  Dtype* mutable_gpu_diff() { return buf(&diff_); }

 private:
  Blob(const Blob&);
  Blob& operator=(const Blob&);
  int dim(size_t i) const { return i < shape_.size() ? shape_[i] : 1; }  // LegacyShape
  Dtype* host(Dtype* const* slot) const {
    Dtype* p = buf(slot);
    cudaDeviceSynchronize();
    return p;
  }
  Dtype* buf(Dtype* const* slot) const {
    Dtype** s = const_cast<Dtype**>(slot);
    if (*s == 0 && capacity_ > 0) {
      void* p = 0;
      const size_t bytes = sizeof(Dtype) * static_cast<size_t>(capacity_);
      CUDA_CHECK(cudaMallocManaged(&p, bytes));
      CUDA_CHECK(cudaMemset(p, 0, bytes));
      CUDA_CHECK(cudaDeviceSynchronize());
      *s = static_cast<Dtype*>(p);
    }
    return *s;
  }
  void release() {
    if (data_) cudaFree(data_);
    if (diff_) cudaFree(diff_);
    data_ = diff_ = 0;
  }
  Dtype* data_;
  Dtype* diff_;
  vector<int> shape_;
  int count_;
  int capacity_;
};
}  // namespace caffe
#endif
