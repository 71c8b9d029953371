// oracle/ref_stub -- TEST INFRASTRUCTURE.  A minimal stand-in for the parts of the Caffe runtime
// that the reference's layer sources touch, so that they compile UNMODIFIED from a reference
// checkout into the libraries under oracle/_ref/ (oracle/Makefile).  Nothing here restates
// reference arithmetic: kernels, LayerSetUp and Reshape are the reference's own object code.
// Stands in for caffe-mnc/include/caffe/common.hpp + util/device_alternate.hpp + glog, with the
// cuBLAS handle the math helpers (math_functions.cu) use.
#ifndef MNC_REF_STUB_COMMON_HPP_
#define MNC_REF_STUB_COMMON_HPP_
#include <cublas_v2.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <memory>
#include <sstream>
#include <string>
#include <vector>

namespace caffe {
using std::shared_ptr;
using std::string;
using std::vector;

namespace stub {
struct Fatal {  // glog LOG(FATAL) / failed CHECK: print and abort
  std::ostringstream os;
  Fatal(const char* f, int l, const char* what) { os << f << ":" << l << " " << what << " "; }
  ~Fatal() {
    std::fprintf(stderr, "[ref_stub] FATAL %s\n", os.str().c_str());
    std::abort();
  }
};
struct Null {
  template <typename T> Null& operator<<(const T&) { return *this; }
};
struct Voidify { template <typename T> void operator&(const T&) {} };
}  // namespace stub
}  // namespace caffe

#define STUB_CHECK_(cond, text) \
  (cond) ? (void)0 : ::caffe::stub::Voidify() & ::caffe::stub::Fatal(__FILE__, __LINE__, text).os
#define CHECK(c) STUB_CHECK_((c), "Check failed: " #c)
#define CHECK_EQ(a, b) STUB_CHECK_((a) == (b), "Check failed: " #a " == " #b)
#define CHECK_NE(a, b) STUB_CHECK_((a) != (b), "Check failed: " #a " != " #b)
#define CHECK_GT(a, b) STUB_CHECK_((a) > (b), "Check failed: " #a " > " #b)
#define CHECK_GE(a, b) STUB_CHECK_((a) >= (b), "Check failed: " #a " >= " #b)
#define CHECK_LT(a, b) STUB_CHECK_((a) < (b), "Check failed: " #a " < " #b)
#define CHECK_LE(a, b) STUB_CHECK_((a) <= (b), "Check failed: " #a " <= " #b)
#define STUB_LOG_INFO ::caffe::stub::Null()
#define STUB_LOG_WARNING ::caffe::stub::Null()
#define STUB_LOG_FATAL ::caffe::stub::Fatal(__FILE__, __LINE__, "").os
#define LOG(sev) STUB_LOG_##sev
#define NOT_IMPLEMENTED LOG(FATAL) << "Not Implemented Yet"
#define DCHECK_GE(a, b) ::caffe::stub::Null()
#define DCHECK_LT(a, b) ::caffe::stub::Null()

#define CUDA_CHECK(condition)                                                   \
  do {                                                                          \
    cudaError_t error = condition;                                              \
    CHECK_EQ(error, cudaSuccess) << " " << cudaGetErrorString(error);           \
  } while (0)
#define CUDA_KERNEL_LOOP(i, n) \
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (n); i += blockDim.x * gridDim.x)
#define CUDA_POST_KERNEL_CHECK CUDA_CHECK(cudaPeekAtLastError())

namespace caffe {
class Caffe {
 public:
  static cublasHandle_t cublas_handle() {
    static cublasHandle_t h = 0;
    if (!h) cublasCreate(&h);
    return h;
  }
};

const int CAFFE_CUDA_NUM_THREADS = 512;  // device_alternate.hpp value for __CUDA_ARCH__ >= 200
inline int CAFFE_GET_BLOCKS(const int N) {
  return (N + CAFFE_CUDA_NUM_THREADS - 1) / CAFFE_CUDA_NUM_THREADS;
}

template <typename Dtype>
inline void caffe_set(const int N, const Dtype alpha, Dtype* Y) {
  for (int i = 0; i < N; ++i) Y[i] = alpha;
}
#ifdef __CUDACC__
template <typename Dtype>
__global__ void stub_set_kernel(const int n, const Dtype alpha, Dtype* y) {
  CUDA_KERNEL_LOOP(index, n) { y[index] = alpha; }
}
template <typename Dtype>
inline void caffe_gpu_set(const int N, const Dtype alpha, Dtype* Y) {
  stub_set_kernel<Dtype><<<CAFFE_GET_BLOCKS(N), CAFFE_CUDA_NUM_THREADS>>>(N, alpha, Y);
}
#endif
}  // namespace caffe

// explicit instantiation / registration macros of common.hpp, layer_factory.hpp
#define INSTANTIATE_CLASS(classname) \
  template class classname<float>;   \
  template class classname<double>
#define INSTANTIATE_LAYER_GPU_FORWARD(classname)                                        \
  template void classname<float>::Forward_gpu(const std::vector<Blob<float>*>& bottom,  \
                                              const std::vector<Blob<float>*>& top);    \
  template void classname<double>::Forward_gpu(const std::vector<Blob<double>*>& bottom, \
                                               const std::vector<Blob<double>*>& top);
#define INSTANTIATE_LAYER_GPU_BACKWARD(classname)                                              \
  template void classname<float>::Backward_gpu(const std::vector<Blob<float>*>& top,           \
                                               const std::vector<bool>& propagate_down,        \
                                               const std::vector<Blob<float>*>& bottom);       \
  template void classname<double>::Backward_gpu(const std::vector<Blob<double>*>& top,         \
                                                const std::vector<bool>& propagate_down,       \
                                                const std::vector<Blob<double>*>& bottom)
#define INSTANTIATE_LAYER_GPU_FUNCS(classname) \
  INSTANTIATE_LAYER_GPU_FORWARD(classname);    \
  INSTANTIATE_LAYER_GPU_BACKWARD(classname)
#define REGISTER_LAYER_CLASS(type)  // no layer registry in the stub: the driver names the class
#endif
