// oracle/ref_stub_loss -- TEST INFRASTRUCTURE.  Definitions of the caffe/util/math_functions.hpp
// helpers the loss layers call, as Caffe's math_functions.cu / .cpp make them: the reductions and
// scalings through cuBLAS (asum, dot, scal, axpy) with a host result, the element-wise device
// kernels, cudaMemcpy(Default), and on the host mkl_alternate.hpp's element loops and the cblas
// stand-in.  The SoftmaxLayer CPU path (gemm / gemv / strided dot) is never run: GPU mode.
#include "caffe/util/math_functions.hpp"

namespace caffe {

#define STUB_CPU_ONLY_UNUSED(name) LOG(FATAL) << #name ": the CPU path is not run"

template <> void caffe_gpu_asum<float>(const int n, const float* x, float* y) {
  CUBLAS_CHECK(cublasSasum(Caffe::cublas_handle(), n, x, 1, y));
}
template <> void caffe_gpu_asum<double>(const int n, const double* x, double* y) {
  CUBLAS_CHECK(cublasDasum(Caffe::cublas_handle(), n, x, 1, y));
}
template <> void caffe_gpu_dot<float>(const int n, const float* x, const float* y, float* out) {
  CUBLAS_CHECK(cublasSdot(Caffe::cublas_handle(), n, x, 1, y, 1, out));
}
template <> void caffe_gpu_dot<double>(const int n, const double* x, const double* y, double* out) {
  CUBLAS_CHECK(cublasDdot(Caffe::cublas_handle(), n, x, 1, y, 1, out));
}
template <> void caffe_gpu_scal<float>(const int N, const float alpha, float* X) {
  CUBLAS_CHECK(cublasSscal(Caffe::cublas_handle(), N, &alpha, X, 1));
}
template <> void caffe_gpu_scal<double>(const int N, const double alpha, double* X) {
  CUBLAS_CHECK(cublasDscal(Caffe::cublas_handle(), N, &alpha, X, 1));
}
template <> void caffe_gpu_axpy<float>(const int N, const float alpha, const float* X, float* Y) {
  CUBLAS_CHECK(cublasSaxpy(Caffe::cublas_handle(), N, &alpha, X, 1, Y, 1));
}
template <> void caffe_gpu_axpy<double>(const int N, const double alpha, const double* X,
                                        double* Y) {
  CUBLAS_CHECK(cublasDaxpy(Caffe::cublas_handle(), N, &alpha, X, 1, Y, 1));
}
template <> void caffe_gpu_axpby<float>(const int N, const float alpha, const float* X,
                                        const float beta, float* Y) {
  caffe_gpu_scal<float>(N, beta, Y);
  caffe_gpu_axpy<float>(N, alpha, X, Y);
}
template <> void caffe_gpu_axpby<double>(const int N, const double alpha, const double* X,
                                         const double beta, double* Y) {
  caffe_gpu_scal<double>(N, beta, Y);
  caffe_gpu_axpy<double>(N, alpha, X, Y);
}

template <typename Dtype>
__global__ void sub_kernel(const int n, const Dtype* a, const Dtype* b, Dtype* y) {
  CUDA_KERNEL_LOOP(index, n) { y[index] = a[index] - b[index]; }
}
template <typename Dtype>
__global__ void mul_kernel(const int n, const Dtype* a, const Dtype* b, Dtype* y) {
  CUDA_KERNEL_LOOP(index, n) { y[index] = a[index] * b[index]; }
}
template <> void caffe_gpu_sub<float>(const int N, const float* a, const float* b, float* y) {
  sub_kernel<float><<<CAFFE_GET_BLOCKS(N), CAFFE_CUDA_NUM_THREADS>>>(N, a, b, y);
}
template <> void caffe_gpu_sub<double>(const int N, const double* a, const double* b, double* y) {
  sub_kernel<double><<<CAFFE_GET_BLOCKS(N), CAFFE_CUDA_NUM_THREADS>>>(N, a, b, y);
}
template <> void caffe_gpu_mul<float>(const int N, const float* a, const float* b, float* y) {
  mul_kernel<float><<<CAFFE_GET_BLOCKS(N), CAFFE_CUDA_NUM_THREADS>>>(N, a, b, y);
}
template <> void caffe_gpu_mul<double>(const int N, const double* a, const double* b, double* y) {
  mul_kernel<double><<<CAFFE_GET_BLOCKS(N), CAFFE_CUDA_NUM_THREADS>>>(N, a, b, y);
}
void caffe_gpu_memcpy(const size_t N, const void* X, void* Y) {
  if (X != Y) CUDA_CHECK(cudaMemcpy(Y, X, N, cudaMemcpyDefault));
}
template <typename Dtype> void caffe_copy(const int N, const Dtype* X, Dtype* Y) {
  if (X != Y) CUDA_CHECK(cudaMemcpy(Y, X, sizeof(Dtype) * N, cudaMemcpyDefault));
}
template void caffe_copy<float>(const int, const float*, float*);
template void caffe_copy<double>(const int, const double*, double*);

template <> void caffe_sub<float>(const int n, const float* a, const float* b, float* y) { vsSub(n, a, b, y); }
template <> void caffe_sub<double>(const int n, const double* a, const double* b, double* y) { vdSub(n, a, b, y); }
template <> void caffe_mul<float>(const int n, const float* a, const float* b, float* y) { vsMul(n, a, b, y); }
template <> void caffe_mul<double>(const int n, const double* a, const double* b, double* y) { vdMul(n, a, b, y); }
template <> void caffe_div<float>(const int n, const float* a, const float* b, float* y) { vsDiv(n, a, b, y); }
template <> void caffe_div<double>(const int n, const double* a, const double* b, double* y) { vdDiv(n, a, b, y); }
template <> void caffe_exp<float>(const int n, const float* a, float* y) { vsExp(n, a, y); }
template <> void caffe_exp<double>(const int n, const double* a, double* y) { vdExp(n, a, y); }
template <> void caffe_scal<float>(const int N, const float alpha, float* X) { cblas_sscal(N, alpha, X, 1); }
template <> void caffe_scal<double>(const int N, const double alpha, double* X) { cblas_dscal(N, alpha, X, 1); }

template <> void caffe_cpu_gemm<float>(const CBLAS_TRANSPOSE, const CBLAS_TRANSPOSE, const int,
    const int, const int, const float, const float*, const float*, const float, float*) {
  STUB_CPU_ONLY_UNUSED(caffe_cpu_gemm);
}
template <> void caffe_cpu_gemm<double>(const CBLAS_TRANSPOSE, const CBLAS_TRANSPOSE, const int,
    const int, const int, const double, const double*, const double*, const double, double*) {
  STUB_CPU_ONLY_UNUSED(caffe_cpu_gemm);
}
template <> void caffe_cpu_gemv<float>(const CBLAS_TRANSPOSE, const int, const int, const float,
    const float*, const float*, const float, float*) {
  STUB_CPU_ONLY_UNUSED(caffe_cpu_gemv);
}
template <> void caffe_cpu_gemv<double>(const CBLAS_TRANSPOSE, const int, const int, const double,
    const double*, const double*, const double, double*) {
  STUB_CPU_ONLY_UNUSED(caffe_cpu_gemv);
}
template <> float caffe_cpu_strided_dot<float>(const int, const float*, const int, const float*,
                                               const int) {
  STUB_CPU_ONLY_UNUSED(caffe_cpu_strided_dot);
  return 0;
}
template <> double caffe_cpu_strided_dot<double>(const int, const double*, const int,
                                                 const double*, const int) {
  STUB_CPU_ONLY_UNUSED(caffe_cpu_strided_dot);
  return 0;
}
}  // namespace caffe
