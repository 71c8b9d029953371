// oracle/ref_stub_heads -- TEST INFRASTRUCTURE.  The caffe/util/math_functions.hpp helpers the head
// layers call beyond those of ref_stub_loss/math_functions.cu: caffe_gpu_gemm / caffe_gpu_gemv on
// row-major operands through cuBLAS's column-major Sgemm / Sgemv (a row-major matrix is its
// transpose in column-major order, so C^T = op(B)^T op(A)^T is computed with the operands swapped),
// and the STOCHASTIC pooling generator, which is never run.
#include "caffe/util/math_functions.hpp"

namespace caffe {

template <> void caffe_gpu_gemm<float>(const CBLAS_TRANSPOSE TransA, const CBLAS_TRANSPOSE TransB,
                                       const int M, const int N, const int K, const float alpha,
                                       const float* A, const float* B, const float beta, float* C) {
  const int lda = (TransA == CblasNoTrans) ? K : M;
  const int ldb = (TransB == CblasNoTrans) ? N : K;
  const cublasOperation_t ta = (TransA == CblasNoTrans) ? CUBLAS_OP_N : CUBLAS_OP_T;
  const cublasOperation_t tb = (TransB == CblasNoTrans) ? CUBLAS_OP_N : CUBLAS_OP_T;
  CUBLAS_CHECK(cublasSgemm(Caffe::cublas_handle(), tb, ta, N, M, K, &alpha, B, ldb, A, lda, &beta,
                           C, N));
}
template <> void caffe_gpu_gemm<double>(const CBLAS_TRANSPOSE, const CBLAS_TRANSPOSE, const int,
                                        const int, const int, const double, const double*,
                                        const double*, const double, double*) {
  LOG(FATAL) << "caffe_gpu_gemm<double>: not run";
}
template <> void caffe_gpu_gemv<float>(const CBLAS_TRANSPOSE TransA, const int M, const int N,
                                       const float alpha, const float* A, const float* x,
                                       const float beta, float* y) {
  const cublasOperation_t t = (TransA == CblasNoTrans) ? CUBLAS_OP_T : CUBLAS_OP_N;
  CUBLAS_CHECK(cublasSgemv(Caffe::cublas_handle(), t, N, M, &alpha, A, N, x, 1, &beta, y, 1));
}
template <> void caffe_gpu_gemv<double>(const CBLAS_TRANSPOSE, const int, const int, const double,
                                        const double*, const double*, const double, double*) {
  LOG(FATAL) << "caffe_gpu_gemv<double>: not run";
}

template <> void caffe_gpu_rng_uniform<float>(const int, const float, const float, float*) {
  LOG(FATAL) << "STOCHASTIC pooling: not run";
}
template <> void caffe_gpu_rng_uniform<double>(const int, const double, const double, double*) {
  LOG(FATAL) << "STOCHASTIC pooling: not run";
}

}  // namespace caffe
