// Head layers of the training net on fp32 Caffe blobs: InnerProduct forward and backward on the
// tensor cores, max Pooling, ReLU and Sigmoid forward and backward.  Replaces
//   InnerProduct  inner_product_layer.cu:9-55 (cuBLAS sgemm / sgemv in the reference)
//   Pooling MAX   pooling_layer.cu:9-44 (MaxPoolForward), MaxPoolBackward; output size
//                 pooling_layer.cpp:90-100
//   ReLU          relu_layer.cu:9-41 (negative_slope 0)
//   Sigmoid       sigmoid_layer.cu:10-40
// DESIGN.md "Head layers for training" states the precision contract and the quirks kept.
//
// The three InnerProduct products are one GEMM shape (gemm_core.cuh), C[p, q] = sum_r A(p, r) * B(q, r),
// on dense operands:
//   forward  p = n, q = m, r = k   A = W (r-contiguous), B = X (r-contiguous)   Y[m, n] = C + b
//   dX       p = k, q = m, r = n   A = W (p-contiguous), B = dY (r-contiguous)  dX[m, k] = C
//   dW       p = n, q = k, r = m   A = dY (p-contiguous), B = X (q-contiguous)  dW[n, k] += C
#include <cfloat>
#include <cstdint>
#include <cuda_runtime.h>

#include "mnc_b200.h"
#include "gemm_core.cuh"
#include "launch_util.h"
#include "sigmoid.cuh"

namespace mnc {
namespace {

// db[n] += sum_m dY[m, n], m ascending, in float32 (the gemv of inner_product_layer.cu:44-46
// with beta 1).
__global__ void __launch_bounds__(256)
fc_bias_grad_kernel(const float* __restrict__ dy, int M, int N, float* __restrict__ db) {
  const int n = blockIdx.x * 256 + threadIdx.x;
  if (n >= N) return;
  float s = 0.f;
  for (int m = 0; m < M; ++m) s = __fadd_rn(s, dy[static_cast<long long>(m) * N + n]);
  db[n] = __fadd_rn(db[n], s);
}

// ------------------------------------------------------------------------------ element-wise
constexpr int kEw = 256;

// MaxPoolForward (pooling_layer.cu:9-44), pad 0: the first maximum in row-major order wins (`>`
// from -FLT_MAX), so a window of NaNs gives -FLT_MAX and mask -1.
__global__ void __launch_bounds__(kEw)
max_pool_kernel(const float* __restrict__ x, long long n, int H, int W, int PH, int PW, int k,
                int stride, float* __restrict__ y, int* __restrict__ mask) {
  for (long long i = blockIdx.x * static_cast<long long>(kEw) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * kEw) {
    const int pw = static_cast<int>(i % PW);
    const int ph = static_cast<int>((i / PW) % PH);
    const long long plane = i / (static_cast<long long>(PW) * PH);
    const int hs = ph * stride, ws = pw * stride;
    const int he = min(hs + k, H), we = min(ws + k, W);
    const float* xp = x + plane * H * W;
    float best = -FLT_MAX;
    int arg = -1;
    for (int h = hs; h < he; ++h)
      for (int w = ws; w < we; ++w)
        if (xp[h * W + w] > best) {
          arg = h * W + w;
          best = xp[arg];
        }
    y[i] = best;
    mask[i] = arg;
  }
}

// MaxPoolBackward: each bottom element gathers, in (ph, pw) order, the diffs of the pooled cells
// that cover it and chose it.
__global__ void __launch_bounds__(kEw)
max_pool_backward_kernel(const float* __restrict__ dy, const int* __restrict__ mask, long long n,
                         int H, int W, int PH, int PW, int k, int stride, float* __restrict__ dx) {
  for (long long i = blockIdx.x * static_cast<long long>(kEw) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * kEw) {
    const int w = static_cast<int>(i % W);
    const int h = static_cast<int>((i / W) % H);
    const long long plane = i / (static_cast<long long>(W) * H);
    const int phs = (h < k) ? 0 : (h - k) / stride + 1;
    const int phe = min(h / stride + 1, PH);
    const int pws = (w < k) ? 0 : (w - k) / stride + 1;
    const int pwe = min(w / stride + 1, PW);
    const float* dp = dy + plane * PH * PW;
    const int* mp = mask + plane * PH * PW;
    float g = 0.f;
    for (int ph = phs; ph < phe; ++ph)
      for (int pw = pws; pw < pwe; ++pw)
        if (mp[ph * PW + pw] == h * W + w) g = __fadd_rn(g, dp[ph * PW + pw]);
    dx[i] = g;
  }
}

// ReLUForward (relu_layer.cu:9-14): x > 0 ? x : x * 0, so a negative input gives -0.0.
__global__ void __launch_bounds__(kEw) relu_kernel(const float* __restrict__ x, long long n,
                                                   float* __restrict__ y) {
  for (long long i = blockIdx.x * static_cast<long long>(kEw) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * kEw) {
    const float v = x[i];
    y[i] = v > 0.f ? v : __fmul_rn(v, 0.f);
  }
}

// ReLUBackward (relu_layer.cu:27-33): dy * ((x > 0) + (x <= 0) * 0), a product, not a select, so a
// non-finite dy over x <= 0 gives NaN.
__global__ void __launch_bounds__(kEw)
relu_backward_kernel(const float* __restrict__ x, const float* __restrict__ dy, long long n,
                     float* __restrict__ dx) {
  for (long long i = blockIdx.x * static_cast<long long>(kEw) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * kEw) {
    const float v = x[i];
    const float f = __fadd_rn(static_cast<float>(v > 0.f), __fmul_rn(static_cast<float>(v <= 0.f), 0.f));
    dx[i] = __fmul_rn(dy[i], f);
  }
}

__global__ void __launch_bounds__(kEw) sigmoid_kernel(const float* __restrict__ x, long long n,
                                                      float* __restrict__ y) {
  for (long long i = blockIdx.x * static_cast<long long>(kEw) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * kEw)
    y[i] = ref_sigmoid(x[i]);
}

// SigmoidBackward (sigmoid_layer.cu:23-28): (dy * y) * (1 - y).
__global__ void __launch_bounds__(kEw)
sigmoid_backward_kernel(const float* __restrict__ y, const float* __restrict__ dy, long long n,
                        float* __restrict__ dx) {
  for (long long i = blockIdx.x * static_cast<long long>(kEw) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * kEw) {
    const float s = y[i];
    dx[i] = __fmul_rn(__fmul_rn(dy[i], s), __fsub_rn(1.f, s));
  }
}

int ew_grid(long long n) { return grid_for(n, kEw, 132 * 16); }

bool pool_args_ok(int N, int C, int H, int W, int kernel, int stride, int pad) {
  return N >= 0 && C >= 0 && H >= 1 && W >= 1 && kernel == 2 && stride == 2 && pad == 0;
}

// pooling_layer.cpp:90-100 with pad 0: ceil((H - k) / stride) + 1.
int pooled_size(int H, int kernel, int stride) {
  const int num = H - kernel;
  return (num <= 0 ? 0 : (num + stride - 1) / stride) + 1;
}

}  // namespace
}  // namespace mnc

using namespace mnc;

extern "C" int mnc_fc_split_k(int rows, int cols, int red) {
  if (rows < 1 || cols < 1 || red < 1) return 0;
  return split_k(rows, cols, red);
}

extern "C" long long mnc_fc_workspace_bytes(int M, int N, int K) {
  if (M < 1 || N < 1 || K < 1) return 0;
  long long b = gemm_workspace(N, M, K);
  const long long dx = gemm_workspace(K, M, N), dw = gemm_workspace(N, K, M);
  if (dx > b) b = dx;
  if (dw > b) b = dw;
  return b;
}

extern "C" int mnc_fc_forward(const float* x, const float* w, const float* b, float* y, int M,
                              int N, int K, void* workspace, long long workspace_bytes,
                              void* stream) {
  if (!x || !w || !y || M < 1 || N < 1 || K < 1) return MNC_ERR_ARG;
  FcOut o;
  o.ptr = y;
  o.sp = 1;
  o.sq = N;
  o.bias = b;
  o.mode = kEpiStore;
  return launch_gemm(operand(w, K, N, true), operand(x, K, M, true), N, M, K, o, workspace,
                     workspace_bytes, static_cast<cudaStream_t>(stream));
}

extern "C" int mnc_fc_backward(const float* x, const float* w, const float* dy, float* dx,
                               float* dw, float* db, int M, int N, int K, void* workspace,
                               long long workspace_bytes, void* stream) {
  if (!dy || M < 1 || N < 1 || K < 1) return MNC_ERR_ARG;
  if ((dw && !x) || (dx && !w)) return MNC_ERR_ARG;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = MNC_OK;
  if (dw) {   // dW[n, k] += sum_m dY[m, n] X[m, k]
    FcOut o;
    o.ptr = dw;
    o.sp = K;
    o.sq = 1;
    o.bias = nullptr;
    o.mode = kEpiAccumulate;
    rc = launch_gemm(operand(dy, N, N, false), operand(x, K, K, false), N, K, M, o, workspace,
                     workspace_bytes, st);
    if (rc != MNC_OK) return rc;
  }
  if (db) {
    fc_bias_grad_kernel<<<(N + 255) / 256, 256, 0, st>>>(dy, M, N, db);
    if ((rc = check_launch()) != MNC_OK) return rc;
  }
  if (dx) {   // dX[m, k] = sum_n dY[m, n] W[n, k]
    FcOut o;
    o.ptr = dx;
    o.sp = 1;
    o.sq = K;
    o.bias = nullptr;
    o.mode = kEpiStore;
    rc = launch_gemm(operand(w, K, K, false), operand(dy, N, M, true), K, M, N, o, workspace,
                     workspace_bytes, st);
  }
  return rc;
}

extern "C" int mnc_max_pool_nchw(const float* x, int N, int C, int H, int W, int kernel,
                                 int stride, int pad, float* y, int* mask, void* stream) {
  if (!x || !y || !mask || !pool_args_ok(N, C, H, W, kernel, stride, pad)) return MNC_ERR_ARG;
  const int PH = pooled_size(H, kernel, stride), PW = pooled_size(W, kernel, stride);
  const long long n = static_cast<long long>(N) * C * PH * PW;
  if (n == 0) return MNC_OK;
  max_pool_kernel<<<ew_grid(n), kEw, 0, static_cast<cudaStream_t>(stream)>>>(x, n, H, W, PH, PW,
                                                                             kernel, stride, y, mask);
  return check_launch();
}

extern "C" int mnc_max_pool_backward_nchw(const float* dy, const int* mask, int N, int C, int H,
                                          int W, int kernel, int stride, int pad, float* dx,
                                          void* stream) {
  if (!dy || !mask || !dx || !pool_args_ok(N, C, H, W, kernel, stride, pad)) return MNC_ERR_ARG;
  const int PH = pooled_size(H, kernel, stride), PW = pooled_size(W, kernel, stride);
  const long long n = static_cast<long long>(N) * C * H * W;
  if (n == 0) return MNC_OK;
  max_pool_backward_kernel<<<ew_grid(n), kEw, 0, static_cast<cudaStream_t>(stream)>>>(
      dy, mask, n, H, W, PH, PW, kernel, stride, dx);
  return check_launch();
}

extern "C" int mnc_relu(const float* x, long long n, float* y, void* stream) {
  if (!x || !y || n < 0) return MNC_ERR_ARG;
  if (n == 0) return MNC_OK;
  relu_kernel<<<ew_grid(n), kEw, 0, static_cast<cudaStream_t>(stream)>>>(x, n, y);
  return check_launch();
}

extern "C" int mnc_relu_backward(const float* x, const float* dy, long long n, float* dx,
                                 void* stream) {
  if (!x || !dy || !dx || n < 0) return MNC_ERR_ARG;
  if (n == 0) return MNC_OK;
  relu_backward_kernel<<<ew_grid(n), kEw, 0, static_cast<cudaStream_t>(stream)>>>(x, dy, n, dx);
  return check_launch();
}

extern "C" int mnc_sigmoid(const float* x, long long n, float* y, void* stream) {
  if (!x || !y || n < 0) return MNC_ERR_ARG;
  if (n == 0) return MNC_OK;
  sigmoid_kernel<<<ew_grid(n), kEw, 0, static_cast<cudaStream_t>(stream)>>>(x, n, y);
  return check_launch();
}

extern "C" int mnc_sigmoid_backward(const float* y, const float* dy, long long n, float* dx,
                                    void* stream) {
  if (!y || !dy || !dx || n < 0) return MNC_ERR_ARG;
  if (n == 0) return MNC_OK;
  sigmoid_backward_kernel<<<ew_grid(n), kEw, 0, static_cast<cudaStream_t>(stream)>>>(y, dy, n, dx);
  return check_launch();
}
