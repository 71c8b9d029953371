// Loss layers of the MNC training net, one image, fp32 device blobs in Caffe layout.  Replaces
//   SoftmaxWithLoss         softmax_loss_layer.cpp:10-86, softmax_loss_layer.cu:11-124 (with the
//                           Softmax GPU arithmetic of softmax_layer.cu:9-120)
//   SmoothL1Loss            smooth_L1_loss_layer.cpp:13-22, smooth_L1_loss_layer.cu:13-136
//   SigmoidCrossEntropyLoss sigmoid_cross_entropy_loss_layer.cpp:31-97 (MNC's weighted form; the
//                           sigmoid is SigmoidForward of sigmoid_layer.cu:9-14)
//   Accuracy                accuracy_layer.cpp:48-103 (forward only, top-1 per class not written)
// DESIGN.md "Loss layers" lists the quirks kept.
//
// Every entry point takes n_valid (device int, NULL: all rows): only the first *n_valid outer rows
// are read, backward writes 0 to the diff of the others, and every normaliser that counts rows
// counts *n_valid.  Loss scalars are reduced in one fixed order: thread t of the one CTA adds the
// float32 terms i = t, t + 1024, ... in float64, then the 1024 partials are added by a halving tree
// (p[t] += p[t + s], s = 512 .. 1); the sum is rounded to float32 once and divided by the
// normaliser in float32.  Terms of padding rows are never formed, so a padded blob with n_valid
// gives the bits of the blob trimmed to n_valid rows.  No atomics; stream-ordered; sync-free.
#include <cfloat>
#include <cuda_runtime.h>

#include "mnc_b200.h"
#include "launch_util.h"
#include "sigmoid.cuh"

namespace mnc {
namespace {

constexpr int kT = 1024;              // threads of the one-CTA kernels
constexpr int kEwThreads = 256;       // element-wise backward

__device__ __forceinline__ int valid_rows(const int* n_valid, int num) {
  if (!n_valid) return num;
  const int v = *n_valid;
  return v < 0 ? 0 : (v > num ? num : v);
}

// The fixed-order float64 sum of the header comment.  Every thread of the CTA calls it.
__device__ double block_sum(double v, double* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = kT / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] = __dadd_rn(sh[threadIdx.x], sh[threadIdx.x + s]);
    __syncthreads();
  }
  const double r = sh[0];
  __syncthreads();
  return r;
}

__device__ int block_count(int v, int* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = kT / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  const int r = sh[0];
  __syncthreads();
  return r;
}

// get_normalizer (softmax_loss_layer.cpp:58-84), valid_count -1 when not counted (the GPU path
// counts only for VALID with an ignore label, softmax_loss_layer.cu:57-61).
__device__ float softmax_normalizer(int mode, int rows, int inner, int valid_count) {
  float n;
  switch (mode) {
    case 0: n = static_cast<float>(rows * inner); break;                      // FULL
    case 1: n = static_cast<float>(valid_count == -1 ? rows * inner : valid_count); break;
    case 2: n = static_cast<float>(rows); break;                              // BATCH_SIZE
    default: n = 1.f; break;                                                  // NONE
  }
  return fmaxf(1.f, n);
}

__device__ __forceinline__ bool is_ignored(int label, int has_ignore, int ignore_label) {
  return has_ignore && label == ignore_label;
}

// ------------------------------------------------------------------ SoftmaxWithLoss
// One thread per (row, inner) position: Caffe's channel max from -FLT_MAX, subtract, expf, channel
// sum in channel order, divide (softmax_layer.cu:86-120, one kernel per step there); then the
// position's loss term -log(max(p_label, FLT_MIN)) (softmax_loss_layer.cu:11-29).
__global__ void __launch_bounds__(kT)
softmax_loss_kernel(const float* __restrict__ x, const float* __restrict__ label, int outer, int C,
                    int inner, const int* __restrict__ n_valid, int has_ignore, int ignore_label,
                    int mode, float* __restrict__ prob, float* __restrict__ loss) {
  __shared__ double shd[kT];
  __shared__ int shi[kT];
  const int rows = valid_rows(n_valid, outer);
  const int npos = rows * inner;
  double acc = 0.0;
  int cnt = 0;
  for (int p = threadIdx.x; p < npos; p += kT) {
    const int n = p / inner, s = p % inner;
    const float* xp = x + static_cast<long long>(n) * C * inner + s;
    float* pp = prob + static_cast<long long>(n) * C * inner + s;
    float m = -FLT_MAX;
    for (int c = 0; c < C; ++c) m = fmaxf(xp[static_cast<long long>(c) * inner], m);
    float sum = 0.f;
    for (int c = 0; c < C; ++c) {
      const float e = expf(__fsub_rn(xp[static_cast<long long>(c) * inner], m));
      pp[static_cast<long long>(c) * inner] = e;
      sum = __fadd_rn(sum, e);
    }
    for (int c = 0; c < C; ++c) {
      float* q = pp + static_cast<long long>(c) * inner;
      *q = __fdiv_rn(*q, sum);
    }
    const int l = static_cast<int>(label[p]);
    if (!is_ignored(l, has_ignore, ignore_label)) {
      ++cnt;
      if (l >= 0 && l < C)   // outside [0, C): counted, no term (DESIGN.md "Loss layers")
        acc = __dadd_rn(acc, static_cast<double>(-logf(fmaxf(pp[static_cast<long long>(l) * inner],
                                                              FLT_MIN))));
    }
  }
  // padding rows of prob: zeros
  const long long total = static_cast<long long>(outer) * C * inner;
  for (long long i = static_cast<long long>(rows) * C * inner + threadIdx.x; i < total; i += kT)
    prob[i] = 0.f;
  const double sum = block_sum(acc, shd);
  const int valid = block_count(cnt, shi);
  if (threadIdx.x == 0) {
    const int vc = (mode == 1 && has_ignore) ? valid : -1;
    loss[0] = __fdiv_rn(static_cast<float>(sum), softmax_normalizer(mode, rows, inner, vc));
  }
}

// softmax_loss_layer.cu:70-124: diff = prob, -1 at the label, 0 in every channel of an ignored
// position; then scaled by top_diff / normaliser (one division, one multiply per element).
__global__ void __launch_bounds__(kT)
softmax_loss_backward_kernel(const float* __restrict__ prob, const float* __restrict__ label,
                             int outer, int C, int inner, const int* __restrict__ n_valid,
                             int has_ignore, int ignore_label, int mode,
                             const float* __restrict__ top_diff, float* __restrict__ diff) {
  __shared__ int shi[kT];
  const int rows = valid_rows(n_valid, outer);
  const int npos = rows * inner;
  int cnt = 0;
  for (int p = threadIdx.x; p < npos; p += kT)
    cnt += !is_ignored(static_cast<int>(label[p]), has_ignore, ignore_label);
  const int valid = block_count(cnt, shi);
  const int vc = (mode == 1 && has_ignore) ? valid : -1;
  const float scale = __fdiv_rn(top_diff[0], softmax_normalizer(mode, rows, inner, vc));
  for (int p = threadIdx.x; p < npos; p += kT) {
    const int n = p / inner, s = p % inner;
    const long long base = static_cast<long long>(n) * C * inner + s;
    const int l = static_cast<int>(label[p]);
    const bool ign = is_ignored(l, has_ignore, ignore_label);
    for (int c = 0; c < C; ++c) {
      const long long i = base + static_cast<long long>(c) * inner;
      float d = ign ? 0.f : prob[i];
      if (!ign && c == l) d = __fsub_rn(d, 1.f);
      diff[i] = __fmul_rn(d, scale);
    }
  }
  const long long total = static_cast<long long>(outer) * C * inner;
  for (long long i = static_cast<long long>(rows) * C * inner + threadIdx.x; i < total; i += kT)
    diff[i] = 0.f;
}

// ------------------------------------------------------------------ SmoothL1Loss
// smooth_L1_loss_layer.cu:13-28,31-63: d = w_in * (b0 - b1) in float; the branch and its value in
// double (1.0 / sigma2, 0.5 * val * val * sigma2, abs_val - 0.5 / sigma2), stored as float; then
// * w_out in float.
__device__ __forceinline__ float smooth_l1_d(const float* b0, const float* b1, const float* w_in,
                                             long long i) {
  const float d = __fsub_rn(b0[i], b1[i]);
  return w_in ? __fmul_rn(w_in[i], d) : d;
}

__global__ void __launch_bounds__(kT)
smooth_l1_loss_kernel(const float* __restrict__ b0, const float* __restrict__ b1,
                      const float* __restrict__ w_in, const float* __restrict__ w_out, int num,
                      int dim, const int* __restrict__ n_valid, float sigma2,
                      float* __restrict__ loss) {
  __shared__ double shd[kT];
  const int rows = valid_rows(n_valid, num);
  const long long n = static_cast<long long>(rows) * dim;
  const double s2 = sigma2;
  double acc = 0.0;
  for (long long i = threadIdx.x; i < n; i += kT) {
    const float val = smooth_l1_d(b0, b1, w_in, i);
    const float abs_val = fabsf(val);
    float e;
    if (static_cast<double>(abs_val) < __ddiv_rn(1.0, s2))
      e = static_cast<float>(__dmul_rn(__dmul_rn(__dmul_rn(0.5, val), val), s2));
    else
      e = static_cast<float>(__dsub_rn(abs_val, __ddiv_rn(0.5, s2)));
    if (w_out) e = __fmul_rn(w_out[i], e);
    acc = __dadd_rn(acc, static_cast<double>(e));
  }
  const double sum = block_sum(acc, shd);
  if (threadIdx.x == 0) loss[0] = __fdiv_rn(static_cast<float>(sum), static_cast<float>(rows));
}

// smooth_L1_loss_layer.cu:67-106, bottom 0: sigma2 * val or sign(val) (threshold in double), times
// alpha = top_diff / num, then * w_in, then * w_out, each rounded.
__global__ void __launch_bounds__(kEwThreads)
smooth_l1_loss_backward_kernel(const float* __restrict__ b0, const float* __restrict__ b1,
                               const float* __restrict__ w_in, const float* __restrict__ w_out,
                               int num, int dim, const int* __restrict__ n_valid, float sigma2,
                               const float* __restrict__ top_diff, float* __restrict__ diff) {
  const int rows = valid_rows(n_valid, num);
  const long long n = static_cast<long long>(rows) * dim;
  const long long total = static_cast<long long>(num) * dim;
  const float alpha = __fdiv_rn(top_diff[0], static_cast<float>(rows));
  const double thresh = __ddiv_rn(1.0, static_cast<double>(sigma2));
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    if (i >= n) {
      diff[i] = 0.f;
      continue;
    }
    const float val = smooth_l1_d(b0, b1, w_in, i);
    const float g = static_cast<double>(fabsf(val)) < thresh
                        ? __fmul_rn(sigma2, val)
                        : static_cast<float>((0.f < val) - (val < 0.f));
    float d = __fmul_rn(alpha, g);
    if (w_in) d = __fmul_rn(w_in[i], d);
    if (w_out) d = __fmul_rn(w_out[i], d);
    diff[i] = d;
  }
}

// ------------------------------------------------------------------ SigmoidCrossEntropyLoss
// One term of sigmoid_cross_entropy_loss_layer.cpp:44-58 as the reference's object evaluates it:
// <math.h> (through mkl_alternate.hpp) puts the float overloads of exp / log in scope, so the
// whole term is float -- expf, 1 + e, logf, a - l, w * (...) -- each operation rounded.
__device__ __forceinline__ float sce_term(float x, float t, const float* w, long long i) {
  const float ge = x >= 0.f ? 1.f : 0.f;
  const float a = __fmul_rn(x, __fsub_rn(t, ge));
  const float b = __fsub_rn(x, __fmul_rn(__fmul_rn(2.f, x), ge));
  const float in = __fsub_rn(a, logf(__fadd_rn(1.f, expf(b))));
  return w ? __fmul_rn(w[i], in) : in;
}

// Loss = -sum w * (...) / sum w (weights) or / num (no weights); with weights and sum w == 0 the
// loss is not written.
__global__ void __launch_bounds__(kT)
sigmoid_ce_loss_kernel(const float* __restrict__ x, const float* __restrict__ t,
                       const float* __restrict__ w, int num, int dim,
                       const int* __restrict__ n_valid, float* __restrict__ loss) {
  __shared__ double shd[kT];
  const int rows = valid_rows(n_valid, num);
  const long long n = static_cast<long long>(rows) * dim;
  double acc = 0.0, wacc = 0.0;
  for (long long i = threadIdx.x; i < n; i += kT) {
    acc = __dadd_rn(acc, static_cast<double>(sce_term(x[i], t[i], w, i)));
    if (w) wacc = __dadd_rn(wacc, static_cast<double>(w[i]));
  }
  const double sum = block_sum(acc, shd);
  const double wsum = w ? block_sum(wacc, shd) : 0.0;
  if (threadIdx.x == 0) {
    const float l = -static_cast<float>(sum);
    if (!w) {
      loss[0] = __fdiv_rn(l, static_cast<float>(rows));
    } else {
      const float ws = static_cast<float>(wsum);
      if (ws > 0.f) loss[0] = __fdiv_rn(l, ws);
    }
  }
}

// :62-92: diff = (s - t) * w, then * (top_diff / sum w) when sum w > 0; without weights
// (s - t) * (top_diff / num).
__global__ void __launch_bounds__(kT)
sigmoid_ce_loss_backward_kernel(const float* __restrict__ x, const float* __restrict__ t,
                                const float* __restrict__ w, int num, int dim,
                                const int* __restrict__ n_valid,
                                const float* __restrict__ top_diff, float* __restrict__ diff) {
  __shared__ double shd[kT];
  const int rows = valid_rows(n_valid, num);
  const long long n = static_cast<long long>(rows) * dim;
  const long long total = static_cast<long long>(num) * dim;
  double wacc = 0.0;
  if (w)
    for (long long i = threadIdx.x; i < n; i += kT) wacc = __dadd_rn(wacc, static_cast<double>(w[i]));
  const float ws = w ? static_cast<float>(block_sum(wacc, shd)) : 0.f;
  const bool scaled = !w || ws > 0.f;
  const float scale = __fdiv_rn(top_diff[0], w ? ws : static_cast<float>(rows));
  for (long long i = threadIdx.x; i < n; i += kT) {
    float d = __fsub_rn(ref_sigmoid(x[i]), t[i]);
    if (w) d = __fmul_rn(d, w[i]);
    if (scaled) d = __fmul_rn(d, scale);
    diff[i] = d;
  }
  for (long long i = n + threadIdx.x; i < total; i += kT) diff[i] = 0.f;
}

// ------------------------------------------------------------------ Accuracy
// accuracy_layer.cpp:48-103.  partial_sort with std::greater<pair<float, int>> ranks equal scores
// by the higher class index, so the label is in the top k iff fewer than k classes have a
// (score, index) pair greater than its own; a label outside [0, C) is never in it.
__global__ void __launch_bounds__(kT)
accuracy_kernel(const float* __restrict__ x, const float* __restrict__ label, int outer, int C,
                int inner, const int* __restrict__ n_valid, int top_k, int has_ignore,
                int ignore_label, float* __restrict__ out) {
  __shared__ int shi[kT];
  const int rows = valid_rows(n_valid, outer);
  const int npos = rows * inner;
  int hits = 0, cnt = 0;
  for (int p = threadIdx.x; p < npos; p += kT) {
    const int l = static_cast<int>(label[p]);
    if (is_ignored(l, has_ignore, ignore_label)) continue;
    ++cnt;
    if (l < 0 || l >= C) continue;
    const int n = p / inner, s = p % inner;
    const float* xp = x + static_cast<long long>(n) * C * inner + s;
    const float sl = xp[static_cast<long long>(l) * inner];
    int greater = 0;
    for (int c = 0; c < C; ++c) {
      const float sc = xp[static_cast<long long>(c) * inner];
      greater += (sl < sc) || (!(sc < sl) && c > l);
    }
    hits += greater < top_k;
  }
  const int h = block_count(hits, shi);
  const int c = block_count(cnt, shi);
  if (threadIdx.x == 0) out[0] = __fdiv_rn(static_cast<float>(h), static_cast<float>(c));
}

}  // namespace
}  // namespace mnc

using namespace mnc;

extern "C" int mnc_softmax_loss(const float* scores, const float* labels, int outer, int channels,
                                int inner, const int* n_valid, int has_ignore, int ignore_label,
                                int normalization, float* prob, float* loss, void* stream) {
  if (outer < 0 || channels <= 0 || inner <= 0 || normalization < 0 || normalization > 3 ||
      !prob || !loss)
    return MNC_ERR_ARG;
  softmax_loss_kernel<<<1, kT, 0, static_cast<cudaStream_t>(stream)>>>(
      scores, labels, outer, channels, inner, n_valid, has_ignore, ignore_label, normalization,
      prob, loss);
  return check_launch();
}

extern "C" int mnc_softmax_loss_backward(const float* prob, const float* labels, int outer,
                                         int channels, int inner, const int* n_valid,
                                         int has_ignore, int ignore_label, int normalization,
                                         const float* top_diff, float* bottom_diff, void* stream) {
  if (outer < 0 || channels <= 0 || inner <= 0 || normalization < 0 || normalization > 3 ||
      !top_diff || !bottom_diff)
    return MNC_ERR_ARG;
  softmax_loss_backward_kernel<<<1, kT, 0, static_cast<cudaStream_t>(stream)>>>(
      prob, labels, outer, channels, inner, n_valid, has_ignore, ignore_label, normalization,
      top_diff, bottom_diff);
  return check_launch();
}

extern "C" int mnc_smooth_l1_loss(const float* pred, const float* target,
                                  const float* inside_weights, const float* outside_weights,
                                  int num, int dim, const int* n_valid, float sigma, float* loss,
                                  void* stream) {
  if (num < 0 || dim <= 0 || !loss || (!inside_weights) != (!outside_weights)) return MNC_ERR_ARG;
  smooth_l1_loss_kernel<<<1, kT, 0, static_cast<cudaStream_t>(stream)>>>(
      pred, target, inside_weights, outside_weights, num, dim, n_valid, sigma * sigma, loss);
  return check_launch();
}

extern "C" int mnc_smooth_l1_loss_backward(const float* pred, const float* target,
                                           const float* inside_weights,
                                           const float* outside_weights, int num, int dim,
                                           const int* n_valid, float sigma, const float* top_diff,
                                           float* bottom_diff, void* stream) {
  if (num < 0 || dim <= 0 || !top_diff || !bottom_diff || (!inside_weights) != (!outside_weights))
    return MNC_ERR_ARG;
  const long long total = static_cast<long long>(num) * dim;
  if (total == 0) return MNC_OK;
  const long long want = (total + kEwThreads - 1) / kEwThreads;
  const int blocks = static_cast<int>(want < 1024 ? want : 1024);
  smooth_l1_loss_backward_kernel<<<blocks, kEwThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      pred, target, inside_weights, outside_weights, num, dim, n_valid, sigma * sigma, top_diff,
      bottom_diff);
  return check_launch();
}

extern "C" int mnc_sigmoid_ce_loss(const float* x, const float* targets, const float* weights,
                                   int num, int dim, const int* n_valid, float* loss,
                                   void* stream) {
  if (num < 0 || dim <= 0 || !loss) return MNC_ERR_ARG;
  sigmoid_ce_loss_kernel<<<1, kT, 0, static_cast<cudaStream_t>(stream)>>>(
      x, targets, weights, num, dim, n_valid, loss);
  return check_launch();
}

extern "C" int mnc_sigmoid_ce_loss_backward(const float* x, const float* targets,
                                            const float* weights, int num, int dim,
                                            const int* n_valid, const float* top_diff,
                                            float* bottom_diff, void* stream) {
  if (num < 0 || dim <= 0 || !top_diff || !bottom_diff) return MNC_ERR_ARG;
  sigmoid_ce_loss_backward_kernel<<<1, kT, 0, static_cast<cudaStream_t>(stream)>>>(
      x, targets, weights, num, dim, n_valid, top_diff, bottom_diff);
  return check_launch();
}

extern "C" int mnc_accuracy(const float* scores, const float* labels, int outer, int channels,
                            int inner, const int* n_valid, int top_k, int has_ignore,
                            int ignore_label, float* accuracy, void* stream) {
  if (outer < 0 || channels <= 0 || inner <= 0 || top_k < 1 || top_k > channels || !accuracy)
    return MNC_ERR_ARG;
  accuracy_kernel<<<1, kT, 0, static_cast<cudaStream_t>(stream)>>>(
      scores, labels, outer, channels, inner, n_valid, top_k, has_ignore, ignore_label, accuracy);
  return check_launch();
}
