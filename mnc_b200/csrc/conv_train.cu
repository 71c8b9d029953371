// Convolution of the training net (the VGG-16 trunk and the RPN) on fp32 NCHW Caffe blobs: forward,
// dX, dW and db on the tensor cores.  Replaces
//   Convolution  conv_layer.cu:10-62 with base_conv_layer.cpp:232-294 (im2col + sgemm per image)
// for the nets' two forms, kernel 3 / pad 1 and kernel 1 / pad 0, stride 1, dilation 1, group 1.
// DESIGN.md "Trunk and RPN convolutions for training" states the mapping and the precision contract.
//
// Every product is the split-bf16 GEMM of gemm_core.cuh, C[p, q] = sum_r A(p, r) * B(q, r), one
// launch per image, with t = kh * 3 + kw the tap of a 3x3 kernel and pix = y * W + x:
//   forward  p = co, q = pix, r = ci * 9 + t   A = W (Cout, Cin * 9) as stored     Y[co, pix] = C + b
//            B = X gathered at (y + kh - 1, x + kw - 1)
//   dX       p = ci, q = pix, r = co * 9 + t   A = W transposed to (Cin, Cout * 9)  dX[ci, pix] = C
//            in the workspace; B = dY gathered at (y - kh + 1, x - kw + 1)
//   dW       p = co, q = ci * 9 + t, r = pix   A = dY (Cout, H * W)                 dW[co, q] += C
//            B = X gathered at (y + kh - 1, x + kw - 1)
// The gather computes each source address in the loader and reads zero outside the image, so no
// column buffer is written.  A 1x1 kernel needs no gather: every operand is a dense matrix.
#include <cstdint>
#include <cuda_runtime.h>

#include "mnc_b200.h"
#include "gemm_core.cuh"
#include "launch_util.h"

namespace mnc {
namespace {

// A 3x3 image operand with the pixel as the row: element (pix, c * 9 + t) is
// img[c, y + kSign * (kh - 1), x + kSign * (kw - 1)], zero outside the H x W image.
// kSign +1: the forward's X; -1: dX's dY.  Consecutive threads walk pixels, so a warp's loads are
// coalesced along image rows.
template <int kSign>
struct GatherPixRows {
  const float* img;
  int H, W;
  int rows;     // H * W

  template <int kRows>
  __device__ __forceinline__ void item(int i, int& row, int& chunk) const {
    const int idx = threadIdx.x + i * kFcThreads;
    row = idx % kRows;
    chunk = idx / kRows;
  }

  template <int kRows>
  __device__ __forceinline__ void load(int row0, int r0, int R, FcStaged<kRows>& s) const {
#pragma unroll
    for (int i = 0; i < FcStaged<kRows>::kItems; ++i) {
      int row, chunk;
      item<kRows>(i, row, chunk);
      const int pix = row0 + row;
      const int y = pix / W, x = pix - y * W;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int r = r0 + chunk * 8 + j;
        const int c = r / 9, t = r - c * 9;
        const int kh = t / 3, kw = t - kh * 3;
        const int yy = y + kSign * (kh - 1), xx = x + kSign * (kw - 1);
        const bool ok = pix < rows && r < R && yy >= 0 && yy < H && xx >= 0 && xx < W;
        s.v[i][j] = ok ? __ldg(img + (static_cast<long long>(c) * H + yy) * W + xx) : 0.f;
      }
    }
  }
};

// A 3x3 image operand with the pixel as the reduction (dW's X): element (ci * 9 + t, pix) is
// X[ci, y + kh - 1, x + kw - 1], zero outside the image.  Consecutive threads walk 8-pixel chunks
// of one row, so the eight loads of a thread, and a warp's loads, follow an image row.
struct GatherPixRed {
  const float* img;
  int H, W;
  int rows;     // Cin * 9

  template <int kRows>
  __device__ __forceinline__ void item(int i, int& row, int& chunk) const {
    const int idx = threadIdx.x + i * kFcThreads;
    row = idx >> 3;
    chunk = idx & 7;
  }

  template <int kRows>
  __device__ __forceinline__ void load(int row0, int r0, int R, FcStaged<kRows>& s) const {
#pragma unroll
    for (int i = 0; i < FcStaged<kRows>::kItems; ++i) {
      int row, chunk;
      item<kRows>(i, row, chunk);
      const int q = row0 + row;
      const int c = q / 9, t = q - c * 9;
      const int dy = t / 3 - 1, dx = t - (t / 3) * 3 - 1;
      const int pix0 = r0 + chunk * 8;
      int y = pix0 / W, x = pix0 - y * W;
      const float* plane = img + static_cast<long long>(c) * H * W;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int yy = y + dy, xx = x + dx;
        const bool ok = q < rows && pix0 + j < R && yy >= 0 && yy < H && xx >= 0 && xx < W;
        s.v[i][j] = ok ? __ldg(plane + yy * W + xx) : 0.f;
        if (++x == W) {
          x = 0;
          ++y;
        }
      }
    }
  }
};

// wt[ci, co * 9 + t] = w[co, ci, t]: the A operand of dX for a 3x3 kernel.
__global__ void __launch_bounds__(256)
conv_transpose_weight_kernel(const float* __restrict__ w, int Cout, int Cin, float* __restrict__ wt) {
  const long long n = static_cast<long long>(Cout) * Cin * 9;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * 256) {
    const int t = static_cast<int>(i % 9);
    const long long cc = i / 9;
    const int ci = static_cast<int>(cc % Cin), co = static_cast<int>(cc / Cin);
    wt[(static_cast<long long>(ci) * Cout + co) * 9 + t] = w[i];
  }
}

// db[co] += sum over images (in order) of sum over pixels of dY[n, co, pix].  The pixel sum of one
// image is fixed-order: thread j adds pixels j, j + 256, ... in order, then a binary tree adds the
// 256 partials (stride 128, 64, ..., 1).  One CTA per channel.
__global__ void __launch_bounds__(256)
conv_bias_grad_kernel(const float* __restrict__ dy, int N, int Cout, int HW, float* __restrict__ db) {
  __shared__ float red[256];
  const int co = blockIdx.x;
  float total = 0.f;
  for (int n = 0; n < N; ++n) {
    const float* p = dy + (static_cast<long long>(n) * Cout + co) * HW;
    float s = 0.f;
    for (int i = threadIdx.x; i < HW; i += 256) s = __fadd_rn(s, p[i]);
    red[threadIdx.x] = s;
    __syncthreads();
    for (int h = 128; h > 0; h >>= 1) {
      if (threadIdx.x < h) red[threadIdx.x] = __fadd_rn(red[threadIdx.x], red[threadIdx.x + h]);
      __syncthreads();
    }
    total = n == 0 ? red[0] : __fadd_rn(total, red[0]);
    __syncthreads();
  }
  if (threadIdx.x == 0) db[co] = __fadd_rn(db[co], total);
}

struct ConvShape {
  int N, Cin, H, W, Cout, k;
  int HW() const { return H * W; }
  int taps() const { return k * k; }
};

bool shape_ok(int N, int Cin, int H, int W, int Cout, int kernel) {
  if (N < 1 || Cin < 1 || H < 1 || W < 1 || Cout < 1) return false;
  if (kernel != 1 && kernel != 3) return false;
  // every index of a product and of a tensor fits an int; one image's operands are addressed with
  // long long where they multiply
  const long long hw = static_cast<long long>(H) * W;
  return hw <= (1 << 30) && static_cast<long long>(Cin) * 9 <= (1 << 30) &&
         static_cast<long long>(Cout) * 9 <= (1 << 30);
}

bool form_ok(int kernel, int pad, int stride) {
  return stride == 1 && ((kernel == 3 && pad == 1) || (kernel == 1 && pad == 0));
}

// Workspace: the split-K partials of the largest of the three products, then (3x3) dX's
// transposed weight, 256-byte aligned.
long long partials_bytes(const ConvShape& s) {
  const int HW = s.HW(), rc = s.Cin * s.taps(), ro = s.Cout * s.taps();
  long long b = gemm_workspace(s.Cout, HW, rc);
  const long long dx = gemm_workspace(s.Cin, HW, ro), dw = gemm_workspace(s.Cout, rc, HW);
  if (dx > b) b = dx;
  if (dw > b) b = dw;
  return (b + 255) / 256 * 256;
}

long long workspace_bytes(const ConvShape& s) {
  const long long wt = s.k == 3 ? static_cast<long long>(s.Cin) * s.Cout * 9 * sizeof(float) : 0;
  return partials_bytes(s) + wt;
}

FcOut out_rows(float* ptr, long long sp, const float* bias, int mode) {
  FcOut o;
  o.ptr = ptr;
  o.sp = sp;
  o.sq = 1;
  o.bias = bias;
  o.mode = mode;
  return o;
}

}  // namespace
}  // namespace mnc

using namespace mnc;

extern "C" long long mnc_conv_workspace_bytes(int N, int Cin, int H, int W, int Cout, int kernel) {
  if (!shape_ok(N, Cin, H, W, Cout, kernel)) return 0;
  return workspace_bytes(ConvShape{N, Cin, H, W, Cout, kernel});
}

extern "C" int mnc_conv_forward(const float* x, const float* w, const float* b, float* y, int N,
                                int Cin, int H, int W, int Cout, int kernel, int pad, int stride,
                                void* workspace, long long workspace_bytes_, void* stream) {
  if (!x || !w || !y || !shape_ok(N, Cin, H, W, Cout, kernel) || !form_ok(kernel, pad, stride))
    return MNC_ERR_ARG;
  const ConvShape s{N, Cin, H, W, Cout, kernel};
  const int HW = s.HW(), R = Cin * s.taps();
  // the forward uses only the split-K partials of its own product, at the start of the workspace
  const long long need = gemm_workspace(Cout, HW, R);
  if (workspace_bytes_ < need || (need > 0 && !workspace)) return MNC_ERR_ARG;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const FcOperand A = operand(w, R, Cout, true);
  int rc = MNC_OK;
  for (int n = 0; n < N && rc == MNC_OK; ++n) {
    const float* xn = x + static_cast<long long>(n) * Cin * HW;
    const FcOut o = out_rows(y + static_cast<long long>(n) * Cout * HW, HW, b, kEpiStore);
    if (kernel == 3)
      rc = launch_gemm(A, GatherPixRows<1>{xn, H, W, HW}, Cout, HW, R, o, workspace,
                       workspace_bytes_, st);
    else
      rc = launch_gemm(A, operand(xn, HW, HW, false), Cout, HW, R, o, workspace, workspace_bytes_, st);
  }
  return rc;
}

extern "C" int mnc_conv_backward(const float* x, const float* w, const float* dy, float* dx,
                                 float* dw, float* db, int N, int Cin, int H, int W, int Cout,
                                 int kernel, int pad, int stride, void* workspace,
                                 long long workspace_bytes_, void* stream) {
  if (!dy || !shape_ok(N, Cin, H, W, Cout, kernel) || !form_ok(kernel, pad, stride))
    return MNC_ERR_ARG;
  if ((dw && !x) || (dx && !w)) return MNC_ERR_ARG;
  const ConvShape s{N, Cin, H, W, Cout, kernel};
  if (workspace_bytes_ < workspace_bytes(s) || (workspace_bytes(s) > 0 && !workspace))
    return MNC_ERR_ARG;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int HW = s.HW(), taps = s.taps();
  int rc = MNC_OK;
  // dW[co, ci * taps + t] += sum_pix dY[co, pix] X[ci, pix + shift(t)], image by image
  for (int n = 0; dw && n < N && rc == MNC_OK; ++n) {
    const FcOperand A = operand(dy + static_cast<long long>(n) * Cout * HW, HW, Cout, true);
    const float* xn = x + static_cast<long long>(n) * Cin * HW;
    const FcOut o = out_rows(dw, static_cast<long long>(Cin) * taps, nullptr, kEpiAccumulate);
    if (kernel == 3)
      rc = launch_gemm(A, GatherPixRed{xn, H, W, Cin * 9}, Cout, Cin * 9, HW, o, workspace,
                       workspace_bytes_, st);
    else
      rc = launch_gemm(A, operand(xn, HW, Cin, true), Cout, Cin, HW, o, workspace, workspace_bytes_, st);
  }
  if (rc != MNC_OK) return rc;
  if (db) {
    conv_bias_grad_kernel<<<Cout, 256, 0, st>>>(dy, N, Cout, HW, db);
    if ((rc = check_launch()) != MNC_OK) return rc;
  }
  if (!dx) return rc;
  // dX[ci, pix] = sum_{co, t} W[co, ci, t] dY[co, pix - shift(t)], overwritten
  FcOperand A;
  if (kernel == 3) {
    float* wt = reinterpret_cast<float*>(static_cast<uint8_t*>(workspace) + partials_bytes(s));
    const long long nw = static_cast<long long>(Cout) * Cin * 9;
    conv_transpose_weight_kernel<<<grid_for(nw, 256, 4 * 132), 256, 0, st>>>(w, Cout, Cin, wt);
    if ((rc = check_launch()) != MNC_OK) return rc;
    A = operand(wt, static_cast<long long>(Cout) * 9, Cin, true);
  } else {
    A = operand(w, Cin, Cin, false);
  }
  for (int n = 0; n < N && rc == MNC_OK; ++n) {
    const float* dyn = dy + static_cast<long long>(n) * Cout * HW;
    const FcOut o = out_rows(dx + static_cast<long long>(n) * Cin * HW, HW, nullptr, kEpiStore);
    if (kernel == 3)
      rc = launch_gemm(A, GatherPixRows<-1>{dyn, H, W, HW}, Cin, HW, Cout * 9, o, workspace,
                       workspace_bytes_, st);
    else
      rc = launch_gemm(A, operand(dyn, HW, HW, false), Cin, HW, Cout, o, workspace,
                       workspace_bytes_, st);
  }
  return rc;
}
