// Head layers of the training net on fp32 Caffe blobs: InnerProduct forward and backward on the
// tensor cores, max Pooling, ReLU and Sigmoid forward and backward.  Replaces
//   InnerProduct  inner_product_layer.cu:9-55 (cuBLAS sgemm / sgemv in the reference)
//   Pooling MAX   pooling_layer.cu:9-44 (MaxPoolForward), MaxPoolBackward; output size
//                 pooling_layer.cpp:90-100
//   ReLU          relu_layer.cu:9-41 (negative_slope 0)
//   Sigmoid       sigmoid_layer.cu:10-40
// DESIGN.md "Head layers for training" states the precision contract and the quirks kept.
//
// The three InnerProduct products are one GEMM shape, C[p, q] = sum_r A(p, r) * B(q, r):
//   forward  p = n, q = m, r = k   A = W (r-contiguous), B = X (r-contiguous)   Y[m, n] = C + b
//   dX       p = k, q = m, r = n   A = W (p-contiguous), B = dY (r-contiguous)  dX[m, k] = C
//   dW       p = n, q = k, r = m   A = dY (p-contiguous), B = X (q-contiguous)  dW[n, k] += C
// Every operand is read as fp32 from global memory by the CTA's own threads and split into
// (hi, lo) bf16 while it is staged: the tile is written reduction-major (64 bf16 = one 128-byte
// row per p or q, 128B swizzle), so one wgmma core (K-major descriptors) serves all three, and
// only the loader's thread-to-element map depends on which dimension is contiguous in memory.
// Per 16-wide k slice: lo*hi, hi*lo, hi*hi, fp32 accumulators in registers.
#include <cfloat>
#include <cstdint>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "mnc_b200.h"
#include "launch_util.h"
#include "ptx.cuh"
#include "sigmoid.cuh"

namespace mnc {
namespace {

// ------------------------------------------------------------------------------ GEMM tiling
constexpr int kFcP = 64;                      // rows of C per CTA (the wgmma M)
constexpr int kFcQ = 128;                     // columns of C per CTA: 64 per consumer warpgroup
constexpr int kFcR = 64;                      // reduction per stage: one 128-byte bf16 row
constexpr int kFcThreads = 256;               // two warpgroups: both load, each runs its 64 columns
constexpr int kFcAPlane = kFcP * kFcR * 2;    // one bf16 plane of the A tile: 8 KB
constexpr int kFcBPlane = kFcQ * kFcR * 2;    // 16 KB
constexpr int kFcStage = 2 * kFcAPlane + 2 * kFcBPlane;   // hi + lo of both: 48 KB
constexpr int kFcSmem = 2 * kFcStage + 1024;  // two stages + alignment: two CTAs per SM
constexpr int kFcSlots = 2 * 132;             // resident CTAs on an H100 SXM (132 SMs)
constexpr int kFcMaxSplit = 32;

// One GEMM operand: element (row, r) at ptr[row * ld + r] (r_contig) or ptr[r * ld + row].
struct FcOperand {
  const float* ptr;
  long long ld;
  int rows;
  int r_contig;
  int vec;          // r_contig, ld % 4 == 0 and ptr 16-byte aligned: float4 loads
};

enum FcEpi { kEpiStore = 0, kEpiAccumulate = 1 };

struct FcOut {
  float* ptr;
  long long sp, sq;     // C[p, q] -> ptr[p * sp + q * sq]
  const float* bias;    // forward: + bias[p] after the product; NULL: none
  int mode;             // FcEpi
};

__device__ __forceinline__ void fc_epilogue(const FcOut& o, int p, int q, float v) {
  float* d = o.ptr + p * o.sp + q * o.sq;
  if (o.mode == kEpiAccumulate) {
    *d = __fadd_rn(*d, v);
  } else {
    *d = o.bias ? __fadd_rn(v, o.bias[p]) : v;
  }
}

// Per-thread staging of a tile: kItems (row, 8-wide r chunk) items of 8 floats.
template <int kRows>
struct FcStaged {
  static constexpr int kItems = kRows * (kFcR / 8) / kFcThreads;
  float v[kItems][8];
};

// Item i of thread t: consecutive threads walk the contiguous dimension of the operand, so every
// load instruction of a warp is coalesced.
template <int kRows>
__device__ __forceinline__ void fc_item(const FcOperand& a, int i, int& row, int& chunk) {
  const int idx = threadIdx.x + i * kFcThreads;
  if (a.r_contig) {
    row = idx >> 3;
    chunk = idx & 7;
  } else {
    row = idx % kRows;
    chunk = idx / kRows;
  }
}

template <int kRows>
__device__ __forceinline__ void fc_load(const FcOperand& a, int row0, int r0, int R,
                                        FcStaged<kRows>& s) {
#pragma unroll
  for (int i = 0; i < FcStaged<kRows>::kItems; ++i) {
    int row, chunk;
    fc_item<kRows>(a, i, row, chunk);
    const int gr = row0 + row, gk = r0 + chunk * 8;
    if (gr < a.rows && a.vec && gk + 8 <= R) {
      const float4* src = reinterpret_cast<const float4*>(a.ptr + gr * a.ld + gk);
      const float4 x0 = __ldg(src), x1 = __ldg(src + 1);
      s.v[i][0] = x0.x; s.v[i][1] = x0.y; s.v[i][2] = x0.z; s.v[i][3] = x0.w;
      s.v[i][4] = x1.x; s.v[i][5] = x1.y; s.v[i][6] = x1.z; s.v[i][7] = x1.w;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const bool ok = gr < a.rows && gk + j < R;
        const long long off = a.r_contig ? gr * a.ld + (gk + j) : (gk + j) * a.ld + gr;
        s.v[i][j] = ok ? __ldg(a.ptr + off) : 0.f;
      }
    }
  }
}

__device__ __forceinline__ uint32_t pack_bf16(__nv_bfloat16 a, __nv_bfloat16 b) {
  return static_cast<uint32_t>(__bfloat16_as_ushort(a)) |
         (static_cast<uint32_t>(__bfloat16_as_ushort(b)) << 16);
}

// hi part of the split: rn_bf16(x), or toward zero where rounding to nearest would overflow to
// infinity (|x| above the largest bf16), so that a finite operand always has finite parts.
__device__ __forceinline__ __nv_bfloat16 split_hi(float x) {
  const __nv_bfloat16 h = __float2bfloat16_rn(x);
  return (__hisinf(h) && isfinite(x)) ? __float2bfloat16_rz(x) : h;
}

// Split each value into hi = split_hi(x), lo = rn_bf16(x - hi) and write both 16-byte chunks with
// the 128B swizzle of a K-major wgmma tile (chunk c of row w at w * 128 + ((c ^ (w & 7)) << 4)).
template <int kRows>
__device__ __forceinline__ void fc_store(const FcOperand& a, const FcStaged<kRows>& s,
                                         uint8_t* hi_plane, uint8_t* lo_plane) {
#pragma unroll
  for (int i = 0; i < FcStaged<kRows>::kItems; ++i) {
    int row, chunk;
    fc_item<kRows>(a, i, row, chunk);
    uint32_t hw[4], lw[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float x0 = s.v[i][2 * e], x1 = s.v[i][2 * e + 1];
      const __nv_bfloat16 h0 = split_hi(x0), h1 = split_hi(x1);
      const __nv_bfloat16 l0 = __float2bfloat16_rn(__fsub_rn(x0, __bfloat162float(h0)));
      const __nv_bfloat16 l1 = __float2bfloat16_rn(__fsub_rn(x1, __bfloat162float(h1)));
      hw[e] = pack_bf16(h0, h1);
      lw[e] = pack_bf16(l0, l1);
    }
    const int off = row * 128 + ((chunk ^ (row & 7)) << 4);
    *reinterpret_cast<uint4*>(hi_plane + off) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
    *reinterpret_cast<uint4*>(lo_plane + off) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
  }
}

// One CTA: a 64 x 128 tile of C over the k-steps [ks0, ks1) of the reduction.  splits == 1: the
// epilogue is applied in place; otherwise the partial goes to part[blockIdx.z][p][q] and
// fc_reduce_kernel applies it.  The loads of stage i + 1 are in flight while stage i's wgmma run.
__global__ void __launch_bounds__(kFcThreads, 2)
fc_gemm_kernel(const FcOperand A, const FcOperand B, int P, int Q, int R, int ksteps_per_split,
               const FcOut o, float* __restrict__ part) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  const int q0 = blockIdx.x * kFcQ, p0 = blockIdx.y * kFcP;
  const int ksteps = (R + kFcR - 1) / kFcR;
  const int ks0 = blockIdx.z * ksteps_per_split;
  const int ks1 = min(ksteps, ks0 + ksteps_per_split);
  const int wg = threadIdx.x >> 7;

  FcStaged<kFcP> sa;
  FcStaged<kFcQ> sb;
  auto stage_ptr = [&](int s) { return smem + s * kFcStage; };
  auto store = [&](int s) {
    uint8_t* st = stage_ptr(s);
    fc_store<kFcP>(A, sa, st, st + kFcAPlane);
    fc_store<kFcQ>(B, sb, st + 2 * kFcAPlane, st + 2 * kFcAPlane + kFcBPlane);
    ptx::fence_proxy_async();   // generic-proxy writes -> visible to the tensor core's async proxy
  };

  float acc[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) acc[j] = 0.f;

  fc_load<kFcP>(A, p0, ks0 * kFcR, R, sa);
  fc_load<kFcQ>(B, q0, ks0 * kFcR, R, sb);
  store(0);
  __syncthreads();
  for (int ks = ks0; ks < ks1; ++ks) {
    const int s = (ks - ks0) & 1;
    const bool more = ks + 1 < ks1;
    if (more) {
      fc_load<kFcP>(A, p0, (ks + 1) * kFcR, R, sa);
      fc_load<kFcQ>(B, q0, (ks + 1) * kFcR, R, sb);
    }
    const uint32_t a_hi = ptx::smem_u32(stage_ptr(s));
    const uint32_t a_lo = a_hi + kFcAPlane;
    const uint32_t b_hi = a_hi + 2 * kFcAPlane + wg * (kFcBPlane / 2);
    const uint32_t b_lo = b_hi + kFcBPlane;
    ptx::wgmma_fence_acc(acc);
    ptx::wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kFcR / 16; ++kk) {
      const uint64_t da_hi = ptx::wgmma_desc_rows<128>(a_hi + kk * 32);
      const uint64_t da_lo = ptx::wgmma_desc_rows<128>(a_lo + kk * 32);
      const uint64_t db_hi = ptx::wgmma_desc_rows<128>(b_hi + kk * 32);
      const uint64_t db_lo = ptx::wgmma_desc_rows<128>(b_lo + kk * 32);
      ptx::wgmma_bf16_n64(acc, da_lo, db_hi, (ks > ks0 || kk > 0) ? 1u : 0u);
      ptx::wgmma_bf16_n64(acc, da_hi, db_lo, 1u);
      ptx::wgmma_bf16_n64(acc, da_hi, db_hi, 1u);
    }
    ptx::wgmma_commit();
    if (more) store(s ^ 1);     // the other stage was read by the previous, completed, wgmma
    ptx::wgmma_wait_all();
    ptx::wgmma_fence_acc(acc);
    __syncthreads();
  }

  // acc[4j + 2h + e] = C[row 16 * warp + lane / 4 + 8h, column 8j + 2 * (lane % 4) + e]
  const int t = threadIdx.x & 127;
  const int pr = p0 + 16 * (t >> 5) + ((t & 31) >> 2);
  const int qc = q0 + wg * 64 + 2 * (t & 3);
  float* dst = part ? part + static_cast<long long>(blockIdx.z) * P * Q : nullptr;
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int p = pr + 8 * h, q = qc + 8 * j + e;
        if (p >= P || q >= Q) continue;
        const float v = acc[4 * j + 2 * h + e];
        if (dst)
          dst[static_cast<long long>(p) * Q + q] = v;
        else
          fc_epilogue(o, p, q, v);
      }
}

// Split-K partials added in split order, then the epilogue.
__global__ void __launch_bounds__(256)
fc_reduce_kernel(const float* __restrict__ part, int P, int Q, int splits, const FcOut o) {
  const long long n = static_cast<long long>(P) * Q;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * 256) {
    float v = part[i];
    for (int s = 1; s < splits; ++s) v = __fadd_rn(v, part[s * n + i]);
    fc_epilogue(o, static_cast<int>(i / Q), static_cast<int>(i % Q), v);
  }
}

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

SmemGrant g_fc_grant;

FcOperand operand(const float* p, long long ld, int rows, bool r_contig) {
  FcOperand a;
  a.ptr = p;
  a.ld = ld;
  a.rows = rows;
  a.r_contig = r_contig ? 1 : 0;
  a.vec = r_contig && ld % 4 == 0 && (reinterpret_cast<uintptr_t>(p) & 15) == 0;
  return a;
}

// k-steps per split: split-K only when the tiles cannot fill the resident CTA slots; then enough
// splits to fill them, at most kFcMaxSplit and never an empty one.
int split_steps(int P, int Q, int R) {
  const long long tiles = static_cast<long long>((P + kFcP - 1) / kFcP) * ((Q + kFcQ - 1) / kFcQ);
  const int ksteps = (R + kFcR - 1) / kFcR;
  if (tiles >= kFcSlots) return ksteps;
  long long s = (kFcSlots + tiles - 1) / tiles;
  if (s > kFcMaxSplit) s = kFcMaxSplit;
  if (s > ksteps) s = ksteps;
  return static_cast<int>((ksteps + s - 1) / s);
}

int split_k(int P, int Q, int R) {
  const int ksteps = (R + kFcR - 1) / kFcR;
  const int per = split_steps(P, Q, R);
  return (ksteps + per - 1) / per;
}

long long gemm_workspace(int P, int Q, int R) {
  const int s = split_k(P, Q, R);
  return s > 1 ? static_cast<long long>(s) * P * Q * sizeof(float) : 0;
}

int launch_gemm(const FcOperand& A, const FcOperand& B, int P, int Q, int R, const FcOut& o,
                void* workspace, long long workspace_bytes, cudaStream_t st) {
  int rc;
  if ((rc = ensure_dynamic_smem(fc_gemm_kernel, kFcSmem, g_fc_grant)) != MNC_OK) return rc;
  const int splits = split_k(P, Q, R);
  const int per = split_steps(P, Q, R);
  float* part = nullptr;
  if (splits > 1) {
    if (!workspace || workspace_bytes < gemm_workspace(P, Q, R)) return MNC_ERR_ARG;
    part = static_cast<float*>(workspace);
  }
  const dim3 grid((Q + kFcQ - 1) / kFcQ, (P + kFcP - 1) / kFcP, splits);
  if (grid.y > 65535) return MNC_ERR_ARG;
  fc_gemm_kernel<<<grid, kFcThreads, kFcSmem, st>>>(A, B, P, Q, R, per, o, part);
  if ((rc = check_launch()) != MNC_OK) return rc;
  if (splits > 1) {
    fc_reduce_kernel<<<grid_for(static_cast<long long>(P) * Q, 256, 4 * 132), 256, 0, st>>>(
        part, P, Q, splits, o);
    rc = check_launch();
  }
  return rc;
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
