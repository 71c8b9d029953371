// The split-bf16 tensor-core GEMM of the training layers (InnerProduct in fc_train.cu, Convolution in
// conv_train.cu), templated on how each operand is read from global memory:
//   C[p, q] = sum_r A(p, r) * B(q, r)
// Every operand is read as fp32 by the CTA's own threads and split into (hi, lo) bf16 while it is
// staged: the tile is written reduction-major (64 bf16 = one 128-byte row per p or q, 128B
// swizzle), so one wgmma core (K-major descriptors) serves every product, and only the operand's
// loader (its thread-to-element map and its addresses) depends on the layout in memory.
// Per 16-wide k slice: lo*hi, hi*lo, hi*hi, fp32 accumulators in registers.
//
// An operand type provides
//   template <int kRows> void item(int i, int& row, int& chunk) const   staging item i of a thread
//   template <int kRows> void load(int row0, int r0, int R, FcStaged<kRows>& s) const
// where load fills s.v[i][j] with element (row0 + row, r0 + 8 * chunk + j), zero outside the
// operand, for the (row, chunk) that item(i) gives.
#pragma once
#include <cstdint>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "mnc_b200.h"
#include "launch_util.h"
#include "ptx.cuh"

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

// Per-thread staging of a tile: kItems (row, 8-wide r chunk) items of 8 floats.
template <int kRows>
struct FcStaged {
  static constexpr int kItems = kRows * (kFcR / 8) / kFcThreads;
  float v[kItems][8];
};

// A dense operand: element (row, r) at ptr[row * ld + r] (r_contig) or ptr[r * ld + row].
struct FcOperand {
  const float* ptr;
  long long ld;
  int rows;
  int r_contig;
  int vec;          // r_contig, ld % 4 == 0 and ptr 16-byte aligned: float4 loads

  // Consecutive threads walk the contiguous dimension of the operand, so every load instruction
  // of a warp is coalesced.
  template <int kRows>
  __device__ __forceinline__ void item(int i, int& row, int& chunk) const {
    const int idx = threadIdx.x + i * kFcThreads;
    if (r_contig) {
      row = idx >> 3;
      chunk = idx & 7;
    } else {
      row = idx % kRows;
      chunk = idx / kRows;
    }
  }

  template <int kRows>
  __device__ __forceinline__ void load(int row0, int r0, int R, FcStaged<kRows>& s) const {
#pragma unroll
    for (int i = 0; i < FcStaged<kRows>::kItems; ++i) {
      int row, chunk;
      item<kRows>(i, row, chunk);
      const int gr = row0 + row, gk = r0 + chunk * 8;
      if (gr < rows && vec && gk + 8 <= R) {
        const float4* src = reinterpret_cast<const float4*>(ptr + gr * ld + gk);
        const float4 x0 = __ldg(src), x1 = __ldg(src + 1);
        s.v[i][0] = x0.x; s.v[i][1] = x0.y; s.v[i][2] = x0.z; s.v[i][3] = x0.w;
        s.v[i][4] = x1.x; s.v[i][5] = x1.y; s.v[i][6] = x1.z; s.v[i][7] = x1.w;
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const bool ok = gr < rows && gk + j < R;
          const long long off = r_contig ? gr * ld + (gk + j) : (gk + j) * ld + gr;
          s.v[i][j] = ok ? __ldg(ptr + off) : 0.f;
        }
      }
    }
  }
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
template <int kRows, class Op>
__device__ __forceinline__ void fc_store(const Op& a, const FcStaged<kRows>& s,
                                         uint8_t* hi_plane, uint8_t* lo_plane) {
#pragma unroll
  for (int i = 0; i < FcStaged<kRows>::kItems; ++i) {
    int row, chunk;
    a.template item<kRows>(i, row, chunk);
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
template <class OpA, class OpB>
__global__ void __launch_bounds__(kFcThreads, 2)
fc_gemm_kernel(const OpA A, const OpB B, int P, int Q, int R, int ksteps_per_split,
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

  A.template load<kFcP>(p0, ks0 * kFcR, R, sa);
  B.template load<kFcQ>(q0, ks0 * kFcR, R, sb);
  store(0);
  __syncthreads();
  for (int ks = ks0; ks < ks1; ++ks) {
    const int s = (ks - ks0) & 1;
    const bool more = ks + 1 < ks1;
    if (more) {
      A.template load<kFcP>(p0, (ks + 1) * kFcR, R, sa);
      B.template load<kFcQ>(q0, (ks + 1) * kFcR, R, sb);
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

// One shared-memory opt-in record per kernel instantiation.
template <class OpA, class OpB>
SmemGrant& gemm_grant() {
  static SmemGrant g;
  return g;
}

template <class OpA, class OpB>
int launch_gemm(const OpA& A, const OpB& B, int P, int Q, int R, const FcOut& o,
                void* workspace, long long workspace_bytes, cudaStream_t st) {
  int rc;
  if ((rc = ensure_dynamic_smem(fc_gemm_kernel<OpA, OpB>, kFcSmem, gemm_grant<OpA, OpB>())) != MNC_OK)
    return rc;
  const int splits = split_k(P, Q, R);
  const int per = split_steps(P, Q, R);
  float* part = nullptr;
  if (splits > 1) {
    if (!workspace || workspace_bytes < gemm_workspace(P, Q, R)) return MNC_ERR_ARG;
    part = static_cast<float*>(workspace);
  }
  const dim3 grid((Q + kFcQ - 1) / kFcQ, (P + kFcP - 1) / kFcP, splits);
  if (grid.y > 65535) return MNC_ERR_ARG;
  fc_gemm_kernel<OpA, OpB><<<grid, kFcThreads, kFcSmem, st>>>(A, B, P, Q, R, per, o, part);
  if ((rc = check_launch()) != MNC_OK) return rc;
  if (splits > 1) {
    fc_reduce_kernel<<<grid_for(static_cast<long long>(P) * Q, 256, 4 * 132), 256, 0, st>>>(
        part, P, Q, splits, o);
    rc = check_launch();
  }
  return rc;
}

}  // namespace
}  // namespace mnc
