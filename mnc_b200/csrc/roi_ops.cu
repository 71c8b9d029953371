// RoI warping, mask resize and mask pooling.
//
// Replaces the three MNC Caffe layers' Forward_gpu:
//   ROIWarping   caffe-mnc/src/caffe/layers/roi_warping_layer.cu:67-107 (+ bilinear :18-64)
//   MaskResize   caffe-mnc/src/caffe/layers/mask_resize_layer.cu:57-73  (+ bilinear :13-54)
//   MaskPooling  caffe-mnc/src/caffe/layers/mask_pooling_layer.cu:13-26
// in two forms:
//   *_nchw  : the layer contract itself (fp32 NCHW blobs in and out) -- what the ROIWarpingLayer /
//             MaskResizeLayer / MaskPoolingLayer host mirrors call and what the HBM microbench
//             (BASELINE.json config 4) times.  One CTA per (RoI, channel slab); the interpolation
//             taps are built once per RoI.  ROIWarping at 28x28 and 14x14 walks the sample rows with
//             the two live feature rows in registers (roi_warp_rowwalk_kernel), other sizes gather
//             the four taps of each output through L1.  Every output element is written exactly once
//             with coalesced streaming stores (the reference writes 3x the bytes: top + argmax_h +
//             argmax_w).
//   *_split : the fused forms the batched engine uses on split-bf16 NHWC activations: warp (+ the
//             2x2 max pool of test.prototxt:494-505) straight to the 14x14 grid and the 7x7 box
//             pool in one pass, never materialising the (R,512,28,28) tensor; mask pooling fused
//             with its 2x2 pool.
// The bilinear arithmetic uses explicit round-to-nearest mul/add in the reference's operation order
// (weights first, then a left-to-right sum), so fp32 results equal the C oracle's bit for bit.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <cstdint>

#include "mnc_b200.h"
#include "roi_geom.cuh"
#include "tri.cuh"

namespace mnc {

__device__ __forceinline__ float bilerp(const AxisTap& th, const AxisTap& tw, float v1, float v2,
                                        float v3, float v4) {
  const float w1 = __fmul_rn(th.h, tw.h), w2 = __fmul_rn(th.h, tw.l);
  const float w3 = __fmul_rn(th.l, tw.h), w4 = __fmul_rn(th.l, tw.l);
  float val = __fmul_rn(w1, v1);
  val = __fadd_rn(val, __fmul_rn(w2, v2));
  val = __fadd_rn(val, __fmul_rn(w3, v3));
  val = __fadd_rn(val, __fmul_rn(w4, v4));
  return val;
}

// ------------------------------------------------------------------------ ROIWarping, NCHW fp32
constexpr int kWarpSlab = 16;    // channels per CTA

// One CTA per (RoI, 16-channel slab).  The per-RoI interpolation tables (row taps, column taps)
// are built once in shared memory; each thread then fixes EPT consecutive outputs of the P x P
// plane and keeps, in registers, their four gather offsets and four bilinear weights (weights
// formed first, as roi_warping_layer.cu:56 does).  The channel loop is then 4 read-only gathers
// (a RoI's window of one channel is <= 9.6 KB, L1-resident after first touch) + 7 un-fused fp32
// ops per output and one vector streaming store per EPT outputs: ~13 instructions per output
// instead of ~50 when offsets and weights are recomputed per element.
// Output bytes are written exactly once, coalesced (the reference also writes argmax_h/argmax_w).
template <int PH, int PW, int EPT>
__global__ void __launch_bounds__(256)
roi_warp_nchw_kernel(const float* __restrict__ feat, int C, int H, int W,
                     const float* __restrict__ rois, float spatial_scale,
                     float* __restrict__ out) {
  constexpr int PP = PH * PW;
  static_assert(PP % EPT == 0, "plane must split into whole vectors");
  constexpr int TPC = PP / EPT;         // threads per channel plane
  constexpr int CLN = 256 / TPC > 0 ? 256 / TPC : 1;  // channel lanes per CTA
  __shared__ AxisTap tap_h[PH], tap_w[PW];
  const int r = blockIdx.x;
  const int c0 = blockIdx.y * kWarpSlab;
  const int tid = threadIdx.x;
  const RoiGeom g = roi_geom(rois + static_cast<long long>(r) * 5, spatial_scale, PH, PW);
  if (tid < PH) tap_h[tid] = axis_tap(__fadd_rn(g.start_h, __fmul_rn(static_cast<float>(tid), g.bin_h)), H);
  if (tid >= 32 && tid < 32 + PW)
    tap_w[tid - 32] = axis_tap(__fadd_rn(g.start_w, __fmul_rn(static_cast<float>(tid - 32), g.bin_w)), W);
  __syncthreads();
  const int q = tid % TPC, cl = tid / TPC;
  if (cl >= CLN) return;
  int off[EPT][4];
  float wgt[EPT][4];
  bool ok[EPT];
#pragma unroll
  for (int e = 0; e < EPT; ++e) {
    const int i = q * EPT + e;
    const int ph = i / PW, pw = i - ph * PW;
    const AxisTap th = tap_h[ph], tw = tap_w[pw];
    ok[e] = th.ok && tw.ok;
    off[e][0] = ok[e] ? th.lo * W + tw.lo : 0;
    off[e][1] = ok[e] ? th.lo * W + tw.hi : 0;
    off[e][2] = ok[e] ? th.hi * W + tw.lo : 0;
    off[e][3] = ok[e] ? th.hi * W + tw.hi : 0;
    wgt[e][0] = __fmul_rn(th.h, tw.h);
    wgt[e][1] = __fmul_rn(th.h, tw.l);
    wgt[e][2] = __fmul_rn(th.l, tw.h);
    wgt[e][3] = __fmul_rn(th.l, tw.l);
  }
  const int nch = min(kWarpSlab, C - c0);
  const int HW = H * W;
  const float* fbase = feat + (static_cast<long long>(g.level) * C + c0) * HW;
  float* obase = out + (static_cast<long long>(r) * C + c0) * PP + q * EPT;
  const bool aligned = (reinterpret_cast<uintptr_t>(obase) & (EPT * 4 - 1)) == 0 && (PP % EPT == 0);
#pragma unroll 2
  for (int c = cl; c < nch; c += CLN) {
    const float* plane = fbase + static_cast<long long>(c) * HW;
    float v[EPT];
#pragma unroll
    for (int e = 0; e < EPT; ++e) {
      const float v1 = __ldg(plane + off[e][0]), v2 = __ldg(plane + off[e][1]);
      const float v3 = __ldg(plane + off[e][2]), v4 = __ldg(plane + off[e][3]);
      float val = __fmul_rn(wgt[e][0], v1);
      val = __fadd_rn(val, __fmul_rn(wgt[e][1], v2));
      val = __fadd_rn(val, __fmul_rn(wgt[e][2], v3));
      val = __fadd_rn(val, __fmul_rn(wgt[e][3], v4));
      v[e] = ok[e] ? val : 0.f;
    }
    float* o = obase + c * PP;
    if (EPT == 4 && aligned) {
      __stcs(reinterpret_cast<float4*>(o), make_float4(v[0], v[EPT > 1 ? 1 : 0], v[EPT > 2 ? 2 : 0], v[EPT > 3 ? 3 : 0]));
    } else if (EPT == 2 && aligned) {
      __stcs(reinterpret_cast<float2*>(o), make_float2(v[0], v[EPT > 1 ? 1 : 0]));
    } else {
#pragma unroll
      for (int e = 0; e < EPT; ++e) __stcs(o + e, v[e]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// ROIWarping by ROW WALK: a warp owns one output plane (RoI, channel); lane = output column pw, and
// the warp walks the P sample rows top to bottom.  The four taps of (ph, pw) are (row lo / hi) x
// (column lo / hi); consecutive sample rows advance by bin_h < 1.4 feature rows, so the two feature
// rows a lane needs are kept in registers and re-read only when the row taps move on -- ~2 loads
// per new feature row instead of 4 per output: 1.5 loads per output for a typical proposal, and
// each load is one coalesced row segment (lanes = neighbouring columns).  Control flow depends only
// on the RoI: the warp never diverges.  The value formula is unchanged (weights first, products
// summed left to right, no FMA): bit-exact with the reference built with -fmad=false.
// Stores: one 4 x P byte row segment per sample row, consecutive rows contiguous (whole plane
// written once, streaming).  P = 14 packs two planes into one warp (lanes 0-13 and 16-29).
template <int P>
__global__ void __launch_bounds__(256)
roi_warp_rowwalk_kernel(const float* __restrict__ feat, int C, int H, int W,
                        const float* __restrict__ rois, float spatial_scale, int ch_per_cta,
                        float* __restrict__ out) {
  constexpr int CH = (P > 16) ? 8 : 4;            // planes walked together by one lane (ILP; the
                                                  // row bookkeeping and the 4 weights are shared)
  constexpr int PP = P * P;
  constexpr int PPW = (P <= 16) ? 2 : 1;          // plane groups per warp
  __shared__ int4 tap_hq[P];                      // {lo (or -1: out of range), hi, bits(h), bits(l)}
  const int r = blockIdx.x;
  const int cbase = blockIdx.y * ch_per_cta;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const RoiGeom g = roi_geom(rois + static_cast<long long>(r) * 5, spatial_scale, P, P);
  if (tid < P) {
    const AxisTap t = axis_tap(__fadd_rn(g.start_h, __fmul_rn(static_cast<float>(tid), g.bin_h)), H);
    tap_hq[tid] = make_int4(t.ok ? t.lo : -1, t.hi, __float_as_int(t.h), __float_as_int(t.l));
  }
  const int sub = (PPW == 2) ? (lane >> 4) : 0;     // which plane group of the warp
  const int pw = (PPW == 2) ? (lane & 15) : lane;
  const bool live = pw < P;
  const AxisTap tw = axis_tap(__fadd_rn(g.start_w, __fmul_rn(static_cast<float>(live ? pw : 0), g.bin_w)), W);
  __syncthreads();
  const int HW = H * W;
  const int nch = min(ch_per_cta, C - cbase);
  const int nwarps = blockDim.x >> 5;
  for (int c = (warp * PPW + sub) * CH; c < nch; c += nwarps * PPW * CH) {
    const float* plane = feat + (static_cast<long long>(g.level) * C + cbase + c) * HW;
    float* o = out + (static_cast<long long>(r) * C + cbase + c) * PP + pw;
    int koff[CH];                                   // plane offsets (a channel tail re-reads plane 0)
#pragma unroll
    for (int k = 0; k < CH; ++k) koff[k] = (c + k < nch ? k : 0) * HW;
    int cur_lo = -1, cur_hi = -1;
    float a_lo[CH], a_hi[CH], b_lo[CH], b_hi[CH];   // rows cur_lo / cur_hi at columns lo / hi
#pragma unroll
    for (int k = 0; k < CH; ++k) a_lo[k] = a_hi[k] = b_lo[k] = b_hi[k] = 0.f;
#pragma unroll 2
    for (int ph = 0; ph < P; ++ph) {
      const int4 tq = tap_hq[ph];
      float val[CH];
#pragma unroll
      for (int k = 0; k < CH; ++k) val[k] = 0.f;
      if (tq.x >= 0) {
        if (tq.x != cur_lo) {
          if (tq.x == cur_hi) {
#pragma unroll
            for (int k = 0; k < CH; ++k) { a_lo[k] = b_lo[k]; a_hi[k] = b_hi[k]; }
          } else {
#pragma unroll
            for (int k = 0; k < CH; ++k) {
              a_lo[k] = __ldg(plane + koff[k] + tq.x * W + tw.lo);
              a_hi[k] = __ldg(plane + koff[k] + tq.x * W + tw.hi);
            }
          }
          cur_lo = tq.x;
          cur_hi = -1;
        }
        if (tq.y != cur_hi) {
          if (tq.y == tq.x) {
#pragma unroll
            for (int k = 0; k < CH; ++k) { b_lo[k] = a_lo[k]; b_hi[k] = a_hi[k]; }
          } else {
#pragma unroll
            for (int k = 0; k < CH; ++k) {
              b_lo[k] = __ldg(plane + koff[k] + tq.y * W + tw.lo);
              b_hi[k] = __ldg(plane + koff[k] + tq.y * W + tw.hi);
            }
          }
          cur_hi = tq.y;
        }
        const float th_h = __int_as_float(tq.z), th_l = __int_as_float(tq.w);
        const float w1 = __fmul_rn(th_h, tw.h), w2 = __fmul_rn(th_h, tw.l);
        const float w3 = __fmul_rn(th_l, tw.h), w4 = __fmul_rn(th_l, tw.l);
#pragma unroll
        for (int k = 0; k < CH; ++k) {
          float v = __fmul_rn(w1, a_lo[k]);
          v = __fadd_rn(v, __fmul_rn(w2, a_hi[k]));
          v = __fadd_rn(v, __fmul_rn(w3, b_lo[k]));
          v = __fadd_rn(v, __fmul_rn(w4, b_hi[k]));
          val[k] = tw.ok ? v : 0.f;
        }
      }
      if (live) {
#pragma unroll
        for (int k = 0; k < CH; ++k)
          if (c + k < nch) __stcs(o + k * PP + ph * P, val[k]);
      }
    }
  }
}

// generic pooled size (runtime), same scheme, scalar stores
__global__ void __launch_bounds__(256)
roi_warp_nchw_generic_kernel(const float* __restrict__ feat, int C, int H, int W,
                             const float* __restrict__ rois, int ph_n, int pw_n,
                             float spatial_scale, float* __restrict__ out) {
  __shared__ AxisTap tap_h[kMaxPooled], tap_w[kMaxPooled];
  const int r = blockIdx.x;
  const int c0 = blockIdx.y * kWarpSlab;
  const int tid = threadIdx.x;
  const RoiGeom g = roi_geom(rois + static_cast<long long>(r) * 5, spatial_scale, ph_n, pw_n);
  if (tid < ph_n) tap_h[tid] = axis_tap(__fadd_rn(g.start_h, __fmul_rn(static_cast<float>(tid), g.bin_h)), H);
  if (tid >= 32 && tid < 32 + pw_n)
    tap_w[tid - 32] = axis_tap(__fadd_rn(g.start_w, __fmul_rn(static_cast<float>(tid - 32), g.bin_w)), W);
  __syncthreads();
  const int pp = ph_n * pw_n;
  const int nch = min(kWarpSlab, C - c0);
  const float* fbase = feat + (static_cast<long long>(g.level) * C + c0) * H * W;
  float* obase = out + (static_cast<long long>(r) * C + c0) * pp;
  for (int i = tid; i < nch * pp; i += 256) {
    const int c = i / pp, rem = i % pp;
    const int ph = rem / pw_n, pw = rem % pw_n;
    const AxisTap th = tap_h[ph], tw = tap_w[pw];
    float val = 0.f;
    if (th.ok && tw.ok) {
      const float* pl = fbase + static_cast<long long>(c) * H * W;
      val = bilerp(th, tw, __ldg(pl + th.lo * W + tw.lo), __ldg(pl + th.lo * W + tw.hi),
                   __ldg(pl + th.hi * W + tw.lo), __ldg(pl + th.hi * W + tw.hi));
    }
    obase[i] = val;
  }
}

// -------------------------------------------------------------- MaskResize / MaskPooling, NCHW
__global__ void mask_resize_nchw_kernel(const float* __restrict__ in, int planes, int ih_n,
                                        int iw_n, int oh_n, int ow_n, float* __restrict__ out) {
  const long long total = static_cast<long long>(planes) * oh_n * ow_n;
  const float ratio_h = __fdiv_rn(static_cast<float>(ih_n), static_cast<float>(oh_n));
  const float ratio_w = __fdiv_rn(static_cast<float>(iw_n), static_cast<float>(ow_n));
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int w = static_cast<int>(i % ow_n);
    const int h = static_cast<int>((i / ow_n) % oh_n);
    const long long p = i / (static_cast<long long>(ow_n) * oh_n);
    const AxisTap th = axis_tap(__fmul_rn(static_cast<float>(h), ratio_h), ih_n);
    const AxisTap tw = axis_tap(__fmul_rn(static_cast<float>(w), ratio_w), iw_n);
    float val = 0.f;
    if (th.ok && tw.ok) {
      const float* b = in + p * ih_n * iw_n;
      val = bilerp(th, tw, b[th.lo * iw_n + tw.lo], b[th.lo * iw_n + tw.hi],
                   b[th.hi * iw_n + tw.lo], b[th.hi * iw_n + tw.hi]);
    }
    out[i] = val;
  }
}

// top[n,c,h,w] = feat[n,c,h,w] * mask[n,0,h,w]; 16-byte streaming loads/stores when hw % 4 == 0.
__global__ void mask_pool_nchw_kernel(const float* __restrict__ feat,
                                      const float* __restrict__ mask, int N, int C, int hw,
                                      float* __restrict__ out) {
  const long long total4 = static_cast<long long>(N) * C * hw / 4;
  const int hw4 = hw / 4;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int q = static_cast<int>(i % hw4);
    const long long n = i / (static_cast<long long>(hw4) * C);
    const float4 f = __ldcs(reinterpret_cast<const float4*>(feat) + i);
    const float4 m = __ldg(reinterpret_cast<const float4*>(mask) + n * hw4 + q);
    __stcs(reinterpret_cast<float4*>(out) + i,
           make_float4(__fmul_rn(f.x, m.x), __fmul_rn(f.y, m.y), __fmul_rn(f.z, m.z),
                       __fmul_rn(f.w, m.w)));
  }
}
__global__ void mask_pool_nchw_scalar_kernel(const float* __restrict__ feat,
                                             const float* __restrict__ mask, int N, int C, int hw,
                                             float* __restrict__ out) {
  const long long total = static_cast<long long>(N) * C * hw;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int q = static_cast<int>(i % hw);
    const long long n = i / (static_cast<long long>(hw) * C);
    out[i] = __fmul_rn(feat[i], mask[n * hw + q]);
  }
}

// ------------------------------------------------------------ fused forms on split-bf16 NHWC
__device__ __forceinline__ float2 ld_split2(const __nv_bfloat16* hi, const __nv_bfloat16* lo,
                                            long long off) {
  const uint32_t h = __ldg(reinterpret_cast<const uint32_t*>(hi + off));
  const uint32_t l = __ldg(reinterpret_cast<const uint32_t*>(lo + off));
  float2 r;
  r.x = __uint_as_float(h << 16) + __uint_as_float(l << 16);
  r.y = __uint_as_float(h & 0xffff0000u) + __uint_as_float(l & 0xffff0000u);
  return r;
}
__device__ __forceinline__ void st_split2(__nv_bfloat16* hi, __nv_bfloat16* lo, long long off,
                                          float a, float b) {
  const __nv_bfloat16 ha = __float2bfloat16_rn(a), hb = __float2bfloat16_rn(b);
  const __nv_bfloat16 la = __float2bfloat16_rn(a - __bfloat162float(ha));
  const __nv_bfloat16 lb = __float2bfloat16_rn(b - __bfloat162float(hb));
  *reinterpret_cast<uint32_t*>(hi + off) =
      static_cast<uint32_t>(__bfloat16_as_ushort(ha)) | (static_cast<uint32_t>(__bfloat16_as_ushort(hb)) << 16);
  *reinterpret_cast<uint32_t*>(lo + off) =
      static_cast<uint32_t>(__bfloat16_as_ushort(la)) | (static_cast<uint32_t>(__bfloat16_as_ushort(lb)) << 16);
}

// One CTA per (RoI, pair of 14x14 output rows).  SUB = 2: warp to 28x28 and take the 2x2 max
// (stage 1, test.prototxt:479-505); SUB = 1: warp straight to 14x14 (stage 2, :809-820).
// Also emits the 7x7 box-branch pool (test.prototxt:571-582).
// The interpolation taps depend only on (RoI, sample row/col): they are computed once per CTA
// into shared memory (2*SUB row taps, 14*SUB column taps).  Threads then run over
// (cell column, 4-channel group): 8-byte loads from each bf16 plane, coalesced along channels.
struct __align__(8) bf4 { uint32_t a, b; };
__device__ __forceinline__ float4 ld_split4(const __nv_bfloat16* hi, const __nv_bfloat16* lo,
                                            long long off) {
  const uint2 h = __ldg(reinterpret_cast<const uint2*>(hi + off));
  const uint2 l = __ldg(reinterpret_cast<const uint2*>(lo + off));
  float4 r;
  r.x = __uint_as_float(h.x << 16) + __uint_as_float(l.x << 16);
  r.y = __uint_as_float(h.x & 0xffff0000u) + __uint_as_float(l.x & 0xffff0000u);
  r.z = __uint_as_float(h.y << 16) + __uint_as_float(l.y << 16);
  r.w = __uint_as_float(h.y & 0xffff0000u) + __uint_as_float(l.y & 0xffff0000u);
  return r;
}
__device__ __forceinline__ uint32_t pack_bf2(__nv_bfloat16 a, __nv_bfloat16 b) {
  return static_cast<uint32_t>(__bfloat16_as_ushort(a)) | (static_cast<uint32_t>(__bfloat16_as_ushort(b)) << 16);
}
__device__ __forceinline__ void st_split4(__nv_bfloat16* hi, __nv_bfloat16* lo, long long off,
                                          const float4 v) {
  const __nv_bfloat16 h0 = __float2bfloat16_rn(v.x), h1 = __float2bfloat16_rn(v.y);
  const __nv_bfloat16 h2 = __float2bfloat16_rn(v.z), h3 = __float2bfloat16_rn(v.w);
  const __nv_bfloat16 l0 = __float2bfloat16_rn(v.x - __bfloat162float(h0));
  const __nv_bfloat16 l1 = __float2bfloat16_rn(v.y - __bfloat162float(h1));
  const __nv_bfloat16 l2 = __float2bfloat16_rn(v.z - __bfloat162float(h2));
  const __nv_bfloat16 l3 = __float2bfloat16_rn(v.w - __bfloat162float(h3));
  // streaming stores: the RoI feature tensors (~1.2 GB per stage) are consumed once by the next
  // GEMM and must not evict conv5_3 (39 MB, re-read by every RoI) from L2
  __stcs(reinterpret_cast<uint2*>(hi + off), make_uint2(pack_bf2(h0, h1), pack_bf2(h2, h3)));
  __stcs(reinterpret_cast<uint2*>(lo + off), make_uint2(pack_bf2(l0, l1), pack_bf2(l2, l3)));
}
// fused-path bilinear: same weights-first formula, evaluated with FMAs (the fused outputs are
// re-quantised to split-bf16 and compared at tolerance; the bit-exact form lives in bilerp()).
__device__ __forceinline__ float4 bilerp4(const float w1, const float w2, const float w3,
                                          const float w4, const float4 v1, const float4 v2,
                                          const float4 v3, const float4 v4) {
  float4 r;
  r.x = fmaf(w4, v4.x, fmaf(w3, v3.x, fmaf(w2, v2.x, w1 * v1.x)));
  r.y = fmaf(w4, v4.y, fmaf(w3, v3.y, fmaf(w2, v2.y, w1 * v1.y)));
  r.z = fmaf(w4, v4.z, fmaf(w3, v3.z, fmaf(w2, v2.z, w1 * v1.z)));
  r.w = fmaf(w4, v4.w, fmaf(w3, v3.w, fmaf(w2, v2.w, w1 * v1.w)));
  return r;
}
__device__ __forceinline__ float4 max4(const float4 a, const float4 b) {
  return make_float4(fmaxf(a.x, b.x), fmaxf(a.y, b.y), fmaxf(a.z, b.z), fmaxf(a.w, b.w));
}

// Work item = (pooled column jp, channel quad).  Everything that depends only on the sample
// position -- the four gather offsets and the four bilinear weights (weights formed first,
// roi_warping_layer.cu:56) -- is computed once per CTA into a shared-memory table (2*SUB sample
// rows x 14*SUB sample columns, 32 B per sample) and read back with two broadcast 128-bit loads.
// The feature map is read as fp32 NHWC (the engine keeps an fp32 copy of conv5_3 = hi + lo, 39 MB
// per batch of 8, so the gathers need no bf16 unpacking): one 16-byte load per tap and quad.
struct __align__(16) SampleTab {
  int off[4];    // element offsets of the 4 taps within the image (channel 0)
  float w[4];    // bilinear weights; all four are 0 for an out-of-range sample
};

// output planes of the fused RoI kernels: split-bf16 (hi, lo) or tri-plane (h, l, c; scale 2^exp)
struct RoiOut {
  void* p14[3];
  void* p7[3];
  float scale;
};
template <bool TRI>
__device__ __forceinline__ void st_feat4(void* const (&pl)[3], long long off, const float4 v, float scale) {
  if (TRI)
    st_tri4(static_cast<__half*>(pl[0]), static_cast<uint8_t*>(pl[1]), static_cast<uint8_t*>(pl[2]), off, v, scale);
  else
    st_split4(static_cast<__nv_bfloat16*>(pl[0]), static_cast<__nv_bfloat16*>(pl[1]), off, v);
}

template <int SUB, bool TRI>
__global__ void __launch_bounds__(256, 4)
roi_warp_split_kernel(const float* __restrict__ feat, int C, int H, int W,
                      const float* __restrict__ rois, float spatial_scale, const RoiOut o) {
  constexpr int P = 14 * SUB;
  constexpr int NS = 2 * SUB * P;  // samples handled by this CTA
  __shared__ SampleTab tab[NS];
  const int r = blockIdx.x;
  const int t = blockIdx.y;  // rows 2t, 2t+1 of the 14x14 grid
  const RoiGeom g = roi_geom(rois + static_cast<long long>(r) * 5, spatial_scale, P, P);
  for (int i = threadIdx.x; i < NS; i += blockDim.x) {
    const int sr = i / P, pw = i - sr * P;
    const int ph = 2 * t * SUB + sr;
    const AxisTap th = axis_tap(__fadd_rn(g.start_h, __fmul_rn(static_cast<float>(ph), g.bin_h)), H);
    const AxisTap tw = axis_tap(__fadd_rn(g.start_w, __fmul_rn(static_cast<float>(pw), g.bin_w)), W);
    const bool ok = th.ok && tw.ok;
    SampleTab e;
    e.off[0] = ok ? (th.lo * W + tw.lo) * C : 0;
    e.off[1] = ok ? (th.lo * W + tw.hi) * C : 0;
    e.off[2] = ok ? (th.hi * W + tw.lo) * C : 0;
    e.off[3] = ok ? (th.hi * W + tw.hi) * C : 0;
    e.w[0] = ok ? __fmul_rn(th.h, tw.h) : 0.f;
    e.w[1] = ok ? __fmul_rn(th.h, tw.l) : 0.f;
    e.w[2] = ok ? __fmul_rn(th.l, tw.h) : 0.f;
    e.w[3] = ok ? __fmul_rn(th.l, tw.l) : 0.f;
    tab[i] = e;
  }
  __syncthreads();
  const float* fimg = feat + static_cast<long long>(g.level) * H * W * C;
  const int c4n = C / 4;
  const float kNeg = -3.402823466e+38f;
  for (int item = threadIdx.x; item < 7 * c4n; item += blockDim.x) {
    const int jp = item / c4n;
    const int c = (item - jp * c4n) * 4;
    const float* fc = fimg + c;
    float4 best7 = make_float4(kNeg, kNeg, kNeg, kNeg);
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const int j = 2 * jp + dx;
        float4 cell = make_float4(kNeg, kNeg, kNeg, kNeg);
#pragma unroll
        for (int sy = 0; sy < SUB; ++sy) {
#pragma unroll
          for (int sx = 0; sx < SUB; ++sx) {
            const SampleTab& e = tab[(dy * SUB + sy) * P + j * SUB + sx];
            const int4 of = *reinterpret_cast<const int4*>(e.off);
            const float4 wg = *reinterpret_cast<const float4*>(e.w);
            const float4 v1 = __ldg(reinterpret_cast<const float4*>(fc + of.x));
            const float4 v2 = __ldg(reinterpret_cast<const float4*>(fc + of.y));
            const float4 v3 = __ldg(reinterpret_cast<const float4*>(fc + of.z));
            const float4 v4 = __ldg(reinterpret_cast<const float4*>(fc + of.w));
            cell = max4(cell, bilerp4(wg.x, wg.y, wg.z, wg.w, v1, v2, v3, v4));
          }
        }
        st_feat4<TRI>(o.p14, ((static_cast<long long>(r) * 14 + (2 * t + dy)) * 14 + j) * C + c, cell, o.scale);
        best7 = max4(best7, cell);
      }
    }
    st_feat4<TRI>(o.p7, ((static_cast<long long>(r) * 7 + t) * 7 + jp) * C + c, best7, o.scale);
  }
}


// ------------------------------------------------------------------------------------------------
// Sibling test graphs (SURVEY.md section 8f row 4).
//   ROIPooling  caffe-mnc/src/caffe/layers/roi_pooling_layer.cu:17-77 (Fast R-CNN max over integer
//               bins; CFM test net, models/VGG16/cfm/test.prototxt:399-465)
//   ROIWarping at 7x7 straight into fc6 (Faster R-CNN test net,
//               models/VGG16/faster_rcnn_end2end/test.prototxt:479-490)
struct PoolBin {
  int h0, h1, w0, w1;
};

// roi_pooling_layer.cu:29-57 for pooled cell (ph, pw)
__device__ __forceinline__ PoolBin roi_pool_bin(const float* roi, float spatial_scale, int H, int W,
                                                int PH, int PW, int ph, int pw) {
  const int sw = static_cast<int>(roundf(__fmul_rn(roi[1], spatial_scale)));
  const int sh = static_cast<int>(roundf(__fmul_rn(roi[2], spatial_scale)));
  const int ew = static_cast<int>(roundf(__fmul_rn(roi[3], spatial_scale)));
  const int eh = static_cast<int>(roundf(__fmul_rn(roi[4], spatial_scale)));
  const int rw = max(ew - sw + 1, 1), rh = max(eh - sh + 1, 1);
  const float bh = __fdiv_rn(static_cast<float>(rh), static_cast<float>(PH));
  const float bw = __fdiv_rn(static_cast<float>(rw), static_cast<float>(PW));
  PoolBin b;
  b.h0 = static_cast<int>(floorf(__fmul_rn(static_cast<float>(ph), bh)));
  b.w0 = static_cast<int>(floorf(__fmul_rn(static_cast<float>(pw), bw)));
  b.h1 = static_cast<int>(ceilf(__fmul_rn(static_cast<float>(ph + 1), bh)));
  b.w1 = static_cast<int>(ceilf(__fmul_rn(static_cast<float>(pw + 1), bw)));
  b.h0 = min(max(b.h0 + sh, 0), H);
  b.h1 = min(max(b.h1 + sh, 0), H);
  b.w0 = min(max(b.w0 + sw, 0), W);
  b.w1 = min(max(b.w1 + sw, 0), W);
  return b;
}

// Layer contract: fp32 NCHW in and out (+ optional argmax, which the reference always writes).
// grid (R, ceil(C/16)); the RoI's PH*PW bins are computed once per CTA into shared memory.
__global__ void __launch_bounds__(256)
roi_pool_nchw_kernel(const float* __restrict__ feat, int C, int H, int W,
                     const float* __restrict__ rois, float spatial_scale, int PH, int PW,
                     float* __restrict__ out, int* __restrict__ argmax) {
  extern __shared__ PoolBin bins[];
  const int r = blockIdx.x;
  const int c0 = blockIdx.y * kWarpSlab;
  const float* roi = rois + static_cast<long long>(r) * 5;
  const int PP = PH * PW;
  for (int i = threadIdx.x; i < PP; i += blockDim.x)
    bins[i] = roi_pool_bin(roi, spatial_scale, H, W, PH, PW, i / PW, i % PW);
  __syncthreads();
  const int level = static_cast<int>(roi[0]);
  const int nc = min(kWarpSlab, C - c0);
  for (int i = threadIdx.x; i < nc * PP; i += blockDim.x) {
    const int c = c0 + i / PP, cell = i % PP;
    const PoolBin b = bins[cell];
    const float* plane = feat + (static_cast<long long>(level) * C + c) * H * W;
    const bool empty = (b.h1 <= b.h0) || (b.w1 <= b.w0);
    float best = empty ? 0.f : -3.402823466e+38f;
    int arg = -1;
    for (int h = b.h0; h < b.h1; ++h)
      for (int w = b.w0; w < b.w1; ++w) {
        const float v = __ldg(plane + h * W + w);
        if (v > best) {
          best = v;
          arg = h * W + w;
        }
      }
    const long long o = (static_cast<long long>(r) * C + c) * PP + cell;
    out[o] = best;
    if (argmax) argmax[o] = arg;
  }
}

// Engine form: fp32 NHWC feature copy in, split-bf16 rows [r][ph][pw][c] out (the K order the FC
// weights are permuted to).  grid (R, P); each thread owns (pw, channel quad) items of row ph.
__global__ void __launch_bounds__(256)
roi_pool_split_kernel(const float* __restrict__ feat, int C, int H, int W,
                      const float* __restrict__ rois, float spatial_scale, int P,
                      __nv_bfloat16* __restrict__ o_hi, __nv_bfloat16* __restrict__ o_lo) {
  __shared__ PoolBin bins[kMaxPooled];
  const int r = blockIdx.x, ph = blockIdx.y;
  const float* roi = rois + static_cast<long long>(r) * 5;
  if (threadIdx.x < P) bins[threadIdx.x] = roi_pool_bin(roi, spatial_scale, H, W, P, P, ph, threadIdx.x);
  __syncthreads();
  const float* fimg = feat + static_cast<long long>(static_cast<int>(roi[0])) * H * W * C;
  const int c4n = C / 4;
  for (int item = threadIdx.x; item < P * c4n; item += blockDim.x) {
    const int pw = item / c4n, c = (item - pw * c4n) * 4;
    const PoolBin b = bins[pw];
    const bool empty = (b.h1 <= b.h0) || (b.w1 <= b.w0);
    const float init = empty ? 0.f : -3.402823466e+38f;
    float4 best = make_float4(init, init, init, init);
    for (int h = b.h0; h < b.h1; ++h)
      for (int w = b.w0; w < b.w1; ++w)
        best = max4(best, __ldg(reinterpret_cast<const float4*>(fimg + (static_cast<long long>(h) * W + w) * C + c)));
    st_split4(o_hi, o_lo, ((static_cast<long long>(r) * P + ph) * P + pw) * C + c, best);
  }
}

// ROIWarping at P x P straight to split-bf16 rows [r][ph][pw][c] (no pooling after it).
__global__ void __launch_bounds__(256)
roi_sample_split_kernel(const float* __restrict__ feat, int C, int H, int W,
                        const float* __restrict__ rois, float spatial_scale, int P,
                        __nv_bfloat16* __restrict__ o_hi, __nv_bfloat16* __restrict__ o_lo) {
  __shared__ SampleTab tab[kMaxPooled];
  const int r = blockIdx.x, ph = blockIdx.y;
  const RoiGeom g = roi_geom(rois + static_cast<long long>(r) * 5, spatial_scale, P, P);
  if (threadIdx.x < P) {
    const int pw = threadIdx.x;
    const AxisTap th = axis_tap(__fadd_rn(g.start_h, __fmul_rn(static_cast<float>(ph), g.bin_h)), H);
    const AxisTap tw = axis_tap(__fadd_rn(g.start_w, __fmul_rn(static_cast<float>(pw), g.bin_w)), W);
    const bool ok = th.ok && tw.ok;
    SampleTab e;
    e.off[0] = ok ? (th.lo * W + tw.lo) * C : 0;
    e.off[1] = ok ? (th.lo * W + tw.hi) * C : 0;
    e.off[2] = ok ? (th.hi * W + tw.lo) * C : 0;
    e.off[3] = ok ? (th.hi * W + tw.hi) * C : 0;
    e.w[0] = ok ? __fmul_rn(th.h, tw.h) : 0.f;
    e.w[1] = ok ? __fmul_rn(th.h, tw.l) : 0.f;
    e.w[2] = ok ? __fmul_rn(th.l, tw.h) : 0.f;
    e.w[3] = ok ? __fmul_rn(th.l, tw.l) : 0.f;
    tab[pw] = e;
  }
  __syncthreads();
  const float* fimg = feat + static_cast<long long>(g.level) * H * W * C;
  const int c4n = C / 4;
  for (int item = threadIdx.x; item < P * c4n; item += blockDim.x) {
    const int pw = item / c4n, c = (item - pw * c4n) * 4;
    const SampleTab& e = tab[pw];
    const int4 of = *reinterpret_cast<const int4*>(e.off);
    const float4 wg = *reinterpret_cast<const float4*>(e.w);
    const float* fc = fimg + c;
    const float4 v = bilerp4(wg.x, wg.y, wg.z, wg.w, __ldg(reinterpret_cast<const float4*>(fc + of.x)),
                             __ldg(reinterpret_cast<const float4*>(fc + of.y)),
                             __ldg(reinterpret_cast<const float4*>(fc + of.z)),
                             __ldg(reinterpret_cast<const float4*>(fc + of.w)));
    st_split4(o_hi, o_lo, ((static_cast<long long>(r) * P + ph) * P + pw) * C + c, v);
  }
}


// sigmoid (sigmoid_layer.cu:10-14) -> mask_proposal (R,1,M,M) -> MaskResize to (R,1,14,14).
// One CTA per RoI; logits row stride given.
__global__ void __launch_bounds__(256)
sigmoid_resize_kernel(const float* __restrict__ logits, int stride, int M, int O,
                      float* __restrict__ mask_proposal, float* __restrict__ mask_resized) {
  extern __shared__ float sm[];  // M*M
  const int r = blockIdx.x;
  const float* x = logits + static_cast<long long>(r) * stride;
  for (int i = threadIdx.x; i < M * M; i += blockDim.x) {
    const float s = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x[i])));
    sm[i] = s;
    mask_proposal[static_cast<long long>(r) * M * M + i] = s;
  }
  __syncthreads();
  const float ratio = __fdiv_rn(static_cast<float>(M), static_cast<float>(O));
  for (int i = threadIdx.x; i < O * O; i += blockDim.x) {
    const int h = i / O, w = i % O;
    const AxisTap th = axis_tap(__fmul_rn(static_cast<float>(h), ratio), M);
    const AxisTap tw = axis_tap(__fmul_rn(static_cast<float>(w), ratio), M);
    float val = 0.f;
    if (th.ok && tw.ok)
      val = bilerp(th, tw, sm[th.lo * M + tw.lo], sm[th.lo * M + tw.hi], sm[th.hi * M + tw.lo],
                   sm[th.hi * M + tw.hi]);
    mask_resized[static_cast<long long>(r) * O * O + i] = val;
  }
}

// MaskPooling + 2x2 max pool on split NHWC: out7[r][t][j][c] = max_{dy,dx} feat14*mask14.
__global__ void __launch_bounds__(256)
mask_pool_split_kernel(const __nv_bfloat16* __restrict__ f_hi, const __nv_bfloat16* __restrict__ f_lo,
                       const float* __restrict__ mask14, int C, __nv_bfloat16* __restrict__ o_hi,
                       __nv_bfloat16* __restrict__ o_lo) {
  const int r = blockIdx.x, t = blockIdx.y;
  __shared__ float m[2][14];
  if (threadIdx.x < 28)
    m[threadIdx.x / 14][threadIdx.x % 14] =
        mask14[static_cast<long long>(r) * 196 + (2 * t + threadIdx.x / 14) * 14 + threadIdx.x % 14];
  __syncthreads();
  for (int c = threadIdx.x * 2; c < C; c += blockDim.x * 2) {
    for (int jp = 0; jp < 7; ++jp) {
      float2 best = make_float2(-3.402823466e+38f, -3.402823466e+38f);
#pragma unroll
      for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
          const int i = 2 * t + dy, j = 2 * jp + dx;
          const float2 f = ld_split2(f_hi, f_lo, ((static_cast<long long>(r) * 14 + i) * 14 + j) * C + c);
          const float mk = m[dy][j];
          best.x = fmaxf(best.x, __fmul_rn(f.x, mk));
          best.y = fmaxf(best.y, __fmul_rn(f.y, mk));
        }
      st_split2(o_hi, o_lo, ((static_cast<long long>(r) * 7 + t) * 7 + jp) * C + c, best.x, best.y);
    }
  }
}

static inline int check_launch() { return cudaGetLastError() == cudaSuccess ? MNC_OK : MNC_ERR_CUDA; }
static inline int grid_for(long long n, int block, int cap) {
  long long g = (n + block - 1) / block;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return static_cast<int>(g);
}

}  // namespace mnc

using namespace mnc;

extern "C" int mnc_roi_warp_nchw(const float* feat, int C, int H, int W, const float* rois, int R,
                                 int pooled_h, int pooled_w, float spatial_scale, float* out,
                                 void* stream) {
  if (R <= 0) return MNC_OK;
  if (pooled_h > kMaxPooled || pooled_w > kMaxPooled || pooled_h <= 0 || pooled_w <= 0)
    return MNC_ERR_ARG;
  auto s = static_cast<cudaStream_t>(stream);
  if (pooled_h == pooled_w && (pooled_h == 28 || pooled_h == 14)) {
    // one pass of the CTA's warps covers threads/32 * (planes per warp) channels: 32 channels per
    // CTA = 4 warps (28x28: 8 planes per lane; 14x14: 2 plane groups x 4), so 128 threads keep
    // every warp of the CTA busy (with 256, half of them only waited at the barrier and held
    // their scheduler slots until the CTA retired)
    constexpr int cpc = 32, threads = 128;
    dim3 wgrid(R, (C + cpc - 1) / cpc);
    if (pooled_h == 28)
      roi_warp_rowwalk_kernel<28><<<wgrid, threads, 0, s>>>(feat, C, H, W, rois, spatial_scale, cpc, out);
    else
      roi_warp_rowwalk_kernel<14><<<wgrid, threads, 0, s>>>(feat, C, H, W, rois, spatial_scale, cpc, out);
    return check_launch();
  }
  dim3 grid(R, (C + kWarpSlab - 1) / kWarpSlab);
  if (pooled_h == 7 && pooled_w == 7)
    roi_warp_nchw_kernel<7, 7, 1><<<grid, 256, 0, s>>>(feat, C, H, W, rois, spatial_scale, out);
  else
    roi_warp_nchw_generic_kernel<<<grid, 256, 0, s>>>(feat, C, H, W, rois, pooled_h, pooled_w,
                                                      spatial_scale, out);
  return check_launch();
}

extern "C" int mnc_mask_resize_nchw(const float* in, int N, int C, int in_h, int in_w, int out_h,
                                    int out_w, float* out, void* stream) {
  const long long total = static_cast<long long>(N) * C * out_h * out_w;
  if (total <= 0) return MNC_OK;
  mask_resize_nchw_kernel<<<grid_for(total, 256, 132 * 8), 256, 0,
                            static_cast<cudaStream_t>(stream)>>>(in, N * C, in_h, in_w, out_h,
                                                                 out_w, out);
  return check_launch();
}

extern "C" int mnc_mask_pool_nchw(const float* feat, const float* mask, int N, int C, int H, int W,
                                  float* out, void* stream) {
  const long long total = static_cast<long long>(N) * C * H * W;
  if (total <= 0) return MNC_OK;
  const int hw = H * W;
  const bool vec = (hw % 4 == 0) && ((reinterpret_cast<uintptr_t>(feat) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(mask) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
  if (vec)
    mask_pool_nchw_kernel<<<grid_for(total / 4, 256, 132 * 16), 256, 0,
                            static_cast<cudaStream_t>(stream)>>>(feat, mask, N, C, hw, out);
  else
    mask_pool_nchw_scalar_kernel<<<grid_for(total, 256, 132 * 16), 256, 0,
                                   static_cast<cudaStream_t>(stream)>>>(feat, mask, N, C, hw, out);
  return check_launch();
}

extern "C" int mnc_roi_warp_split(const float* feat_nhwc, int C, int H, int W, const float* rois,
                                  int R, int sub, float spatial_scale, void* o14_hi, void* o14_lo,
                                  void* o7_hi, void* o7_lo, void* stream) {
  if (R <= 0) return MNC_OK;
  if (C % 4 != 0 || (sub != 1 && sub != 2) || (reinterpret_cast<uintptr_t>(feat_nhwc) & 15))
    return MNC_ERR_ARG;
  auto s = static_cast<cudaStream_t>(stream);
  RoiOut o;
  o.p14[0] = o14_hi; o.p14[1] = o14_lo; o.p14[2] = nullptr;
  o.p7[0] = o7_hi; o.p7[1] = o7_lo; o.p7[2] = nullptr;
  o.scale = 1.0f;
  dim3 grid(R, 7);
  if (sub == 2)
    roi_warp_split_kernel<2, false><<<grid, 256, 0, s>>>(feat_nhwc, C, H, W, rois, spatial_scale, o);
  else
    roi_warp_split_kernel<1, false><<<grid, 256, 0, s>>>(feat_nhwc, C, H, W, rois, spatial_scale, o);
  return check_launch();
}

// Same, writing tri-plane outputs (fp16 value, e4m3 residual, e4m3 copy) scaled by `scale` = 2^exp.
extern "C" int mnc_roi_warp_tri(const float* feat_nhwc, int C, int H, int W, const float* rois,
                                int R, int sub, float spatial_scale, float scale, void* o14_h,
                                void* o14_l, void* o14_c, void* o7_h, void* o7_l, void* o7_c,
                                void* stream) {
  if (R <= 0) return MNC_OK;
  if (C % 4 != 0 || (sub != 1 && sub != 2) || (reinterpret_cast<uintptr_t>(feat_nhwc) & 15) ||
      !tri_planes_aligned(o14_h, o14_l, o14_c) || !tri_planes_aligned(o7_h, o7_l, o7_c))
    return MNC_ERR_ARG;
  auto s = static_cast<cudaStream_t>(stream);
  RoiOut o;
  o.p14[0] = o14_h; o.p14[1] = o14_l; o.p14[2] = o14_c;
  o.p7[0] = o7_h; o.p7[1] = o7_l; o.p7[2] = o7_c;
  o.scale = scale;
  dim3 grid(R, 7);
  if (sub == 2)
    roi_warp_split_kernel<2, true><<<grid, 256, 0, s>>>(feat_nhwc, C, H, W, rois, spatial_scale, o);
  else
    roi_warp_split_kernel<1, true><<<grid, 256, 0, s>>>(feat_nhwc, C, H, W, rois, spatial_scale, o);
  return check_launch();
}

extern "C" int mnc_roi_pool_nchw(const float* feat, int C, int H, int W, const float* rois, int R,
                                 int pooled_h, int pooled_w, float spatial_scale, float* out,
                                 int* argmax, void* stream) {
  if (R <= 0) return MNC_OK;
  if (C <= 0 || pooled_h <= 0 || pooled_w <= 0) return MNC_ERR_ARG;
  const int smem = pooled_h * pooled_w * static_cast<int>(sizeof(PoolBin));
  if (smem > 48 * 1024) return MNC_ERR_ARG;
  dim3 grid(R, (C + kWarpSlab - 1) / kWarpSlab);
  roi_pool_nchw_kernel<<<grid, 256, smem, static_cast<cudaStream_t>(stream)>>>(
      feat, C, H, W, rois, spatial_scale, pooled_h, pooled_w, out, argmax);
  return check_launch();
}

extern "C" int mnc_roi_pool_split(const float* feat_nhwc, int C, int H, int W, const float* rois,
                                  int R, int pooled, float spatial_scale, void* o_hi, void* o_lo,
                                  void* stream) {
  if (R <= 0) return MNC_OK;
  if (C % 4 != 0 || pooled <= 0 || pooled > kMaxPooled ||
      (reinterpret_cast<uintptr_t>(feat_nhwc) & 15))
    return MNC_ERR_ARG;
  roi_pool_split_kernel<<<dim3(R, pooled), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      feat_nhwc, C, H, W, rois, spatial_scale, pooled, static_cast<__nv_bfloat16*>(o_hi),
      static_cast<__nv_bfloat16*>(o_lo));
  return check_launch();
}

extern "C" int mnc_roi_sample_split(const float* feat_nhwc, int C, int H, int W, const float* rois,
                                    int R, int pooled, float spatial_scale, void* o_hi, void* o_lo,
                                    void* stream) {
  if (R <= 0) return MNC_OK;
  if (C % 4 != 0 || pooled <= 0 || pooled > kMaxPooled ||
      (reinterpret_cast<uintptr_t>(feat_nhwc) & 15))
    return MNC_ERR_ARG;
  roi_sample_split_kernel<<<dim3(R, pooled), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      feat_nhwc, C, H, W, rois, spatial_scale, pooled, static_cast<__nv_bfloat16*>(o_hi),
      static_cast<__nv_bfloat16*>(o_lo));
  return check_launch();
}

extern "C" int mnc_sigmoid_mask_resize(const float* logits, int stride, int R, int mask_size,
                                       int out_size, float* mask_proposal, float* mask_resized,
                                       void* stream) {
  if (R <= 0) return MNC_OK;
  sigmoid_resize_kernel<<<R, 256, mask_size * mask_size * sizeof(float),
                          static_cast<cudaStream_t>(stream)>>>(logits, stride, mask_size, out_size,
                                                               mask_proposal, mask_resized);
  return check_launch();
}

extern "C" int mnc_mask_pool_split(const void* f_hi, const void* f_lo, const float* mask14, int R,
                                   int C, void* o_hi, void* o_lo, void* stream) {
  if (R <= 0) return MNC_OK;
  if (C % 2 != 0) return MNC_ERR_ARG;
  dim3 grid(R, 7);
  mask_pool_split_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(f_hi), static_cast<const __nv_bfloat16*>(f_lo), mask14, C,
      static_cast<__nv_bfloat16*>(o_hi), static_cast<__nv_bfloat16*>(o_lo));
  return check_launch();
}
