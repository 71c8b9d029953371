// Backward passes of the four Caffe layers, fp32 NCHW device blobs.  Replaces Backward_gpu of
//   ROIWarping   caffe-mnc/src/caffe/layers/roi_warping_layer.cu:379-436
//                (feature gradient :125-245, coordinate gradient :247-361 + thrust reduce :409-434)
//   MaskResize   caffe-mnc/src/caffe/layers/mask_resize_layer.cu:86-183
//   MaskPooling  caffe-mnc/src/caffe/layers/mask_pooling_layer.cu:43-99
//   ROIPooling   caffe-mnc/src/caffe/layers/roi_pooling_layer.cu:94-184
// The reference's arithmetic is kept exactly (DESIGN.md "Backward semantics"): every float
// operation it rounds separately is written with __fmul_rn / __fadd_rn / __fsub_rn / __fdiv_rn,
// its double sub-expressions with __dmul_rn / __dadd_rn / __dsub_rn, in its operation order, so the
// feature and mask gradients equal the reference built with -fmad=false bit for bit.
//
// Every kernel is a gather: each output element is written by exactly one thread, which sums its
// terms in the reference's order.  No float atomics, so two calls on the same inputs give the same
// bits.
//   * Feature gradients of ROIWarping / ROIPooling: the reference runs one thread per bottom
//     element and loops over EVERY RoI of the batch.  Here a CTA owns a tile of 8 x 32 bottom
//     positions of one image and a slab of 8 channels; it compacts, in ascending index order, the
//     RoIs of its image whose rectangle meets the tile, stages their geometry (and, for
//     ROIWarping, the per-(RoI, ph) and per-(RoI, pw) bilinear factors) in shared memory, and each
//     thread then walks only that list, accumulating its 8 channels side by side.
//   * Coordinate gradient of ROIWarping: the reference writes an R*5*C*P*P float buffer, copies it
//     into a thrust::device_vector and reduces it with reduce_by_key.  Here a CTA per (RoI,
//     64-channel slab) sums its terms in double in a fixed order, and a second kernel adds the
//     slabs in a fixed order: R * slabs * 4 doubles of workspace instead of two 0.5 GB buffers.
#include <cuda_runtime.h>

#include "mnc_b200.h"
#include "roi_geom.cuh"

namespace mnc {
namespace {

constexpr int kTileH = 8, kTileW = 32;           // bottom positions per CTA, one per thread
constexpr int kTileThreads = kTileH * kTileW;    // 256: one warp per tile row
constexpr int kSlab = 8;                         // channels per CTA, accumulated side by side
constexpr int kChunk = 16;                       // RoIs whose tables are staged at once
constexpr int kCoordSlab = 64;                   // channels per CTA of the coordinate gradient
constexpr int kCoordThreads = 256;

inline int check_launch() { return cudaGetLastError() == cudaSuccess ? MNC_OK : MNC_ERR_CUDA; }

// Ordered compaction over the block (kTileThreads threads): returns how many threads have `hit`
// set and gives each such thread its rank among them in `pos` (ranks follow thread order).  The
// caller writes its entry at `pos` and then synchronises.
__device__ __forceinline__ int compact_ordered(bool hit, int* wcount, int& pos) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, hit);
  if (lane == 0) wcount[warp] = __popc(m);
  __syncthreads();
  int off = 0, total = 0;
#pragma unroll
  for (int k = 0; k < kTileThreads / 32; ++k) {
    const int c = wcount[k];
    off += k < warp ? c : 0;
    total += c;
  }
  pos = off + __popc(m & ((1u << lane) - 1u));
  return total;
}

// ------------------------------------------------------------------ ROIWarping, feature gradient
// One sample row (or column) of a RoI as the backward pass sees it.  The forward pass stores the
// clamped sample coordinate `a` as argmax (roi_warping_layer.cu:26-47, 61); get_feature_gradient
// (:126-173) re-derives the taps lo / hi from it and weights bottom row lo by (lo + 1 - a) and row
// hi by (a + 1 - hi).  lo = -1 marks a sample outside the map (argmax -1: no gradient).
struct GradTap {
  int lo, hi;
  float f_lo, f_hi;
};

__device__ __forceinline__ GradTap grad_tap(float x, int dim) {
  GradTap t;
  if (x < -0.5 || x > dim - 0.5) {
    t.lo = t.hi = -1;
    t.f_lo = t.f_hi = 0.f;
    return t;
  }
  if (x <= 0) x = 0;
  int lo = static_cast<int>(x), hi;
  if (lo >= dim - 1) {
    hi = lo = dim - 1;
    x = static_cast<float>(lo);
  } else {
    hi = lo + 1;
  }
  t.lo = lo;
  t.hi = hi;
  t.f_lo = __fsub_rn(static_cast<float>(lo + 1), x);      // (h + 1 - argmax_h), :158
  t.f_hi = __fsub_rn(__fadd_rn(x, 1.f), static_cast<float>(hi));   // (argmax_h + 1 - h), :166
  return t;
}

// The factor of bottom index `i` for tap t: get_feature_gradient tests lo first (:156, :164).
__device__ __forceinline__ float tap_factor(const GradTap& t, int i) {
  return i == t.lo ? t.f_lo : (i == t.hi ? t.f_hi : 0.f);
}

// A RoI as ROIWarpingBackwardFeature sees it (roi_warping_layer.cu:197-223).
struct WarpRoi {
  int r;                       // RoI index
  float x0, x1, y0, y1;        // in_roi rectangle: floor(start), ceil(end) (:203-204)
  float sw, sh;                // rounded start
  float bin_w, bin_h;          // max(end - start + 1, 1) / pooled (:218-223)
};

__device__ __forceinline__ void warp_rect(const float* roi, float ss, float& sw, float& sh,
                                          float& ew, float& eh) {
  sw = roundf(__fmul_rn(roi[1], ss));
  sh = roundf(__fmul_rn(roi[2], ss));
  ew = roundf(__fmul_rn(roi[3], ss));
  eh = roundf(__fmul_rn(roi[4], ss));
}

__global__ void __launch_bounds__(kTileThreads)
roi_warp_bwd_feat_kernel(const float* __restrict__ rois, int R, int C, int H, int W, int PH, int PW,
                         float ss, const float* __restrict__ top_diff, float* __restrict__ feat_diff) {
  __shared__ int s_list[kTileThreads];
  __shared__ int s_wcount[kTileThreads / 32];
  __shared__ WarpRoi s_roi[kChunk];
  __shared__ GradTap s_th[kChunk][kMaxPooled], s_tw[kChunk][kMaxPooled];
  const int tiles_w = (W + kTileW - 1) / kTileW;
  const int h0 = (blockIdx.x / tiles_w) * kTileH, w0 = (blockIdx.x % tiles_w) * kTileW;
  const int c0 = blockIdx.y * kSlab, n = blockIdx.z;
  const int tid = threadIdx.x;
  const int h = h0 + tid / kTileW, w = w0 + tid % kTileW;
  const float hf = static_cast<float>(h), wf = static_cast<float>(w);
  const int nk = min(kSlab, C - c0);
  const int PP = PH * PW;
  float acc[kSlab];
#pragma unroll
  for (int k = 0; k < kSlab; ++k) acc[k] = 0.f;
  for (int base = 0; base < R; base += kTileThreads) {
    const int i = base + tid;
    bool hit = false;
    if (i < R) {
      const float* roi = rois + static_cast<long long>(i) * 5;
      float sw, sh, ew, eh;
      warp_rect(roi, ss, sw, sh, ew, eh);
      // some position of the tile lies in the RoI's in_roi rectangle (a superset test: the exact
      // per-position test below decides)
      hit = static_cast<int>(roi[0]) == n && floorf(sw) <= static_cast<float>(w0 + kTileW - 1) &&
            ceilf(ew) >= static_cast<float>(w0) && floorf(sh) <= static_cast<float>(h0 + kTileH - 1) &&
            ceilf(eh) >= static_cast<float>(h0);
    }
    int pos;
    const int cnt = compact_ordered(hit, s_wcount, pos);
    if (hit) s_list[pos] = i;
    __syncthreads();
    for (int j0 = 0; j0 < cnt; j0 += kChunk) {
      const int nj = min(kChunk, cnt - j0);
      if (tid < nj) {
        const int r = s_list[j0 + tid];
        float sw, sh, ew, eh;
        warp_rect(rois + static_cast<long long>(r) * 5, ss, sw, sh, ew, eh);
        WarpRoi q;
        q.r = r;
        q.x0 = floorf(sw);
        q.x1 = ceilf(ew);
        q.y0 = floorf(sh);
        q.y1 = ceilf(eh);
        q.sw = sw;
        q.sh = sh;
        q.bin_w = __fdiv_rn(fmaxf(__fadd_rn(__fsub_rn(ew, sw), 1.f), 1.f), static_cast<float>(PW));
        q.bin_h = __fdiv_rn(fmaxf(__fadd_rn(__fsub_rn(eh, sh), 1.f), 1.f), static_cast<float>(PH));
        s_roi[tid] = q;
      }
      // forward sample positions (roi_warping_layer.cu:78-99) -> backward taps
      for (int e = tid; e < nj * (PH + PW); e += kTileThreads) {
        const int j = e / (PH + PW), p = e % (PH + PW);
        const RoiGeom g = roi_geom(rois + static_cast<long long>(s_list[j0 + j]) * 5, ss, PH, PW);
        if (p < PH)
          s_th[j][p] = grad_tap(__fadd_rn(g.start_h, __fmul_rn(static_cast<float>(p), g.bin_h)), H);
        else
          s_tw[j][p - PH] = grad_tap(__fadd_rn(g.start_w, __fmul_rn(static_cast<float>(p - PH), g.bin_w)), W);
      }
      __syncthreads();
      if (h < H && w < W) {
        for (int j = 0; j < nj; ++j) {
          const WarpRoi q = s_roi[j];
          if (!(wf >= q.x0 && wf <= q.x1 && hf >= q.y0 && hf <= q.y1)) continue;
          // feasible pooled cells (roi_warping_layer.cu:225-233)
          const int phs = min(max(static_cast<int>(floorf(__fsub_rn(__fdiv_rn(__fsub_rn(__fsub_rn(hf, q.sh), 1.f), q.bin_h), 1.f))), 0), PH);
          const int phe = min(max(static_cast<int>(ceilf(__fdiv_rn(__fadd_rn(__fsub_rn(hf, q.sh), 1.f), q.bin_h))), 0), PH);
          const int pws = min(max(static_cast<int>(floorf(__fsub_rn(__fdiv_rn(__fsub_rn(__fsub_rn(wf, q.sw), 1.f), q.bin_w), 1.f))), 0), PW);
          const int pwe = min(max(static_cast<int>(ceilf(__fdiv_rn(__fadd_rn(__fsub_rn(wf, q.sw), 1.f), q.bin_w))), 0), PW);
          const float* td = top_diff + (static_cast<long long>(q.r) * C + c0) * PP;
          for (int ph = phs; ph < phe; ++ph) {
            const GradTap th = s_th[j][ph];
            if (th.lo < 0) continue;                 // argmax -1: weight 0 (:128-132)
            const float fh = tap_factor(th, h);
            if (fh == 0.f) continue;                 // zero terms leave a finite sum unchanged
            for (int pw = pws; pw < pwe; ++pw) {
              const GradTap tw = s_tw[j][pw];
              if (tw.lo < 0) continue;
              const float fw = tap_factor(tw, w);
              if (fw == 0.f) continue;
              const float wt = __fmul_rn(fh, fw);
              const float* t = td + ph * PW + pw;
#pragma unroll
              for (int k = 0; k < kSlab; ++k)
                if (k < nk) acc[k] = __fadd_rn(acc[k], __fmul_rn(wt, __ldg(t + k * PP)));
            }
          }
        }
      }
      __syncthreads();
    }
  }
  if (h < H && w < W) {
    float* o = feat_diff + ((static_cast<long long>(n) * C + c0) * H + h) * W + w;
#pragma unroll
    for (int k = 0; k < kSlab; ++k)
      if (k < nk) o[static_cast<long long>(k) * H * W] = acc[k];
  }
}

// --------------------------------------------------------------- ROIWarping, coordinate gradient
// Per sample row (or column): what get_coordinate_gradient (roi_warping_layer.cu:248-304) and its
// caller (:331-358) derive from the argmax coordinate a.  arg < 0: the term is 0 -- either the
// reference returns 0 (tap arg + 1 past the map, :255-257), or the sample lies outside the map
// (argmax -1), where the reference reads outside the sampled plane and we contribute 0.
struct CoordTap {
  int arg;        // (int) a
  float a;
  double A;       // 1.0 - a + arg
  double B;       // a - arg, rounded in float
  double m_lo;    // 0.5 - map_ratio
  double m_hi;    // -0.5 + map_ratio
};

__device__ __forceinline__ CoordTap coord_tap(float x, int dim, int start, float bin, int pooled) {
  CoordTap t;
  t.arg = -1;
  t.a = 0.f;
  t.A = t.B = t.m_lo = t.m_hi = 0.0;
  if (x < -0.5 || x > dim - 0.5) return t;
  if (x <= 0) x = 0;
  const int lo = static_cast<int>(x);
  if (lo >= dim - 1) x = static_cast<float>(dim - 1);
  const int arg = static_cast<int>(x);
  if (arg + 1 > dim - 1) return t;
  t.arg = arg;
  t.a = x;
  t.A = __dadd_rn(__dsub_rn(1.0, static_cast<double>(x)), static_cast<double>(arg));
  t.B = static_cast<double>(__fsub_rn(x, static_cast<float>(arg)));
  // output_h = (ih - roi_start_h) / bin_size_h (:356); map_ratio_h = output_h / pooled (:259)
  const float out = __fdiv_rn(__fsub_rn(x, static_cast<float>(start)), bin);
  const double ratio = static_cast<double>(__fdiv_rn(out, static_cast<float>(pooled)));
  t.m_lo = __dsub_rn(0.5, ratio);
  t.m_hi = __dadd_rn(-0.5, ratio);
  return t;
}

// acc = (float)((double)acc + term), one `+=` of :270-288
__device__ __forceinline__ float acc_d(float acc, double term) {
  return __double2float_rn(__dadd_rn(static_cast<double>(acc), term));
}

__global__ void __launch_bounds__(kCoordThreads)
roi_warp_bwd_coord_kernel(const float* __restrict__ feat, int B, int C, int H, int W,
                          const float* __restrict__ rois, int PH, int PW, float ss,
                          const float* __restrict__ top_diff, double* __restrict__ partial) {
  __shared__ CoordTap s_th[kMaxPooled], s_tw[kMaxPooled];
  __shared__ double s_part[kCoordThreads / 32][4];
  const int r = blockIdx.x, c0 = blockIdx.y * kCoordSlab, tid = threadIdx.x;
  const float* roi = rois + static_cast<long long>(r) * 5;
  const int level = static_cast<int>(roi[0]);
  if (tid < PH + PW) {
    // forward sample position (float start and bin, :78-99) ...
    const RoiGeom g = roi_geom(roi, ss, PH, PW);
    // ... and the coordinate kernel's int start / end and bin (:333-342)
    const int sw = static_cast<int>(roundf(__fmul_rn(roi[1], ss)));
    const int sh = static_cast<int>(roundf(__fmul_rn(roi[2], ss)));
    const int ew = static_cast<int>(roundf(__fmul_rn(roi[3], ss)));
    const int eh = static_cast<int>(roundf(__fmul_rn(roi[4], ss)));
    const float bin_w = __fdiv_rn(static_cast<float>(max(ew - sw + 1, 1)), static_cast<float>(PW));
    const float bin_h = __fdiv_rn(static_cast<float>(max(eh - sh + 1, 1)), static_cast<float>(PH));
    if (tid < PH)
      s_th[tid] = coord_tap(__fadd_rn(g.start_h, __fmul_rn(static_cast<float>(tid), g.bin_h)), H, sh, bin_h, PH);
    else
      s_tw[tid - PH] = coord_tap(__fadd_rn(g.start_w, __fmul_rn(static_cast<float>(tid - PH), g.bin_w)), W, sw, bin_w, PW);
  }
  __syncthreads();
  double s1 = 0.0, s2 = 0.0, s3 = 0.0, s4 = 0.0;
  if (level >= 0 && level < B) {
    const int PP = PH * PW;
    const int nc = min(kCoordSlab, C - c0);
    const float* fbase = feat + (static_cast<long long>(level) * C + c0) * H * W;
    const float* tbase = top_diff + (static_cast<long long>(r) * C + c0) * PP;
    for (int i = tid; i < nc * PP; i += kCoordThreads) {
      const int c = i / PP, p = i - c * PP;
      const CoordTap th = s_th[p / PW], tw = s_tw[p % PW];
      if (th.arg < 0 || tw.arg < 0) continue;
      const float* pl = fbase + static_cast<long long>(c) * H * W + th.arg * W + tw.arg;
      const double v1 = __ldg(pl), v2 = __ldg(pl + 1), v3 = __ldg(pl + W), v4 = __ldg(pl + W + 1);
      float dxc = 0.f, dyc = 0.f, dw = 0.f, dh = 0.f;
      dxc = acc_d(dxc, __dmul_rn(-th.A, v1));                   // :270-273
      dxc = acc_d(dxc, __dmul_rn(th.A, v2));
      dxc = acc_d(dxc, __dmul_rn(-th.B, v3));
      dxc = acc_d(dxc, __dmul_rn(th.B, v4));
      dyc = acc_d(dyc, __dmul_rn(-tw.A, v1));                   // :275-278
      dyc = acc_d(dyc, __dmul_rn(-tw.B, v2));
      dyc = acc_d(dyc, __dmul_rn(tw.A, v3));
      dyc = acc_d(dyc, __dmul_rn(tw.B, v4));
      dw = acc_d(dw, __dmul_rn(__dmul_rn(tw.m_lo, th.A), v1));  // :280-283
      dw = acc_d(dw, __dmul_rn(__dmul_rn(tw.m_hi, th.A), v2));
      dw = acc_d(dw, __dmul_rn(__dmul_rn(tw.m_lo, th.B), v3));
      dw = acc_d(dw, __dmul_rn(__dmul_rn(tw.m_hi, th.B), v4));
      dh = acc_d(dh, __dmul_rn(__dmul_rn(th.m_lo, tw.A), v1));  // :285-288
      dh = acc_d(dh, __dmul_rn(__dmul_rn(th.m_lo, tw.B), v2));
      dh = acc_d(dh, __dmul_rn(__dmul_rn(th.m_hi, tw.A), v3));
      dh = acc_d(dh, __dmul_rn(__dmul_rn(th.m_hi, tw.B), v4));
      const double hx = __dmul_rn(0.5, static_cast<double>(dxc));
      const double hy = __dmul_rn(0.5, static_cast<double>(dyc));
      const float w1 = __double2float_rn(__dsub_rn(hx, static_cast<double>(dw)));   // :290-302
      const float w2 = __double2float_rn(__dsub_rn(hy, static_cast<double>(dh)));
      const float w3 = __double2float_rn(__dadd_rn(hx, static_cast<double>(dw)));
      const float w4 = __double2float_rn(__dadd_rn(hy, static_cast<double>(dh)));
      const float td = __ldg(tbase + i);                                            // :358-359
      s1 = __dadd_rn(s1, static_cast<double>(__fmul_rn(__fmul_rn(ss, w1), td)));
      s2 = __dadd_rn(s2, static_cast<double>(__fmul_rn(__fmul_rn(ss, w2), td)));
      s3 = __dadd_rn(s3, static_cast<double>(__fmul_rn(__fmul_rn(ss, w3), td)));
      s4 = __dadd_rn(s4, static_cast<double>(__fmul_rn(__fmul_rn(ss, w4), td)));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s1 = __dadd_rn(s1, __shfl_down_sync(0xffffffffu, s1, o));
    s2 = __dadd_rn(s2, __shfl_down_sync(0xffffffffu, s2, o));
    s3 = __dadd_rn(s3, __shfl_down_sync(0xffffffffu, s3, o));
    s4 = __dadd_rn(s4, __shfl_down_sync(0xffffffffu, s4, o));
  }
  if ((tid & 31) == 0) {
    s_part[tid >> 5][0] = s1;
    s_part[tid >> 5][1] = s2;
    s_part[tid >> 5][2] = s3;
    s_part[tid >> 5][3] = s4;
  }
  __syncthreads();
  if (tid < 4) {
    double s = 0.0;
    for (int k = 0; k < kCoordThreads / 32; ++k) s = __dadd_rn(s, s_part[k][tid]);
    partial[(static_cast<long long>(r) * gridDim.y + blockIdx.y) * 4 + tid] = s;
  }
}

// rois_diff[r] = {0, sum over slabs of the four partial sums}, slabs in ascending order.
__global__ void roi_warp_bwd_coord_sum_kernel(const double* __restrict__ partial, int R, int slabs,
                                              float* __restrict__ rois_diff) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * 5) return;
  const int r = i / 5, k = i % 5;
  double s = 0.0;
  if (k > 0)
    for (int b = 0; b < slabs; ++b) s = __dadd_rn(s, partial[(static_cast<long long>(r) * slabs + b) * 4 + k - 1]);
  rois_diff[i] = __double2float_rn(s);
}

// ------------------------------------------------------------------------------- MaskResize
// getGradientWeight (mask_resize_layer.cu:87-133).
__device__ __forceinline__ float resize_grad_weight(float ah, float aw, int h, int w, int H, int W) {
  if (ah < -0.5 || ah > (H - 0.5) || aw < -0.5 || aw > (W - 0.5)) return 0.f;
  if (ah < 0) ah = 0;
  if (aw < 0) aw = 0;
  int hl = static_cast<int>(ah), wl = static_cast<int>(aw), hh, wh;
  if (hl >= H - 1) {
    hh = hl = H - 1;
    ah = static_cast<float>(hl);
  } else {
    hh = hl + 1;
  }
  if (wl >= W - 1) {
    wh = wl = W - 1;
    aw = static_cast<float>(wl);
  } else {
    wh = wl + 1;
  }
  const float fh_lo = __fsub_rn(static_cast<float>(h + 1), ah);
  const float fh_hi = __fsub_rn(__fadd_rn(ah, 1.f), static_cast<float>(h));
  const float fw_lo = __fsub_rn(static_cast<float>(w + 1), aw);
  const float fw_hi = __fsub_rn(__fadd_rn(aw, 1.f), static_cast<float>(w));
  if (h == hl) {
    if (w == wl) return __fmul_rn(fh_lo, fw_lo);
    if (w == wh) return __fmul_rn(fh_lo, fw_hi);
  } else if (h == hh) {
    if (w == wl) return __fmul_rn(fh_hi, fw_lo);
    if (w == wh) return __fmul_rn(fh_hi, fw_hi);
  }
  return 0.f;
}

// MaskResizeBackward (mask_resize_layer.cu:135-173): one thread per input element, at most 2 x 2
// output cells.
__global__ void mask_resize_bwd_kernel(const float* __restrict__ top_diff, long long planes,
                                       int ih_n, int iw_n, int oh_n, int ow_n,
                                       float* __restrict__ in_diff) {
  const long long total = planes * ih_n * iw_n;
  const float ratio_h = __fdiv_rn(static_cast<float>(ih_n), static_cast<float>(oh_n));
  const float ratio_w = __fdiv_rn(static_cast<float>(iw_n), static_cast<float>(ow_n));
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int w = static_cast<int>(i % iw_n);
    const int h = static_cast<int>((i / iw_n) % ih_n);
    const long long p = i / (static_cast<long long>(iw_n) * ih_n);
    const int hs = static_cast<int>(floorf(__fdiv_rn(static_cast<float>(h), ratio_h)));
    const int ws = static_cast<int>(floorf(__fdiv_rn(static_cast<float>(w), ratio_w)));
    const float* td = top_diff + p * oh_n * ow_n;
    float g = 0.f;
    for (int ph = hs; ph <= hs + 1; ++ph) {
      for (int pw = ws; pw <= ws + 1; ++pw) {
        const float iw = __fmul_rn(static_cast<float>(pw), ratio_w);
        const float ih = __fmul_rn(static_cast<float>(ph), ratio_h);
        if (fabsf(__fsub_rn(iw, static_cast<float>(w))) >= 1.f ||
            fabsf(__fsub_rn(ih, static_cast<float>(h))) >= 1.f)
          continue;
        // ph == oh_n or pw == ow_n samples at >= dim - 0.5 and so has weight 0; the reference
        // multiplies that 0 by an element past the row (or the plane), which adds nothing
        if (ph >= oh_n || pw >= ow_n) continue;
        const float wt = resize_grad_weight(ih, iw, h, w, ih_n, iw_n);
        if (wt == 0.f) continue;
        g = __fadd_rn(g, __fmul_rn(wt, td[ph * ow_n + pw]));
      }
    }
    in_diff[i] = g;
  }
}

// ------------------------------------------------------------------------------- MaskPooling
// MaskPoolingBackwardFeature (mask_pooling_layer.cu:43-58): feat_diff = top_diff * mask.
__global__ void mask_pool_bwd_feat_kernel(const float* __restrict__ top_diff,
                                          const float* __restrict__ mask, int C, int hw,
                                          long long total, float* __restrict__ feat_diff) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int q = static_cast<int>(i % hw);
    const long long n = i / (static_cast<long long>(hw) * C);
    feat_diff[i] = __fmul_rn(top_diff[i], mask[n * hw + q]);
  }
}

// MaskPoolingBackwardMask (:60-76): one thread per mask element sums over channels c = 0..C-1.
__global__ void mask_pool_bwd_mask_kernel(const float* __restrict__ top_diff,
                                          const float* __restrict__ feat, int C, int hw,
                                          long long total, float* __restrict__ mask_diff) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int q = static_cast<int>(i % hw);
    const long long n = i / hw;
    const float* t = top_diff + n * C * hw + q;
    const float* f = feat + n * C * hw + q;
    float g = 0.f;
#pragma unroll 8
    for (int c = 0; c < C; ++c)
      g = __fadd_rn(g, __fmul_rn(__ldg(t + static_cast<long long>(c) * hw), __ldg(f + static_cast<long long>(c) * hw)));
    mask_diff[i] = g;
  }
}

// ------------------------------------------------------------------------------- ROIPooling
// A RoI as ROIPoolBackward sees it (roi_pooling_layer.cu:117-143).
struct PoolRoi {
  int r, sw, sh, ew, eh;
  float bin_w, bin_h;
};

__device__ __forceinline__ void pool_rect(const float* roi, float ss, int& sw, int& sh, int& ew, int& eh) {
  sw = static_cast<int>(roundf(__fmul_rn(roi[1], ss)));
  sh = static_cast<int>(roundf(__fmul_rn(roi[2], ss)));
  ew = static_cast<int>(roundf(__fmul_rn(roi[3], ss)));
  eh = static_cast<int>(roundf(__fmul_rn(roi[4], ss)));
}

__global__ void __launch_bounds__(kTileThreads)
roi_pool_bwd_kernel(const float* __restrict__ rois, int R, int C, int H, int W, int PH, int PW,
                    float ss, const float* __restrict__ top_diff, const int* __restrict__ argmax,
                    float* __restrict__ feat_diff) {
  __shared__ int s_wcount[kTileThreads / 32];
  __shared__ PoolRoi s_roi[kTileThreads];
  const int tiles_w = (W + kTileW - 1) / kTileW;
  const int h0 = (blockIdx.x / tiles_w) * kTileH, w0 = (blockIdx.x % tiles_w) * kTileW;
  const int c0 = blockIdx.y * kSlab, n = blockIdx.z;
  const int tid = threadIdx.x;
  const int h = h0 + tid / kTileW, w = w0 + tid % kTileW;
  const int nk = min(kSlab, C - c0);
  const int PP = PH * PW;
  const int idx = h * W + w;
  float acc[kSlab];
#pragma unroll
  for (int k = 0; k < kSlab; ++k) acc[k] = 0.f;
  for (int base = 0; base < R; base += kTileThreads) {
    const int i = base + tid;
    bool hit = false;
    int sw = 0, sh = 0, ew = 0, eh = 0;
    if (i < R) {
      const float* roi = rois + static_cast<long long>(i) * 5;
      pool_rect(roi, ss, sw, sh, ew, eh);
      hit = static_cast<int>(roi[0]) == n && sw <= w0 + kTileW - 1 && ew >= w0 &&
            sh <= h0 + kTileH - 1 && eh >= h0;
    }
    int pos;
    const int cnt = compact_ordered(hit, s_wcount, pos);
    if (hit) {
      PoolRoi q;
      q.r = i;
      q.sw = sw;
      q.sh = sh;
      q.ew = ew;
      q.eh = eh;
      q.bin_w = __fdiv_rn(static_cast<float>(max(ew - sw + 1, 1)), static_cast<float>(PW));
      q.bin_h = __fdiv_rn(static_cast<float>(max(eh - sh + 1, 1)), static_cast<float>(PH));
      s_roi[pos] = q;
    }
    __syncthreads();
    if (h < H && w < W) {
      for (int j = 0; j < cnt; ++j) {
        const PoolRoi q = s_roi[j];
        if (!(w >= q.sw && w <= q.ew && h >= q.sh && h <= q.eh)) continue;   // :123-127
        // feasible pooled cells (:145-153)
        const int phs = min(max(static_cast<int>(floorf(__fdiv_rn(static_cast<float>(h - q.sh), q.bin_h))), 0), PH);
        const int phe = min(max(static_cast<int>(ceilf(__fdiv_rn(static_cast<float>(h - q.sh + 1), q.bin_h))), 0), PH);
        const int pws = min(max(static_cast<int>(floorf(__fdiv_rn(static_cast<float>(w - q.sw), q.bin_w))), 0), PW);
        const int pwe = min(max(static_cast<int>(ceilf(__fdiv_rn(static_cast<float>(w - q.sw + 1), q.bin_w))), 0), PW);
        const long long off = (static_cast<long long>(q.r) * C + c0) * PP;
        for (int ph = phs; ph < phe; ++ph)
          for (int pw = pws; pw < pwe; ++pw) {
            const long long o = off + ph * PW + pw;
#pragma unroll
            for (int k = 0; k < kSlab; ++k)
              if (k < nk && __ldg(argmax + o + k * PP) == idx)
                acc[k] = __fadd_rn(acc[k], __ldg(top_diff + o + k * PP));   // :157-159
          }
      }
    }
    __syncthreads();
  }
  if (h < H && w < W) {
    float* o = feat_diff + ((static_cast<long long>(n) * C + c0) * H + h) * W + w;
#pragma unroll
    for (int k = 0; k < kSlab; ++k)
      if (k < nk) o[static_cast<long long>(k) * H * W] = acc[k];
  }
}

inline int grid_for(long long n, int block, int cap) {
  long long g = (n + block - 1) / block;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return static_cast<int>(g);
}

inline dim3 tile_grid(int B, int C, int H, int W) {
  return dim3(((H + kTileH - 1) / kTileH) * ((W + kTileW - 1) / kTileW), (C + kSlab - 1) / kSlab, B);
}

}  // namespace
}  // namespace mnc

using namespace mnc;

extern "C" int mnc_roi_warp_backward_nchw(const float* feat, int B, int C, int H, int W,
                                          const float* rois, int R, int pooled_h, int pooled_w,
                                          float spatial_scale, const float* top_diff,
                                          float* feat_diff, float* rois_diff, void* stream) {
  if (R <= 0) return MNC_OK;
  if (pooled_h <= 0 || pooled_w <= 0 || pooled_h > kMaxPooled || pooled_w > kMaxPooled ||
      B <= 0 || C <= 0 || H <= 0 || W <= 0 || B > 65535)
    return MNC_ERR_ARG;
  auto s = static_cast<cudaStream_t>(stream);
  if (feat_diff) {
    roi_warp_bwd_feat_kernel<<<tile_grid(B, C, H, W), kTileThreads, 0, s>>>(
        rois, R, C, H, W, pooled_h, pooled_w, spatial_scale, top_diff, feat_diff);
    if (check_launch() != MNC_OK) return MNC_ERR_CUDA;
  }
  if (rois_diff) {
    const int slabs = (C + kCoordSlab - 1) / kCoordSlab;
    double* partial = nullptr;
    if (cudaMallocAsync(reinterpret_cast<void**>(&partial),
                        sizeof(double) * 4 * static_cast<size_t>(R) * slabs, s) != cudaSuccess)
      return MNC_ERR_CUDA;
    roi_warp_bwd_coord_kernel<<<dim3(R, slabs), kCoordThreads, 0, s>>>(
        feat, B, C, H, W, rois, pooled_h, pooled_w, spatial_scale, top_diff, partial);
    roi_warp_bwd_coord_sum_kernel<<<grid_for(5LL * R, 256, 1 << 30), 256, 0, s>>>(partial, R, slabs, rois_diff);
    const int rc = check_launch();
    if (cudaFreeAsync(partial, s) != cudaSuccess || rc != MNC_OK) return MNC_ERR_CUDA;
  }
  return MNC_OK;
}

extern "C" int mnc_mask_resize_backward_nchw(const float* top_diff, int N, int C, int in_h,
                                             int in_w, int out_h, int out_w, float* in_diff,
                                             void* stream) {
  const long long total = static_cast<long long>(N) * C * in_h * in_w;
  if (total <= 0) return MNC_OK;
  if (out_h <= 0 || out_w <= 0) return MNC_ERR_ARG;
  mask_resize_bwd_kernel<<<grid_for(total, 256, 132 * 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      top_diff, static_cast<long long>(N) * C, in_h, in_w, out_h, out_w, in_diff);
  return check_launch();
}

extern "C" int mnc_mask_pool_backward_nchw(const float* feat, const float* mask,
                                           const float* top_diff, int N, int C, int H, int W,
                                           float* feat_diff, float* mask_diff, void* stream) {
  const long long total = static_cast<long long>(N) * C * H * W;
  if (total <= 0) return MNC_OK;
  auto s = static_cast<cudaStream_t>(stream);
  const int hw = H * W;
  if (feat_diff)
    mask_pool_bwd_feat_kernel<<<grid_for(total, 256, 132 * 16), 256, 0, s>>>(top_diff, mask, C, hw,
                                                                             total, feat_diff);
  if (mask_diff) {
    const long long nm = static_cast<long long>(N) * hw;
    mask_pool_bwd_mask_kernel<<<grid_for(nm, 128, 132 * 16), 128, 0, s>>>(top_diff, feat, C, hw, nm,
                                                                          mask_diff);
  }
  return check_launch();
}

extern "C" int mnc_roi_pool_backward_nchw(const float* top_diff, const int* argmax, int B, int C,
                                          int H, int W, const float* rois, int R, int pooled_h,
                                          int pooled_w, float spatial_scale, float* feat_diff,
                                          void* stream) {
  if (R <= 0) return MNC_OK;
  if (pooled_h <= 0 || pooled_w <= 0 || pooled_h > kMaxPooled || pooled_w > kMaxPooled ||
      B <= 0 || C <= 0 || H <= 0 || W <= 0 || B > 65535)
    return MNC_ERR_ARG;
  if (!feat_diff) return MNC_OK;
  roi_pool_bwd_kernel<<<tile_grid(B, C, H, W), kTileThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      rois, R, C, H, W, pooled_h, pooled_w, spatial_scale, top_diff, argmax, feat_diff);
  return check_launch();
}
