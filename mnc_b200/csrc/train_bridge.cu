// TRAIN phase of the two cascade bridge layers, one image, fp32 device blobs.  Replaces the
// reference's numpy/cv2 Python layers
//   StageBridgeLayer  lib/pylayer/stage_bridge_layer.py:131-235 (forward_train), :82-129 (backward)
//   MaskLayer         lib/pylayer/mask_layer.py:56-93 (forward_train), :50-54 (backward)
// with the helpers they call (lib/transform/bbox_transform.py:39-203, mask_transform.py:16-80,
// lib/utils/bbox.pyx).  Both layers are deterministic, so the arithmetic is kept exactly: float64
// where numpy promotes to float64, float32 where it stays in float32, every operation rounded
// separately (__dmul_rn / __fadd_rn ...) in numpy's order, np.around as rint (half to even).
// DESIGN.md "Training-phase bridge layers" lists the reference's quirks kept here.
//
// Stream-ordered and sync-free: StageBridge keeps every row (K = n + G, foreground first), so every
// output size is known on the host and forward + backward can be captured in a CUDA graph.
//   * stage_bridge_rows_kernel (one CTA) decodes, clips and assigns every row twice: a first pass
//     counts the foreground rows, the second places each row by a block scan (stable partition)
//     and writes its outputs and the state the backward reads.
//   * stage_bridge_masks_kernel (one CTA per output row) restates intersect_mask
//     (mask_target.cuh, shared with ProposalTargetLayer in rpn_train.cu).
//   * stage_bridge_backward_kernel: one warp per bottom row writes that whole row through the
//     inverse permutation -- no memset, no atomics.
//   * mask_layer_train_kernel (one CTA per RoI) counts mask_overlap's pixels with integers.
#include <cuda_runtime.h>

#include "mnc_b200.h"
#include "cv_resize.cuh"
#include "mask_target.cuh"
#include "launch_util.h"

namespace mnc {
namespace {

constexpr int kRowThreads = 512;
constexpr int kMaskThreads = 256;

struct BridgeCfg {
  double mean[4], std_[4];
  int normalize;
  float inside[4];
  double bbox_thresh;
  float binarize_thresh;
};

// Exclusive rank of `flag` among the block's threads (thread order) and the block's total.
__device__ __forceinline__ int block_rank(bool flag, int* wcount, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, flag);
  __syncthreads();                                   // wcount may still be read by the last call
  if (lane == 0) wcount[warp] = __popc(m);
  __syncthreads();
  int off = 0;
  total = 0;
#pragma unroll
  for (int k = 0; k < kRowThreads / 32; ++k) {
    const int c = wcount[k];
    off += k < warp ? c : 0;
    total += c;
  }
  return off + __popc(m & ((1u << lane) - 1u));
}

struct Row {
  double b[4];   // clipped box
  int keep;      // clip_boxes' keep: the unclipped box lies inside the image
  int a;         // gt assignment (first maximum)
  int reg;       // regression label (rows < n)
  bool fg;
};

// One row of all_rois (stage_bridge_layer.py:141-165) and its assignment (_sample_output
// :188-195).  Rows < n are RoIs decoded with the regression label's deltas, rows >= n the gt boxes.
__device__ Row bridge_row(int i, const float* __restrict__ rois, int n,
                          const float* __restrict__ bbox_pred, const float* __restrict__ seg, int C,
                          const float* __restrict__ gt, int G, const float* __restrict__ im_info,
                          double bbox_thresh) {
  Row r;
  r.reg = 0;
  double x1, y1, x2, y2;
  if (i < n) {
    const float* s = seg + static_cast<long long>(i) * C;
    int best = 1;                                    // argmax over classes 1..C-1, first max
    for (int c = 2; c < C; ++c)
      if (s[c] > s[best]) best = c;
    r.reg = best;
    const float* d = bbox_pred + static_cast<long long>(i) * 4 * C + 4 * best;
    const float* b = rois + static_cast<long long>(i) * 5;
    // bbox_transform_inv (bbox_transform.py:64-99) on float64: the deltas are float64 (:153)
    const double bx1 = b[1], by1 = b[2], bx2 = b[3], by2 = b[4];
    const double w = __dadd_rn(__dsub_rn(bx2, bx1), 1.0), h = __dadd_rn(__dsub_rn(by2, by1), 1.0);
    const double cx = __dadd_rn(bx1, __dmul_rn(0.5, w)), cy = __dadd_rn(by1, __dmul_rn(0.5, h));
    const double pcx = __dadd_rn(__dmul_rn(static_cast<double>(d[0]), w), cx);
    const double pcy = __dadd_rn(__dmul_rn(static_cast<double>(d[1]), h), cy);
    const double pw = __dmul_rn(exp(static_cast<double>(d[2])), w);
    const double ph = __dmul_rn(exp(static_cast<double>(d[3])), h);
    x1 = __dsub_rn(pcx, __dmul_rn(0.5, pw));
    y1 = __dsub_rn(pcy, __dmul_rn(0.5, ph));
    x2 = __dadd_rn(pcx, __dmul_rn(0.5, pw));
    y2 = __dadd_rn(pcy, __dmul_rn(0.5, ph));
  } else {
    const float* g = gt + static_cast<long long>(i - n) * 5;
    x1 = g[0];
    y1 = g[1];
    x2 = g[2];
    y2 = g[3];
  }
  // clip_boxes (bbox_transform.py:102-120); im_shape - 1 is float32 arithmetic
  const double hm1 = __fsub_rn(im_info[0], 1.f), wm1 = __fsub_rn(im_info[1], 1.f);
  r.keep = x1 >= 0 && x2 <= wm1 && y1 >= 0 && y2 <= hm1;
  r.b[0] = fmax(fmin(x1, wm1), 0.0);
  r.b[1] = fmax(fmin(y1, hm1), 0.0);
  r.b[2] = fmax(fmin(x2, wm1), 0.0);
  r.b[3] = fmax(fmin(y2, hm1), 0.0);
  // bbox_overlaps (bbox.pyx:15-55) against every gt box, first maximum
  double best = 0.0;
  r.a = 0;
  const double area = __dmul_rn(__dadd_rn(__dsub_rn(r.b[2], r.b[0]), 1.0),
                                __dadd_rn(__dsub_rn(r.b[3], r.b[1]), 1.0));
  for (int k = 0; k < G; ++k) {
    const float* g = gt + k * 5;
    const double q0 = g[0], q1 = g[1], q2 = g[2], q3 = g[3];
    const double qa = __dmul_rn(__dadd_rn(__dsub_rn(q2, q0), 1.0), __dadd_rn(__dsub_rn(q3, q1), 1.0));
    double ov = 0.0;
    const double iw = __dadd_rn(__dsub_rn(fmin(r.b[2], q2), fmax(r.b[0], q0)), 1.0);
    if (iw > 0) {
      const double ih = __dadd_rn(__dsub_rn(fmin(r.b[3], q3), fmax(r.b[1], q1)), 1.0);
      if (ih > 0) {
        const double ua = __dsub_rn(__dadd_rn(area, qa), __dmul_rn(iw, ih));
        ov = __ddiv_rn(__dmul_rn(iw, ih), ua);
      }
    }
    if (k == 0 || ov > best) {
      best = ov;
      r.a = k;
    }
  }
  r.fg = best >= bbox_thresh;
  return r;
}

// grid 1, kRowThreads threads.
__global__ void __launch_bounds__(kRowThreads)
stage_bridge_rows_kernel(const float* __restrict__ rois, int n, const float* __restrict__ bbox_pred,
                         const float* __restrict__ seg, int C, const float* __restrict__ gt, int G,
                         const float* __restrict__ im_info, const int* __restrict__ mask_info,
                         BridgeCfg cfg, float* __restrict__ rois_out, float* __restrict__ labels,
                         float* __restrict__ info_out, float* __restrict__ bbox_targets,
                         float* __restrict__ bbox_inside, float* __restrict__ bbox_outside,
                         int* __restrict__ state) {
  __shared__ int wcount[kRowThreads / 32];
  const int K = n + G;
  int nfg = 0;
  for (int base = 0; base < K; base += kRowThreads) {
    const int i = base + threadIdx.x;
    const bool fg = i < K && bridge_row(i, rois, n, bbox_pred, seg, C, gt, G, im_info,
                                        cfg.bbox_thresh).fg;
    int total;
    block_rank(fg, wcount, total);
    nfg += total;
  }
  int* keep = state;
  int* inv = state + K;
  int* reg = state + 2 * K;
  int* clip = state + 2 * K + n;
  if (threadIdx.x == 0) state[2 * K + 2 * n] = nfg;
  const float im_scale = im_info[2];
  int fg_before = 0;
  for (int base = 0; base < K; base += kRowThreads) {
    const int i = base + threadIdx.x;
    Row r;
    r.fg = false;
    if (i < K) r = bridge_row(i, rois, n, bbox_pred, seg, C, gt, G, im_info, cfg.bbox_thresh);
    int total;
    const int rank = block_rank(i < K && r.fg, wcount, total);
    if (i < K) {
      // stable partition (:195-197): foreground rows, then background rows, each in index order
      const int p = r.fg ? fg_before + rank : nfg + (i - fg_before - rank);
      keep[p] = i;
      inv[i] = p;
      if (i < n) {
        reg[i] = r.reg;
        clip[i] = r.keep;
      }
      float* ro = rois_out + static_cast<long long>(p) * 5;
      ro[0] = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) ro[k + 1] = static_cast<float>(r.b[k]);
      const float* g = gt + r.a * 5;
      const float label = r.fg ? g[4] : 0.f;         // background clamped to 0 (:201)
      labels[p] = label;

      // bbox_compute_targets / get_bbox_regression_label (bbox_transform.py:39-61,157-203)
      const int C4 = 4 * C;
      float* bt = bbox_targets + static_cast<long long>(p) * C4;
      float* bi = bbox_inside + static_cast<long long>(p) * C4;
      float* bo = bbox_outside + static_cast<long long>(p) * C4;
      for (int c = 0; c < C4; ++c) bt[c] = bi[c] = bo[c] = 0.f;
      if (label > 0.f) {
        const double ew = __dadd_rn(__dsub_rn(r.b[2], r.b[0]), 1.0);
        const double eh = __dadd_rn(__dsub_rn(r.b[3], r.b[1]), 1.0);
        const double ecx = __dadd_rn(r.b[0], __dmul_rn(0.5, ew));
        const double ecy = __dadd_rn(r.b[1], __dmul_rn(0.5, eh));
        const float gw = __fadd_rn(__fsub_rn(g[2], g[0]), 1.f);   // float32 gt side
        const float gh = __fadd_rn(__fsub_rn(g[3], g[1]), 1.f);
        const float gcx = __fadd_rn(g[0], __fmul_rn(0.5f, gw));
        const float gcy = __fadd_rn(g[1], __fmul_rn(0.5f, gh));
        double t[4];
        t[0] = __ddiv_rn(__dsub_rn(static_cast<double>(gcx), ecx), ew);
        t[1] = __ddiv_rn(__dsub_rn(static_cast<double>(gcy), ecy), eh);
        t[2] = log(__ddiv_rn(static_cast<double>(gw), ew));
        t[3] = log(__ddiv_rn(static_cast<double>(gh), eh));
        const int start = static_cast<int>(__fmul_rn(4.f, label));
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const double v = cfg.normalize ? __ddiv_rn(__dsub_rn(t[k], cfg.mean[k]), cfg.std_[k]) : t[k];
          const int c = start + k;
          if (c < 0 || c >= C4) continue;
          bt[c] = static_cast<float>(v);
          bi[c] = cfg.inside[k];
          bo[c] = cfg.inside[k] > 0.f ? 1.f : 0.f;
        }
      }

      // gt_mask_info (:211-233): ex box in float64, gt box float32 / im_scale, np.around
      float* mi = info_out + static_cast<long long>(p) * 12;
      if (r.fg) {
        mi[0] = static_cast<float>(r.a);
        mi[1] = static_cast<float>(mask_info[r.a * 2 + 0]);
        mi[2] = static_cast<float>(mask_info[r.a * 2 + 1]);
        mi[3] = label;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          mi[4 + k] = static_cast<float>(static_cast<int>(rint(__ddiv_rn(r.b[k], static_cast<double>(im_scale)))));
          mi[8 + k] = static_cast<float>(static_cast<int>(rintf(__fdiv_rn(g[k], im_scale))));
        }
      } else {
#pragma unroll
        for (int k = 0; k < 12; ++k) mi[k] = -1.f;
      }
    }
    fg_before += total;
  }
}

// grid K, kMaskThreads threads: the mask target of row p (mask_target.cuh); mask_weight 1 for the
// first nfg rows (:172-173).
__global__ void __launch_bounds__(kMaskThreads)
stage_bridge_masks_kernel(const float* __restrict__ info, const int* __restrict__ state, int K,
                          int n, const float* __restrict__ gt_masks, int G, int Hm, int Wm, int M,
                          float thresh, float* __restrict__ targets, float* __restrict__ weight) {
  const int p = blockIdx.x;
  const int MM = M * M;
  const bool fg = p < state[2 * K + 2 * n];
  float* t = targets + static_cast<long long>(p) * MM;
  float* w = weight + static_cast<long long>(p) * MM;
  mask_target_row(info + static_cast<long long>(p) * 12, fg, gt_masks, G, Hm, Wm, M, thresh, t, w);
}

// grid ceil(n / 8), 256 threads: one warp per bottom row i (stage_bridge_layer.py:82-129).
__global__ void __launch_bounds__(256)
stage_bridge_backward_kernel(const float* __restrict__ top_diff, const int* __restrict__ state,
                             int n, int K, const float* __restrict__ rois,
                             const float* __restrict__ bbox_pred, int C, float clip_thresh,
                             float* __restrict__ rois_diff, float* __restrict__ bbox_diff) {
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= n) return;
  const int p = state[K + i], l = state[2 * K + i], keep = state[2 * K + n + i];
  const float* td = top_diff + static_cast<long long>(p) * 5;
  const float* d = bbox_pred + static_cast<long long>(i) * 4 * C + 4 * l;
  const float* b = rois + static_cast<long long>(i) * 5;
  // np.exp on float32, correctly rounded
  const float ew = static_cast<float>(exp(static_cast<double>(d[2])));
  const float eh = static_cast<float>(exp(static_cast<double>(d[3])));
  if (rois_diff && lane < 5) {
    float v = 0.f;
    if (lane == 1 || lane == 2) v = td[lane];
    if (lane == 3) v = __fmul_rn(td[3], __fadd_rn(d[0], ew));   // delta_x, not delta_w (:107)
    if (lane == 4) v = __fmul_rn(td[4], __fadd_rn(d[1], eh));
    rois_diff[static_cast<long long>(i) * 5 + lane] = v;
  }
  if (bbox_diff) {
    // W_old / H_old index the 5-column blob: y1 - batch index and x2 - x1 (:93-94)
    const float W_old = __fsub_rn(b[2], b[0]), H_old = __fsub_rn(b[3], b[1]);
    float g[4];
    g[0] = __fmul_rn(td[1], W_old);
    g[1] = __fmul_rn(td[2], H_old);
    g[2] = __fmul_rn(__fmul_rn(td[3], ew), W_old);
    g[3] = __fmul_rn(__fmul_rn(td[4], eh), H_old);
    float* out = bbox_diff + static_cast<long long>(i) * 4 * C;
    for (int c = lane; c < 4 * C; c += 32) {
      float v = 0.f;
      if (keep && c >= 4 * l && c < 4 * l + 4) {
        v = g[c - 4 * l];
        if (clip_thresh > 0.f) v = fminf(fmaxf(v, -clip_thresh), clip_thresh);
      }
      out[c] = v;
    }
  }
}

__device__ __forceinline__ int block_sum(int v, int* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  int s = 0;
#pragma unroll
  for (int k = 0; k < kMaskThreads / 32; ++k) s += red[k];
  return s;
}

// grid N, kMaskThreads threads: MaskLayer.forward_train (mask_layer.py:68-83) for RoI i.
__global__ void __launch_bounds__(kMaskThreads)
mask_layer_train_kernel(const float* __restrict__ pred, int M, const float* __restrict__ gt_masks,
                        int G, int Hm, int Wm, const float* __restrict__ info, float thresh,
                        double fg_thresh, float* __restrict__ labels) {
  __shared__ int red[kMaskThreads / 32];
  const int i = blockIdx.x;
  const float* mi = info + static_cast<long long>(i) * 12;
  if (mi[0] == -1.f) {
    if (threadIdx.x == 0) labels[i] = 0.f;
    return;
  }
  // float-valued entries used as indices truncate; the boxes go through np.round
  const int a = static_cast<int>(mi[0]), mh = static_cast<int>(mi[1]), mw = static_cast<int>(mi[2]);
  const int ex1 = static_cast<int>(rintf(mi[4])), ey1 = static_cast<int>(rintf(mi[5]));
  const int ex2 = static_cast<int>(rintf(mi[6])), ey2 = static_cast<int>(rintf(mi[7]));
  const int gx1 = static_cast<int>(rintf(mi[8])), gy1 = static_cast<int>(rintf(mi[9]));
  const int gx2 = static_cast<int>(rintf(mi[10])), gy2 = static_cast<int>(rintf(mi[11]));
  const int ew = ex2 - ex1 + 1, eh = ey2 - ey1 + 1;
  const int ix1 = max(ex1, gx1), iy1 = max(ey1, gy1), ix2 = min(ex2, gx2), iy2 = min(ey2, gy2);
  const bool has_gt = a >= 0 && a < G;
  const float* m = gt_masks + static_cast<long long>(a) * Hm * Wm;
  const float* mp = pred + static_cast<long long>(i) * M * M;
  int m1 = 0, inter = 0, m2 = 0;
  if (ew > 0 && eh > 0) {
    for (long long s = threadIdx.x; s < static_cast<long long>(ew) * eh; s += blockDim.x) {
      const int dx = static_cast<int>(s % ew), dy = static_cast<int>(s / ew);
      int x0, x1, y0, y1;
      float ax0, ax1, ay0, ay1;
      cv_tap(dx, static_cast<double>(M) / ew, M, x0, x1, ax0, ax1);
      cv_tap(dy, static_cast<double>(M) / eh, M, y0, y1, ay0, ay1);
      const float r0 = __fadd_rn(__fmul_rn(mp[y0 * M + x0], ax0), __fmul_rn(mp[y0 * M + x1], ax1));
      const float r1 = __fadd_rn(__fmul_rn(mp[y1 * M + x0], ax0), __fmul_rn(mp[y1 * M + x1], ax1));
      if (__fadd_rn(__fmul_rn(r0, ay0), __fmul_rn(r1, ay1)) >= thresh) {
        ++m1;
        const int x = ex1 + dx, y = ey1 + dy;
        if (has_gt && x >= ix1 && x <= ix2 && y >= iy1 && y <= iy2 &&
            gt_plane(m, Hm, Wm, mh, mw, gx1, gy1, x, y) != 0.f)
          ++inter;
      }
    }
  }
  if (has_gt) {
    const int ch = min(mh, Hm), cw = min(mw, Wm);
    for (long long s = threadIdx.x; s < static_cast<long long>(max(ch, 0)) * max(cw, 0); s += blockDim.x)
      m2 += m[(s / cw) * Wm + s % cw] != 0.f;
  }
  m1 = block_sum(m1, red);
  inter = block_sum(inter, red);
  m2 = block_sum(m2, red);
  if (threadIdx.x != 0) return;
  // mask_overlap (mask_transform.py:16-46): 0 for disjoint boxes or a union below 1
  double iou = 0.0;
  if (ix1 <= ix2 && iy1 <= iy2) {
    const double uni = static_cast<double>(m1) + m2 - inter;
    if (!(uni < 1.0)) iou = static_cast<double>(inter) / uni;
  }
  labels[i] = iou < fg_thresh ? 0.f : mi[3];
}

// mask_layer.py:50-54: rows with a positive label copy the top diff, the others are 0.
__global__ void mask_layer_backward_kernel(const float* __restrict__ top_diff,
                                           const float* __restrict__ labels, long long total, int S,
                                           float* __restrict__ bottom_diff) {
  for (long long j = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; j < total;
       j += static_cast<long long>(gridDim.x) * blockDim.x)
    bottom_diff[j] = labels[j / S] > 0.f ? top_diff[j] : 0.f;
}

}  // namespace
}  // namespace mnc

extern "C" int mnc_stage_bridge_train(
    const float* rois, int n, const float* bbox_pred, const float* seg_cls_prob, int num_classes,
    const float* gt_boxes, int G, const float* gt_masks, int mask_h, int mask_w,
    const float* im_info, const int* mask_info, const double* means, const double* stds,
    const float* inside_weights, double bbox_thresh, int mask_size, float binarize_thresh,
    float* rois_out, float* labels, float* mask_targets, float* mask_weight, float* gt_mask_info,
    float* bbox_targets, float* bbox_inside_weights, float* bbox_outside_weights, int* state,
    void* stream) {
  if (n < 0 || G <= 0 || num_classes < 2 || mask_h <= 0 || mask_w <= 0 || mask_size <= 0 ||
      !inside_weights || (means == nullptr) != (stds == nullptr))
    return MNC_ERR_ARG;
  mnc::BridgeCfg cfg;
  cfg.normalize = means != nullptr;
  for (int k = 0; k < 4; ++k) {
    cfg.mean[k] = means ? means[k] : 0.0;
    cfg.std_[k] = stds ? stds[k] : 1.0;
    cfg.inside[k] = inside_weights[k];
  }
  cfg.bbox_thresh = bbox_thresh;
  cfg.binarize_thresh = binarize_thresh;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int K = n + G;
  mnc::stage_bridge_rows_kernel<<<1, mnc::kRowThreads, 0, s>>>(
      rois, n, bbox_pred, seg_cls_prob, num_classes, gt_boxes, G, im_info, mask_info, cfg,
      rois_out, labels, gt_mask_info, bbox_targets, bbox_inside_weights, bbox_outside_weights,
      state);
  mnc::stage_bridge_masks_kernel<<<K, mnc::kMaskThreads, 0, s>>>(
      gt_mask_info, state, K, n, gt_masks, G, mask_h, mask_w, mask_size, binarize_thresh,
      mask_targets, mask_weight);
  return mnc::check_launch();
}

extern "C" int mnc_stage_bridge_train_backward(const float* top_diff, const int* state,
                                               const float* rois, const float* bbox_pred, int n,
                                               int G, int num_classes, float clip_thresh,
                                               float* rois_diff, float* bbox_pred_diff,
                                               void* stream) {
  if (n < 0 || G <= 0 || num_classes < 2 || clip_thresh < 0.f) return MNC_ERR_ARG;
  if (n == 0 || (!rois_diff && !bbox_pred_diff)) return MNC_OK;
  mnc::stage_bridge_backward_kernel<<<(n + 7) / 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      top_diff, state, n, n + G, rois, bbox_pred, num_classes, clip_thresh, rois_diff,
      bbox_pred_diff);
  return mnc::check_launch();
}

extern "C" int mnc_mask_layer_train(const float* mask_pred, int N, int mask_size,
                                    const float* gt_masks, int G, int mask_h, int mask_w,
                                    const float* gt_masks_info, float binarize_thresh,
                                    double fg_seg_thresh, float* labels, void* stream) {
  if (N < 0 || mask_size <= 0 || G <= 0 || mask_h <= 0 || mask_w <= 0) return MNC_ERR_ARG;
  if (N == 0) return MNC_OK;
  mnc::mask_layer_train_kernel<<<N, mnc::kMaskThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      mask_pred, mask_size, gt_masks, G, mask_h, mask_w, gt_masks_info, binarize_thresh,
      fg_seg_thresh, labels);
  return mnc::check_launch();
}

extern "C" int mnc_mask_layer_train_backward(const float* top_diff, const float* labels, int N,
                                             int mask_size, float* bottom_diff, void* stream) {
  if (N < 0 || mask_size <= 0) return MNC_ERR_ARG;
  if (N == 0) return MNC_OK;
  const long long total = static_cast<long long>(N) * mask_size * mask_size;
  const int grid = static_cast<int>(total / 256 + 1 < 1024 ? total / 256 + 1 : 1024);
  mnc::mask_layer_backward_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      top_diff, labels, total, mask_size * mask_size, bottom_diff);
  return mnc::check_launch();
}
