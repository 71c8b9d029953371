// TRAIN phase of the three RPN-stage Python layers, one image, fp32 device blobs.  Replaces
//   ProposalLayer        lib/pylayer/proposal_layer.py:52-175 (TRAIN tops), :177-230 (backward)
//   ProposalTargetLayer  lib/pylayer/proposal_target_layer.py:62-216, backward :109-115
//   AnchorTargetLayer    lib/pylayer/anchor_target_layer.py:51-209 (its backward is a no-op)
// with the helpers they call (lib/transform/bbox_transform.py, mask_transform.py:49-80,
// lib/utils/bbox.pyx).  Arithmetic follows numpy's dtypes operation by operation, as in
// train_bridge.cu; DESIGN.md "RPN-stage training layers" lists the quirks kept.
//
// Random sampling is an input.  Where the reference draws npr.choice(cands, size, replace=False)
// and uses only the chosen SET, the set here is the `size` candidates with the smallest
// (key, index) pairs, keys being uint32 the caller supplies (i.i.d. uniform keys give a uniform
// random subset, numpy's distribution).  select_smallest() finds it with an 8-bit radix select over
// the keys (integer histogram counts, so order-free) and a block scan over the tie-breaking index.
//
// Stream-ordered, sync-free, deterministic: data-dependent counts stay on the device; the outputs of
// ProposalTargetLayer are written at a capacity Kmax the host computes from the config.
#include <cuda_runtime.h>

#include "mnc_b200.h"
#include "bbox_decode.cuh"
#include "mask_target.cuh"
#include "launch_util.h"

namespace mnc {
namespace {

constexpr int kA = 9;                 // anchors per position (generate_anchors)
constexpr int kSelThreads = 1024;
constexpr int kMaskThreads = 256;
constexpr int kMaxCats = 4;

struct AnchorTable {
  float v[kA][4];
};

// bbox.pyx:15-55 for one box pair, float64.
__device__ __forceinline__ double iou64(double b0, double b1, double b2, double b3, const float* q) {
  const double q0 = q[0], q1 = q[1], q2 = q[2], q3 = q[3];
  const double qa = __dmul_rn(__dadd_rn(__dsub_rn(q2, q0), 1.0), __dadd_rn(__dsub_rn(q3, q1), 1.0));
  const double iw = __dadd_rn(__dsub_rn(fmin(b2, q2), fmax(b0, q0)), 1.0);
  if (!(iw > 0)) return 0.0;
  const double ih = __dadd_rn(__dsub_rn(fmin(b3, q3), fmax(b1, q1)), 1.0);
  if (!(ih > 0)) return 0.0;
  const double area = __dmul_rn(__dadd_rn(__dsub_rn(b2, b0), 1.0), __dadd_rn(__dsub_rn(b3, b1), 1.0));
  const double ua = __dsub_rn(__dadd_rn(area, qa), __dmul_rn(iw, ih));
  return __ddiv_rn(__dmul_rn(iw, ih), ua);
}

// Block-wide helpers for one CTA of kSelThreads threads.
struct SelShared {
  int hist[256];
  int wcount[kSelThreads / 32];
  int total;
  int digit, need;
};

__device__ int block_count(bool flag, SelShared& sh) {
  const unsigned m = __ballot_sync(0xffffffffu, flag);
  __syncthreads();
  if (threadIdx.x == 0) sh.total = 0;
  __syncthreads();
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(&sh.total, __popc(m));
  __syncthreads();
  return sh.total;
}

// Exclusive rank of `flag` among the block's threads (thread order) and the block's total.
__device__ int block_rank(bool flag, SelShared& sh, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, flag);
  __syncthreads();
  if (lane == 0) sh.wcount[warp] = __popc(m);
  __syncthreads();
  int off = 0;
  total = 0;
#pragma unroll 8
  for (int k = 0; k < kSelThreads / 32; ++k) {
    const int c = sh.wcount[k];
    off += k < warp ? c : 0;
    total += c;
  }
  return off + __popc(m & ((1u << lane) - 1u));
}

// Number of i < N with cand(i).
template <class Cand>
__device__ int count_cands(int N, Cand cand, SelShared& sh) {
  int c = 0;
  for (int base = 0; base < N; base += kSelThreads) {
    const int i = base + threadIdx.x;
    c += block_count(i < N && cand(i), sh);
  }
  return c;
}

// Calls take(i) for the cnt candidates with the smallest (keys[i], i); 0 <= cnt <= #candidates.
template <class Cand, class Take>
__device__ void select_smallest(const unsigned* __restrict__ keys, int N, int cnt, Cand cand,
                                Take take, SelShared& sh) {
  if (cnt <= 0) return;                              // block-uniform
  unsigned prefix = 0, mask = 0;
  int need = cnt;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int b = threadIdx.x; b < 256; b += kSelThreads) sh.hist[b] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < N; i += kSelThreads) {
      if (!cand(i)) continue;
      const unsigned k = keys[i];
      if ((k & mask) == prefix) atomicAdd(&sh.hist[(k >> shift) & 255u], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int cum = 0, d = 0;
      for (; d < 255 && cum + sh.hist[d] < need; ++d) cum += sh.hist[d];
      sh.digit = d;
      sh.need = need - cum;
    }
    __syncthreads();
    prefix |= static_cast<unsigned>(sh.digit) << shift;
    mask |= 255u << shift;
    need = sh.need;
    __syncthreads();
  }
  // every key below `prefix`, and the first `need` (by index) of those equal to it
  int before = 0;
  for (int base = 0; base < N; base += kSelThreads) {
    const int i = base + threadIdx.x;
    const bool c = i < N && cand(i);
    const unsigned k = c ? keys[i] : 0u;
    int total;
    const int r = block_rank(c && k == prefix, sh, total);
    if (c && (k < prefix || (k == prefix && before + r < need))) take(i);
    before += total;
  }
  __syncthreads();
}

// =============================================================================== ProposalLayer
// One thread per kept row k < R: proposal_index (the anchor index t in (h, w, a) order of the k-th
// RoI, proposal_layer.py:168-170) and the backward's state {t, weight_out_proposal *
// weight_out_anchor} -- clip_boxes' keep tests (bbox_transform.py:110) on the unclipped fp32
// proposal and on the float64 anchor (:105-106, :118-122).  Rows k >= count get index -1.
__global__ void proposal_train_state_kernel(const int* __restrict__ order,
                                            const int* __restrict__ keep,
                                            const int* __restrict__ num_keep, int R,
                                            const float* __restrict__ bbox, int H, int W,
                                            int feat_stride, const float* __restrict__ im_info,
                                            const AnchorTable anchors,
                                            float* __restrict__ proposal_index,
                                            int* __restrict__ state) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= R) return;
  if (k >= min(num_keep[0], R)) {
    proposal_index[k] = -1.f;
    state[2 * k] = -1;
    state[2 * k + 1] = 0;
    return;
  }
  const int t = order[keep[k]];
  const int a = t % kA, pix = t / kA;
  const int y = pix / W, x = pix % W;
  const long long HW = static_cast<long long>(H) * W;
  const float* d = bbox + static_cast<long long>(4 * a) * HW + pix;
  const float sx = static_cast<float>(x * feat_stride), sy = static_cast<float>(y * feat_stride);
  const float ax1 = anchors.v[a][0] + sx, ay1 = anchors.v[a][1] + sy;
  const float ax2 = anchors.v[a][2] + sx, ay2 = anchors.v[a][3] + sy;
  float cx, cy, pw, ph;
  decode_center(ax1, ay1, ax2, ay2, d[0], d[HW], d[2 * HW], d[3 * HW], cx, cy, pw, ph);
  const float px1 = __fsub_rn(cx, __fmul_rn(0.5f, pw)), py1 = __fsub_rn(cy, __fmul_rn(0.5f, ph));
  const float px2 = __fadd_rn(cx, __fmul_rn(0.5f, pw)), py2 = __fadd_rn(cy, __fmul_rn(0.5f, ph));
  const float wm1 = __fsub_rn(im_info[1], 1.f), hm1 = __fsub_rn(im_info[0], 1.f);
  const bool in_p = px1 >= 0.f && px2 <= wm1 && py1 >= 0.f && py2 <= hm1;
  const bool in_a = ax1 >= 0.f && ax2 <= wm1 && ay1 >= 0.f && ay2 <= hm1;   // exact integers
  proposal_index[k] = static_cast<float>(t);
  state[2 * k] = t;
  state[2 * k + 1] = in_p && in_a;
}

// One thread per kept row (proposal_layer.py:177-230); the diff was zeroed.  Row indices are unique
// anchors, so writes never collide.
__global__ void proposal_backward_kernel(const float* __restrict__ top_diff, int R,
                                         const int* __restrict__ state,
                                         const float* __restrict__ bbox, int H, int W,
                                         const AnchorTable anchors, float clip_thresh,
                                         float* __restrict__ bbox_diff) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= R) return;
  const int t = state[2 * k];
  if (t < 0) return;
  const float* td = top_diff + static_cast<long long>(k) * 5;
  bool nz = false;
#pragma unroll
  for (int j = 0; j < 5; ++j) nz |= fabsf(td[j]) > 0.f;   // top_non_zero_ind (:182)
  if (!nz) return;
  const double wgt = state[2 * k + 1] ? 1.0 : 0.0;
  const int c = t % kA, pix = t / kA;
  const long long HW = static_cast<long long>(H) * W;
  // anchor_w / anchor_h: float64 differences of the (integer) base anchors
  const double aw = static_cast<double>(anchors.v[c][2]) - static_cast<double>(anchors.v[c][0]);
  const double ah = static_cast<double>(anchors.v[c][3]) - static_cast<double>(anchors.v[c][1]);
  const float d1 = td[1], d2 = td[2], d3 = td[3], d4 = td[4];
  const float dxc = __fadd_rn(d1, d3), dyc = __fadd_rn(d2, d4);
  const float dfw = __fmul_rn(0.5f, __fsub_rn(d3, d1)), dfh = __fmul_rn(0.5f, __fsub_rn(d4, d2));
  const float* b = bbox + static_cast<long long>(4 * c) * HW + pix;
  const float ew = static_cast<float>(exp(static_cast<double>(b[2 * HW])));   // np.exp on float32
  const float eh = static_cast<float>(exp(static_cast<double>(b[3 * HW])));
  float v[4];
  v[0] = static_cast<float>(__dmul_rn(__dmul_rn(static_cast<double>(dxc), aw), wgt));
  v[1] = static_cast<float>(__dmul_rn(__dmul_rn(static_cast<double>(dyc), ah), wgt));
  v[2] = static_cast<float>(__dmul_rn(__dmul_rn(static_cast<double>(__fmul_rn(dfw, ew)), aw), wgt));
  v[3] = static_cast<float>(__dmul_rn(__dmul_rn(static_cast<double>(__fmul_rn(dfh, eh)), ah), wgt));
  float* out = bbox_diff + static_cast<long long>(4 * c) * HW + pix;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float x = v[j];
    if (clip_thresh > 0.f) x = fminf(fmaxf(x, -clip_thresh), clip_thresh);
    out[j * HW] = x;
  }
}

// ========================================================================= ProposalTargetLayer
struct PtCfg {
  int batch;                          // cfg.TRAIN.BATCH_SIZE (one image)
  int nfg, nbg;                       // category counts
  double fg_frac[kMaxCats], fg_lo[kMaxCats], fg_hi[kMaxCats];
  double bg_frac[kMaxCats], bg_lo[kMaxCats], bg_hi[kMaxCats];
  int normalize;
  double mean[4], std_[4];
  float inside[4];
};

// Layout of the int32 state buffer (N = n + G rows of all_rois):
//   fgpos[N] bgpos[N]   output position of row i in the fg / bg part of keep_inds, or -1
//   asg[N]              gt_assignment (first maximum)
//   sel[N]              bit 0 fg-sampled, bit 1 bg-sampled
//   keep[Kmax]          keep_inds, padded with -1
//   (8-byte aligned) max_overlaps[N] double
__host__ __device__ inline long long pt_mo_offset(int N, int Kmax) { return (4LL * N + Kmax + 1) & ~1LL; }
__host__ __device__ inline long long pt_state_ints(int N, int Kmax) { return pt_mo_offset(N, Kmax) + 2LL * N; }

// One CTA: overlaps, sampling, keep_inds and every per-row output except the mask targets.
__global__ void __launch_bounds__(kSelThreads)
proposal_target_kernel(const float* __restrict__ rpn_rois, int n,
                       const float* __restrict__ rois_index, const int* __restrict__ n_valid,
                       const float* __restrict__ gt, int G,
                       const int* __restrict__ mask_info, const float* __restrict__ im_info,
                       const unsigned* __restrict__ keys, PtCfg cfg, int C, int Kmax,
                       float* __restrict__ rois_out, float* __restrict__ labels,
                       float* __restrict__ bbox_targets, float* __restrict__ bbox_inside,
                       float* __restrict__ bbox_outside, float* __restrict__ info_out,
                       float* __restrict__ fg_inds, float* __restrict__ bg_inds,
                       int* __restrict__ counts, int* __restrict__ state) {
  __shared__ SelShared sh;
  const int N = n + G;
  int* fgpos = state;
  int* bgpos = state + N;
  int* asg = state + 2 * N;
  int* sel = state + 3 * N;
  int* keep = state + 4 * N;
  double* mo = reinterpret_cast<double*>(state + pt_mo_offset(N, Kmax));
  // rows [nv, n) are padding (ProposalLayer kept fewer than n): absent from all_rois, their max
  // overlap -inf puts them in no category
  const int nv = n_valid ? max(0, min(n_valid[0], n)) : n;

  // all_rois = rpn_rois ++ gt rows (:76-80); bbox_overlaps against every gt box (:127-132)
  for (int i = threadIdx.x; i < N; i += kSelThreads) {
    const float* b = i < n ? rpn_rois + static_cast<long long>(i) * 5 + 1 : gt + (i - n) * 5;
    const double b0 = b[0], b1 = b[1], b2 = b[2], b3 = b[3];
    double best = 0.0;
    int a = 0;
    for (int g = 0; g < G; ++g) {
      const double ov = iou64(b0, b1, b2, b3, gt + g * 5);
      if (g == 0 || ov > best) {
        best = ov;
        a = g;
      }
    }
    mo[i] = i >= nv && i < n ? -INFINITY : best;
    asg[i] = a;
    sel[i] = 0;
  }
  __syncthreads();

  // foreground categories (:137-146), then background (:148-159); np.round is half to even
  for (int c = 0; c < cfg.nfg; ++c) {
    const double lo = cfg.fg_lo[c], hi = cfg.fg_hi[c];
    auto cand = [&](int i) { return mo[i] >= lo && mo[i] <= hi; };
    const int size = count_cands(N, cand, sh);
    const double want = rint(static_cast<double>(cfg.batch) * cfg.fg_frac[c]);
    const int cnt = static_cast<int>(fmin(static_cast<double>(size), fmax(want, 0.0)));
    select_smallest(keys + static_cast<long long>(c) * N, N, cnt, cand,
                    [&](int i) { sel[i] |= 1; }, sh);
  }
  const int nfg = count_cands(N, [&](int i) { return (sel[i] & 1) != 0; }, sh);
  for (int c = 0; c < cfg.nbg; ++c) {
    const double lo = cfg.bg_lo[c], hi = cfg.bg_hi[c];
    auto cand = [&](int i) { return mo[i] >= lo && mo[i] <= hi; };
    const int size = count_cands(N, cand, sh);
    const double want = rint(static_cast<double>(cfg.batch - nfg) * cfg.bg_frac[c]);
    const int cnt = static_cast<int>(fmin(static_cast<double>(size), fmax(want, 0.0)));
    select_smallest(keys + static_cast<long long>(cfg.nfg + c) * N, N, cnt, cand,
                    [&](int i) { sel[i] |= 2; }, sh);
  }

  // keep_inds = unique(fg) ++ unique(bg) (:162); a row may sit in both parts
  int fg_before = 0, bg_before = 0, nbg = 0;
  for (int base = 0; base < N; base += kSelThreads) {
    const int i = base + threadIdx.x;
    const int s = i < N ? sel[i] : 0;
    int tf, tb;
    const int rf = block_rank(s & 1, sh, tf);
    const int rb = block_rank(s & 2, sh, tb);
    if (i < N) {
      fgpos[i] = (s & 1) ? fg_before + rf : -1;
      bgpos[i] = (s & 2) ? nfg + bg_before + rb : -1;
      if (s & 1) keep[fg_before + rf] = i;
      if (s & 2) keep[nfg + bg_before + rb] = i;
    }
    fg_before += tf;
    bg_before += tb;
  }
  nbg = bg_before;
  const int K = nfg + nbg;
  // fg rows of gt boxes (>= n) are last in the sorted fg part: the MIX_INDEX fg list is a prefix
  int nfg_mix = 0;
  for (int base = 0; base < N; base += kSelThreads) {
    const int i = base + threadIdx.x;
    nfg_mix += block_count(i < n && (sel[i] & 1), sh);
  }
  for (int p = K + threadIdx.x; p < Kmax; p += kSelThreads) keep[p] = -1;
  if (threadIdx.x == 0) {
    counts[0] = K;
    counts[1] = nfg_mix;
    counts[2] = nbg;
    counts[3] = nfg;
  }
  __syncthreads();

  const float im_scale = im_info[2];
  const int C4 = 4 * C;
  for (int p = threadIdx.x; p < Kmax; p += kSelThreads) {
    float* ro = rois_out + static_cast<long long>(p) * 5;
    float* bt = bbox_targets + static_cast<long long>(p) * C4;
    float* bi = bbox_inside + static_cast<long long>(p) * C4;
    float* bo = bbox_outside + static_cast<long long>(p) * C4;
    float* mi = info_out + static_cast<long long>(p) * 12;
    for (int c = 0; c < C4; ++c) bt[c] = bi[c] = bo[c] = 0.f;
    // MIX_INDEX lists (:96-105): rois_index of the fg rows < n, of every bg row
    if (p < nfg_mix) fg_inds[p] = rois_index[keep[p]];
    else fg_inds[p] = -1.f;
    if (p < nbg) {
      const int i = keep[nfg + p];
      bg_inds[p] = i < n ? rois_index[i] : -1.f;     // a gt row here is an IndexError upstream
    } else {
      bg_inds[p] = -1.f;
    }
    if (p >= K) {                                    // padded row
      for (int k = 0; k < 5; ++k) ro[k] = 0.f;
      labels[p] = -1.f;
      for (int k = 0; k < 12; ++k) mi[k] = -1.f;
      continue;
    }
    const int i = keep[p];
    const bool fg = p < nfg;
    const int a = asg[i];
    const float* g = gt + a * 5;
    const float* r = i < n ? rpn_rois + static_cast<long long>(i) * 5 : nullptr;
    float b[4];
    ro[0] = r ? r[0] : 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      b[k] = r ? r[k + 1] : gt[(i - n) * 5 + k];
      ro[k + 1] = b[k];
    }
    const float label = fg ? g[4] : 0.f;             // bg labels clamped to 0 (:166)
    labels[p] = label;
    // bbox_compute_targets on float32 rois and gt boxes (bbox_transform.py:39-61,160-176), then
    // get_bbox_regression_label (:179-203)
    if (label > 0.f) {
      const float ew = __fadd_rn(__fsub_rn(b[2], b[0]), 1.f), eh = __fadd_rn(__fsub_rn(b[3], b[1]), 1.f);
      const float ecx = __fadd_rn(b[0], __fmul_rn(0.5f, ew)), ecy = __fadd_rn(b[1], __fmul_rn(0.5f, eh));
      const float gw = __fadd_rn(__fsub_rn(g[2], g[0]), 1.f), gh = __fadd_rn(__fsub_rn(g[3], g[1]), 1.f);
      const float gcx = __fadd_rn(g[0], __fmul_rn(0.5f, gw)), gcy = __fadd_rn(g[1], __fmul_rn(0.5f, gh));
      float t[4];
      t[0] = __fdiv_rn(__fsub_rn(gcx, ecx), ew);
      t[1] = __fdiv_rn(__fsub_rn(gcy, ecy), eh);
      t[2] = static_cast<float>(log(static_cast<double>(__fdiv_rn(gw, ew))));
      t[3] = static_cast<float>(log(static_cast<double>(__fdiv_rn(gh, eh))));
      const int start = static_cast<int>(__fmul_rn(4.f, label));
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float v = cfg.normalize
            ? static_cast<float>(__ddiv_rn(__dsub_rn(static_cast<double>(t[k]), cfg.mean[k]), cfg.std_[k]))
            : t[k];
        const int c = start + k;
        if (c < 0 || c >= C4) continue;
        bt[c] = v;
        bi[c] = cfg.inside[k];
        bo[c] = cfg.inside[k] > 0.f ? 1.f : 0.f;
      }
    }
    // top_mask_info (:190-214): boxes / im_scale in float32, np.around
    if (fg) {
      mi[0] = static_cast<float>(a);
      mi[1] = static_cast<float>(mask_info[a * 2 + 0]);
      mi[2] = static_cast<float>(mask_info[a * 2 + 1]);
      mi[3] = label;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        mi[4 + k] = static_cast<float>(static_cast<int>(rintf(__fdiv_rn(b[k], im_scale))));
        mi[8 + k] = static_cast<float>(static_cast<int>(rintf(__fdiv_rn(g[k], im_scale))));
      }
    } else {
#pragma unroll
      for (int k = 0; k < 12; ++k) mi[k] = -1.f;
    }
  }
}

// grid Kmax, kMaskThreads threads: mask targets of the fg rows (:186-214), weight 1 for them.
__global__ void __launch_bounds__(kMaskThreads)
proposal_target_masks_kernel(const float* __restrict__ info, const int* __restrict__ counts,
                             const float* __restrict__ gt_masks, int G, int Hm, int Wm, int M,
                             float thresh, float* __restrict__ targets, float* __restrict__ weight) {
  const int p = blockIdx.x;
  const long long MM = static_cast<long long>(M) * M;
  mask_target_row(info + static_cast<long long>(p) * 12, p < counts[3], gt_masks, G, Hm, Wm, M,
                  thresh, targets + p * MM, weight + p * MM);
}

// rpn_rois diff row i (:109-115): top row p copied where keep_inds[p] == i, the last such p winning
// as numpy's fancy assignment does; with bp_all off only the fg part counts.  One thread per value.
__global__ void proposal_target_backward_kernel(const float* __restrict__ top_diff,
                                                const int* __restrict__ state, int n, int G,
                                                int bp_all, float* __restrict__ rois_diff) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n * 5) return;
  const int i = j / 5, col = j - 5 * (j / 5);
  const int N = n + G;
  int p = bp_all ? state[N + i] : -1;
  if (p < 0) p = state[i];
  rois_diff[j] = p >= 0 ? top_diff[static_cast<long long>(p) * 5 + col] : 0.f;
}

// ========================================================================== AnchorTargetLayer
struct AtCfg {
  int border;
  double neg, pos;                    // RPN_NEGATIVE_OVERLAP, RPN_POSITIVE_OVERLAP
  int clobber;                        // RPN_CLOBBER_POSITIVES
  int num_fg, batch;                  // int(RPN_FG_FRACTION * RPN_BATCHSIZE), RPN_BATCHSIZE
  double pos_weight;                  // RPN_POSITIVE_WEIGHT
  float inside[4];                    // RPN_BBOX_INSIDE_WEIGHTS
};

// Scratch: lab int8 [T] (-2 outside the image, else the working label), argmax int32 [T],
// gt_max uint64 [G] (float64 bits; overlaps are >= 0 so integer order is value order),
// weights float [2].
__host__ __device__ inline long long at_ws_bytes(int T, int G) {
  return ((static_cast<long long>(T) + 7) & ~7LL) + 4LL * ((T + 1) & ~1) + 8LL * G + 16;
}

struct AtWs {
  signed char* lab;
  int* arg;
  unsigned long long* gmax;
  float* w;
};

inline AtWs at_ws(void* ws, int T, int G) {
  char* p = static_cast<char*>(ws);
  AtWs s;
  s.lab = reinterpret_cast<signed char*>(p);
  p += (static_cast<long long>(T) + 7) & ~7LL;
  s.arg = reinterpret_cast<int*>(p);
  p += 4LL * ((T + 1) & ~1);
  s.gmax = reinterpret_cast<unsigned long long*>(p);
  p += 8LL * G;
  s.w = reinterpret_cast<float*>(p);
  return s;
}

__device__ __forceinline__ void anchor_box(const AnchorTable& an, int t, int W, int feat_stride,
                                           double b[4]) {
  const int a = t % kA, pix = t / kA;
  const double sx = static_cast<double>((pix % W) * feat_stride);
  const double sy = static_cast<double>((pix / W) * feat_stride);
  b[0] = an.v[a][0] + sx;
  b[1] = an.v[a][1] + sy;
  b[2] = an.v[a][2] + sx;
  b[3] = an.v[a][3] + sy;
}

// One thread per anchor: inside test (:80-85), argmax / max over gt (:96-97), column maxima.
__global__ void anchor_overlaps_kernel(int T, int W, int feat_stride, const AnchorTable an,
                                       const float* __restrict__ gt, int G,
                                       const float* __restrict__ im_info, AtCfg cfg, AtWs ws) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  double b[4];
  anchor_box(an, t, W, feat_stride, b);
  const double xl = __fadd_rn(im_info[1], static_cast<float>(cfg.border));
  const double yl = __fadd_rn(im_info[0], static_cast<float>(cfg.border));
  const bool inside = b[0] >= -cfg.border && b[1] >= -cfg.border && b[2] < xl && b[3] < yl;
  if (!inside) {
    ws.lab[t] = -2;
    return;
  }
  double best = 0.0;
  int arg = 0;
  for (int g = 0; g < G; ++g) {
    const double ov = iou64(b[0], b[1], b[2], b[3], gt + g * 5);
    if (g == 0 || ov > best) {
      best = ov;
      arg = g;
    }
    atomicMax(&ws.gmax[g], static_cast<unsigned long long>(__double_as_longlong(ov)));
  }
  ws.arg[t] = arg;
  ws.lab[t] = -1;
}

// One thread per inside anchor: the label before sampling (:100-113) and the targets (:138-139).
__global__ void anchor_labels_kernel(int T, int H, int W, int feat_stride, const AnchorTable an,
                                     const float* __restrict__ gt, int G, AtCfg cfg, AtWs ws,
                                     float* __restrict__ bbox_targets) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const int a = t % kA, pix = t / kA;
  const long long HW = static_cast<long long>(H) * W;
  float* bt = bbox_targets + static_cast<long long>(4 * a) * HW + pix;
  if (ws.lab[t] == -2) {
#pragma unroll
    for (int k = 0; k < 4; ++k) bt[k * HW] = 0.f;
    return;
  }
  double b[4];
  anchor_box(an, t, W, feat_stride, b);
  bool gt_arg = false;
  double best = 0.0;
  for (int g = 0; g < G; ++g) {
    const double ov = iou64(b[0], b[1], b[2], b[3], gt + g * 5);
    // np.where(overlaps == gt_max_overlaps)[0]: a tie with ANY column's maximum (:98)
    gt_arg |= ov == __longlong_as_double(static_cast<long long>(ws.gmax[g]));
    if (g == 0 || ov > best) best = ov;
  }
  int lab = -1;
  if (!cfg.clobber && best < cfg.neg) lab = 0;
  if (gt_arg) lab = 1;
  if (best >= cfg.pos) lab = 1;
  if (cfg.clobber && best < cfg.neg) lab = 0;
  ws.lab[t] = static_cast<signed char>(lab);
  // bbox_transform(anchor float64, gt float32).astype(float32) (anchor_target_layer.py:199-209)
  const float* g = gt + ws.arg[t] * 5;
  const double ew = __dadd_rn(__dsub_rn(b[2], b[0]), 1.0), eh = __dadd_rn(__dsub_rn(b[3], b[1]), 1.0);
  const double ecx = __dadd_rn(b[0], __dmul_rn(0.5, ew)), ecy = __dadd_rn(b[1], __dmul_rn(0.5, eh));
  const float gw = __fadd_rn(__fsub_rn(g[2], g[0]), 1.f), gh = __fadd_rn(__fsub_rn(g[3], g[1]), 1.f);
  const float gcx = __fadd_rn(g[0], __fmul_rn(0.5f, gw)), gcy = __fadd_rn(g[1], __fmul_rn(0.5f, gh));
  bt[0] = static_cast<float>(__ddiv_rn(__dsub_rn(static_cast<double>(gcx), ecx), ew));
  bt[HW] = static_cast<float>(__ddiv_rn(__dsub_rn(static_cast<double>(gcy), ecy), eh));
  bt[2 * HW] = static_cast<float>(log(__ddiv_rn(static_cast<double>(gw), ew)));
  bt[3 * HW] = static_cast<float>(log(__ddiv_rn(static_cast<double>(gh), eh)));
}

// One CTA: surplus fg / bg disabled by the key-based choice (:115-134), the MIX_INDEX override
// (:136-150) and the outside weights' denominators (:155-169).
__global__ void __launch_bounds__(kSelThreads)
anchor_sample_kernel(int T, const unsigned* __restrict__ keys, const float* __restrict__ fg_inds,
                     const float* __restrict__ bg_inds, const int* __restrict__ mix_counts,
                     int mix_cap, AtCfg cfg, AtWs ws) {
  __shared__ SelShared sh;
  signed char* lab = ws.lab;
  auto is_fg = [&](int i) { return lab[i] == 1; };
  const int nfg = count_cands(T, is_fg, sh);
  if (nfg > cfg.num_fg)
    select_smallest(keys, T, nfg - cfg.num_fg, is_fg, [&](int i) { lab[i] = -1; }, sh);
  const int num_bg = cfg.batch - count_cands(T, is_fg, sh);
  auto is_bg = [&](int i) { return lab[i] == 0; };
  const int nbg = count_cands(T, is_bg, sh);
  if (nbg > num_bg)
    select_smallest(keys, T, nbg - num_bg, is_bg, [&](int i) { lab[i] = -1; }, sh);
  if (mix_counts) {
    // anchors of bg_inds first, then fg_inds, when inside the image (float == int compare)
    for (int pass = 0; pass < 2; ++pass) {
      const float* v = pass ? fg_inds : bg_inds;
      const int cnt = min(mix_counts[pass ? 1 : 2], mix_cap);
      for (int j = threadIdx.x; j < cnt; j += kSelThreads) {
        const float f = v[j];
        const int t = static_cast<int>(f);
        if (f >= 0.f && t < T && static_cast<float>(t) == f && lab[t] != -2)
          lab[t] = pass ? 1 : 0;
      }
      __syncthreads();
    }
  }
  const int npos = count_cands(T, is_fg, sh);
  const int nneg = count_cands(T, is_bg, sh);
  if (threadIdx.x == 0) {
    if (cfg.pos_weight < 0) {
      const float w = static_cast<float>(1.0 / static_cast<double>(npos + nneg));
      ws.w[0] = ws.w[1] = w;
    } else {
      ws.w[0] = static_cast<float>(cfg.pos_weight / static_cast<double>(npos));
      ws.w[1] = static_cast<float>((1.0 - cfg.pos_weight) / static_cast<double>(nneg));
    }
  }
}

// One thread per anchor: the four tops in Caffe layout, unmap'ed (:171-209).
__global__ void anchor_write_kernel(int T, int H, int W, AtCfg cfg, AtWs ws,
                                    float* __restrict__ labels, float* __restrict__ inside_w,
                                    float* __restrict__ outside_w) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const int a = t % kA, pix = t / kA;
  const long long HW = static_cast<long long>(H) * W;
  const int l = ws.lab[t];
  labels[static_cast<long long>(a) * HW + pix] = l == -2 ? -1.f : static_cast<float>(l);
  const float ow = l == 1 ? ws.w[0] : (l == 0 ? ws.w[1] : 0.f);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    inside_w[(4 * a + k) * HW + pix] = l == 1 ? cfg.inside[k] : 0.f;
    outside_w[(4 * a + k) * HW + pix] = ow;
  }
}

AnchorTable anchor_table() {
  float f[36];
  mnc_generate_anchors(f);
  AnchorTable t;
  for (int i = 0; i < kA; ++i)
    for (int k = 0; k < 4; ++k) t.v[i][k] = f[i * 4 + k];
  return t;
}

}  // namespace
}  // namespace mnc

extern "C" int mnc_proposal_train_state(const int* order, const int* keep, const int* num_keep,
                                        int R, const float* rpn_bbox_pred, int H, int W,
                                        int feat_stride, const float* im_info,
                                        float* proposal_index, int* state, void* stream) {
  if (R < 0 || H <= 0 || W <= 0 || feat_stride <= 0) return MNC_ERR_ARG;
  if (R == 0) return MNC_OK;
  mnc::proposal_train_state_kernel<<<(R + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      order, keep, num_keep, R, rpn_bbox_pred, H, W, feat_stride, im_info, mnc::anchor_table(),
      proposal_index, state);
  return mnc::check_launch();
}

extern "C" int mnc_proposal_backward(const float* top_diff, int R, const int* state,
                                     const float* rpn_bbox_pred, int H, int W, float clip_thresh,
                                     float* bbox_pred_diff, void* stream) {
  if (R < 0 || H <= 0 || W <= 0 || clip_thresh < 0.f) return MNC_ERR_ARG;
  if (!bbox_pred_diff) return MNC_OK;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int rc = mnc::cuda_status(cudaMemsetAsync(bbox_pred_diff, 0, sizeof(float) * 4 * mnc::kA * H * W, s));
  if (rc != MNC_OK) return rc;
  if (R > 0)
    mnc::proposal_backward_kernel<<<(R + 127) / 128, 128, 0, s>>>(
        top_diff, R, state, rpn_bbox_pred, H, W, mnc::anchor_table(), clip_thresh, bbox_pred_diff);
  return mnc::check_launch();
}

extern "C" long long mnc_proposal_target_state_ints(int n, int G, int k_max) {
  return mnc::pt_state_ints(n + G, k_max);
}

extern "C" int mnc_proposal_target_capacity(int batch_size, int n_fg_cats, int n_bg_cats) {
  return batch_size + n_fg_cats + n_bg_cats;
}

extern "C" int mnc_proposal_target(
    const float* rpn_rois, int n, const float* rpn_rois_index, const int* n_valid,
    const float* gt_boxes, int G, const float* gt_masks, int mask_h, int mask_w,
    const int* mask_info, const float* im_info, const unsigned* keys, int batch_size, int n_fg_cats, const double* fg_fraction,
    const double* fg_thresh_lo, const double* fg_thresh_hi, int n_bg_cats,
    const double* bg_fraction, const double* bg_thresh_lo, const double* bg_thresh_hi,
    const double* means, const double* stds, const float* inside_weights, int mask_size,
    float binarize_thresh, int num_classes, int k_max, float* rois, float* labels,
    float* bbox_targets, float* bbox_inside_weights, float* bbox_outside_weights,
    float* mask_targets, float* mask_weight, float* gt_masks_info, float* fg_inds,
    float* bg_inds, int* counts, int* state, void* stream) {
  if (n < 0 || G <= 0 || batch_size <= 0 || num_classes < 2 || mask_h <= 0 || mask_w <= 0 ||
      mask_size <= 0 || n_fg_cats < 0 || n_fg_cats > mnc::kMaxCats || n_bg_cats < 0 ||
      n_bg_cats > mnc::kMaxCats || !inside_weights || (means == nullptr) != (stds == nullptr) ||
      k_max != mnc_proposal_target_capacity(batch_size, n_fg_cats, n_bg_cats) ||
      (n > 0 && !rpn_rois_index))
    return MNC_ERR_ARG;
  mnc::PtCfg cfg;
  cfg.batch = batch_size;
  cfg.nfg = n_fg_cats;
  cfg.nbg = n_bg_cats;
  double fsum = 0.0, bsum = 0.0;
  for (int c = 0; c < mnc::kMaxCats; ++c) {
    cfg.fg_frac[c] = c < n_fg_cats ? fg_fraction[c] : 0.0;
    cfg.fg_lo[c] = c < n_fg_cats ? fg_thresh_lo[c] : 0.0;
    cfg.fg_hi[c] = c < n_fg_cats ? fg_thresh_hi[c] : 0.0;
    cfg.bg_frac[c] = c < n_bg_cats ? bg_fraction[c] : 0.0;
    cfg.bg_lo[c] = c < n_bg_cats ? bg_thresh_lo[c] : 0.0;
    cfg.bg_hi[c] = c < n_bg_cats ? bg_thresh_hi[c] : 0.0;
    if (cfg.fg_frac[c] < 0.0 || cfg.bg_frac[c] < 0.0) return MNC_ERR_ARG;
    fsum += cfg.fg_frac[c];
    bsum += cfg.bg_frac[c];
  }
  // each np.round adds at most 1/2, so K <= BATCH_SIZE (1 + eps) + #categories / 2 < k_max; eps
  // lets a list whose decimal fractions add to 1 in real numbers pass its rounded sum
  if (fsum > 1.0 + 1e-9 || bsum > 1.0 + 1e-9 || batch_size > (1 << 28)) return MNC_ERR_ARG;
  cfg.normalize = means != nullptr;
  for (int k = 0; k < 4; ++k) {
    cfg.mean[k] = means ? means[k] : 0.0;
    cfg.std_[k] = stds ? stds[k] : 1.0;
    cfg.inside[k] = inside_weights[k];
  }
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  mnc::proposal_target_kernel<<<1, mnc::kSelThreads, 0, s>>>(
      rpn_rois, n, rpn_rois_index, n_valid, gt_boxes, G, mask_info, im_info, keys, cfg, num_classes,
      k_max,
      rois, labels, bbox_targets, bbox_inside_weights, bbox_outside_weights, gt_masks_info,
      fg_inds, bg_inds, counts, state);
  mnc::proposal_target_masks_kernel<<<k_max, mnc::kMaskThreads, 0, s>>>(
      gt_masks_info, counts, gt_masks, G, mask_h, mask_w, mask_size, binarize_thresh, mask_targets,
      mask_weight);
  return mnc::check_launch();
}

extern "C" int mnc_proposal_target_backward(const float* top_diff, const int* state, int n, int G,
                                            int bp_all, float* rpn_rois_diff, void* stream) {
  if (n < 0 || G <= 0) return MNC_ERR_ARG;
  if (n == 0 || !rpn_rois_diff) return MNC_OK;
  mnc::proposal_target_backward_kernel<<<(5 * n + 255) / 256, 256, 0,
                                         static_cast<cudaStream_t>(stream)>>>(
      top_diff, state, n, G, bp_all, rpn_rois_diff);
  return mnc::check_launch();
}

extern "C" long long mnc_anchor_target_workspace_bytes(int H, int W, int G) {
  return mnc::at_ws_bytes(H * W * mnc::kA, G);
}

extern "C" int mnc_anchor_target(
    int H, int W, int feat_stride, int allowed_border, const float* gt_boxes, int G,
    const float* im_info, const unsigned* keys, const float* fg_inds, const float* bg_inds,
    const int* mix_counts, int mix_cap, double negative_overlap, double positive_overlap,
    int clobber_positives, double fg_fraction, int batch_size, double positive_weight,
    const float* inside_weights, void* workspace, float* labels, float* bbox_targets,
    float* bbox_inside_weights, float* bbox_outside_weights, void* stream) {
  if (H <= 0 || W <= 0 || feat_stride <= 0 || G <= 0 || batch_size <= 0 || !inside_weights ||
      !workspace || (mix_counts && (!fg_inds || !bg_inds || mix_cap < 0)) ||
      (positive_weight >= 0 && !(positive_weight > 0 && positive_weight < 1)) ||
      !(fg_fraction >= 0.0 && fg_fraction <= 1.0))   // above 1, RPN_BATCHSIZE - #fg goes negative
    return MNC_ERR_ARG;
  mnc::AtCfg cfg;
  cfg.border = allowed_border;
  cfg.neg = negative_overlap;
  cfg.pos = positive_overlap;
  cfg.clobber = clobber_positives;
  cfg.num_fg = static_cast<int>(fg_fraction * batch_size);
  cfg.batch = batch_size;
  cfg.pos_weight = positive_weight;
  for (int k = 0; k < 4; ++k) cfg.inside[k] = inside_weights[k];
  const int T = H * W * mnc::kA;
  const mnc::AtWs ws = mnc::at_ws(workspace, T, G);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int rc = mnc::cuda_status(cudaMemsetAsync(ws.gmax, 0, 8LL * G, s));
  if (rc != MNC_OK) return rc;
  const mnc::AnchorTable an = mnc::anchor_table();
  const int grid = (T + 255) / 256;
  mnc::anchor_overlaps_kernel<<<grid, 256, 0, s>>>(T, W, feat_stride, an, gt_boxes, G, im_info,
                                                   cfg, ws);
  mnc::anchor_labels_kernel<<<grid, 256, 0, s>>>(T, H, W, feat_stride, an, gt_boxes, G, cfg, ws,
                                                 bbox_targets);
  mnc::anchor_sample_kernel<<<1, mnc::kSelThreads, 0, s>>>(T, keys, fg_inds, bg_inds, mix_counts,
                                                          mix_cap, cfg, ws);
  mnc::anchor_write_kernel<<<grid, 256, 0, s>>>(T, H, W, cfg, ws, labels, bbox_inside_weights,
                                                bbox_outside_weights);
  return mnc::check_launch();
}
