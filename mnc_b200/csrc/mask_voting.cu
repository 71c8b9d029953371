// GPU mask voting.
//
// Replaces `_mv` (lib/nms/mv_kernel.cu: kernels :36-240, host wrapper :242-348) and the host loop
// of gpu_mask_voting that feeds it (lib/transform/mask_transform.py:242-274, with
// lib/utils/bbox.pyx:15-55 for the float64 IoU).
//
// The reference renders every one of the nb input masks to image size (nb*H*W floats: 1.44 GB at
// 600x1000, nb = 600) and then aggregates.  Here nothing image-sized is ever stored:
//   mv_aggregate : for each result instance, CTAs sweep the union bounding region of its
//                  candidates, evaluate  sum_i w_i * render_i(h, w)  on the fly in candidate-list
//                  order, and reduce the tight bounding box of {agg > 0.4} with warp shuffles +
//                  atomicMin/Max (4 ints per result).  (An inward band scan that stops at the first
//                  hit was tried: exact, but its serialised rounds were 2.5x slower on real
//                  detections, whose union regions have wide empty borders.)
//   mv_finalize  : resamples the aggregate back to MxM, evaluating it at the <= 4 pixels each
//                  output needs.
// Per-pixel arithmetic mirrors the reference expression by expression (same last-row / last-col
// nearest rule, same W/2, H/2 defaults for an empty mask).
#include <cuda_runtime.h>
#include <climits>
#include <cstdint>

#include "mnc_b200.h"
#include "launch_util.h"

namespace mnc {

constexpr float kBinarizeThresh = 0.4f;  // mv_kernel.cu:13
constexpr int kMaxBoxes = 1024;          // nb limit of the device pipeline (2 stages x 300 = 600)

// (mask_size / box_width, mask_size / box_height) exactly as mv_kernel.cu:55-58 computes them;
// evaluated once per candidate instead of once per pixel (two IEEE divisions saved per render).
__device__ __forceinline__ float2 mv_ratio(const float4 box, int mask_size) {
  const float box_width = box.z - box.x + 1.0;
  const float box_height = box.w - box.y + 1.0;
  return make_float2((float)mask_size / box_width, (float)mask_size / box_height);
}

// One pixel of one candidate's 21x21 mask pasted into its box -- the value `mask_render` produces
// (mv_kernel.cu:36-91).  The operation order inside each expression is the reference's (products
// of the two 1-D weights first, then the four weighted taps summed left to right) because results
// are compared bit for bit with the reference built without FMA contraction; the structure is
// ours: outside test, 1-D cell / fraction per axis, last-cell rule, 4-tap blend.
struct MvAxis {
  int cell;     // floor of the mask coordinate
  float frac;   // coordinate - cell
};
__device__ __forceinline__ MvAxis mv_axis(int p, float box_lo, float ratio) {
  const float pos = ((float)p - box_lo) * ratio;
  MvAxis a;
  a.cell = floor(pos);
  a.frac = pos - a.cell;
  return a;
}
__device__ __forceinline__ float mv_render(const float4 box, const float2 ratio,
                                           const float* __restrict__ mask, int mask_size, int h,
                                           int w) {
  if (w < box.x || w > box.z || h < box.y || h > box.w) return 0.0f;   // unrounded box, float compare
  const MvAxis ax = mv_axis(w, box.x, ratio.x);
  const MvAxis ay = mv_axis(h, box.y, ratio.y);
  const int last = mask_size - 1;
  // a sample in the last mask row or column is not interpolated along either axis (:66-74)
  if (ax.cell == last || ay.cell == last)
    return __ldg(mask + (ax.cell == last && ay.cell == last ? last * mask_size + last
                                                           : ay.cell * mask_size + ax.cell));
  const float* tap = mask + ay.cell * mask_size + ax.cell;
  const float w00 = (1 - ax.frac) * (1 - ay.frac);
  const float w01 = ax.frac * (1 - ay.frac);
  const float w10 = (1 - ax.frac) * ay.frac;
  const float w11 = ax.frac * ay.frac;
  return w00 * __ldg(tap) + w01 * __ldg(tap + 1) + w10 * __ldg(tap + mask_size) +
         w11 * __ldg(tap + mask_size + 1);
}

struct CandList {
  float4* box;   // shared
  float* wgt;    // shared
  int* ind;      // shared
  float2* ratio; // shared: (mask_size / box_width, mask_size / box_height), mv_kernel.cu:55-58
  float* suf;    // shared: suf[i] = sum of wgt[i..n)
  int n;
};

// mask_aggregate (mv_kernel.cu:93-112) at one pixel: sum in candidate-list order.
__device__ __forceinline__ float agg_at(const CandList& cl, const float* __restrict__ masks,
                                        int mask_size, int h, int w) {
  float val = 0.0f;
  for (int i = 0; i < cl.n; ++i) {
    const float4 b = cl.box[i];
    if (w < b.x || w > b.z || h < b.y || h > b.w) continue;  // render == 0: adds nothing
    val += (mv_render(b, cl.ratio[i], masks + static_cast<long long>(cl.ind[i]) * mask_size * mask_size,
                      mask_size, h, w) * cl.wgt[i]);
  }
  return val;
}

// The predicate  agg_at(...) > 0.4  without always finishing the sum.  Valid when every mask value
// of the image lies in [0, 1] and every weight is >= 0 (checked on the device by mv_range_kernel):
// the terms are then non-negative, so fp32 partial sums never decrease -- once one exceeds the
// threshold the final sum does too; and the final sum is at most partial + remaining weights
// (render <= 1), so when even that (with a 1e-4 margin, >> the accumulated rounding) cannot reach
// the threshold the pixel is off.  Same answer as comparing the full candidate-order sum.
__device__ __forceinline__ bool agg_exceeds_unit(const CandList& cl, const float* __restrict__ masks,
                                                 int mask_size, int h, int w) {
  float val = 0.0f;
  for (int i = 0; i < cl.n; ++i) {
    if (val + cl.suf[i] * 1.0001f <= kBinarizeThresh) return false;
    const float4 b = cl.box[i];
    if (w < b.x || w > b.z || h < b.y || h > b.w) continue;
    val += (mv_render(b, cl.ratio[i], masks + static_cast<long long>(cl.ind[i]) * mask_size * mask_size,
                      mask_size, h, w) * cl.wgt[i]);
    if (val > kBinarizeThresh) return true;
  }
  return val > kBinarizeThresh;
}

__device__ __forceinline__ void load_cands(CandList& cl, const float* __restrict__ boxes,
                                           int box_dim, const int* __restrict__ cand_inds,
                                           const float* __restrict__ cand_weights, int begin,
                                           int end, int mask_size) {
  cl.n = end - begin;
  for (int i = threadIdx.x; i < cl.n; i += blockDim.x) {
    const int ind = cand_inds[begin + i];
    const float* b = boxes + static_cast<long long>(ind) * box_dim;
    cl.box[i] = make_float4(b[0], b[1], b[2], b[3]);
    cl.wgt[i] = cand_weights[begin + i];
    cl.ind[i] = ind;
    cl.ratio[i] = mv_ratio(cl.box[i], mask_size);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float acc = 0.f;
    for (int i = cl.n - 1; i >= 0; --i) {
      acc += cl.wgt[i];
      cl.suf[i] = acc;
    }
  }
  __syncthreads();
}

// unit[img] = 1 iff all mask values of the image are in [0,1] and all candidate weights are >= 0
// (NaNs fail the test).  grid (32, batch); unit[] preset to 1.
__global__ void __launch_bounds__(256)
mv_range_kernel(const float* __restrict__ masks, long long masks_per_img,
                const float* __restrict__ cand_weights, long long cand_img_stride,
                const int* __restrict__ cand_begin, const int* __restrict__ cand_end,
                const int* __restrict__ n_res, int max_results, int* __restrict__ unit) {
  const int img = blockIdx.y;
  const float* m = masks + img * masks_per_img;
  bool ok = true;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < masks_per_img;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float v = m[i];
    ok &= (v >= 0.f && v <= 1.f);
  }
  if (blockIdx.x == 0) {
    // only the entries of the lists themselves: the gaps between lists are never written
    const int nr = min(n_res[img], max_results);
    for (int t = 0; t < nr; ++t) {
      const int lo = cand_begin[img * max_results + t], hi = cand_end[img * max_results + t];
      for (int i = lo + threadIdx.x; i < hi; i += blockDim.x)
        ok &= (cand_weights[img * cand_img_stride + i] >= 0.f);
    }
  }
  if (!__syncthreads_and(ok) && threadIdx.x == 0) atomicAnd(&unit[img], 0);
}

__global__ void mv_init_bbox_kernel(int* __restrict__ bbox, int total, int* __restrict__ unit,
                                    int batch) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < batch) unit[i] = 1;
  if (i < total) {
    bbox[i * 4 + 0] = INT_MAX;
    bbox[i * 4 + 1] = INT_MAX;
    bbox[i * 4 + 2] = INT_MIN;
    bbox[i * 4 + 3] = INT_MIN;
  }
}

// grid (chunks, max_results, batch); 256 threads.  Launched twice per call:
//   pass 1 (stride 6, refine 0): every 6th pixel of every 6th row -- 1/36 of the evaluations --
//           gives an inner bounding box (each of its four sides comes from a real "on" pixel);
//   pass 2 (stride 1, refine 1): all pixels EXCEPT those inside the box pass 1 left in `bbox`
//           (a pixel inside a box spanned by "on" pixels cannot move the final box), i.e. only the
//           border between the search region and the aggregate's support is evaluated exactly.
// The result is the same tight box as a full sweep; a voted mask fills most of its box, so the
// border is a small fraction of the region.  When the image's masks are in [0,1] and the weights
// >= 0 (unit[img]) the search region is first cut down from the union of the candidate boxes to
// the columns / rows whose covering weight  sum_i w_i [x_i0 <= w <= x_i1]  can exceed the threshold
// at all (render <= 1, so agg(h, w) <= that sum; same 1e-4 margin as agg_exceeds_unit).
__global__ void __launch_bounds__(256)
mv_aggregate_kernel(const float* __restrict__ boxes, const float* __restrict__ masks, int nb,
                    int box_dim, int mask_size, const int* __restrict__ cand_inds,
                    const float* __restrict__ cand_weights, long long cand_img_stride,
                    const int* __restrict__ cand_begin, const int* __restrict__ cand_end,
                    const int* __restrict__ n_res, int max_results, const int* __restrict__ im_hw,
                    const int* __restrict__ unit, int* __restrict__ bbox, int stride, int refine) {
  extern __shared__ unsigned char smraw[];
  const int img = blockIdx.z, t = blockIdx.y;
  if (t >= n_res[img]) return;
  CandList cl;
  cl.box = reinterpret_cast<float4*>(smraw);
  cl.wgt = reinterpret_cast<float*>(cl.box + nb);
  cl.ind = reinterpret_cast<int*>(cl.wgt + nb);
  cl.ratio = reinterpret_cast<float2*>(cl.ind + nb);
  cl.suf = reinterpret_cast<float*>(cl.ratio + nb);
  const float* pboxes = boxes + static_cast<long long>(img) * nb * box_dim;
  const float* pmasks = masks + static_cast<long long>(img) * nb * mask_size * mask_size;
  const int rt = img * max_results + t;
  // pass 2: the box pass 1 found (read before any of this pass's updates matter: every value this
  // word ever holds is a side of a box spanned by "on" pixels, so any snapshot is safe to skip)
  int in_x0 = INT_MAX, in_y0 = INT_MAX, in_x1 = INT_MIN, in_y1 = INT_MIN;
  if (refine) {
    in_x0 = bbox[rt * 4 + 0];
    in_y0 = bbox[rt * 4 + 1];
    in_x1 = bbox[rt * 4 + 2];
    in_y1 = bbox[rt * 4 + 3];
  }
  load_cands(cl, pboxes, box_dim, cand_inds + img * cand_img_stride,
             cand_weights + img * cand_img_stride, cand_begin[rt], cand_end[rt], mask_size);
  const int H = im_hw[img * 2 + 0], W = im_hw[img * 2 + 1];
  // union region of the candidate boxes (a superset of every pixel with a non-zero render)
  __shared__ int reg[4], core[4];
  if (threadIdx.x == 0) {
    reg[0] = core[0] = INT_MAX;
    reg[1] = core[1] = INT_MAX;
    reg[2] = core[2] = INT_MIN;
    reg[3] = core[3] = INT_MIN;
  }
  __syncthreads();
  {
    int x0 = INT_MAX, y0 = INT_MAX, x1 = INT_MIN, y1 = INT_MIN;
    for (int i = threadIdx.x; i < cl.n; i += blockDim.x) {
      const float4 b = cl.box[i];
      x0 = min(x0, static_cast<int>(floorf(b.x)));
      y0 = min(y0, static_cast<int>(floorf(b.y)));
      x1 = max(x1, static_cast<int>(ceilf(b.z)));
      y1 = max(y1, static_cast<int>(ceilf(b.w)));
    }
    if (x0 != INT_MAX) {
      atomicMin(&reg[0], x0);
      atomicMin(&reg[1], y0);
      atomicMax(&reg[2], x1);
      atomicMax(&reg[3], y1);
    }
  }
  __syncthreads();
  int rx0 = max(reg[0], 0), ry0 = max(reg[1], 0);
  int rx1 = min(reg[2], W - 1), ry1 = min(reg[3], H - 1);
  if (cl.n == 0 || rx1 < rx0 || ry1 < ry0) return;
  const bool unit_range = unit[img] != 0;
  if (unit_range) {
    // columns, then rows, whose covering weight can reach the threshold
    int lo = INT_MAX, hi = INT_MIN;
    for (int w = rx0 + threadIdx.x; w <= rx1; w += blockDim.x) {
      float u = 0.f;
      for (int i = 0; i < cl.n; ++i) {
        const float4 b = cl.box[i];
        if (!(w < b.x || w > b.z)) u += cl.wgt[i];
      }
      if (u * 1.0001f > kBinarizeThresh) {
        lo = min(lo, w);
        hi = max(hi, w);
      }
    }
    if (lo != INT_MAX) {
      atomicMin(&core[0], lo);
      atomicMax(&core[2], hi);
    }
    lo = INT_MAX;
    hi = INT_MIN;
    for (int h = ry0 + threadIdx.x; h <= ry1; h += blockDim.x) {
      float u = 0.f;
      for (int i = 0; i < cl.n; ++i) {
        const float4 b = cl.box[i];
        if (!(h < b.y || h > b.w)) u += cl.wgt[i];
      }
      if (u * 1.0001f > kBinarizeThresh) {
        lo = min(lo, h);
        hi = max(hi, h);
      }
    }
    if (lo != INT_MAX) {
      atomicMin(&core[1], lo);
      atomicMax(&core[3], hi);
    }
    __syncthreads();
    if (core[0] == INT_MAX || core[1] == INT_MAX) return;   // nowhere can the sum exceed 0.4
    rx0 = core[0];
    ry0 = core[1];
    rx1 = core[2];
    ry1 = core[3];
  }
  const int gw = (rx1 - rx0) / stride + 1, gh = (ry1 - ry0) / stride + 1;
  const long long npix = static_cast<long long>(gw) * gh;
  int bx0 = INT_MAX, by0 = INT_MAX, bx1 = INT_MIN, by1 = INT_MIN;
  for (long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; p < npix;
       p += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int h = ry0 + static_cast<int>(p / gw) * stride;
    const int w = rx0 + static_cast<int>(p % gw) * stride;
    if (w >= in_x0 && w <= in_x1 && h >= in_y0 && h <= in_y1) continue;   // inside pass 1's box
    // reduce_mask_col/row, mv_kernel.cu:114-142 (strict >)
    const bool on = unit_range ? agg_exceeds_unit(cl, pmasks, mask_size, h, w)
                               : agg_at(cl, pmasks, mask_size, h, w) > kBinarizeThresh;
    if (on) {
      bx0 = min(bx0, w);
      bx1 = max(bx1, w);
      by0 = min(by0, h);
      by1 = max(by1, h);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    bx0 = min(bx0, __shfl_xor_sync(0xffffffffu, bx0, o));
    by0 = min(by0, __shfl_xor_sync(0xffffffffu, by0, o));
    bx1 = max(bx1, __shfl_xor_sync(0xffffffffu, bx1, o));
    by1 = max(by1, __shfl_xor_sync(0xffffffffu, by1, o));
  }
  if ((threadIdx.x & 31) == 0 && bx0 != INT_MAX) {
    atomicMin(&bbox[rt * 4 + 0], bx0);
    atomicMin(&bbox[rt * 4 + 1], by0);
    atomicMax(&bbox[rt * 4 + 2], bx1);
    atomicMax(&bbox[rt * 4 + 3], by1);
  }
}

// grid (max_results, batch); 256 threads.  reduce_bounding_x/y defaults (mv_kernel.cu:144-190)
// and mask_resize (:193-240).
__global__ void __launch_bounds__(256)
mv_finalize_kernel(const float* __restrict__ boxes, const float* __restrict__ masks, int nb,
                   int box_dim, int mask_size, const int* __restrict__ cand_inds,
                   const float* __restrict__ cand_weights, long long cand_img_stride,
                   const int* __restrict__ cand_begin, const int* __restrict__ cand_end,
                   const int* __restrict__ n_res, int max_results, const int* __restrict__ im_hw,
                   const int* __restrict__ bbox, float* __restrict__ out_mask,
                   int* __restrict__ out_box) {
  extern __shared__ unsigned char smraw[];
  const int img = blockIdx.y, t = blockIdx.x;
  if (t >= n_res[img]) return;
  CandList cl;
  cl.box = reinterpret_cast<float4*>(smraw);
  cl.wgt = reinterpret_cast<float*>(cl.box + nb);
  cl.ind = reinterpret_cast<int*>(cl.wgt + nb);
  cl.ratio = reinterpret_cast<float2*>(cl.ind + nb);
  cl.suf = reinterpret_cast<float*>(cl.ratio + nb);
  const float* pboxes = boxes + static_cast<long long>(img) * nb * box_dim;
  const float* pmasks = masks + static_cast<long long>(img) * nb * mask_size * mask_size;
  const int rt = img * max_results + t;
  load_cands(cl, pboxes, box_dim, cand_inds + img * cand_img_stride,
             cand_weights + img * cand_img_stride, cand_begin[rt], cand_end[rt], mask_size);
  const int image_height = im_hw[img * 2 + 0], image_width = im_hw[img * 2 + 1];
  int bbox_x1 = bbox[rt * 4 + 0], bbox_y1 = bbox[rt * 4 + 1];
  int bbox_x2 = bbox[rt * 4 + 2], bbox_y2 = bbox[rt * 4 + 3];
  if (bbox_x1 == INT_MAX) {  // nothing above the threshold: both axes take their defaults
    bbox_x1 = bbox_x2 = image_width / 2;
    bbox_y1 = bbox_y2 = image_height / 2;
  }
  if (threadIdx.x == 0) {
    out_box[rt * 4 + 0] = bbox_x1;
    out_box[rt * 4 + 1] = bbox_y1;
    out_box[rt * 4 + 2] = bbox_x2;
    out_box[rt * 4 + 3] = bbox_y2;
  }
  for (int index = threadIdx.x; index < mask_size * mask_size; index += blockDim.x) {
    int w = index % mask_size;
    int h = index / mask_size;
    float bbox_width = bbox_x2 - bbox_x1 + 1.0;
    float bbox_height = bbox_y2 - bbox_y1 + 1.0;
    float ratio_w = bbox_width / static_cast<float>(mask_size);
    float ratio_h = bbox_height / static_cast<float>(mask_size);
    float inverse_x = bbox_x1 + static_cast<float>(w) * ratio_w;
    float inverse_y = bbox_y1 + static_cast<float>(h) * ratio_h;
    int start_x = floor(inverse_x);
    int start_y = floor(inverse_y);
    float val;
    if (start_x == image_width - 1 && start_y == image_height - 1) {
      val = agg_at(cl, pmasks, mask_size, image_height - 1, image_width - 1);
    } else if (start_x == image_width - 1 || start_y == image_height - 1) {
      val = agg_at(cl, pmasks, mask_size, start_y, start_x);
    } else {
      float top_left_weight = (1 - (inverse_x - start_x)) * (1 - (inverse_y - start_y));
      float top_right_weight = (inverse_x - start_x) * (1 - (inverse_y - start_y));
      float bot_left_weight = (1 - (inverse_x - start_x)) * (inverse_y - start_y);
      float bot_right_weight = (inverse_x - start_x) * (inverse_y - start_y);
      val = top_left_weight * agg_at(cl, pmasks, mask_size, start_y, start_x) +
            top_right_weight * agg_at(cl, pmasks, mask_size, start_y, start_x + 1) +
            bot_left_weight * agg_at(cl, pmasks, mask_size, start_y + 1, start_x) +
            bot_right_weight * agg_at(cl, pmasks, mask_size, start_y + 1, start_x + 1);
    }
    out_mask[static_cast<long long>(rt) * mask_size * mask_size + index] = val;
  }
}

// ------------------------------------------------------------------ candidate-list construction
// One CTA per image.  From the per-class NMS keep lists pick the global score threshold
// (mask_transform.py:242-244) and enumerate result instances in (class, score-rank) order
// (:253-270).  kept entry e = (class c, k): original box index = order[c][keep[c][k]].
//   1. all entries gathered in one round (keep -> order -> score: three dependent loads, every
//      entry in flight at once instead of class by class);
//   2. thresh = the min(total, max_per_image)-th largest score by a 4-pass byte-wise radix select on
//      order-preserving keys (an all-pairs rank count was 2000 x 2000 compares on one SM);
//   3. entries with score >= thresh are emitted in entry order by a ballot / prefix-count
//      compaction (was a 2000-step loop of one thread); class_bar[p] = results before the end of
//      class p's entries.
__device__ __forceinline__ uint32_t vote_sort_key(float f) {
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__global__ void __launch_bounds__(1024)
vote_select_kernel(const float* __restrict__ scores, int nb, int ncls,
                   const int* __restrict__ order, const int* __restrict__ keep, int keep_stride,
                   const int* __restrict__ num_keep, int max_per_image, int max_results,
                   int* __restrict__ res_box_idx, int* __restrict__ res_class,
                   float* __restrict__ res_score, int* __restrict__ n_res,
                   int* __restrict__ class_bar, int* __restrict__ overflow) {
  extern __shared__ unsigned char smraw[];
  const int img = blockIdx.x;
  const int nprob = ncls - 1;
  const int cap = nprob * max_per_image;
  float* s_score = reinterpret_cast<float*>(smraw);      // cap
  int* s_orig = reinterpret_cast<int*>(s_score + cap);    // cap
  int* s_pref = s_orig + cap;                             // cap: class of the entry, later the
                                                          //      number of flagged entries before it
  int* s_off = s_pref + cap;                              // nprob + 1
  __shared__ float s_thresh;
  __shared__ int s_total, s_need, s_run;
  __shared__ uint32_t s_prefix, s_hist[256];
  __shared__ int s_warp[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* pscores = scores + static_cast<long long>(img) * nb * ncls;
  if (tid == 0) {
    int off = 0;
    for (int p = 0; p < nprob; ++p) {
      s_off[p] = off;
      off += min(num_keep[img * nprob + p], max_per_image);
    }
    s_off[nprob] = off;
    s_total = off;
    s_run = 0;
  }
  __syncthreads();
  const int total = s_total;
  if (total == 0) {
    if (tid == 0) n_res[img] = 0;
    for (int p = tid; p < nprob; p += blockDim.x) class_bar[img * nprob + p] = 0;
    return;
  }
  for (int e = tid; e < total; e += blockDim.x) {
    int p = 0;
    while (e >= s_off[p + 1]) ++p;                        // class of entry e (nprob <= 20 steps)
    const int prob = img * nprob + p;
    const int pos = keep[static_cast<long long>(prob) * keep_stride + (e - s_off[p])];
    const int orig = order[static_cast<long long>(prob) * nb + pos];
    s_orig[e] = orig;
    s_pref[e] = p;
    s_score[e] = pscores[static_cast<long long>(orig) * ncls + (p + 1)];
  }
  if (tid == 0) {
    s_prefix = 0u;
    s_need = min(total, max_per_image);                   // thresh = the s_need-th largest score
  }
  __syncthreads();
  for (int pass = 3; pass >= 0; --pass) {
    if (tid < 256) s_hist[tid] = 0u;
    __syncthreads();
    const uint32_t prefix = s_prefix;
    const int sh = 8 * pass;
    for (int e = tid; e < total; e += blockDim.x) {
      const uint32_t key = vote_sort_key(s_score[e]);
      if (pass == 3 || (key >> (sh + 8)) == (prefix >> (sh + 8))) atomicAdd(&s_hist[(key >> sh) & 255u], 1u);
    }
    __syncthreads();
    if (tid == 0) {
      int need = s_need, cum = 0, bin = 255;
      for (; bin > 0; --bin) {
        if (cum + static_cast<int>(s_hist[bin]) >= need) break;
        cum += s_hist[bin];
      }
      s_prefix = prefix | (static_cast<uint32_t>(bin) << sh);
      s_need = need - cum;
    }
    __syncthreads();
  }
  const uint32_t tkey = s_prefix;
  for (int e = tid; e < total; e += blockDim.x)
    if (vote_sort_key(s_score[e]) == tkey) s_thresh = s_score[e];   // same bits from every writer
  __syncthreads();
  const float thresh = s_thresh;
  // compaction in entry order; results beyond max_results are dropped and reported
  for (int base = 0; base < total; base += blockDim.x) {
    const int e = base + tid;
    const bool flag = e < total && s_score[e] >= thresh;
    const int cls = e < total ? s_pref[e] + 1 : 0;
    const unsigned bal = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    int t = s_run;
    for (int w = 0; w < warp; ++w) t += s_warp[w];
    t += __popc(bal & ((1u << lane) - 1u));
    if (e < total) s_pref[e] = t;                         // flagged entries before e
    if (flag) {
      if (t < max_results) {
        res_box_idx[img * max_results + t] = s_orig[e];
        res_class[img * max_results + t] = cls;
        res_score[img * max_results + t] = s_score[e];
      } else {
        atomicExch(overflow, 1);
      }
    }
    __syncthreads();
    if (tid == 0) {
      int tot = 0;
      for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) tot += s_warp[w];
      s_run += tot;
    }
    __syncthreads();
  }
  const int flagged = s_run;
  for (int p = tid; p < nprob; p += blockDim.x) {
    const int end = s_off[p + 1];
    class_bar[img * nprob + p] = min(end < total ? s_pref[end] : flagged, max_results);
  }
  if (tid == 0) n_res[img] = min(flagged, max_results);
}

// grid (max_results, batch), kMaxBoxes threads.  For result t with query box q = boxes[res_box_idx]:
// candidates = {i : IoU64(boxes[i], q) >= iou_thresh} in index order (bbox.pyx:38-54,
// mask_transform.py:262-263); weights = scores[i, c] / fp32(sum_fp64(scores[cands, c])) (:265-267,
// numpy-1.x semantics, see oracle/oracle.py).
__global__ void __launch_bounds__(kMaxBoxes)
vote_candidates_kernel(const float* __restrict__ boxes, const float* __restrict__ scores,
                       const unsigned char* __restrict__ box_valid, int nb,
                       int ncls, const int* __restrict__ res_box_idx,
                       const int* __restrict__ res_class, const int* __restrict__ n_res,
                       int max_results, double iou_thresh, int* __restrict__ cand_inds,
                       float* __restrict__ cand_weights, int* __restrict__ cand_begin,
                       int* __restrict__ cand_end) {
  const int img = blockIdx.y, t = blockIdx.x;
  const int rt = img * max_results + t;
  if (t >= n_res[img]) {
    if (threadIdx.x == 0) {
      cand_begin[rt] = t * nb;
      cand_end[rt] = t * nb;
    }
    return;
  }
  __shared__ int s_warp[kMaxBoxes / 32];
  __shared__ int s_list[kMaxBoxes];
  __shared__ float s_sum;
  __shared__ int s_cnt;
  const float* pboxes = boxes + static_cast<long long>(img) * nb * 4;
  const float* pscores = scores + static_cast<long long>(img) * nb * ncls;
  const int qi = res_box_idx[rt];
  const int c = res_class[rt];
  const double q0 = pboxes[qi * 4 + 0], q1 = pboxes[qi * 4 + 1], q2 = pboxes[qi * 4 + 2],
               q3 = pboxes[qi * 4 + 3];
  const double box_area = __dmul_rn(q2 - q0 + 1, q3 - q1 + 1);
  const int i = threadIdx.x;
  int flag = 0;
  if (i < nb) {
    const double b0 = pboxes[i * 4 + 0], b1 = pboxes[i * 4 + 1], b2 = pboxes[i * 4 + 2],
                 b3 = pboxes[i * 4 + 3];
    double ov = 0.0;
    const double iw = fmin(b2, q2) - fmax(b0, q0) + 1;
    if (iw > 0) {
      const double ih = fmin(b3, q3) - fmax(b1, q1) + 1;
      if (ih > 0) {
        const double ua = __dsub_rn(__dadd_rn(__dmul_rn(b2 - b0 + 1, b3 - b1 + 1), box_area),
                                    __dmul_rn(iw, ih));
        ov = __ddiv_rn(__dmul_rn(iw, ih), ua);
      }
    }
    flag = (ov >= iou_thresh) ? 1 : 0;
    if (box_valid && !box_valid[static_cast<long long>(img) * nb + i]) flag = 0;  // padding rows
  }
  // block-wide exclusive scan of flags (index order)
  const unsigned bal = __ballot_sync(0xffffffffu, flag);
  const int lane = i & 31, wid = i >> 5;
  if (lane == 0) s_warp[wid] = __popc(bal);
  __syncthreads();
  if (i == 0) {
    int run = 0;
    for (int w2 = 0; w2 < kMaxBoxes / 32; ++w2) {
      const int v = s_warp[w2];
      s_warp[w2] = run;
      run += v;
    }
    s_cnt = run;
  }
  __syncthreads();
  const int pos = s_warp[wid] + __popc(bal & ((1u << lane) - 1u));
  if (flag) s_list[pos] = i;
  __syncthreads();
  const int cnt = s_cnt;
  if (i == 0) {
    double total = 0.0;
    for (int k = 0; k < cnt; ++k)
      total = __dadd_rn(total, static_cast<double>(pscores[static_cast<long long>(s_list[k]) * ncls + c]));
    s_sum = static_cast<float>(total);
    cand_begin[rt] = t * nb;
    cand_end[rt] = t * nb + cnt;
  }
  __syncthreads();
  const float denom = s_sum;
  int* ci = cand_inds + static_cast<long long>(img) * max_results * nb + static_cast<long long>(t) * nb;
  float* cw = cand_weights + static_cast<long long>(img) * max_results * nb + static_cast<long long>(t) * nb;
  if (i < cnt) {
    const int ind = s_list[i];
    ci[i] = ind;
    cw[i] = __fdiv_rn(pscores[static_cast<long long>(ind) * ncls + c], denom);
  }
}

static inline int check_launch() { return cudaGetLastError() == cudaSuccess ? MNC_OK : MNC_ERR_CUDA; }

}  // namespace mnc

using namespace mnc;

// 1 (default): coarse pass + exact border pass; 0: one full sweep of the region (A/B and
// cross-check switch, mnc_mv_set_two_pass).  Identical results.
static int g_mv_two_pass = 1;
extern "C" int mnc_mv_set_two_pass(int on) {
  const int prev = g_mv_two_pass;
  g_mv_two_pass = on ? 1 : 0;
  return prev;
}
extern "C" int mnc_mv_device_launches() { return g_mv_two_pass ? 5 : 4; }

// launch shape of the two passes (A/B knob): stride of the coarse pass,
// CTAs per result of the coarse / the exact border pass
static int g_mv_stride = 6, g_mv_chunks1 = 2, g_mv_chunks2 = 16;
extern "C" int mnc_mv_set_shape(int stride, int chunks_coarse, int chunks_border) {
  if (stride < 1 || stride > 64 || chunks_coarse < 1 || chunks_border < 1 || chunks_coarse > 1024 ||
      chunks_border > 1024)
    return MNC_ERR_ARG;
  g_mv_stride = stride;
  g_mv_chunks1 = chunks_coarse;
  g_mv_chunks2 = chunks_border;
  return MNC_OK;
}

extern "C" int mnc_mv_device(const float* boxes, const float* masks, int nb, int box_dim,
                             int mask_size, const int* cand_inds, const float* cand_weights,
                             long long cand_img_stride, const int* cand_begin, const int* cand_end,
                             const int* n_res, int max_results, int batch, const int* im_hw,
                             int* bbox_ws, float* out_mask, int* out_box, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (nb <= 0 || max_results <= 0 || batch <= 0) return MNC_ERR_ARG;
  const int smem = nb * (16 + 4 + 4 + 8 + 4);
  if (smem > 200 * 1024) return MNC_ERR_ARG;
  static SmemGrant grant_agg, grant_fin;   // (static shared memory counts against the 48 KB default)
  if (!ensure_dynamic_smem(mv_aggregate_kernel, smem, grant_agg) ||
      !ensure_dynamic_smem(mv_finalize_kernel, smem, grant_fin))
    return MNC_ERR_CUDA;
  const int total = batch * max_results;
  int* unit = bbox_ws + static_cast<long long>(total) * 4;   // [batch] flags after the boxes
  mv_init_bbox_kernel<<<(total + 255) / 256, 256, 0, stream>>>(bbox_ws, total, unit, batch);
  mv_range_kernel<<<dim3(32, batch), 256, 0, stream>>>(
      masks, static_cast<long long>(nb) * mask_size * mask_size, cand_weights, cand_img_stride,
      cand_begin, cand_end, n_res, max_results, unit);
  if (g_mv_two_pass) {
    mv_aggregate_kernel<<<dim3(g_mv_chunks1, max_results, batch), 256, smem, stream>>>(
        boxes, masks, nb, box_dim, mask_size, cand_inds, cand_weights, cand_img_stride, cand_begin,
        cand_end, n_res, max_results, im_hw, unit, bbox_ws, g_mv_stride, 0);
  }
  const int chunks = g_mv_two_pass ? g_mv_chunks2 : 24;
  mv_aggregate_kernel<<<dim3(chunks, max_results, batch), 256, smem, stream>>>(
      boxes, masks, nb, box_dim, mask_size, cand_inds, cand_weights, cand_img_stride, cand_begin,
      cand_end, n_res, max_results, im_hw, unit, bbox_ws, 1, g_mv_two_pass);
  mv_finalize_kernel<<<dim3(max_results, batch), 256, smem, stream>>>(
      boxes, masks, nb, box_dim, mask_size, cand_inds, cand_weights, cand_img_stride, cand_begin,
      cand_end, n_res, max_results, im_hw, bbox_ws, out_mask, out_box);
  return check_launch();
}

extern "C" int mnc_vote_select(const float* scores, int nb, int ncls, const int* order,
                               const int* keep, int keep_stride, const int* num_keep,
                               int max_per_image, int max_results, int batch, int* res_box_idx,
                               int* res_class, float* res_score, int* n_res, int* class_bar,
                               int* overflow, void* stream_) {
  const int cap = (ncls - 1) * max_per_image;
  const int smem = cap * 12 + (ncls + 1) * 4;
  if (smem > 48 * 1024) return MNC_ERR_ARG;
  vote_select_kernel<<<batch, 1024, smem, static_cast<cudaStream_t>(stream_)>>>(
      scores, nb, ncls, order, keep, keep_stride, num_keep, max_per_image, max_results,
      res_box_idx, res_class, res_score, n_res, class_bar, overflow);
  return check_launch();
}

extern "C" int mnc_vote_candidates(const float* boxes, const float* scores,
                                   const unsigned char* box_valid, int nb, int ncls,
                                   const int* res_box_idx, const int* res_class, const int* n_res,
                                   int max_results, int batch, double iou_thresh, int* cand_inds,
                                   float* cand_weights, int* cand_begin, int* cand_end,
                                   void* stream_) {
  if (nb > kMaxBoxes) return MNC_ERR_ARG;
  vote_candidates_kernel<<<dim3(max_results, batch), kMaxBoxes, 0,
                           static_cast<cudaStream_t>(stream_)>>>(
      boxes, scores, box_valid, nb, ncls, res_box_idx, res_class, n_res, max_results, iou_thresh,
      cand_inds, cand_weights, cand_begin, cand_end);
  return check_launch();
}

// ---------------------------------------------------------------------------------------------
// Reference-compatible host entry point: same arguments and meaning as
//   void _mv(const float* all_boxes, const float* all_masks, int all_boxes_num,
//            const int* candidate_inds, const int* candidate_start,
//            const float* candidate_weights, int candidate_num, int image_height,
//            int image_width, int box_dim, int mask_size, int result_num,
//            float* finalize_output_mask, int* finalize_output_box, int device_id)
//   (lib/nms/gpu_mv.hpp:1-4; candidate_start holds END offsets, mv_kernel.cu:101-102)
// plus an int status.  Unlike the reference, device_id is honoured.
extern "C" int mnc_mv_host(const float* all_boxes, const float* all_masks, int all_boxes_num,
                           const int* candidate_inds, const int* candidate_start,
                           const float* candidate_weights, int candidate_num, int image_height,
                           int image_width, int box_dim, int mask_size, int result_num,
                           float* finalize_output_mask, int* finalize_output_box, int device_id) {
  if (result_num == 0) return MNC_OK;
  if (all_boxes_num <= 0 || box_dim < 4 || mask_size <= 0 || result_num < 0 || candidate_num < 0)
    return MNC_ERR_ARG;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return MNC_ERR_NOGPU;
  int cur = 0;
  cudaGetDevice(&cur);
  if (cur != device_id && cudaSetDevice(device_id) != cudaSuccess) return MNC_ERR_CUDA;
  const size_t nb = all_boxes_num, mm = static_cast<size_t>(mask_size) * mask_size;
  auto al = [](size_t b) { return (b + 255) & ~static_cast<size_t>(255); };
  const size_t o_boxes = 0;
  const size_t o_masks = o_boxes + al(nb * box_dim * 4);
  const size_t o_inds = o_masks + al(nb * mm * 4);
  const size_t o_wgt = o_inds + al(static_cast<size_t>(candidate_num) * 4 + 4);
  const size_t o_begin = o_wgt + al(static_cast<size_t>(candidate_num) * 4 + 4);
  const size_t o_end = o_begin + al(static_cast<size_t>(result_num) * 4);
  const size_t o_nres = o_end + al(static_cast<size_t>(result_num) * 4);
  const size_t o_hw = o_nres + 256;
  const size_t o_bbox = o_hw + 256;
  const size_t o_omask = o_bbox + al(static_cast<size_t>(result_num) * 16 + 4);  // + unit flag
  const size_t o_obox = o_omask + al(static_cast<size_t>(result_num) * mm * 4);
  const size_t total = o_obox + al(static_cast<size_t>(result_num) * 16);
  char* base = nullptr;
  if (cudaMalloc(&base, total) != cudaSuccess) return MNC_ERR_CUDA;
  int rc = MNC_OK;
  int* h_begin = new int[result_num];
  for (int n = 0; n < result_num; ++n) h_begin[n] = (n == 0) ? 0 : candidate_start[n - 1];
  const int h_hw[2] = {image_height, image_width};
  bool ok = true;
  ok &= cudaMemcpy(base + o_boxes, all_boxes, nb * box_dim * 4, cudaMemcpyHostToDevice) == cudaSuccess;
  ok &= cudaMemcpy(base + o_masks, all_masks, nb * mm * 4, cudaMemcpyHostToDevice) == cudaSuccess;
  if (candidate_num > 0) {
    ok &= cudaMemcpy(base + o_inds, candidate_inds, static_cast<size_t>(candidate_num) * 4, cudaMemcpyHostToDevice) == cudaSuccess;
    ok &= cudaMemcpy(base + o_wgt, candidate_weights, static_cast<size_t>(candidate_num) * 4, cudaMemcpyHostToDevice) == cudaSuccess;
  }
  ok &= cudaMemcpy(base + o_begin, h_begin, static_cast<size_t>(result_num) * 4, cudaMemcpyHostToDevice) == cudaSuccess;
  ok &= cudaMemcpy(base + o_end, candidate_start, static_cast<size_t>(result_num) * 4, cudaMemcpyHostToDevice) == cudaSuccess;
  ok &= cudaMemcpy(base + o_nres, &result_num, 4, cudaMemcpyHostToDevice) == cudaSuccess;
  ok &= cudaMemcpy(base + o_hw, h_hw, 8, cudaMemcpyHostToDevice) == cudaSuccess;
  delete[] h_begin;
  if (ok) {
    rc = mnc_mv_device(reinterpret_cast<float*>(base + o_boxes),
                       reinterpret_cast<float*>(base + o_masks), all_boxes_num, box_dim, mask_size,
                       reinterpret_cast<int*>(base + o_inds),
                       reinterpret_cast<float*>(base + o_wgt), 0,
                       reinterpret_cast<int*>(base + o_begin), reinterpret_cast<int*>(base + o_end),
                       reinterpret_cast<int*>(base + o_nres), result_num, 1,
                       reinterpret_cast<int*>(base + o_hw), reinterpret_cast<int*>(base + o_bbox),
                       reinterpret_cast<float*>(base + o_omask),
                       reinterpret_cast<int*>(base + o_obox), nullptr);
    if (rc == MNC_OK) {
      ok &= cudaMemcpy(finalize_output_mask, base + o_omask, static_cast<size_t>(result_num) * mm * 4, cudaMemcpyDeviceToHost) == cudaSuccess;
      ok &= cudaMemcpy(finalize_output_box, base + o_obox, static_cast<size_t>(result_num) * 16, cudaMemcpyDeviceToHost) == cudaSuccess;
    }
  }
  cudaFree(base);
  if (!ok) return MNC_ERR_CUDA;
  return rc;
}

// utils.cython_bbox.bbox_overlaps (lib/utils/bbox.pyx:15-55): float64 IoU matrix, host buffers.
namespace mnc {
__global__ void bbox_overlaps_kernel(const double* __restrict__ boxes, int N,
                                     const double* __restrict__ query, int K,
                                     double* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(N) * K) return;
  const int n = static_cast<int>(i / K), k = static_cast<int>(i % K);
  const double* b = boxes + 4 * n;
  const double* q = query + 4 * k;
  const double box_area = __dmul_rn(q[2] - q[0] + 1, q[3] - q[1] + 1);
  double ov = 0.0;
  const double iw = fmin(b[2], q[2]) - fmax(b[0], q[0]) + 1;
  if (iw > 0) {
    const double ih = fmin(b[3], q[3]) - fmax(b[1], q[1]) + 1;
    if (ih > 0) {
      const double ua = __dsub_rn(__dadd_rn(__dmul_rn(b[2] - b[0] + 1, b[3] - b[1] + 1), box_area),
                                  __dmul_rn(iw, ih));
      ov = __ddiv_rn(__dmul_rn(iw, ih), ua);
    }
  }
  out[i] = ov;
}
}  // namespace mnc

extern "C" int mnc_bbox_overlaps_host(const double* boxes, int N, const double* query, int K,
                                      double* out) {
  if (N <= 0 || K <= 0) return MNC_OK;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return MNC_ERR_NOGPU;
  double *d_b = nullptr, *d_q = nullptr, *d_o = nullptr;
  bool ok = cudaMalloc(&d_b, sizeof(double) * 4 * N) == cudaSuccess &&
            cudaMalloc(&d_q, sizeof(double) * 4 * K) == cudaSuccess &&
            cudaMalloc(&d_o, sizeof(double) * static_cast<size_t>(N) * K) == cudaSuccess;
  if (ok) {
    ok &= cudaMemcpy(d_b, boxes, sizeof(double) * 4 * N, cudaMemcpyHostToDevice) == cudaSuccess;
    ok &= cudaMemcpy(d_q, query, sizeof(double) * 4 * K, cudaMemcpyHostToDevice) == cudaSuccess;
    const long long total = static_cast<long long>(N) * K;
    mnc::bbox_overlaps_kernel<<<static_cast<unsigned>((total + 255) / 256), 256>>>(d_b, N, d_q, K, d_o);
    ok &= cudaGetLastError() == cudaSuccess;
    ok &= cudaMemcpy(out, d_o, sizeof(double) * static_cast<size_t>(N) * K, cudaMemcpyDeviceToHost) == cudaSuccess;
  }
  cudaFree(d_b);
  cudaFree(d_q);
  cudaFree(d_o);
  return ok ? MNC_OK : MNC_ERR_CUDA;
}
