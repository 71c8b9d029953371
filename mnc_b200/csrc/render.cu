// Result rendering on the device (SURVEY.md section 8f row 3): the step right after mask voting in
// tools/demo.py:153-158 and lib/utils/vis_seg.py:101-131 (_convert_pred_to_image): every kept
// instance's 21x21 mask is resized to its (rounded, clipped) box with cv2.resize INTER_LINEAR,
// binarised at cfg.BINARIZE_THRESH and painted, in list order, into an instance-id image and a
// class-id image; each box outline is then drawn into the class image with the value 150.
//
// The reference paints instance after instance over whole sub-arrays; here one thread owns one
// pixel and walks the instance list backwards, stopping at the last writer of that pixel -- the
// same result without the n read-modify-write passes over the image.
//
// cv2.resize is restated in cv_resize.cuh.
#include <cuda_runtime.h>
#include <cstdint>

#include "mnc_b200.h"
#include "cv_resize.cuh"
#include "launch_util.h"

namespace mnc {

struct InstRec {
  int x1, y1, x2, y2;  // np.round(box).astype(int), clipped to the image (vis_seg.py:106-114)
  int cls;
};

// numpy slice [a-1 : a+1] along an axis: rows/cols {a-1, a}; empty when a == 0 (start -1 wraps to
// the last element, past the stop).
__device__ __forceinline__ bool in_edge_band(int v, int a) { return a >= 1 && (v == a - 1 || v == a); }

constexpr int kRenderChunk = 256;

// grid (ceil(W/128), H, batch); 128 threads, one pixel each.
__global__ void __launch_bounds__(128)
paste_instances_kernel(const float* __restrict__ boxes, int box_dim, const float* __restrict__ masks,
                       const int* __restrict__ cls, const int* __restrict__ counts, int max_n, int M,
                       int H, int W, float thresh, int* __restrict__ inst_img,
                       int* __restrict__ cls_img, unsigned char* __restrict__ bgr) {
  __shared__ InstRec recs[kRenderChunk];
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y;
  const int b = blockIdx.z;
  const int n = min(counts[b], max_n);
  const float* pboxes = boxes + static_cast<long long>(b) * max_n * box_dim;
  const float* pmasks = masks + static_cast<long long>(b) * max_n * M * M;
  const int* pcls = cls + static_cast<long long>(b) * max_n;

  int inst_val = 0, cls_val = 0;
  bool inst_done = false, cls_done = false;
  // chunks from the end of the list towards its start
  for (int hi = n; hi > 0; hi -= kRenderChunk) {
    const int lo = max(hi - kRenderChunk, 0);
    __syncthreads();
    for (int i = lo + threadIdx.x; i < hi; i += blockDim.x) {
      const float* bx = pboxes + static_cast<long long>(i) * box_dim;
      InstRec r;
      r.x1 = min(max(static_cast<int>(rintf(bx[0])), 0), W - 1);
      r.y1 = min(max(static_cast<int>(rintf(bx[1])), 0), H - 1);
      r.x2 = min(max(static_cast<int>(rintf(bx[2])), 0), W - 1);
      r.y2 = min(max(static_cast<int>(rintf(bx[3])), 0), H - 1);
      r.cls = pcls[i];
      recs[i - lo] = r;
    }
    __syncthreads();
    const bool all_done = (x >= W) || (inst_done && cls_done);
    if (__syncthreads_and(all_done)) break;
    if (x >= W) continue;
    for (int i = hi - 1; i >= lo && !(inst_done && cls_done); --i) {
      const InstRec r = recs[i - lo];
      const int bw = r.x2 - r.x1 + 1, bh = r.y2 - r.y1 + 1;
      if (bw <= 0 || bh <= 0) continue;  // cv2.resize would reject an empty size; nothing painted
      const bool in_x = x >= r.x1 && x <= r.x2, in_y = y >= r.y1 && y <= r.y2;
      // outline, drawn after this instance's mask (vis_seg.py:123-126)
      if (!cls_done) {
        const bool edge = (in_y && (in_edge_band(x, r.x1) || in_edge_band(x, r.x2))) ||
                          (in_x && (in_edge_band(y, r.y1) || in_edge_band(y, r.y2)));
        if (edge) {
          cls_val = 150;
          cls_done = true;
        }
      }
      if (!(in_x && in_y)) continue;
      int x0, x1i, y0, y1i;
      float ax0, ax1, ay0, ay1;
      cv_tap(x - r.x1, static_cast<double>(M) / bw, M, x0, x1i, ax0, ax1);
      cv_tap(y - r.y1, static_cast<double>(M) / bh, M, y0, y1i, ay0, ay1);
      const float* m = pmasks + static_cast<long long>(i) * M * M;
      const float r0 = __fadd_rn(__fmul_rn(m[y0 * M + x0], ax0), __fmul_rn(m[y0 * M + x1i], ax1));
      const float r1 = __fadd_rn(__fmul_rn(m[y1i * M + x0], ax0), __fmul_rn(m[y1i * M + x1i], ax1));
      const float v = __fadd_rn(__fmul_rn(r0, ay0), __fmul_rn(r1, ay1));
      if (v >= thresh) {
        if (!inst_done) {
          inst_val = i + 1;
          inst_done = true;
        }
        if (!cls_done) {
          cls_val = r.cls;
          cls_done = true;
        }
      }
    }
  }
  if (x >= W) return;
  const long long o = (static_cast<long long>(b) * H + y) * W + x;
  if (inst_img) inst_img[o] = inst_val;
  if (cls_img) cls_img[o] = cls_val;
  if (bgr) {
    // _get_voc_color_map (vis_seg.py:133-148): bit j of each colour channel comes from bits
    // 3j, 3j+1, 3j+2 of the class id, most significant first; stored BGR as demo.py:163 does.
    int cid = cls_val & 255, r = 0, g = 0, bl = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      r |= (cid & 1) << (7 - j);
      g |= ((cid >> 1) & 1) << (7 - j);
      bl |= ((cid >> 2) & 1) << (7 - j);
      cid >>= 3;
    }
    bgr[o * 3 + 0] = static_cast<unsigned char>(bl);
    bgr[o * 3 + 1] = static_cast<unsigned char>(g);
    bgr[o * 3 + 2] = static_cast<unsigned char>(r);
  }
}

// Binarised, box-sized masks packed one after another (voc_eval.py:249-251 resizes every
// prediction this way before mask_overlap): out[offset[i] + dy * bw + dx] = resized >= thresh.
// grid (ceil(max_area/256), n).
__global__ void __launch_bounds__(256)
binarize_masks_kernel(const int* __restrict__ rboxes, const float* __restrict__ masks, int M,
                      float thresh, const long long* __restrict__ offsets,
                      unsigned char* __restrict__ out) {
  const int i = blockIdx.y;
  const int x1 = rboxes[i * 4 + 0], y1 = rboxes[i * 4 + 1];
  const int bw = rboxes[i * 4 + 2] - x1 + 1, bh = rboxes[i * 4 + 3] - y1 + 1;
  if (bw <= 0 || bh <= 0) return;
  const float* m = masks + static_cast<long long>(i) * M * M;
  for (long long p = blockIdx.x * blockDim.x + threadIdx.x; p < static_cast<long long>(bw) * bh;
       p += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int dx = static_cast<int>(p % bw), dy = static_cast<int>(p / bw);
    int x0, x1i, y0, y1i;
    float ax0, ax1, ay0, ay1;
    cv_tap(dx, static_cast<double>(M) / bw, M, x0, x1i, ax0, ax1);
    cv_tap(dy, static_cast<double>(M) / bh, M, y0, y1i, ay0, ay1);
    const float r0 = __fadd_rn(__fmul_rn(m[y0 * M + x0], ax0), __fmul_rn(m[y0 * M + x1i], ax1));
    const float r1 = __fadd_rn(__fmul_rn(m[y1i * M + x0], ax0), __fmul_rn(m[y1i * M + x1i], ax1));
    const float v = __fadd_rn(__fmul_rn(r0, ay0), __fmul_rn(r1, ay1));
    out[offsets[i] + p] = v >= thresh ? 1 : 0;
  }
}

}  // namespace mnc

extern "C" int mnc_paste_instances(const float* boxes, int box_dim, const float* masks,
                                   const int* cls, const int* counts, int batch, int max_n,
                                   int mask_size, int H, int W, float thresh, int* inst_img,
                                   int* cls_img, unsigned char* bgr, void* stream) {
  if (batch <= 0 || max_n < 0 || box_dim < 4 || mask_size <= 0 || H <= 0 || W <= 0)
    return MNC_ERR_ARG;
  dim3 grid((W + 127) / 128, H, batch);
  mnc::paste_instances_kernel<<<grid, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      boxes, box_dim, masks, cls, counts, max_n, mask_size, H, W, thresh, inst_img, cls_img, bgr);
  return mnc::check_launch();
}

extern "C" int mnc_binarize_masks(const int* rboxes, const float* masks, int n, int mask_size,
                                  float thresh, const long long* offsets, int max_area,
                                  unsigned char* out, void* stream) {
  if (n < 0 || mask_size <= 0) return MNC_ERR_ARG;
  if (n == 0 || max_area <= 0) return MNC_OK;
  int gx = (max_area + 255) / 256;
  if (gx > 1024) gx = 1024;
  mnc::binarize_masks_kernel<<<dim3(gx, n), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      rboxes, masks, mask_size, thresh, offsets, out);
  return mnc::check_launch();
}
