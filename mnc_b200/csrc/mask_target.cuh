// The mask target of one foreground row, shared by the two TRAIN layers that write one:
// StageBridgeLayer (train_bridge.cu) and ProposalTargetLayer (rpn_train.cu).  Both call
// intersect_mask (lib/transform/mask_transform.py:49-80) on a row's rounded ex box and gt box and
// describe the row by the same 12-float gt_mask_info record (gt index, mask height, width, label,
// ex box, gt box), so the restatement reads only that record and the gt mask.
#pragma once

#include <cuda_runtime.h>

#include "cv_resize.cuh"

namespace mnc {

// The value the gt-mask crop puts at image position (x, y) inside the box intersection; 0 outside
// the crop (mask_info) and outside the stored mask.
__device__ __forceinline__ float gt_plane(const float* __restrict__ m, int Hm, int Wm, int mh,
                                          int mw, int gx1, int gy1, int x, int y) {
  const int gx = x - gx1, gy = y - gy1;
  return (gx < mw && gy < mh && gx < Wm && gy < Hm) ? m[gy * Wm + gx] : 0.f;
}

// Called by every thread of a CTA for output row p: intersect_mask of the row described by its
// gt_mask_info record `mi`, resized to M x M and binarised into t, and the mask weight (1 for
// foreground rows) into w.  Each of the M x M cv2.resize samples reads its <= 4 taps straight from
// the gt mask (or 0); the ex-box sized plane of the reference is never materialised.
__device__ __forceinline__ void mask_target_row(const float* __restrict__ mi, bool fg,
                                                const float* __restrict__ gt_masks, int G, int Hm,
                                                int Wm, int M, float thresh, float* __restrict__ t,
                                                float* __restrict__ w) {
  const int MM = M * M;
  const int a = static_cast<int>(mi[0]), mh = static_cast<int>(mi[1]), mw = static_cast<int>(mi[2]);
  const int ex1 = static_cast<int>(mi[4]), ey1 = static_cast<int>(mi[5]);
  const int ex2 = static_cast<int>(mi[6]), ey2 = static_cast<int>(mi[7]);
  const int gx1 = static_cast<int>(mi[8]), gy1 = static_cast<int>(mi[9]);
  const int ix1 = max(ex1, gx1), iy1 = max(ey1, gy1);
  const int ix2 = min(ex2, static_cast<int>(mi[10])), iy2 = min(ey2, static_cast<int>(mi[11]));
  const bool live = fg && ix1 <= ix2 && iy1 <= iy2 && a >= 0 && a < G;
  const int ew = ex2 - ex1 + 1, eh = ey2 - ey1 + 1;
  const float* m = gt_masks + static_cast<long long>(a) * Hm * Wm;
  for (int s = threadIdx.x; s < MM; s += blockDim.x) {
    w[s] = fg ? 1.f : 0.f;
    float out = 0.f;
    if (live) {
      const int dy = s / M, dx = s % M;
      int x0, x1, y0, y1;
      float ax0, ax1, ay0, ay1;
      cv_tap(dx, static_cast<double>(ew) / M, ew, x0, x1, ax0, ax1);
      cv_tap(dy, static_cast<double>(eh) / M, eh, y0, y1, ay0, ay1);
      float v[2][2];
      const int ys[2] = {y0, y1}, xs[2] = {x0, x1};
#pragma unroll
      for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int x = ex1 + xs[q], y = ey1 + ys[u];
          v[u][q] = (x >= ix1 && x <= ix2 && y >= iy1 && y <= iy2)
                        ? gt_plane(m, Hm, Wm, mh, mw, gx1, gy1, x, y) : 0.f;
        }
      const float r0 = __fadd_rn(__fmul_rn(v[0][0], ax0), __fmul_rn(v[0][1], ax1));
      const float r1 = __fadd_rn(__fmul_rn(v[1][0], ax0), __fmul_rn(v[1][1], ax1));
      out = __fadd_rn(__fmul_rn(r0, ay0), __fmul_rn(r1, ay1)) >= thresh ? 1.f : 0.f;
    }
    t[s] = out;
  }
}

}  // namespace mnc
