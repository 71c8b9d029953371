// RoI sampling geometry shared by the ROIWarping forward kernels (roi_ops.cu) and their backward
// passes (roi_backward.cu): the RoI's rounded start and forward bin size, and the bilinear taps of
// one sample coordinate along one axis.
#pragma once

#include <cuda_runtime.h>

namespace mnc {

constexpr int kMaxPooled = 32;   // pooled_h, pooled_w <= 32

struct AxisTap {
  int lo, hi;   // indices of the two taps along the axis (lo == hi at the last row / column)
  float l, h;   // l = frac, h = 1 - frac
  int ok;       // 0: sample out of range -> output 0
};

// roi_warping_layer.cu:18-47 for one axis.
__device__ __forceinline__ AxisTap axis_tap(float x, int dim) {
  AxisTap t;
  t.ok = !(x < -0.5 || x > dim - 0.5);
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
  t.l = __fsub_rn(x, static_cast<float>(lo));
  t.h = __fsub_rn(1.f, t.l);
  return t;
}

struct RoiGeom {
  int level;
  float start_h, start_w, bin_h, bin_w;
};

// roi_warping_layer.cu:78-90
__device__ __forceinline__ RoiGeom roi_geom(const float* roi, float spatial_scale, int ph_n,
                                            int pw_n) {
  RoiGeom g;
  g.level = static_cast<int>(roi[0]);
  const float sw = roundf(__fmul_rn(roi[1], spatial_scale));
  const float sh = roundf(__fmul_rn(roi[2], spatial_scale));
  const float ew = roundf(__fmul_rn(roi[3], spatial_scale));
  const float eh = roundf(__fmul_rn(roi[4], spatial_scale));
  const float rw = fmaxf(__fsub_rn(ew, sw), 0.f);
  const float rh = fmaxf(__fsub_rn(eh, sh), 0.f);
  g.start_h = sh;
  g.start_w = sw;
  g.bin_h = __fdiv_rn(rh, static_cast<float>(ph_n));
  g.bin_w = __fdiv_rn(rw, static_cast<float>(pw_n));
  return g;
}

}  // namespace mnc
