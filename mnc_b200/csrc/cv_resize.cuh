// cv2.resize INTER_LINEAR (OpenCV, a dependency of the reference, not part of it), one axis, shared
// by the result rendering (render.cu) and the training bridge layers (train_bridge.cu): destination
// index d of an axis resized from n source samples with scale = n / dst.  Restated as in
// preprocess.cu: fx = fma(d + 0.5, scale, -0.5) in double (one rounding), floor, clamp (sx < 0 ->
// 0, frac 0; sx >= n - 1 -> n - 1, frac 0).  The caller runs the horizontal pass, then the
// vertical one, in fp32 with separately rounded products and sums.  tests/cv_resize.py models
// this rule bit for bit; the tests hold every kernel that uses it to that model.
#pragma once

#include <cuda_runtime.h>

namespace mnc {

__device__ __forceinline__ void cv_tap(int d, double scale, int n, int& i0, int& i1, float& a0,
                                       float& a1) {
  const double fd = fma(d + 0.5, scale, -0.5);  // fused, as nvcc contracts it; see preprocess.cu
  int s = static_cast<int>(floor(fd));
  float f = static_cast<float>(fd - s);
  if (s < 0) {
    f = 0.f;
    s = 0;
  }
  if (s >= n - 1) {
    i0 = i1 = n - 1;
    f = 0.f;
  } else {
    i0 = s;
    i1 = s + 1;
  }
  a0 = 1.f - f;
  a1 = f;
}

}  // namespace mnc
