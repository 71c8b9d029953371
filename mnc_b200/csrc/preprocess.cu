// Input preparation on the device: prep_im_for_blob + im_list_to_blob
// (reference lib/utils/blob.py:17-50): uint8 BGR HWC image -> float32, minus cfg.PIXEL_MEANS,
// cv2.resize(fx = fy = scale, INTER_LINEAR), HWC -> NCHW blob.
//
// OpenCV's float INTER_LINEAR rule is restated (OpenCV is a dependency of the reference, not part
// of it): source coordinate fx = fma(dx + 0.5, 1 / scale, -0.5) in double, sx = floor(fx); sx < 0 ->
// (0, frac 0); sx >= W-1 -> (W-1, frac 0); horizontal interpolation first, then vertical, in fp32
// with separately rounded products and sums.  This is the device's rule, pinned bit for bit by
// tests/cv_resize.py; cv2's own bits depend on whether IPP runs and on the CPU (DESIGN.md §6).
#include <cuda_runtime.h>
#include <cstdint>

#include "mnc_b200.h"
#include "launch_util.h"

namespace mnc {

struct LinTap {
  int i0, i1;
  float a0, a1;
};

__device__ __forceinline__ LinTap lin_tap(int d, double inv_scale, int n) {
  // the coordinate is one fused multiply-add in double (written out, so that the rule does not
  // depend on nvcc's contraction) and the fraction is rounded to fp32 once; an fp32 coordinate
  // would lose 1e-5 of the fraction at x ~ 200 and 3e-3 of a pixel value -- measured against cv2
  const double fd = fma(d + 0.5, inv_scale, -0.5);
  int s = static_cast<int>(floor(fd));
  float f = static_cast<float>(fd - s);
  if (s < 0) {
    f = 0.f;
    s = 0;
  }
  LinTap t;
  if (s >= n - 1) {
    t.i0 = t.i1 = n - 1;
    f = 0.f;
  } else {
    t.i0 = s;
    t.i1 = s + 1;
  }
  t.a0 = 1.f - f;
  t.a1 = f;
  return t;
}

// grid (ceil(out_w/128), out_h, batch); one thread per output pixel, 3 channels.
__global__ void __launch_bounds__(128)
prep_image_kernel(const uint8_t* __restrict__ img, int H, int W, double m0, double m1, double m2,
                  double inv_scale, int out_h, int out_w, float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y;
  const int b = blockIdx.z;
  if (x >= out_w) return;
  const LinTap tx = lin_tap(x, inv_scale, W);
  const LinTap ty = lin_tap(y, inv_scale, H);
  const uint8_t* base = img + static_cast<long long>(b) * H * W * 3;
  const double means[3] = {m0, m1, m2};
  float* ob = out + static_cast<long long>(b) * 3 * out_h * out_w + static_cast<long long>(y) * out_w + x;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    // `im = im.astype(np.float32); im -= pixel_means`: float32(double(pixel) - mean)
    const float p00 = static_cast<float>(static_cast<double>(base[(static_cast<long long>(ty.i0) * W + tx.i0) * 3 + c]) - means[c]);
    const float p01 = static_cast<float>(static_cast<double>(base[(static_cast<long long>(ty.i0) * W + tx.i1) * 3 + c]) - means[c]);
    const float p10 = static_cast<float>(static_cast<double>(base[(static_cast<long long>(ty.i1) * W + tx.i0) * 3 + c]) - means[c]);
    const float p11 = static_cast<float>(static_cast<double>(base[(static_cast<long long>(ty.i1) * W + tx.i1) * 3 + c]) - means[c]);
    const float r0 = __fadd_rn(__fmul_rn(p00, tx.a0), __fmul_rn(p01, tx.a1));
    const float r1 = __fadd_rn(__fmul_rn(p10, tx.a0), __fmul_rn(p11, tx.a1));
    ob[static_cast<long long>(c) * out_h * out_w] = __fadd_rn(__fmul_rn(r0, ty.a0), __fmul_rn(r1, ty.a1));
  }
}

}  // namespace mnc

extern "C" int mnc_prep_images(const unsigned char* img_bgr_hwc, int batch, int H, int W,
                               const double* pixel_means3, double scale, int out_h, int out_w,
                               float* out_nchw, void* stream) {
  if (batch <= 0 || H <= 0 || W <= 0 || out_h <= 0 || out_w <= 0 || scale <= 0) return MNC_ERR_ARG;
  dim3 grid((out_w + 127) / 128, out_h, batch);
  mnc::prep_image_kernel<<<grid, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      img_bgr_hwc, H, W, pixel_means3[0], pixel_means3[1], pixel_means3[2], 1.0 / scale, out_h,
      out_w, out_nchw);
  return mnc::check_launch();
}
