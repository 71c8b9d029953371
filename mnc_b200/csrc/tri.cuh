// Tri-plane ("precision mode 1") element conversions shared by the kernels that produce or consume
// operands of the FP8-corrected tensor-core path (igemm_tc.cu has the format's definition).
#pragma once
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cstdint>

namespace mnc {

struct Tri2 {
  uint32_t h;      // two fp16
  uint16_t l, c;   // two e4m3 each
};

// (x0, x1) * scale -> fp16 value, e4m3 residual (x 2^6), e4m3 copy (x 2^-5); all saturating.
__device__ __forceinline__ Tri2 tri_pack2(float x0, float x1, float scale) {
  const float a0 = fminf(fmaxf(x0 * scale, -65504.f), 65504.f);
  const float a1 = fminf(fmaxf(x1 * scale, -65504.f), 65504.f);
  const __half2 h = __floats2half2_rn(a0, a1);
  const float2 hf = __half22float2(h);
  Tri2 t;
  t.h = *reinterpret_cast<const uint32_t*>(&h);
  t.l = __nv_cvt_float2_to_fp8x2(make_float2((a0 - hf.x) * 64.f, (a1 - hf.y) * 64.f), __NV_SATFINITE, __NV_E4M3);
  t.c = __nv_cvt_float2_to_fp8x2(make_float2(a0 * 0.03125f, a1 * 0.03125f), __NV_SATFINITE, __NV_E4M3);
  return t;
}

// value carried by the two precise planes, still scaled by 2^exp: h + l / 2^6
__device__ __forceinline__ float2 tri_unpack2(uint32_t h, uint16_t l) {
  const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&h));
  const __half2_raw lr = __nv_cvt_fp8x2_to_halfraw2(l, __NV_E4M3);
  const float2 lf = __half22float2(*reinterpret_cast<const __half2*>(&lr));
  return make_float2(fmaf(lf.x, 0.015625f, hf.x), fmaf(lf.y, 0.015625f, hf.y));
}

// four consecutive channels at element offset `off` (off % 4 == 0)
__device__ __forceinline__ void st_tri4(__half* h, uint8_t* l, uint8_t* c, long long off,
                                        const float4 v, float scale) {
  const Tri2 a = tri_pack2(v.x, v.y, scale), b = tri_pack2(v.z, v.w, scale);
  __stcs(reinterpret_cast<uint2*>(h + off), make_uint2(a.h, b.h));
  __stcs(reinterpret_cast<unsigned int*>(l + off), static_cast<uint32_t>(a.l) | (static_cast<uint32_t>(b.l) << 16));
  __stcs(reinterpret_cast<unsigned int*>(c + off), static_cast<uint32_t>(a.c) | (static_cast<uint32_t>(b.c) << 16));
}
__device__ __forceinline__ float4 ld_tri4(const __half* h, const uint8_t* l, long long off) {
  const uint2 hw = __ldg(reinterpret_cast<const uint2*>(h + off));
  const uint32_t lw = __ldg(reinterpret_cast<const unsigned int*>(l + off));
  const float2 a = tri_unpack2(hw.x, static_cast<uint16_t>(lw & 0xffffu));
  const float2 b = tri_unpack2(hw.y, static_cast<uint16_t>(lw >> 16));
  return make_float4(a.x, a.y, b.x, b.y);
}

// Host-side argument check of the entry points that use st_tri4 / ld_tri4: four elements move at a
// time, 8 bytes of the fp16 plane and 4 bytes of each e4m3 plane (c may be null: not accessed).
inline bool tri_planes_aligned(const void* h, const void* l, const void* c) {
  return reinterpret_cast<uintptr_t>(h) % 8 == 0 && reinterpret_cast<uintptr_t>(l) % 4 == 0 &&
         (c == nullptr || reinterpret_cast<uintptr_t>(c) % 4 == 0);
}

}  // namespace mnc
