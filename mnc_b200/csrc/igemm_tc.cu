// Implicit-GEMM convolution / inner-product on the sm_90a tensor cores (wgmma).
//
// Replaces, for the MNC inference path, Caffe's Convolution layer
// (caffe-mnc/src/caffe/layers/cudnn_conv_layer.cu:11-54, conv_layer.cu:8-23 +
// util/im2col.cu:9-39) and InnerProduct layer (inner_product_layer.cu:21-27).
//
// Design:
//  * activations live in HBM as NHWC, split into two bf16 planes (hi, lo) with
//    x ~= hi + lo (16 mantissa bits).  Weights likewise, stored [Cout][tap][Cin].
//  * one persistent CTA per SM, three warpgroups: warpgroup 0 is the producer (one warp issues
//    TMA loads into a ring of stages and the group gives its registers back), warpgroups 1 and 2
//    are consumers: each owns 64 of the tile's 128 pixel rows, issues wgmma on the stage's
//    shared-memory operands and keeps its fp32 accumulators (64 x BN) in registers.
//  * im2col is folded into the TMA descriptor: the A tile for filter tap (dy,dx)
//    is the 4-D box [1, TH, TW, 64ch] at (h0+dy, w0+dx); out-of-image rows/cols
//    are zero-filled by TMA, which *is* the conv zero padding.
//  * fp32-class accuracy on bf16 tensor cores: D += Ahi*Bhi + Ahi*Blo + Alo*Bhi
//    (the dropped Alo*Blo term is ~2^-18 relative).
//  * epilogue: the consumers pass their accumulator fragments through shared memory so that a
//    thread owns one pixel row of a 32-channel chunk -> +bias -> ReLU -> re-split to (hi, lo)
//    bf16 NHWC (staged and written by TMA stores), or raw fp32 (split-K partials / final logits).
//    The producer keeps filling the ring for the next tile meanwhile.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>

#include "mnc_b200.h"
#include "ptx.cuh"
#include "tri.cuh"
#include "launch_util.h"

namespace mnc {

struct IgemmArgs {
  int batch, H, W;
  int Cin, Cout;
  int taps;  // 1 (inner product / 1x1) or 9 (3x3, pad 1, stride 1)
  int tiles_h, tiles_w, tiles_n;
  int k_steps;  // taps * Cin / 64
  int split_k;
  int relu;
  // 0: split bf16 (hi, lo); 1: fp32; 2: split bf16 after a fused 2x2/2 ceil-mode max pool;
  // 4: tri-plane (fp16 hi, e4m3 lo, e4m3 hi copy -- see "precision mode 1" below); 5: tri-plane
  // after the fused max pool
  int out_mode;
  const float* bias;
  __nv_bfloat16* out_hi;   // modes 4/5: the fp16 plane
  __nv_bfloat16* out_lo;   // modes 4/5: the e4m3 residual plane
  uint8_t* out_x;          // modes 4/5: the e4m3 copy of the value
  float* out_f32;
  float acc_scale;         // accumulator -> true value (1 for bf16 operands; 2^-(ea+ew) in mode 1)
  float out_scale;         // modes 4/5: 2^ea of the tensor being written
  unsigned int* amax;      // optional: atomicMax of |output| as float bits (scale calibration)
  long long out_pix_stride;  // elements between consecutive pixels (rows)
  int out_ch_offset;
  long long split_stride;  // elements between split-K partial planes (fp32 mode)
  int vec_ok;              // 16-byte vector stores are aligned
  int tma_store;           // out_modes 0 / 4: epilogue stages tiles in smem and TMA-stores them
};

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;   // K elements per stage: 128-byte rows of the 2-byte planes
constexpr int kSmemMax = 227 * 1024;   // opt-in shared memory of one sm_90 CTA

// epilogue shared memory: the accumulator exchange (two 32-channel chunks of 128 rows, fp32, rows
// padded to 33 words so that both the fragment writes and the row reads spread over the banks)
// and the TMA-store staging (one buffer per consumer warpgroup x (hi, lo) x 128 rows x 64 B) share
// one region: a chunk passes through the exchange before it is staged, so the exchange waits for
// the previous chunk's stores to have read the staging instead of taking 33 KB of its own.  That
// leaves the operand ring of conv tiles a third stage at BN = 128 (and a fourth at BN = 64).
constexpr int kXchgStride = 33;
constexpr int kXchgBytes = 2 * 128 * kXchgStride * 4;
constexpr int kStagingBytes = 2 * 2 * 128 * 64;
constexpr int kEpiBytes = kXchgBytes > kStagingBytes ? kXchgBytes : kStagingBytes;
constexpr int kBarrierBytes = 1024;

// A stage holds one 2-byte and one 2-byte (mode 0) or two 1-byte (mode 1) planes of the A tile
// and of the B tile: the same bytes in both precision modes.
template <int BN, int TH = 8>
struct IgemmCfg {
  static constexpr int kABytes = kBlockM * kBlockK * 2;  // one 2-byte plane of the A tile
  static constexpr int kBBytes = BN * kBlockK * 2;       // one 2-byte plane of the B tile
  static constexpr int kStageBytes = 2 * kABytes + 2 * kBBytes;
  static constexpr int kFixedBytes = 1024 /*align*/ + kBarrierBytes + kEpiBytes;
  static constexpr int kStagesRaw = (kSmemMax - kFixedBytes) / kStageBytes;
  // the deeper ring pays for conv tiles only: measured on the H100, linear tiles (TH = 1) with a
  // third / fourth stage made the whole step 6 % slower, so they run two / three
  static constexpr int kCap = TH == 1 ? (BN == 128 ? 2 : 3) : 8;
  static constexpr int kStages = kStagesRaw > kCap ? kCap : kStagesRaw;
  static constexpr int kSmemBytes = kStages * kStageBytes + kFixedBytes;
  static_assert(kStages >= 2, "the ring needs two stages");
};
static_assert(IgemmCfg<128>::kStages == 3 && IgemmCfg<64>::kStages == 4,
              "conv tiles run 3 operand stages at BN = 128 and 4 at BN = 64");

struct Tile {
  int img, h0, w0, n0, ks;
  int kb, kn, kstride;   // this work item's k-steps: kb, kb + kstride, ... (kn of them)
};

__device__ __forceinline__ Tile decode_tile(const IgemmArgs& p, int t, int TH, int TW, int BN) {
  const int per_img = p.tiles_h * p.tiles_w;
  const int spatial = p.batch * per_img;
  const int sp = t % spatial;
  const int rest = t / spatial;
  const int nt = rest % p.tiles_n;
  Tile tl;
  tl.ks = rest / p.tiles_n;
  tl.img = sp / per_img;
  const int r = sp % per_img;
  tl.h0 = (r / p.tiles_w) * TH;
  tl.w0 = (r % p.tiles_w) * TW;
  tl.n0 = nt * BN;
  // Split-K work items take INTERLEAVED k-steps (ks, ks + split, ks + 2*split, ...): the CTAs that
  // share a row tile start together and advance in step, so at any moment they read adjacent
  // 128-byte segments of the same activation rows -- DRAM sees ~split*128 contiguous bytes per row
  // instead of isolated 128-byte touches 200 KB apart (fc6_maskest: K = 100352).
  tl.kb = tl.ks;
  tl.kstride = p.split_k;
  tl.kn = (p.k_steps - tl.ks + p.split_k - 1) / p.split_k;
  return tl;
}

// ---------------------------------------------------------------------- precision mode 1 format
// "tri-plane" activations / weights (DESIGN.md section 3): a tensor with per-tensor exponent e is
// stored as   h = fp16(x * 2^e)            (main operand, fp16 wgmma)
//             l = e4m3((x*2^e - h) * 2^6)  (residual, 2^-11 of h at most)
//             c = e4m3(x * 2^e * 2^-5)     (low-precision copy of the value)
// for activations, and with the residual scaled by 2^5 / the copy by 2^-6 for weights, so that
//   X.W * 2^(ex+ew) = Xh.Wh  +  Xl.Wc  +  Xc.Wl      (2^6 * 2^-6 = 2^-5 * 2^5 = 1)
// The first product runs as fp16 MMAs, the two corrections as ONE K-concatenated chain of FP8
// MMAs at twice the rate: 2 tensor-work units per MAC instead of the 3 of the split-bf16 scheme,
// at 1.1e-5 relative error per layer (scripts/fp8_correction_model.py; measured in tests).
// The FP8 chain has an accumulator of its own, added to the fp16 one in the epilogue: the
// corrections are 2^-11 of the result, so whatever precision the FP8 path keeps in its adds is
// spent on them alone and never on the main product.
// (element conversions: tri.cuh)

// ---------------------------------------------------------------------------------- epilogue
// One tile's accumulators -> global memory (bias, ReLU, optional 2x2 ceil-mode max pool, re-split,
// store), run by the 256 consumer threads.  Consumer warpgroup `grp` holds rows [64 grp, 64 grp +
// 64) in wgmma fragment order; per 64-column block both groups write their fragments to the
// exchange buffer and then group g takes the block's 32-column chunk g with one thread per pixel
// row (row = thread index in the group), which is the unit the stores and the pool window want.
struct EpiState {
  int chunk_ctr;
  float amx;   // max |output| seen by this thread (valid pixels only)
};

template <int TH, int TW, int BN>
__device__ __forceinline__ void epilogue_tile(const IgemmArgs& p, const CUtensorMap* tm_o_hi_p,
                                              const CUtensorMap* tm_o_lo_p,
                                              const CUtensorMap* tm_o_x_p, uint8_t* staging,
                                              float (&acc)[BN / 64][32], const Tile& tl, int grp,
                                              EpiState& st) {
  const int tid = threadIdx.x & 127;
  const int lane = threadIdx.x & 31;
  constexpr int NBUF = 1;             // staging buffers per group
  const int lead = 128 + grp * 128;   // the group's bulk-store thread
  const int row = tid;
  int& chunk_ctr = st.chunk_ctr;
  float& amx = st.amx;
  const float asc = p.acc_scale;
  const int img = tl.img, h0 = tl.h0, w0 = tl.w0, n0 = tl.n0, ks = tl.ks;
  const int h = h0 + row / TW;
  const int w = w0 + row % TW;
  const bool valid = (h < p.H) && (w < p.W);
  const long long pix = (static_cast<long long>(img) * p.H + h) * p.W + w;
  // fragment coordinates of this thread (ptx.cuh, wgmma_*_n64)
  const int frow = grp * 64 + (tid >> 5) * 16 + (lane >> 2);
  const int fcol = (lane & 3) * 2;
#pragma unroll
  for (int nb = 0; nb < BN / 64; ++nb) {
    const int c0 = nb * 64 + grp * 32;
    uint32_t r[32];
    {
      float* xchg = reinterpret_cast<float*>(staging);
      // the exchange overwrites the staging buffers: the previous chunk's stores must have read them
      if (p.tma_store) {
        if (threadIdx.x == lead) ptx::tma_store_wait_read<0>();
        ptx::named_bar_sync(1, 256);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int col = j * 8 + fcol;
        float* d0 = xchg + ((col >> 5) * 128 + frow) * kXchgStride + (col & 31);
        d0[0] = acc[nb][4 * j];
        d0[1] = acc[nb][4 * j + 1];
        d0[8 * kXchgStride] = acc[nb][4 * j + 2];
        d0[8 * kXchgStride + 1] = acc[nb][4 * j + 3];
      }
      ptx::named_bar_sync(1, 256);
      const float* s0 = xchg + (grp * 128 + row) * kXchgStride;
#pragma unroll
      for (int j = 0; j < 32; ++j) r[j] = __float_as_uint(s0[j]);
      ptx::named_bar_sync(2, 256);   // the buffer may be rewritten
    }
      const int ch0 = n0 + c0;
      if (p.out_mode == 3) continue;  // diagnostic: accumulators are drained and discarded
      if (p.out_mode == 2 || p.out_mode == 5) {
        // Fused 2x2 stride-2 ceil-mode max pool (pooling_layer.cu:11-47).  A warp holds 32/TW
        // whole image rows of the pixel tile (TW = 16: two rows, TW = 8: four), so the pool window
        // of an even (row, column) is lanes {l, l^1, l^TW, l^(TW+1)}: two shuffles per channel.
        // Each of the 4 lanes of a window then stores 8 of the chunk's 32 channels.
        // The 4 lanes of a window end up with 8 channels each by a reduce-scatter: exchange halves
        // with the x neighbour (16 shuffles), then quarters with the y neighbour (8) -- 24 shuffles
        // and 24 max per chunk instead of 64 + 64 for all-channels-everywhere.
        const bool odd_x = (lane & 1) != 0;
        const bool odd_y = ((lane / TW) & 1) != 0;
        const int part = (odd_x ? 2 : 0) | (odd_y ? 1 : 0);   // this lane stores channels part*8 .. +7
        const int hl = (row / TW) & ~1;   // tile-local top row / left column of this lane's window
        const int wl = (row % TW) & ~1;
        // max commutes with the monotone epilogue  x -> relu(x * scale + bias)  (scale > 0), so the
        // window maximum is taken on the RAW accumulators and the epilogue arithmetic runs on the 8
        // surviving channels of each lane only (bit-identical: fma and max are monotone / exact)
        float x[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) x[j] = __uint_as_float(r[j]);
        if (!__all_sync(0xffffffffu, valid)) {   // ragged tile: rows outside the image never win
#pragma unroll
          for (int j = 0; j < 32; ++j) x[j] = valid ? x[j] : -3.402823466e+38f;
        }
        float y[16], m[8];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float keep = odd_x ? x[j + 16] : x[j];
          const float send = odd_x ? x[j] : x[j + 16];
          y[j] = fmaxf(keep, __shfl_xor_sync(0xffffffffu, send, 1));
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float keep = odd_y ? y[j + 8] : y[j];
          const float send = odd_y ? y[j] : y[j + 8];
          m[j] = fmaxf(keep, __shfl_xor_sync(0xffffffffu, send, TW));
        }
        const int hp = (h0 + hl) >> 1;
        const int wp = (w0 + wl) >> 1;
        const int Ho = (p.H + 1) >> 1, Wo = (p.W + 1) >> 1;
        const int chp = ch0 + part * 8;
        if (hp < Ho && wp < Wo && (h0 + hl) < p.H && (w0 + wl) < p.W &&
            chp < p.Cout) {
          const long long ppix = (static_cast<long long>(img) * Ho + hp) * Wo + wp;
          const long long poff = ppix * p.out_pix_stride + p.out_ch_offset + chp;
          float bv[8];
          if (p.bias != nullptr && chp + 8 <= p.Cout && (reinterpret_cast<uintptr_t>(p.bias + chp) & 15) == 0) {
            const float4 b0 = __ldg(reinterpret_cast<const float4*>(p.bias + chp));
            const float4 b1 = __ldg(reinterpret_cast<const float4*>(p.bias + chp) + 1);
            bv[0] = b0.x, bv[1] = b0.y, bv[2] = b0.z, bv[3] = b0.w;
            bv[4] = b1.x, bv[5] = b1.y, bv[6] = b1.z, bv[7] = b1.w;
          } else {
#pragma unroll
            for (int j = 0; j < 8; ++j)
              bv[j] = (p.bias != nullptr && chp + j < p.Cout) ? __ldg(p.bias + chp + j) : 0.f;
          }
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            m[j] = m[j] * asc + bv[j];
            if (p.relu) m[j] = fmaxf(m[j], 0.f);
            if (chp + j < p.Cout) amx = fmaxf(amx, fabsf(m[j]));   // max |pooled output|
          }
          if (p.out_mode == 5) {
            uint32_t hw[4], lw[2], cw[2];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const Tri2 tr = tri_pack2(m[2 * e], m[2 * e + 1], p.out_scale);
              hw[e] = tr.h;
              if (e & 1) {
                lw[e >> 1] |= static_cast<uint32_t>(tr.l) << 16;
                cw[e >> 1] |= static_cast<uint32_t>(tr.c) << 16;
              } else {
                lw[e >> 1] = tr.l;
                cw[e >> 1] = tr.c;
              }
            }
            *reinterpret_cast<uint4*>(reinterpret_cast<__half*>(p.out_hi) + poff) =
                make_uint4(hw[0], hw[1], hw[2], hw[3]);
            *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(p.out_lo) + poff) = make_uint2(lw[0], lw[1]);
            *reinterpret_cast<uint2*>(p.out_x + poff) = make_uint2(cw[0], cw[1]);
            continue;
          }
          __nv_bfloat16* ph = p.out_hi + poff;
          __nv_bfloat16* pl = p.out_lo + poff;
          uint32_t hw[4], lw[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float x0 = m[2 * e], x1 = m[2 * e + 1];
            const __nv_bfloat16 h0b = __float2bfloat16_rn(x0);
            const __nv_bfloat16 h1b = __float2bfloat16_rn(x1);
            const __nv_bfloat16 l0b = __float2bfloat16_rn(x0 - __bfloat162float(h0b));
            const __nv_bfloat16 l1b = __float2bfloat16_rn(x1 - __bfloat162float(h1b));
            hw[e] = static_cast<uint32_t>(__bfloat16_as_ushort(h0b)) |
                    (static_cast<uint32_t>(__bfloat16_as_ushort(h1b)) << 16);
            lw[e] = static_cast<uint32_t>(__bfloat16_as_ushort(l0b)) |
                    (static_cast<uint32_t>(__bfloat16_as_ushort(l1b)) << 16);
          }
          *reinterpret_cast<uint4*>(ph) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
          *reinterpret_cast<uint4*>(pl) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
        }
      } else if (p.tma_store) {
        // ---- out_mode 0 / 4 via shared-memory staging + TMA store: each thread owns one pixel row
        // of the 128 x 32-channel chunk (64 B per 2-byte plane, written with the 64B-swizzle
        // pattern so the 16-byte stores are bank-conflict free; the one-byte planes of mode 4 are
        // 32 B per row, unswizzled); one elected thread then issues the bulk tensor stores.  TMA
        // clips ragged tiles and channel tails, and the global writes
        // are whole rows.
        const bool tri = (p.out_mode == 4);
        const int buf = chunk_ctr % NBUF;
        uint8_t* sb = staging + (grp * NBUF + buf) * (2 * 128 * 64);
        // (the previous store from this buffer was waited for before the exchange)
        if (ch0 < p.Cout) {
          // bias: 8 x 16-byte loads when the chunk is whole and aligned (the usual case)
          float bv[32];
          if (p.bias != nullptr && ch0 + 32 <= p.Cout &&
              (reinterpret_cast<uintptr_t>(p.bias + ch0) & 15) == 0) {
#pragma unroll
            for (int j4 = 0; j4 < 8; ++j4) {
              const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.bias + ch0) + j4);
              bv[4 * j4] = b4.x;
              bv[4 * j4 + 1] = b4.y;
              bv[4 * j4 + 2] = b4.z;
              bv[4 * j4 + 3] = b4.w;
            }
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
              bv[j] = (p.bias != nullptr && ch0 + j < p.Cout) ? __ldg(p.bias + ch0 + j) : 0.f;
          }
          float mx = 0.f;
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            uint32_t hw[4], lw[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              float x0 = __uint_as_float(r[g * 8 + 2 * e]) * asc + bv[g * 8 + 2 * e];
              float x1 = __uint_as_float(r[g * 8 + 2 * e + 1]) * asc + bv[g * 8 + 2 * e + 1];
              if (p.relu) {
                x0 = fmaxf(x0, 0.f);
                x1 = fmaxf(x1, 0.f);
              }
              mx = fmaxf(mx, fmaxf(fabsf(x0), fabsf(x1)));
              if (tri) {
                const Tri2 tr = tri_pack2(x0, x1, p.out_scale);
                hw[e] = tr.h;
                // lw[0..1]: residual bytes, lw[2..3]: copy bytes (8 channels each)
                if (e & 1) {
                  lw[e >> 1] |= static_cast<uint32_t>(tr.l) << 16;
                  lw[2 + (e >> 1)] |= static_cast<uint32_t>(tr.c) << 16;
                } else {
                  lw[e >> 1] = tr.l;
                  lw[2 + (e >> 1)] = tr.c;
                }
              } else {
                // packed conversions: (x0, x1) -> bf16x2 in one instruction; the hi values come
                // back as floats by a shift / mask of the packed word
                const __nv_bfloat162 hp = __floats2bfloat162_rn(x0, x1);
                const uint32_t hbits = *reinterpret_cast<const uint32_t*>(&hp);
                const float f0 = __uint_as_float(hbits << 16);
                const float f1 = __uint_as_float(hbits & 0xffff0000u);
                const __nv_bfloat162 lp = __floats2bfloat162_rn(x0 - f0, x1 - f1);
                hw[e] = hbits;
                lw[e] = *reinterpret_cast<const uint32_t*>(&lp);
              }
            }
            const int off = row * 64 + ((g ^ ((row >> 1) & 3)) << 4);
            *reinterpret_cast<uint4*>(sb + off) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
            if (tri) {
              *reinterpret_cast<uint2*>(sb + 128 * 64 + row * 32 + g * 8) = make_uint2(lw[0], lw[1]);
              *reinterpret_cast<uint2*>(sb + 128 * 96 + row * 32 + g * 8) = make_uint2(lw[2], lw[3]);
            } else {
              *reinterpret_cast<uint4*>(sb + 128 * 64 + off) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
            }
          }
          if (valid) amx = fmaxf(amx, mx);
        }
        ptx::fence_proxy_async();
        ptx::named_bar_sync(3 + grp, 128);
        if (threadIdx.x == lead && ch0 < p.Cout) {
          ptx::tma_store_4d(tm_o_hi_p, sb, ch0, w0, h0, img);
          ptx::tma_store_4d(tm_o_lo_p, sb + 128 * 64, ch0, w0, h0, img);
          if (tri) ptx::tma_store_4d(tm_o_x_p, sb + 128 * 96, ch0, w0, h0, img);
          ptx::tma_store_commit();
        }
        ++chunk_ctr;
      } else if (valid && ch0 < p.Cout) {
        float v[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          float x = __uint_as_float(r[j]) * asc;
          if (p.bias != nullptr && ch0 + j < p.Cout) x += __ldg(p.bias + ch0 + j);
          if (p.relu) x = fmaxf(x, 0.f);
          v[j] = x;
          if (ch0 + j < p.Cout) amx = fmaxf(amx, fabsf(x));
        }
        const bool fullchunk = (ch0 + 32 <= p.Cout) && p.vec_ok;
        if (p.out_mode == 0) {
          __nv_bfloat16* ph = p.out_hi + pix * p.out_pix_stride + p.out_ch_offset + ch0;
          __nv_bfloat16* pl = p.out_lo + pix * p.out_pix_stride + p.out_ch_offset + ch0;
          if (fullchunk) {
#pragma unroll
            for (int g = 0; g < 4; ++g) {
              uint32_t hw[4], lw[4];
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float x0 = v[g * 8 + 2 * e], x1 = v[g * 8 + 2 * e + 1];
                const __nv_bfloat16 h0b = __float2bfloat16_rn(x0);
                const __nv_bfloat16 h1b = __float2bfloat16_rn(x1);
                const __nv_bfloat16 l0b = __float2bfloat16_rn(x0 - __bfloat162float(h0b));
                const __nv_bfloat16 l1b = __float2bfloat16_rn(x1 - __bfloat162float(h1b));
                hw[e] = static_cast<uint32_t>(__bfloat16_as_ushort(h0b)) |
                        (static_cast<uint32_t>(__bfloat16_as_ushort(h1b)) << 16);
                lw[e] = static_cast<uint32_t>(__bfloat16_as_ushort(l0b)) |
                        (static_cast<uint32_t>(__bfloat16_as_ushort(l1b)) << 16);
              }
              *reinterpret_cast<uint4*>(ph + g * 8) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
              *reinterpret_cast<uint4*>(pl + g * 8) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
            }
          } else {
            for (int j = 0; j < 32 && ch0 + j < p.Cout; ++j) {
              const __nv_bfloat16 hb = __float2bfloat16_rn(v[j]);
              ph[j] = hb;
              pl[j] = __float2bfloat16_rn(v[j] - __bfloat162float(hb));
            }
          }
        } else {
          float* po = p.out_f32 + ks * p.split_stride + pix * p.out_pix_stride +
                      p.out_ch_offset + ch0;
          if (fullchunk) {
#pragma unroll
            for (int g = 0; g < 8; ++g)
              *reinterpret_cast<float4*>(po + g * 4) =
                  make_float4(v[g * 4], v[g * 4 + 1], v[g * 4 + 2], v[g * 4 + 3]);
          } else {
            for (int j = 0; j < 32 && ch0 + j < p.Cout; ++j) po[j] = v[j];
          }
        }
      }
  }
}

__device__ __forceinline__ void epilogue_finish(const IgemmArgs& p, int grp, const EpiState& st) {
  if (threadIdx.x == 128 + grp * 128) ptx::tma_store_wait_read<0>();  // smem must outlive the bulk stores
  if (p.amax != nullptr) {
    float amx = st.amx;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amx = fmaxf(amx, __shfl_xor_sync(0xffffffffu, amx, o));
    if ((threadIdx.x & 31) == 0 && amx > 0.f) atomicMax(p.amax, __float_as_uint(amx));
  }
}

// PM (precision mode): 0 = split-bf16 operands (planes hi, lo; 3 bf16 MMAs per k slice);
// 1 = tri-plane operands (fp16 value, e4m3 residual, e4m3 copy; see above): per 64 K-elements
// 4 fp16 MMAs + 4 FP8 MMAs (K = 32 each, double rate) instead of 12 bf16 MMAs.  A stage holds
// A:[h | l | c] then B:[h | c | l] -- same bytes as mode 0 (one 2-byte and two 1-byte planes).
template <int TH, int TW, int BN, int PM>
__global__ void __launch_bounds__(384, 1)
igemm_tc_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                const __grid_constant__ CUtensorMap tm_a_x,
                const __grid_constant__ CUtensorMap tm_b_hi, const __grid_constant__ CUtensorMap tm_b_lo,
                const __grid_constant__ CUtensorMap tm_b_x,
                const __grid_constant__ CUtensorMap tm_o_hi, const __grid_constant__ CUtensorMap tm_o_lo,
                const __grid_constant__ CUtensorMap tm_o_x,
                const IgemmArgs p) {
  static_assert(TH * TW == kBlockM, "pixel tile must have 128 rows");
  using Cfg = IgemmCfg<BN, TH>;
  constexpr int kStages = Cfg::kStages;
  constexpr int kABytes = Cfg::kABytes;
  constexpr int kBBytes = Cfg::kBBytes;
  constexpr int NB = BN / 64;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * Cfg::kStageBytes);
  uint64_t* empty_bar = full_bar + kStages;
  uint8_t* staging = smem + kStages * Cfg::kStageBytes + kBarrierBytes;  // 1024-aligned

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  const int total_tiles = p.split_k * p.tiles_n * p.batch * p.tiles_h * p.tiles_w;
  const int kchunks = p.Cin / kBlockK;
  const int first = blockIdx.x;
  const int stride = gridDim.x;

  if (warp == 0 && lane == 0) {
    ptx::prefetch_tmap(&tm_a_hi);
    ptx::prefetch_tmap(&tm_a_lo);
    ptx::prefetch_tmap(&tm_b_hi);
    ptx::prefetch_tmap(&tm_b_lo);
    if (PM == 1) {
      ptx::prefetch_tmap(&tm_a_x);
      ptx::prefetch_tmap(&tm_b_x);
    }
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < kStages; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 2);   // one arrival per consumer warpgroup
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    ptx::setmaxnreg_dec<40>();
    if (warp == 0) {
      // ------------------------------------------------------------ TMA producer
      // whole warp, warp-uniform arguments; one lane is elected inside each issue (ptx.cuh)
      int stage = 0;
      uint32_t phase = 0;
      // B planes: mode 0 [hi | lo] of kBBytes each; mode 1 [h (kBBytes) | c | l (kBBytes/2 each)]
      constexpr int kNP = (PM == 0) ? 2 : 3;
      const CUtensorMap* amaps[3] = {&tm_a_hi, &tm_a_lo, &tm_a_x};
      const CUtensorMap* bmaps[3] = {&tm_b_hi, &tm_b_lo, &tm_b_x};
      for (int t = first; t < total_tiles; t += stride) {
        const Tile tl = decode_tile(p, t, TH, TW, BN);
        for (int i = 0, k = tl.kb; i < tl.kn; ++i, k += tl.kstride) {
          ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* st = smem + stage * Cfg::kStageBytes;
          ptx::mbar_arrive_expect_tx_w(&full_bar[stage], Cfg::kStageBytes);
          const int tap = k / kchunks;
          const int kc = k - tap * kchunks;
          int dy = 0, dx = 0;
          if (p.taps == 9) {
            dy = tap / 3 - 1;
            dx = tap % 3 - 1;
          }
#pragma unroll
          for (int pl = 0; pl < kNP; ++pl) {
            const int aoff = (PM == 0) ? pl * kABytes : (pl == 0 ? 0 : kABytes + (pl - 1) * (kABytes / 2));
            const int boff = (PM == 0) ? pl * kBBytes : (pl == 0 ? 0 : kBBytes + (pl - 1) * (kBBytes / 2));
            ptx::tma_load_4d_w(st + aoff, amaps[pl], &full_bar[stage], kc * kBlockK, tl.w0 + dx,
                               tl.h0 + dy, tl.img);
            ptx::tma_load_2d_w(st + 2 * kABytes + boff, bmaps[pl], &full_bar[stage],
                               tap * p.Cin + kc * kBlockK, tl.n0);
          }
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ------------------------------------------------- consumers: wgmma main loop + epilogue
    ptx::setmaxnreg_inc<232>();
    const int grp = wg - 1;
    const int tid = threadIdx.x & 127;
    float acc[NB][32];
    float accc[PM == 1 ? NB : 1][32];   // mode 1: the FP8 correction chain
    EpiState est = {0, 0.f};
    int stage = 0;
    uint32_t phase = 0;
    for (int t = first; t < total_tiles; t += stride) {
      const Tile tl = decode_tile(p, t, TH, TW, BN);
      for (int i = 0; i < tl.kn; ++i) {
        ptx::mbar_wait(&full_bar[stage], phase);
        // this group's 64 rows of every A plane; 64-row blocks of the B planes
        const uint32_t a_hi = ptx::smem_u32(smem + stage * Cfg::kStageBytes) + grp * (kABytes / 2);
        const uint32_t b_hi = ptx::smem_u32(smem + stage * Cfg::kStageBytes) + 2 * kABytes;
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) {
          ptx::wgmma_fence_acc(acc[nb]);
          if (PM == 1) ptx::wgmma_fence_acc(accc[nb]);
        }
        ptx::wgmma_fence();
        if (PM == 0) {
          const uint32_t a_lo = a_hi + kABytes;
          const uint32_t b_lo = b_hi + kBBytes;
#pragma unroll
          for (int kk = 0; kk < kBlockK / 16; ++kk) {
            const uint64_t da_hi = ptx::wgmma_desc_rows<128>(a_hi + kk * 32);
            const uint64_t da_lo = ptx::wgmma_desc_rows<128>(a_lo + kk * 32);
            const uint32_t acc0 = (i > 0 || kk > 0) ? 1u : 0u;
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) {
              const uint64_t db_hi = ptx::wgmma_desc_rows<128>(b_hi + nb * (64 * 128) + kk * 32);
              const uint64_t db_lo = ptx::wgmma_desc_rows<128>(b_lo + nb * (64 * 128) + kk * 32);
              // small cross terms first, then the dominant product
              ptx::wgmma_bf16_n64(acc[nb], da_lo, db_hi, acc0);
              ptx::wgmma_bf16_n64(acc[nb], da_hi, db_lo, 1u);
              ptx::wgmma_bf16_n64(acc[nb], da_hi, db_hi, 1u);
            }
          }
        } else {
          const uint32_t a_l = ptx::smem_u32(smem + stage * Cfg::kStageBytes) + kABytes + grp * (kABytes / 4);
          const uint32_t a_c = a_l + kABytes / 2;
          const uint32_t b_c = b_hi + kBBytes, b_l = b_c + kBBytes / 2;
          // corrections (FP8, K = 32 per instruction): residual x copy, copy x residual
#pragma unroll
          for (int kk = 0; kk < kBlockK / 32; ++kk) {
            const uint64_t da_l = ptx::wgmma_desc_rows<64>(a_l + kk * 32);
            const uint64_t da_c = ptx::wgmma_desc_rows<64>(a_c + kk * 32);
            const uint32_t acc0 = (i > 0 || kk > 0) ? 1u : 0u;
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) {
              const uint64_t db_c = ptx::wgmma_desc_rows<64>(b_c + nb * (64 * 64) + kk * 32);
              const uint64_t db_l = ptx::wgmma_desc_rows<64>(b_l + nb * (64 * 64) + kk * 32);
              ptx::wgmma_e4m3_n64(accc[nb], da_l, db_c, acc0);
              ptx::wgmma_e4m3_n64(accc[nb], da_c, db_l, 1u);
            }
          }
          // main product (fp16, K = 16 per instruction)
#pragma unroll
          for (int kk = 0; kk < kBlockK / 16; ++kk) {
            const uint64_t da = ptx::wgmma_desc_rows<128>(a_hi + kk * 32);
            const uint32_t acc0 = (i > 0 || kk > 0) ? 1u : 0u;
#pragma unroll
            for (int nb = 0; nb < NB; ++nb)
              ptx::wgmma_f16_n64(acc[nb], da, ptx::wgmma_desc_rows<128>(b_hi + nb * (64 * 128) + kk * 32), acc0);
          }
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait_all();
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) {
          ptx::wgmma_fence_acc(acc[nb]);
          if (PM == 1) ptx::wgmma_fence_acc(accc[nb]);
        }
        if (tid == 0) ptx::mbar_arrive(&empty_bar[stage]);   // the stage's operands have been read
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
      if (PM == 1) {
#pragma unroll
        for (int nb = 0; nb < NB; ++nb)
#pragma unroll
          for (int j = 0; j < 32; ++j) acc[nb][j] += accc[nb][j];
      }
      epilogue_tile<TH, TW, BN>(p, &tm_o_hi, &tm_o_lo, &tm_o_x, staging, acc, tl, grp, est);
    }
    epilogue_finish(p, grp, est);
  }
}

// ------------------------------------------------------------------------------ conv1_1
// conv1_1 (3 -> 64 channels, K = 27) on the tensor cores: as an MMA the layer is a few
// instructions per tile and the kernel is bound by writing its output.  There is nothing for TMA
// to im2col (3 channels), so a producer warpgroup builds the A tile itself: thread p gathers the
// 27-value patch of pixel p from the fp32 NCHW blob (coalesced along the row; neighbours' re-reads
// hit L1), splits each value into (hi, lo) bf16, pads K to 32 and writes the two 64-byte rows of
// the tile with the 64B swizzle pattern the wgmma descriptor (64-byte rows, K-major) expects.
// Weights: one [hi(64) ; lo(64)] x 32 tile, loaded once by TMA; per 16-wide k slice the two
// consumer warpgroups run A_lo x B_hi, A_hi x B_lo, A_hi x B_hi on their 64 rows, and
// epilogue_tile is reused unchanged (bias, ReLU, re-split, swizzled staging, TMA store).  The image
// batch is viewed as batch*H one-row images so that a tile is 128 consecutive pixels of a row.
constexpr int kC11K = 32;                       // 27 padded
constexpr int kC11ABytes = kBlockM * kC11K * 2; // one bf16 plane of the A tile: 8 KB
constexpr int kC11Stages = 2;
constexpr int kC11BBytes = 128 * kC11K * 2;     // stacked weight tile: 8 KB
constexpr int kC11Ring = kC11Stages * 2 * kC11ABytes + kC11BBytes;  // 40 KB
constexpr int kC11Smem = kC11Ring + kBarrierBytes + kEpiBytes + 1024 /*align*/;
constexpr int kC11Threads = 384;   // producer warpgroup + two consumer warpgroups

__global__ void __launch_bounds__(kC11Threads, 1)
conv1_1_tc_kernel(const float* __restrict__ data, int B, int H, int W,
                  const __grid_constant__ CUtensorMap tm_b, const __grid_constant__ CUtensorMap tm_o_hi,
                  const __grid_constant__ CUtensorMap tm_o_lo, const __grid_constant__ CUtensorMap tm_o_x,
                  const IgemmArgs p) {
  constexpr int BN = 64;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* a_ring = smem;
  uint8_t* b_tile = smem + kC11Stages * 2 * kC11ABytes;
  uint64_t* a_full = reinterpret_cast<uint64_t*>(smem + kC11Ring);
  uint64_t* a_empty = a_full + kC11Stages;
  uint64_t* b_full = a_empty + kC11Stages;
  uint8_t* staging = smem + kC11Ring + kBarrierBytes;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  const int total_tiles = p.batch * p.tiles_w;   // p.batch = B*H one-row images
  const int first = blockIdx.x, stride = gridDim.x;

  if (warp == 0 && lane == 0) ptx::prefetch_tmap(&tm_b);
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < kC11Stages; ++s) {
      ptx::mbar_init(&a_full[s], 128);
      ptx::mbar_init(&a_empty[s], 2);
    }
    ptx::mbar_init(b_full, 1);
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    if (warp == 0) {   // weights: once per CTA
      ptx::mbar_arrive_expect_tx_w(b_full, kC11BBytes);
      ptx::tma_load_2d_w(b_tile, &tm_b, b_full, 0, 0);
    }
    // -------------------------------------------------------------- A producers (128 threads)
    const int pr = threadIdx.x;   // tile row = pixel within the 128-pixel row segment
    const long long plane = static_cast<long long>(H) * W;
    int as = 0;
    uint32_t aph = 0;
    for (int t = first; t < total_tiles; t += stride) {
      const int img = t / p.tiles_w;             // one-row image index = b*H + h
      const int w = (t - img * p.tiles_w) * 128 + pr;
      const int b = img / H, h = img - b * H;
      // gather the patch first (global-load latency overlaps the wait for the stage)
      float v[27];
      const float* xb = data + static_cast<long long>(b) * 3 * plane;
#pragma unroll
      for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int ky = 0; ky < 3; ++ky)
#pragma unroll
          for (int kx = 0; kx < 3; ++kx) {
            const int hh = h + ky - 1, ww = w + kx - 1;
            const bool ok = hh >= 0 && hh < H && ww >= 0 && ww < W && w < W;
            v[c * 9 + ky * 3 + kx] = ok ? __ldg(xb + c * plane + static_cast<long long>(hh) * W + ww) : 0.f;
          }
      uint32_t hw[16], lw[16];   // 32 bf16 each, k = 27..31 are zero
#pragma unroll
      for (int e = 0; e < 16; ++e) {
        const float x0 = (2 * e < 27) ? v[2 * e] : 0.f;
        const float x1 = (2 * e + 1 < 27) ? v[(2 * e + 1 < 27) ? 2 * e + 1 : 0] : 0.f;
        const __nv_bfloat16 h0 = __float2bfloat16_rn(x0), h1 = __float2bfloat16_rn(x1);
        const __nv_bfloat16 l0 = __float2bfloat16_rn(x0 - __bfloat162float(h0));
        const __nv_bfloat16 l1 = __float2bfloat16_rn(x1 - __bfloat162float(h1));
        hw[e] = static_cast<uint32_t>(__bfloat16_as_ushort(h0)) |
                (static_cast<uint32_t>(__bfloat16_as_ushort(h1)) << 16);
        lw[e] = static_cast<uint32_t>(__bfloat16_as_ushort(l0)) |
                (static_cast<uint32_t>(__bfloat16_as_ushort(l1)) << 16);
      }
      ptx::mbar_wait(&a_empty[as], aph ^ 1);
      uint8_t* sa = a_ring + as * 2 * kC11ABytes;
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        const int off = pr * 64 + ((g ^ ((pr >> 1) & 3)) << 4);   // SWIZZLE_64B
        *reinterpret_cast<uint4*>(sa + off) = make_uint4(hw[4 * g], hw[4 * g + 1], hw[4 * g + 2], hw[4 * g + 3]);
        *reinterpret_cast<uint4*>(sa + kC11ABytes + off) =
            make_uint4(lw[4 * g], lw[4 * g + 1], lw[4 * g + 2], lw[4 * g + 3]);
      }
      ptx::fence_proxy_async();      // generic-proxy writes -> visible to the tensor core's async proxy
      ptx::mbar_arrive(&a_full[as]);
      if (++as == kC11Stages) {
        as = 0;
        aph ^= 1;
      }
    }
  } else {
    // -------------------------------------------------------------- consumers
    const int grp = wg - 1;
    const int tid = threadIdx.x & 127;
    float acc[1][32];
    EpiState est = {0, 0.f};
    ptx::mbar_wait(b_full, 0);
    const uint32_t b_hi = ptx::smem_u32(b_tile);
    const uint32_t b_lo = b_hi + 64 * (kC11K * 2);
    int as = 0;
    uint32_t aph = 0;
    for (int t = first; t < total_tiles; t += stride) {
      const Tile tl = decode_tile(p, t, 1, 128, BN);
      ptx::mbar_wait(&a_full[as], aph);
      const uint32_t a_hi = ptx::smem_u32(a_ring + as * 2 * kC11ABytes) + grp * (kC11ABytes / 2);
      const uint32_t a_lo = a_hi + kC11ABytes;
      ptx::wgmma_fence_acc(acc[0]);
      ptx::wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kC11K / 16; ++kk) {
        const uint64_t da_hi = ptx::wgmma_desc_rows<64>(a_hi + kk * 32);
        const uint64_t da_lo = ptx::wgmma_desc_rows<64>(a_lo + kk * 32);
        const uint64_t db_hi = ptx::wgmma_desc_rows<64>(b_hi + kk * 32);
        const uint64_t db_lo = ptx::wgmma_desc_rows<64>(b_lo + kk * 32);
        ptx::wgmma_bf16_n64(acc[0], da_lo, db_hi, kk > 0 ? 1u : 0u);
        ptx::wgmma_bf16_n64(acc[0], da_hi, db_lo, 1u);
        ptx::wgmma_bf16_n64(acc[0], da_hi, db_hi, 1u);
      }
      ptx::wgmma_commit();
      ptx::wgmma_wait_all();
      ptx::wgmma_fence_acc(acc[0]);
      if (tid == 0) ptx::mbar_arrive(&a_empty[as]);
      if (++as == kC11Stages) {
        as = 0;
        aph ^= 1;
      }
      epilogue_tile<1, 128, BN>(p, &tm_o_hi, &tm_o_lo, &tm_o_x, staging, acc, tl, grp, est);
    }
    epilogue_finish(p, grp, est);
  }
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) !=
            cudaSuccess ||
        qres != cudaDriverEntryPointSuccess) {
      return nullptr;
    }
    fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

static CUtensorMapSwizzle swizzle_for_row(int row_bytes) {
  return row_bytes >= 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                          : (row_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

// [N][H][W][C] activation plane of `eb`-byte elements (2: bf16 / fp16, 1: e4m3), box
// [1][TH][TW][bk], swizzle mode = the box row width (bk * eb bytes), zero OOB fill.
static int make_act_map(CUtensorMap* m, const void* base, int N, int H, int W, int C, int TH,
                        int TW, int bk, int eb = 2) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return MNC_ERR_DRIVER;
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)C * eb, (cuuint64_t)W * C * eb, (cuuint64_t)H * W * C * eb};
  cuuint32_t box[4] = {(cuuint32_t)bk, (cuuint32_t)TW, (cuuint32_t)TH, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(m, eb == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 4,
                   const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle_for_row(bk * eb), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? MNC_OK : MNC_ERR_DRIVER;
}

// [Cout][Ktot] weight plane, box [box_rows][bk].
static int make_wgt_map(CUtensorMap* m, const void* base, int Cout, long long Ktot, int box_rows,
                        int bk, int eb = 2) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return MNC_ERR_DRIVER;
  cuuint64_t dims[2] = {(cuuint64_t)Ktot, (cuuint64_t)Cout};
  cuuint64_t strides[1] = {(cuuint64_t)Ktot * eb};
  cuuint32_t box[2] = {(cuuint32_t)bk, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, eb == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 2,
                   const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle_for_row(bk * eb), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? MNC_OK : MNC_ERR_DRIVER;
}

// output plane seen as [N][H][W][Cout] with pixel stride `pix_stride` elements; box
// [1][TH][TW][32]: 2-byte planes with the 64-byte swizzle of the epilogue's staging layout,
// 1-byte planes (32-byte rows) unswizzled.
static int make_out_map(CUtensorMap* m, const void* base, int N, int H, int W, int Cout,
                        long long pix_stride, int TH, int TW, int eb = 2) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return MNC_ERR_DRIVER;
  cuuint64_t dims[4] = {(cuuint64_t)Cout, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)pix_stride * eb, (cuuint64_t)W * pix_stride * eb,
                           (cuuint64_t)H * W * pix_stride * eb};
  cuuint32_t box[4] = {32, (cuuint32_t)TW, (cuuint32_t)TH, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(m, eb == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 4,
                   const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   eb == 2 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE,
                   CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? MNC_OK : MNC_ERR_DRIVER;
}

static int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  }
  return n;
}

struct Maps {
  CUtensorMap a[3], b[3], o[3];
};

template <int TH, int TW, int BN, int PM>
static int launch_igemm(const Maps& m, const IgemmArgs& a, int max_ctas, cudaStream_t stream) {
  using Cfg = IgemmCfg<BN, TH>;
  auto kern = igemm_tc_kernel<TH, TW, BN, PM>;
  static SmemGrant grant;
  if (!ensure_dynamic_smem(kern, Cfg::kSmemBytes, grant)) return MNC_ERR_CUDA;
  const int total = a.split_k * a.tiles_n * a.batch * a.tiles_h * a.tiles_w;
  int grid = sm_count();
  if (max_ctas > 0 && max_ctas < grid) grid = max_ctas;
  if (total < grid) grid = total;
  kern<<<grid, 384, Cfg::kSmemBytes, stream>>>(m.a[0], m.a[1], m.a[2], m.b[0], m.b[1], m.b[2], m.o[0],
                                               m.o[1], m.o[2], a);
  return cudaGetLastError() == cudaSuccess ? MNC_OK : MNC_ERR_CUDA;
}

}  // namespace mnc

using namespace mnc;

// General form.  in_fmt 0: operands are split-bf16 planes (a0 = hi, a1 = lo; w0 = hi, w1 = lo);
// in_fmt 1: tri-plane operands (a0 = fp16 value, a1 = e4m3 residual, a2 = e4m3 copy; w0 = fp16,
// w1 = e4m3 copy, w2 = e4m3 residual -- layouts above).  out_mode 0 / 2: split-bf16 (out0 = hi,
// out1 = lo), 1: fp32 (out0), 4 / 5: tri-plane (out0 = fp16, out1 = residual, out2 = copy) with
// exponent scale `out_scale`; 2 and 5 apply the fused 2x2 ceil-mode max pool.  acc_scale turns the
// accumulator into the true value (2^-(ea+ew) for tri-plane operands, 1 otherwise).  amax
// (optional, device) receives atomicMax(|output|) as float bits.
extern "C" int mnc_igemm_tc2(int in_fmt, const void* a0, const void* a1, const void* a2, int batch,
                             int H, int W, int Cin, const void* w0, const void* w1, const void* w2,
                             int Cout, int taps, const float* bias, int relu, int out_mode,
                             void* out0, void* out1, void* out2, long long out_pix_stride,
                             int out_ch_offset, int split_k, long long split_stride, int bn,
                             int max_ctas, float acc_scale, float out_scale, unsigned int* amax,
                             void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (Cin % 64 != 0 || (taps != 1 && taps != 9) || batch <= 0 || H <= 0 || W <= 0 || Cout <= 0)
    return MNC_ERR_ARG;
  if (in_fmt != 0 && in_fmt != 1) return MNC_ERR_ARG;
  if (out_mode != 0 && out_mode != 1 && out_mode != 2 && out_mode != 3 && out_mode != 4 && out_mode != 5)
    return MNC_ERR_ARG;
  const bool tri_out = (out_mode == 4 || out_mode == 5);
  const bool pooled = (out_mode == 2 || out_mode == 5);
  if (split_k < 1) split_k = 1;
  if (split_k > 1 && out_mode != 1) return MNC_ERR_ARG;
  if (pooled && (taps != 9 || Cout % 8 != 0 || out_pix_stride % 8 != 0 || out_ch_offset % 8 != 0))
    return MNC_ERR_ARG;
  if (tri_out && (out_pix_stride % 16 != 0 || out_ch_offset % 16 != 0 ||
                  (reinterpret_cast<uintptr_t>(out0) | reinterpret_cast<uintptr_t>(out1) |
                   reinterpret_cast<uintptr_t>(out2)) % 16 != 0))
    return MNC_ERR_ARG;
  const bool conv = (taps == 9);
  if (bn != 0 && bn != 64 && bn != 128 && bn != 192 && bn != 256) return MNC_ERR_ARG;
  // the accumulators of a tile live in the consumers' registers: 128 columns is the widest tile
  // that leaves room for the second (FP8) accumulator of precision mode 1, so wider requests
  // run as 128
  if (bn == 0) bn = (Cout <= 64) ? 64 : 128;
  if (bn > 128) bn = 128;
  const int TH = conv ? 8 : 1, TW = conv ? 16 : 128;
  const int bk = kBlockK;

  IgemmArgs a;
  a.batch = batch;
  a.H = H;
  a.W = W;
  a.Cin = Cin;
  a.Cout = Cout;
  a.taps = taps;
  a.tiles_h = (H + TH - 1) / TH;
  a.tiles_w = (W + TW - 1) / TW;
  a.tiles_n = (Cout + bn - 1) / bn;
  a.k_steps = taps * (Cin / bk);
  if (split_k > a.k_steps) split_k = a.k_steps;
  a.split_k = split_k;
  a.relu = relu;
  a.out_mode = out_mode;
  a.bias = bias;
  a.out_hi = static_cast<__nv_bfloat16*>(out0);
  a.out_lo = static_cast<__nv_bfloat16*>(out1);
  a.out_x = static_cast<uint8_t*>(out2);
  a.out_f32 = static_cast<float*>(out0);
  a.out_pix_stride = out_pix_stride;
  a.out_ch_offset = out_ch_offset;
  a.split_stride = split_stride;
  a.acc_scale = acc_scale;
  a.out_scale = out_scale;
  a.amax = amax;
  const int vec = (out_mode == 1) ? 4 : 8;
  a.vec_ok = (out_pix_stride % vec == 0) && (out_ch_offset % vec == 0) &&
             (reinterpret_cast<uintptr_t>(out0) % 16 == 0) &&
             (out_mode == 1 || reinterpret_cast<uintptr_t>(out1) % 16 == 0) &&
             (split_stride % vec == 0);

  Maps m;
  int rc;
  if ((rc = make_act_map(&m.a[0], a0, batch, H, W, Cin, TH, TW, bk, 2)) != MNC_OK) return rc;
  if ((rc = make_act_map(&m.a[1], a1, batch, H, W, Cin, TH, TW, bk, in_fmt ? 1 : 2)) != MNC_OK)
    return rc;
  m.a[2] = m.a[1];
  if (in_fmt == 1 && (rc = make_act_map(&m.a[2], a2, batch, H, W, Cin, TH, TW, bk, 1)) != MNC_OK)
    return rc;
  const long long ktot = static_cast<long long>(taps) * Cin;
  // epilogue through shared memory + TMA store when the output planes allow a tensor map
  m.o[0] = m.a[0];  // placeholders when unused
  m.o[1] = m.a[1];
  m.o[2] = m.a[1];
  a.tma_store = 0;
  if (out_mode == 0 && out_pix_stride % 8 == 0 && out_ch_offset % 8 == 0 &&
      reinterpret_cast<uintptr_t>(out0) % 16 == 0 && reinterpret_cast<uintptr_t>(out1) % 16 == 0) {
    const __nv_bfloat16* bh = static_cast<const __nv_bfloat16*>(out0) + out_ch_offset;
    const __nv_bfloat16* bl = static_cast<const __nv_bfloat16*>(out1) + out_ch_offset;
    if (make_out_map(&m.o[0], bh, batch, H, W, Cout, out_pix_stride, TH, TW) == MNC_OK &&
        make_out_map(&m.o[1], bl, batch, H, W, Cout, out_pix_stride, TH, TW) == MNC_OK)
      a.tma_store = 1;
  }
  if (out_mode == 4) {
    const __nv_bfloat16* bh = static_cast<const __nv_bfloat16*>(out0) + out_ch_offset;
    const uint8_t* bl = static_cast<const uint8_t*>(out1) + out_ch_offset;
    const uint8_t* bc = static_cast<const uint8_t*>(out2) + out_ch_offset;
    if (make_out_map(&m.o[0], bh, batch, H, W, Cout, out_pix_stride, TH, TW, 2) != MNC_OK ||
        make_out_map(&m.o[1], bl, batch, H, W, Cout, out_pix_stride, TH, TW, 1) != MNC_OK ||
        make_out_map(&m.o[2], bc, batch, H, W, Cout, out_pix_stride, TH, TW, 1) != MNC_OK)
      return MNC_ERR_DRIVER;
    a.tma_store = 1;
  }
  if ((rc = make_wgt_map(&m.b[0], w0, Cout, ktot, bn, bk, 2)) != MNC_OK) return rc;
  if ((rc = make_wgt_map(&m.b[1], w1, Cout, ktot, bn, bk, in_fmt ? 1 : 2)) != MNC_OK) return rc;
  m.b[2] = m.b[1];
  if (in_fmt == 1 && (rc = make_wgt_map(&m.b[2], w2, Cout, ktot, bn, bk, 1)) != MNC_OK) return rc;

#define MNC_LAUNCH(TH_, TW_, BN_)                                                        \
  return in_fmt == 1 ? launch_igemm<TH_, TW_, BN_, 1>(m, a, max_ctas, stream)             \
                     : launch_igemm<TH_, TW_, BN_, 0>(m, a, max_ctas, stream)
  if (conv) {
    if (bn == 64) MNC_LAUNCH(8, 16, 64);
    MNC_LAUNCH(8, 16, 128);
  }
  if (bn == 64) MNC_LAUNCH(1, 128, 64);
  MNC_LAUNCH(1, 128, 128);
#undef MNC_LAUNCH
}

// Split-bf16 operands, outputs 0 / 1 / 2 (the round-1 entry point; kept for its callers).
extern "C" int mnc_igemm_tc(const void* a_hi, const void* a_lo, int batch, int H, int W, int Cin,
                            const void* w_hi, const void* w_lo, int Cout, int taps,
                            const float* bias, int relu, int out_mode, void* out0, void* out1,
                            long long out_pix_stride, int out_ch_offset, int split_k,
                            long long split_stride, int bn, int max_ctas, void* stream_) {
  return mnc_igemm_tc2(0, a_hi, a_lo, nullptr, batch, H, W, Cin, w_hi, w_lo, nullptr, Cout, taps,
                       bias, relu, out_mode, out0, out1, nullptr, out_pix_stride, out_ch_offset,
                       split_k, split_stride, bn, max_ctas, 1.0f, 1.0f, nullptr, stream_);
}

// conv1_1 on the tensor cores.  w_stacked: bf16 [128][32] = rows 0..63 the hi plane, 64..127 the lo
// plane of weight.reshape(64, 27) (k = c*9 + ky*3 + kx), columns 27..31 zero.
// out_mode 0: split-bf16 planes (out0 = hi, out1 = lo); 4: tri-plane (out0 = fp16, out1 = e4m3
// residual, out2 = e4m3 copy) scaled by out_scale.  amax (optional, device): atomicMax(|output|).
extern "C" int mnc_conv1_1_tc2(const float* data_nchw, int batch, int H, int W, const void* w_stacked,
                               const float* bias, int out_mode, void* out0, void* out1, void* out2,
                               float out_scale, unsigned int* amax, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (batch <= 0 || H <= 0 || W <= 0 || (out_mode != 0 && out_mode != 4)) return MNC_ERR_ARG;
  if ((reinterpret_cast<uintptr_t>(out0) | reinterpret_cast<uintptr_t>(out1) |
       reinterpret_cast<uintptr_t>(w_stacked)) % 16 != 0)
    return MNC_ERR_ARG;
  if (out_mode == 4 && (out2 == nullptr || reinterpret_cast<uintptr_t>(out2) % 16 != 0)) return MNC_ERR_ARG;
  IgemmArgs a;
  a.batch = batch * H;   // one-row images
  a.H = 1;
  a.W = W;
  a.Cin = 32;
  a.Cout = 64;
  a.taps = 1;
  a.tiles_h = 1;
  a.tiles_w = (W + 127) / 128;
  a.tiles_n = 1;
  a.k_steps = 1;
  a.split_k = 1;
  a.relu = 1;
  a.out_mode = out_mode;
  a.bias = bias;
  a.out_hi = static_cast<__nv_bfloat16*>(out0);
  a.out_lo = static_cast<__nv_bfloat16*>(out1);
  a.out_f32 = nullptr;
  a.out_pix_stride = 64;
  a.out_ch_offset = 0;
  a.split_stride = 0;
  a.vec_ok = 1;
  a.tma_store = 1;
  a.out_x = static_cast<uint8_t*>(out2);
  a.acc_scale = 1.0f;
  a.out_scale = out_scale;
  a.amax = amax;
  CUtensorMap tb, to_hi, to_lo, to_x;
  int rc;
  const int eb = (out_mode == 4) ? 1 : 2;
  if ((rc = make_wgt_map(&tb, w_stacked, 128, 32, 128, 32)) != MNC_OK) return rc;
  if ((rc = make_out_map(&to_hi, out0, a.batch, 1, W, 64, 64, 1, 128, 2)) != MNC_OK) return rc;
  if ((rc = make_out_map(&to_lo, out1, a.batch, 1, W, 64, 64, 1, 128, eb)) != MNC_OK) return rc;
  to_x = to_lo;
  if (out_mode == 4 && (rc = make_out_map(&to_x, out2, a.batch, 1, W, 64, 64, 1, 128, 1)) != MNC_OK) return rc;
  static SmemGrant grant;
  if (!ensure_dynamic_smem(conv1_1_tc_kernel, kC11Smem, grant)) return MNC_ERR_CUDA;
  const int total = a.batch * a.tiles_w;
  int grid = sm_count();
  if (total < grid) grid = total;
  conv1_1_tc_kernel<<<grid, kC11Threads, kC11Smem, stream>>>(data_nchw, batch, H, W, tb, to_hi, to_lo,
                                                             to_x, a);
  return cudaGetLastError() == cudaSuccess ? MNC_OK : MNC_ERR_CUDA;
}

extern "C" int mnc_conv1_1_tc(const float* data_nchw, int batch, int H, int W, const void* w_stacked,
                              const float* bias, void* out_hi, void* out_lo, void* stream_) {
  return mnc_conv1_1_tc2(data_nchw, batch, H, W, w_stacked, bias, 0, out_hi, out_lo, nullptr, 1.0f,
                         nullptr, stream_);
}
