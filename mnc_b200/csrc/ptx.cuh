// Thin inline-PTX wrappers for the sm_90a features the MNC hot path uses:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA, operands in shared memory,
// fp32 accumulators in registers), setmaxnreg.
// Hand-written for sm_90a only; there is no fallback path.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace mnc {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ----------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---------------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tmap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}

// TMA store (shared -> global), bulk-group completion.
__device__ __forceinline__ void tma_store_4d(const void* tmap, const void* smem_src, int c0, int c1,
                                             int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
      ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int kPending>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(kPending) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ------------------------------------------------------------------ warp-convergent issue
// cp.async.bulk.tensor takes its operands from UNIFORM registers.  When the issuing code sits
// inside `if (lane == 0) { ... }` the compiler treats every value in that region as per-thread
// and wraps each instruction in an election + R2UR + branch sequence.  The `_w` forms below are
// meant to be executed by ALL 32 lanes of a converged warp with warp-uniform arguments: the
// election happens inside the asm block, so the operands are computed on the uniform datapath and
// reach the instruction directly.
__device__ __forceinline__ void mbar_arrive_expect_tx_w(uint64_t* bar, uint32_t bytes) {
  asm volatile(
      "{\n\t.reg .pred q;\n\t"
      "elect.sync _|q, 0xffffffff;\n\t"
      "@q mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n\t}" ::"r"(smem_u32(bar)),
      "r"(bytes)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d_w(void* smem_dst, const void* tmap, uint64_t* bar,
                                              int c0, int c1, int c2, int c3) {
  asm volatile(
      "{\n\t.reg .pred q;\n\t"
      "elect.sync _|q, 0xffffffff;\n\t"
      "@q cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];\n\t}"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d_w(void* smem_dst, const void* tmap, uint64_t* bar,
                                              int c0, int c1) {
  asm volatile(
      "{\n\t.reg .pred q;\n\t"
      "elect.sync _|q, 0xffffffff;\n\t"
      "@q cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];\n\t}"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// ------------------------------------------------------------------ register budget
// A warpgroup hands registers back (producer) or takes more (consumers holding accumulators).
template <int kRegs>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs));
}
template <int kRegs>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs));
}

// ------------------------------------------------------------------ wgmma
// Shared-memory matrix descriptor of a K-major operand tile whose rows are kRowBytes (128 / 64 /
// 32) long and swizzled with the mode of the same width, as TMA writes them: 8-row atoms of
// 8 * kRowBytes.  Fields: [0,14) address >> 4, [16,30) leading byte offset >> 4 (unused for
// swizzled K-major), [32,46) stride byte offset >> 4 (between 8-row atoms), [62,64) swizzle
// (1 = 128B, 2 = 64B, 3 = 32B).  A k slice inside the swizzle atom is addressed by advancing the
// start address (32 bytes per slice).
template <int kRowBytes>
__device__ __forceinline__ uint64_t wgmma_desc_rows(uint32_t smem_addr) {
  static_assert(kRowBytes == 128 || kRowBytes == 64 || kRowBytes == 32, "row width");
  constexpr uint64_t kMode = kRowBytes == 128 ? 1 : (kRowBytes == 64 ? 2 : 3);
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>((8u * kRowBytes) >> 4) << 32;
  d |= kMode << 62;
  return d;
}

__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_wait_all() {
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
}
// keeps the compiler from moving uses of an accumulator across the asynchronous MMAs
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[32]) {
#pragma unroll
  for (int j = 0; j < 32; ++j) asm volatile("" : "+f"(d[j])::"memory");
}

// D[64 x 64, fp32 registers] (+)= A[64 x K, smem] * B[64 x K, smem]^T, both K-major.
// Thread t of the warpgroup holds, for j = 0..7: d[4j], d[4j+1] = row 16*(t/32) + (t%32)/4,
// columns 8j + 2*(t%4) + {0, 1}; d[4j+2], d[4j+3] = the same columns of row + 8.
#define MNC_WGMMA_D32                                                                          \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                    \
  "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}"
#define MNC_WGMMA_D32_OPS(d)                                                                   \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),          \
      "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]),  \
      "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),            \
      "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]),            \
      "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])

// bf16 operands, K = 16 per instruction.
__device__ __forceinline__ void wgmma_bf16_n64(float (&d)[32], uint64_t desc_a, uint64_t desc_b,
                                               uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 " MNC_WGMMA_D32
      ", %32, %33, p, 1, 1, 0, 0;\n\t}"
      : MNC_WGMMA_D32_OPS(d)
      : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}
// fp16 operands, K = 16 per instruction.
__device__ __forceinline__ void wgmma_f16_n64(float (&d)[32], uint64_t desc_a, uint64_t desc_b,
                                              uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " MNC_WGMMA_D32
      ", %32, %33, p, 1, 1, 0, 0;\n\t}"
      : MNC_WGMMA_D32_OPS(d)
      : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}
// E4M3 operands (one byte per element in shared memory), K = 32 per instruction: twice the MAC
// rate of the 16-bit kinds.
__device__ __forceinline__ void wgmma_e4m3_n64(float (&d)[32], uint64_t desc_a, uint64_t desc_b,
                                               uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k32.f32.e4m3.e4m3 " MNC_WGMMA_D32
      ", %32, %33, p, 1, 1;\n\t}"
      : MNC_WGMMA_D32_OPS(d)
      : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}
#undef MNC_WGMMA_D32
#undef MNC_WGMMA_D32_OPS

}  // namespace ptx
}  // namespace mnc
