// Bitmask NMS with warp ballots, a device-side greedy scan, and a rank (counting) sort.
//
// Replaces `_nms` (lib/nms/nms_kernel.cu:34-78 kernel, :91-144 host wrapper) and the
// `scores.argsort()[::-1]` calls in front of it (lib/nms/gpu_nms.pyx:25-26,
// lib/pylayer/proposal_layer.py:139).  Differences in design, not in result:
//  * suppression words are built with __ballot_sync (lanes = 32 columns, loop over rows);
//  * only the upper triangle is computed;
//  * the greedy reduce runs on the device (one warp per problem) and stops at `max_keep`, so the
//    n x n/64 word matrix never crosses PCIe (the reference copies 4.5 MB D->H for n = 6000);
//  * many problems (images x classes) are batched in one launch, with per-problem counts read
//    from device memory (counts are data dependent: they come from the min-size filter).
// Semantics kept exactly: IoU with the +1 convention, suppress when IoU > thresh (strict),
// boxes visited in the given (score-sorted) order.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdlib>
#include <cstring>

#include "mnc_b200.h"
#include "launch_util.h"

namespace mnc {

// Intersection I and union U of devIoU (nms_kernel.cu:24-32) for a, the earlier (row) box, and cb,
// the later (column) box -- argument order of nms_kernel.cu:66-71.  The reference's
// interS / (Sa + Sb - interS) leaves the rounding of the union to nvcc's FMA contraction: in the
// reference binary the row box is invariant in the column loop, so Sa is a plain product and the
// column box's product is fused into the sum, U = fl(fma(bw, bh, Sa) - I).  The same source
// compiled in these kernels, where the later box is the invariant one, fuses the other product,
// which moves U, and with it fl(I / U), by an ulp where the areas are inexact.  So the reference's
// rounding is pinned here with intrinsics, and every NMS kernel decides with these I and U.  The
// earlier box's product now takes one FMUL per pair that the contracted form folded into its FFMA
// (on the H100: no change in the capped forms, about 2% in nms_mask + nms_scan).
__device__ __forceinline__ void nms_inter_union(const float* a, const float (&cb)[4], float& inter,
                                                float& uni) {
  const float width = max(min(a[2], cb[2]) - max(a[0], cb[0]) + 1, 0.f);
  const float height = max(min(a[3], cb[3]) - max(a[1], cb[1]) + 1, 0.f);
  inter = __fmul_rn(width, height);
  const float sa = __fmul_rn(a[2] - a[0] + 1, a[3] - a[1] + 1);
  uni = __fsub_rn(__fmaf_rn(cb[2] - cb[0] + 1, cb[3] - cb[1] + 1, sa), inter);
}

// disjoint boxes: interS == 0 exactly, and 0 / x > thresh is false for every x (NaN included) when
// thresh >= 0, so the division can be skipped without changing the result
__device__ __forceinline__ bool nms_disjoint(const float* a, const float (&cb)[4]) {
  return (min(a[2], cb[2]) - max(a[0], cb[0]) + 1 <= 0.f) ||
         (min(a[3], cb[3]) - max(a[1], cb[1]) + 1 <= 0.f);
}

// fl(I / U) > thresh: a, the earlier box, suppresses cb
__device__ __forceinline__ bool nms_suppresses(const float* a, const float (&cb)[4], float thresh) {
  if (nms_disjoint(a, cb) && !(thresh < 0.f)) return false;
  float inter, uni;
  nms_inter_union(a, cb, inter, uni);
  // Decide fl(I / U) > thresh without the division whenever the answer is not within rounding of
  // the threshold: q = fl(I / U) differs from I / U by at most 2^-24 relative, so
  // I > t*U*(1 + 1e-6) implies q > t and I < t*U*(1 - 1e-6) implies q < t (the margin also covers
  // the rounding of t*U).  Everything else -- U <= 0, NaNs, a ratio within 1e-6 of the
  // threshold -- takes the division.
  if (uni > 0.f && thresh >= 0.f) {
    const float tu = __fmul_rn(thresh, uni);
    if (inter > __fmul_rn(tu, 1.000001f)) return true;
    if (inter < __fmul_rn(tu, 0.999999f)) return false;
  }
  return __fdiv_rn(inter, uni) > thresh;
}

// mask layout: [problem][row][col_block] (u64), row in [0, n_max): a kept row's words are
// contiguous, which is what the scan's critical path reads.
// grid (col_blocks, row_blocks, problems), 128 threads.
__global__ void __launch_bounds__(128)
nms_mask_kernel(const float* __restrict__ boxes, int box_stride, long long problem_stride,
                const int* __restrict__ counts, int n_max, float thresh,
                unsigned long long* __restrict__ mask) {
  const int col_blk = blockIdx.x, row_blk = blockIdx.y, prob = blockIdx.z;
  if (col_blk < row_blk) return;
  const int n = min(counts ? counts[prob] : n_max, n_max);
  if (row_blk * 64 >= n || col_blk * 64 >= n) return;
  const float* pb = boxes + prob * problem_stride;
  __shared__ float row_boxes[64][4];
  __shared__ uint32_t halves[64][2];
  const int tid = threadIdx.x;
  if (tid < 64) {
    const int r = row_blk * 64 + tid;
#pragma unroll
    for (int k = 0; k < 4; ++k) row_boxes[tid][k] = (r < n) ? pb[(long long)r * box_stride + k] : 0.f;
  }
  const int warp = tid >> 5, lane = tid & 31;
  const int half = warp & 1;          // which 32 columns of the tile
  const int row_base = (warp >> 1) * 32;
  const int col = col_blk * 64 + half * 32 + lane;
  float cb[4] = {0.f, 0.f, 0.f, 0.f};
  const bool col_ok = col < n;
  if (col_ok) {
#pragma unroll
    for (int k = 0; k < 4; ++k) cb[k] = pb[(long long)col * box_stride + k];
  }
  __syncthreads();
#pragma unroll 4
  for (int i = 0; i < 32; ++i) {
    const int rl = row_base + i;
    const int r = row_blk * 64 + rl;
    // reference: row box is `cur_box` (a), column box is block_boxes (b); within the diagonal
    // tile only columns j > i are tested (nms_kernel.cu:66-69)
    bool sup = false;
    if (col_ok && r < n && col > r && (!nms_disjoint(row_boxes[rl], cb) || thresh < 0.f)) {
      // always the division: on the H100 the division-free test of nms_suppresses made this
      // kernel slower
      float inter, uni;
      nms_inter_union(row_boxes[rl], cb, inter, uni);
      sup = __fdiv_rn(inter, uni) > thresh;
    }
    const uint32_t bits = __ballot_sync(0xffffffffu, sup);
    if (lane == 0) halves[rl][half] = bits;
  }
  __syncthreads();
  if (tid < 64) {
    const int r = row_blk * 64 + tid;
    if (r < n) {
      const unsigned long long word =
          static_cast<unsigned long long>(halves[tid][0]) |
          (static_cast<unsigned long long>(halves[tid][1]) << 32);
      const int col_blocks = (n_max + 63) / 64;
      mask[(static_cast<long long>(prob) * n_max + r) * col_blocks + col_blk] = word;
    }
  }
}

// One CTA (256 threads) per problem.  Walks 64-box blocks: thread 0 resolves the block's internal
// dependencies from the 64 diagonal words (staged in shared memory), then every thread ORs the
// kept rows into its own later column word (row-major words: one coalesced read per kept row).
__global__ void __launch_bounds__(256)
nms_scan_kernel(const unsigned long long* __restrict__ mask, const int* __restrict__ counts,
                int n_max, int max_keep, int* __restrict__ keep_out, int keep_stride,
                int* __restrict__ num_out) {
  extern __shared__ unsigned long long remv[];  // col_blocks words
  __shared__ unsigned long long diag[2][64];
  __shared__ int s_rows[64];
  __shared__ int s_nk, s_num;
  const int prob = blockIdx.x;
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const int n = min(counts ? counts[prob] : n_max, n_max);
  const int cb_max = (n_max + 63) / 64;
  const int col_blocks = (n + 63) / 64;
  const unsigned long long* pm = mask + static_cast<long long>(prob) * n_max * cb_max;
  int* keep = keep_out + static_cast<long long>(prob) * keep_stride;
  for (int c = tid; c < col_blocks; c += blockDim.x) remv[c] = 0ull;
  if (tid == 0) s_num = 0;
  if (tid < 64) diag[0][tid] = (tid < n) ? pm[static_cast<long long>(tid) * cb_max] : 0ull;
  __syncthreads();
  for (int blk = 0; blk < col_blocks; ++blk) {
    const int r0 = blk * 64;
    const int buf = blk & 1;
    if (tid == 0) {
      // greedy pass over the 64 candidates of this block (bit i of diag[i'] = i' suppresses i)
      unsigned long long cur = remv[blk];
      int num = s_num, nk = 0;
      const int rows = min(64, n - r0);
      const unsigned long long rowmask = rows == 64 ? ~0ull : ((1ull << rows) - 1ull);
      // visit only the candidates that are still alive: one iteration per KEPT box (typically a
      // handful per block), not one per candidate
      unsigned long long avail = ~cur & rowmask;
      while (avail && num < max_keep) {
        const int i = __ffsll(static_cast<long long>(avail)) - 1;
        keep[num++] = r0 + i;
        s_rows[nk++] = r0 + i;
        cur |= diag[buf][i];
        avail = ~cur & rowmask & ~((2ull << i) - 1ull);   // alive candidates after i
      }
      s_nk = nk;
      s_num = num;
    } else if (tid >= 64 && tid < 128 && blk + 1 < col_blocks) {
      // meanwhile: the next block's diagonal words (independent of what is kept here)
      const int r = r0 + 64 + (tid - 64);
      diag[buf ^ 1][tid - 64] = (r < n) ? pm[static_cast<long long>(r) * cb_max + blk + 1] : 0ull;
    }
    __syncthreads();
    if (s_num >= max_keep) break;
    // OR the kept rows into the running suppression words of the later column blocks.  Lanes
    // run along a row (coalesced 8-byte loads), warps split the kept rows; a warp's <= 8 loads
    // per column chunk are independent, so the whole phase costs about one memory round trip.
    const int nk = s_nk;
    if (nk > 0) {
      for (int c0 = blk + 1; c0 < col_blocks; c0 += 32) {
        const int c = c0 + lane;
        unsigned long long acc = 0ull;
        if (c < col_blocks) {
#pragma unroll 8
          for (int q = warp; q < nk; q += nwarps)
            acc |= __ldg(pm + static_cast<long long>(s_rows[q]) * cb_max + c);
          if (acc) atomicOr(&remv[c], acc);
        }
      }
    }
    __syncthreads();
  }
  if (tid == 0) num_out[prob] = s_num;
}

// ---------------------------------------------------------------------------------------------
// Capped NMS (max_keep << n, the ProposalLayer case: 6000 candidates, 300 survivors,
// proposal_layer.py:147-152) WITHOUT the n x n/64 suppression matrix.  The greedy result only ever
// consults IoU(kept box, later candidate): at most n * max_keep pairs plus the 64 x 64 triangle
// inside each 64-candidate block -- ~1.3 M pairs for 6000 / 300 against the 18 M of the full upper
// triangle that nms_mask_kernel builds (and 5 M against 50 M for configs[4]'s 10 000 boxes).  So:
// one CTA per problem walks the candidates in blocks of 64, keeps the kept boxes in shared memory,
// and per block
//   A. all warps: lanes = candidates (two 32-lane halves), warp pairs stride over the kept list
//      (broadcast 16-byte shared-memory reads) and over the block's own rows; suppression bits are
//      collected with __ballot_sync (I and U as in nms_mask_kernel);
//   B. thread 0 resolves the block serially from the 64 diagonal words -- one iteration per KEPT
//      box -- and appends the survivors to the kept list; the next block's boxes were prefetched
//      into registers during A.
// It stops at max_keep survivors.  Same keep list as nms_mask + nms_scan (tests compare them on
// clustered and sparse boxes); only 1 SM per image is busy, so in the pipelined engine the other
// in-flight batch's tensor kernels run beside it instead of waiting for a full-GPU mask launch.
constexpr int kLazyThreads = 1024;
constexpr int kLazyGroups = kLazyThreads / 64;   // warp pairs striding over kept boxes / block rows

__global__ void __launch_bounds__(kLazyThreads)
nms_lazy_kernel(const float* __restrict__ boxes, int box_stride, long long problem_stride,
                const int* __restrict__ counts, int n_max, float thresh, int max_keep,
                int* __restrict__ keep_out, int keep_stride, int* __restrict__ num_out) {
  extern __shared__ float4 kept_box[];             // max_keep entries
  __shared__ float4 cand[2][64];
  __shared__ uint32_t sup_bits[2];                 // candidates suppressed by an earlier kept box
  __shared__ uint32_t diag_half[64][2];            // bit j of row i: candidate i suppresses j (j > i)
  __shared__ int s_num;
  const int prob = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int half = warp & 1, grp = warp >> 1;
  const int c = half * 32 + lane;                  // this thread's candidate within the block
  const int n = min(counts ? counts[prob] : n_max, n_max);
  const float* pb = boxes + prob * problem_stride;
  int* keep = keep_out + static_cast<long long>(prob) * keep_stride;
  if (tid == 0) {
    s_num = 0;
    sup_bits[0] = sup_bits[1] = 0u;
  }
  if (tid < 64) {
    float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
    if (tid < n) {
      const float* s = pb + static_cast<long long>(tid) * box_stride;
      b = make_float4(s[0], s[1], s[2], s[3]);
    }
    cand[0][tid] = b;
  }
  __syncthreads();
  const int blocks = (n + 63) / 64;
  for (int blk = 0; blk < blocks; ++blk) {
    const int r0 = blk * 64, buf = blk & 1;
    const int num = s_num;
    // prefetch the next block's boxes (the last warp pair; the loads complete under phase A)
    float4 nxt = make_float4(0.f, 0.f, 0.f, 0.f);
    const bool fetch = grp == kLazyGroups - 1 && blk + 1 < blocks;
    if (fetch && r0 + 64 + c < n) {
      const float* s = pb + static_cast<long long>(r0 + 64 + c) * box_stride;
      nxt = make_float4(s[0], s[1], s[2], s[3]);
    }
    // ---- phase A
    const float4 cv = cand[buf][c];
    const float cb[4] = {cv.x, cv.y, cv.z, cv.w};
    const bool c_ok = r0 + c < n;
    bool sup = false;
    for (int k = grp; k < num; k += kLazyGroups)
      sup |= nms_suppresses(reinterpret_cast<const float*>(&kept_box[k]), cb, thresh);
    const uint32_t sb = __ballot_sync(0xffffffffu, sup && c_ok);
    if (lane == 0 && sb) atomicOr(&sup_bits[half], sb);
#pragma unroll
    for (int q = 0; q < 64 / kLazyGroups; ++q) {
      const int i = grp * (64 / kLazyGroups) + q;  // row of the diagonal tile
      bool s = false;
      if (c_ok && c > i) s = nms_suppresses(reinterpret_cast<const float*>(&cand[buf][i]), cb, thresh);
      const uint32_t bits = __ballot_sync(0xffffffffu, s);
      if (lane == 0) diag_half[i][half] = bits;
    }
    if (fetch) cand[buf ^ 1][c] = nxt;
    __syncthreads();
    // ---- phase B
    if (tid == 0) {
      unsigned long long cur = static_cast<unsigned long long>(sup_bits[0]) |
                               (static_cast<unsigned long long>(sup_bits[1]) << 32);
      const int rows = min(64, n - r0);
      const unsigned long long rowmask = rows == 64 ? ~0ull : ((1ull << rows) - 1ull);
      unsigned long long avail = ~cur & rowmask;
      int nk = num;
      while (avail && nk < max_keep) {
        const int i = __ffsll(static_cast<long long>(avail)) - 1;
        keep[nk] = r0 + i;
        kept_box[nk] = cand[buf][i];
        ++nk;
        cur |= static_cast<unsigned long long>(diag_half[i][0]) |
               (static_cast<unsigned long long>(diag_half[i][1]) << 32);
        avail = ~cur & rowmask & ~((2ull << i) - 1ull);   // alive candidates after i
      }
      s_num = nk;
      sup_bits[0] = sup_bits[1] = 0u;
    }
    __syncthreads();
    if (s_num >= max_keep) break;
  }
  if (tid == 0) num_out[prob] = s_num;
}

// The same walk spread over a thread-block CLUSTER of 8 CTAs (8 SMs) per problem: phase A is
// compute-bound on one SM (64 x kept pair tests per block), so each CTA tests the block's 64 candidates
// against every 8th part of the kept list and builds 8 of the 64 diagonal rows; the suppression
// bits are OR-ed into, and the diagonal words stored to, EVERY CTA's shared memory through
// distributed shared memory (double-buffered by block parity), one cluster barrier publishes them,
// and then every CTA runs the same serial resolve on the same words -- so each keeps an identical
// kept list locally and nothing has to be broadcast back.  CTA 0 writes the result.
namespace cg = cooperative_groups;
constexpr int kLazyClusterSize = 8;
constexpr int kLazyClusterThreads = 256;
constexpr int kLazyClusterGroups = kLazyClusterThreads / 64;   // warp pairs per CTA

__global__ void __cluster_dims__(kLazyClusterSize, 1, 1) __launch_bounds__(kLazyClusterThreads)
nms_lazy_cluster_kernel(const float* __restrict__ boxes, int box_stride, long long problem_stride,
                        const int* __restrict__ counts, int n_max, float thresh, int max_keep,
                        int* __restrict__ keep_out, int keep_stride, int* __restrict__ num_out) {
  constexpr int S = kLazyClusterSize, G = kLazyClusterGroups;
  constexpr int kRowsPerCta = 64 / S, kRowsPerGroup = kRowsPerCta / G;
  static_assert(kRowsPerGroup >= 1 && kRowsPerGroup * G * S == 64, "diagonal rows must tile");
  extern __shared__ float4 kept_box[];             // max_keep entries (every CTA holds the full list)
  int* kept_idx = reinterpret_cast<int*>(kept_box + max_keep);   // their positions (written out at the end:
                                                   // cluster.sync() carries a GPU-scope fence, which
                                                   // would wait for global stores issued in the loop)
  __shared__ float4 cand[2][64];
  __shared__ uint32_t sup_bits[2][2];              // [block parity][half]
  __shared__ uint32_t diag_half[2][64][2];         // [block parity][row][half]
  __shared__ int s_num;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = static_cast<int>(cluster.block_rank());
  const int prob = blockIdx.x / S;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int half = warp & 1, grp = warp >> 1;
  const int c = half * 32 + lane;
  const int n = min(counts ? counts[prob] : n_max, n_max);
  const float* pb = boxes + prob * problem_stride;
  int* keep = keep_out + static_cast<long long>(prob) * keep_stride;
  if (tid == 0) {
    s_num = 0;
    sup_bits[0][0] = sup_bits[0][1] = sup_bits[1][0] = sup_bits[1][1] = 0u;
  }
  if (tid < 64) {
    float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
    if (tid < n) {
      const float* s = pb + static_cast<long long>(tid) * box_stride;
      b = make_float4(s[0], s[1], s[2], s[3]);
    }
    cand[0][tid] = b;
  }
  cluster.sync();                                  // every CTA's words are zeroed before any peer ORs into them
  const int blocks = (n + 63) / 64;
  for (int blk = 0; blk < blocks; ++blk) {
    const int r0 = blk * 64, buf = blk & 1;
    const int num = s_num;
    float4 nxt = make_float4(0.f, 0.f, 0.f, 0.f);
    const bool fetch = grp == G - 1 && blk + 1 < blocks;
    if (fetch && r0 + 64 + c < n) {
      const float* s = pb + static_cast<long long>(r0 + 64 + c) * box_stride;
      nxt = make_float4(s[0], s[1], s[2], s[3]);
    }
    // ---- phase A: this CTA's share of the kept list and of the diagonal rows
    const float4 cv = cand[buf][c];
    const float cb[4] = {cv.x, cv.y, cv.z, cv.w};
    const bool c_ok = r0 + c < n;
    bool sup = false;
    for (int k = rank * G + grp; k < num; k += S * G)
      sup |= nms_suppresses(reinterpret_cast<const float*>(&kept_box[k]), cb, thresh);
    const uint32_t sb = __ballot_sync(0xffffffffu, sup && c_ok);
    if (sb && lane < S) atomicOr(cluster.map_shared_rank(&sup_bits[buf][half], lane), sb);
#pragma unroll
    for (int q = 0; q < kRowsPerGroup; ++q) {
      const int i = rank * kRowsPerCta + grp * kRowsPerGroup + q;
      bool s = false;
      if (c_ok && c > i) s = nms_suppresses(reinterpret_cast<const float*>(&cand[buf][i]), cb, thresh);
      const uint32_t bits = __ballot_sync(0xffffffffu, s);
      if (lane < S) *cluster.map_shared_rank(&diag_half[buf][i][half], lane) = bits;
    }
    if (fetch) cand[buf ^ 1][c] = nxt;
    cluster.sync();                                // remote ORs / stores of this block are visible
    // ---- phase B: the same serial resolve in every CTA
    if (tid == 0) {
      unsigned long long cur = static_cast<unsigned long long>(sup_bits[buf][0]) |
                               (static_cast<unsigned long long>(sup_bits[buf][1]) << 32);
      const int rows = min(64, n - r0);
      const unsigned long long rowmask = rows == 64 ? ~0ull : ((1ull << rows) - 1ull);
      unsigned long long avail = ~cur & rowmask;
      int nk = num;
      while (avail && nk < max_keep) {
        const int i = __ffsll(static_cast<long long>(avail)) - 1;
        kept_idx[nk] = r0 + i;
        kept_box[nk] = cand[buf][i];
        ++nk;
        cur |= static_cast<unsigned long long>(diag_half[buf][i][0]) |
               (static_cast<unsigned long long>(diag_half[buf][i][1]) << 32);
        avail = ~cur & rowmask & ~((2ull << i) - 1ull);
      }
      s_num = nk;
      // this parity's words are next written by peers in block blk + 2, i.e. after they passed the
      // barrier of block blk + 1, which this CTA reaches only after this reset
      sup_bits[buf][0] = sup_bits[buf][1] = 0u;
    }
    __syncthreads();
    if (s_num >= max_keep) break;                  // identical in every CTA of the cluster
  }
  if (rank == 0) {
    const int num = s_num;
    for (int i = tid; i < num; i += blockDim.x) keep[i] = kept_idx[i];
    if (tid == 0) num_out[prob] = num;
  }
}

// 256 candidates per round instead of 64 (mode 3).  The 64-candidate cluster form spends most of a
// round in the cluster barrier (a GPU-scope fence) and the hand-over to the serial
// resolve -- 94 rounds for 6000 candidates; with 256-candidate rounds there are 24.  One thread per
// candidate (256 threads per CTA, 8 suppression words per row): each CTA tests all 256 candidates
// against every 8th kept box and builds 32 of the 256 diagonal rows (warps whose candidates all
// precede a row skip it: the matrix is strictly upper triangular); its 1 KB slab of diagonal words
// goes to the 7 peers with 16-byte distributed-shared-memory stores, suppression bits by remote
// atomic OR; then the same serial resolve in every CTA, now over 8 words.
constexpr int kWideBlock = 256;                  // candidates per round
constexpr int kWideWords = kWideBlock / 32;      // suppression words per row
constexpr int kWideRowsPerCta = kWideBlock / kLazyClusterSize;
constexpr int kWideMaxKeep = 1024;               // 24.1 KB static + 20 B per kept box <= 48 KB

__global__ void __cluster_dims__(kLazyClusterSize, 1, 1) __launch_bounds__(kWideBlock)
nms_lazy_cluster_wide_kernel(const float* __restrict__ boxes, int box_stride, long long problem_stride,
                             const int* __restrict__ counts, int n_max, float thresh, int max_keep,
                             int* __restrict__ keep_out, int keep_stride, int* __restrict__ num_out) {
  constexpr int S = kLazyClusterSize, CB = kWideBlock, NW = kWideWords, RPC = kWideRowsPerCta;
  static_assert(CB == 256 && NW == 8 && RPC == 32, "one warp per suppression word, 32 rows per CTA");
  extern __shared__ float4 kept_box[];             // max_keep entries (every CTA holds the full list)
  int* kept_idx = reinterpret_cast<int*>(kept_box + max_keep);
  __shared__ float4 cand[2][CB];
  __shared__ __align__(16) uint32_t sup_bits[2][NW];      // [round parity][word]
  __shared__ __align__(16) uint32_t diag[2][CB][NW];      // [round parity][row][word]
  __shared__ int s_num;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = static_cast<int>(cluster.block_rank());
  const int prob = blockIdx.x / S;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int c = tid;                               // this thread's candidate within the round
  const int n = min(counts ? counts[prob] : n_max, n_max);
  const float* pb = boxes + prob * problem_stride;
  int* keep = keep_out + static_cast<long long>(prob) * keep_stride;
  if (tid == 0) s_num = 0;
  if (tid < 2 * NW) (&sup_bits[0][0])[tid] = 0u;
  {
    float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < n) {
      const float* s = pb + static_cast<long long>(c) * box_stride;
      b = make_float4(s[0], s[1], s[2], s[3]);
    }
    cand[0][c] = b;
  }
  cluster.sync();                                  // every CTA's words are zeroed before any peer ORs into them
  const int rounds = (n + CB - 1) / CB;
  for (int blk = 0; blk < rounds; ++blk) {
    const int r0 = blk * CB, buf = blk & 1;
    const int num = s_num;
    float4 nxt = make_float4(0.f, 0.f, 0.f, 0.f);
    const bool fetch = blk + 1 < rounds;
    if (fetch && r0 + CB + c < n) {
      const float* s = pb + static_cast<long long>(r0 + CB + c) * box_stride;
      nxt = make_float4(s[0], s[1], s[2], s[3]);
    }
    // ---- phase A: every 8th kept box, and 32 of the 256 diagonal rows
    const float4 cv = cand[buf][c];
    const float cb[4] = {cv.x, cv.y, cv.z, cv.w};
    const bool c_ok = r0 + c < n;
    bool sup = false;
    for (int k = rank; k < num; k += S)
      sup |= nms_suppresses(reinterpret_cast<const float*>(&kept_box[k]), cb, thresh);
    const uint32_t sb = __ballot_sync(0xffffffffu, sup && c_ok);
    if (sb && lane < S) atomicOr(cluster.map_shared_rank(&sup_bits[buf][warp], lane), sb);
    const int row0 = rank * RPC;
    for (int q = 0; q < RPC; ++q) {
      const int i = row0 + q;
      uint32_t bits = 0u;
      if (i < 32 * warp + 31) {                    // warp-uniform: some candidate of this warp follows row i
        bool s = false;
        if (c_ok && c > i) s = nms_suppresses(reinterpret_cast<const float*>(&cand[buf][i]), cb, thresh);
        bits = __ballot_sync(0xffffffffu, s);
      }
      if (lane == 0) diag[buf][i][warp] = bits;
    }
    if (fetch) cand[buf ^ 1][c] = nxt;
    __syncthreads();                               // this CTA's slab of diagonal words is complete
    {
      // slab = rows row0 .. row0+31 = 64 uint4; 32 threads per peer, 2 uint4 each
      const int peer = tid >> 5;
      if (peer != rank) {
        const uint4* src = reinterpret_cast<const uint4*>(&diag[buf][row0][0]);
        uint4* dst = cluster.map_shared_rank(reinterpret_cast<uint4*>(&diag[buf][row0][0]), peer);
        dst[lane] = src[lane];
        dst[lane + 32] = src[lane + 32];
      }
    }
    cluster.sync();                                // remote ORs / stores of this round are visible
    // ---- phase B: the same serial resolve in every CTA
    if (tid == 0) {
      uint32_t cur[NW];
#pragma unroll
      for (int w = 0; w < NW; ++w) cur[w] = sup_bits[buf][w];
      const int rows = min(CB, n - r0);
      int nk = num;
#pragma unroll
      for (int w = 0; w < NW; ++w) {
        const int valid = min(max(rows - 32 * w, 0), 32);
        const uint32_t rowmask = valid == 32 ? 0xffffffffu : ((1u << valid) - 1u);
        while (nk < max_keep) {
          const uint32_t alive = ~cur[w] & rowmask;
          if (!alive) break;
          const int ib = __ffs(static_cast<int>(alive)) - 1;
          const int i = 32 * w + ib;
          kept_idx[nk] = r0 + i;
          kept_box[nk] = cand[buf][i];
          ++nk;
          const uint4 d0 = *reinterpret_cast<const uint4*>(&diag[buf][i][0]);
          const uint4 d1 = *reinterpret_cast<const uint4*>(&diag[buf][i][4]);
          cur[0] |= d0.x; cur[1] |= d0.y; cur[2] |= d0.z; cur[3] |= d0.w;
          cur[4] |= d1.x; cur[5] |= d1.y; cur[6] |= d1.z; cur[7] |= d1.w;
          cur[w] |= 1u << ib;                      // visited
        }
      }
      s_num = nk;
      // this parity's words are next written by peers in round blk + 2, i.e. after they passed the
      // barrier of round blk + 1, which this CTA reaches only after this reset
#pragma unroll
      for (int w = 0; w < NW; ++w) sup_bits[buf][w] = 0u;
    }
    __syncthreads();
    if (s_num >= max_keep) break;                  // identical in every CTA of the cluster
  }
  if (rank == 0) {
    const int num = s_num;
    for (int i = tid; i < num; i += blockDim.x) keep[i] = kept_idx[i];
    if (tid == 0) num_out[prob] = num;
  }
}

// 1: mnc_nms_sorted uses nms_lazy_kernel when max_keep is small against n (default); 0: always the
// mask + scan pair (A/B and cross-check switch, mnc_nms_set_lazy).
static int g_nms_lazy = 2;           // 2: the cluster form of the capped NMS (default), 1: one CTA per problem
constexpr int kLazyMaxKeep = 2048;   // kept boxes in shared memory: 32 KB
constexpr int kLazyMinN = 1024;

// Bitonic sort in shared memory, one CTA per problem, n <= 32768: (key desc, index asc).
// Keys are mapped to order-preserving uint32 (0 is reserved for invalid / padding entries).
__device__ __forceinline__ uint32_t f32_sort_key(float f) {
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__global__ void __launch_bounds__(1024)
bitonic_sort_desc_kernel(const float* __restrict__ keys, long long outer_stride,
                         long long inner_stride, int inner, int key_stride,
                         const unsigned char* __restrict__ valid, int n, int np2,
                         int* __restrict__ order, int* __restrict__ n_valid) {
  extern __shared__ uint32_t sk[];                          // np2 keys
  uint16_t* si = reinterpret_cast<uint16_t*>(sk + np2);     // np2 indices
  __shared__ int s_cnt;
  const int prob = blockIdx.x;
  const int tid = threadIdx.x;
  const float* pk = keys + (prob / inner) * outer_stride + (prob % inner) * inner_stride;
  const unsigned char* pv = valid ? valid + static_cast<long long>(prob) * n : nullptr;
  if (tid == 0) s_cnt = 0;
  __syncthreads();
  int local = 0;
  for (int i = tid; i < np2; i += blockDim.x) {
    uint32_t k = 0u;
    uint16_t ix = 0xFFFFu;
    if (i < n && (pv ? pv[i] != 0 : true)) {
      k = f32_sort_key(pk[static_cast<long long>(i) * key_stride]);
      ix = static_cast<uint16_t>(i);
      ++local;
    }
    sk[i] = k;
    si[i] = ix;
  }
  if (local) atomicAdd(&s_cnt, local);
  __syncthreads();
  for (int k = 2; k <= np2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = tid; t < (np2 >> 1); t += blockDim.x) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        const int l = i | j;
        const uint32_t ka = sk[i], kb = sk[l];
        const uint16_t ia = si[i], ib = si[l];
        const bool a_first = (ka > kb) || (ka == kb && ia < ib);
        const bool b_first = (kb > ka) || (ka == kb && ib < ia);
        const bool up = (i & k) == 0;
        if (up ? b_first : a_first) {
          sk[i] = kb;
          sk[l] = ka;
          si[i] = ib;
          si[l] = ia;
        }
      }
      __syncthreads();
    }
  }
  const int cnt = s_cnt;
  for (int i = tid; i < cnt; i += blockDim.x) order[static_cast<long long>(prob) * n + i] = si[i];
  if (tid == 0 && n_valid) n_valid[prob] = cnt;
}

// Top-k selection + sort, one CTA per problem: order[prob][0..min(n_valid, k)) = indices of the k
// best entries in (key desc, index asc) order -- all that `scores.argsort()[::-1][:pre_nms_topN]`
// (proposal_layer.py:139-142) ever uses.  Sorting all 21546 anchors (32768-slot bitonic network,
// every stage through shared memory) is far more work; here
//   1. keys -> order-preserving u32 in shared memory,
//   2. 4-pass byte-wise radix select finds T = the k-th largest key,
//   3. entries above T are compacted (any order), entries equal to T are taken in index order
//      until k are selected (the tie rule),
//   4. the <= 8192 selected (key, ~index) pairs are bitonic-sorted as packed u64.
constexpr int kTopkThreads = 1024;

__global__ void __launch_bounds__(kTopkThreads)
topk_sort_desc_kernel(const float* __restrict__ keys, long long outer_stride,
                      long long inner_stride, int inner, int key_stride,
                      const unsigned char* __restrict__ valid, int n, int k, int np2,
                      int* __restrict__ order, int order_stride, int* __restrict__ n_out) {
  extern __shared__ unsigned long long sbuf[];               // np2 packed pairs
  uint32_t* skey = reinterpret_cast<uint32_t*>(sbuf + np2);  // n keys
  __shared__ uint32_t hist[256];
  __shared__ int s_nv, s_pos, s_warp[32], s_run;
  __shared__ uint32_t s_prefix;
  __shared__ int s_need, s_eq;
  const int prob = blockIdx.x, tid = threadIdx.x;
  const float* pk = keys + (prob / inner) * outer_stride + (prob % inner) * inner_stride;
  const unsigned char* pv = valid ? valid + static_cast<long long>(prob) * n : nullptr;
  if (tid == 0) {
    s_nv = 0;
    s_pos = 0;
    s_run = 0;
  }
  __syncthreads();
  int local = 0;
  for (int i = tid; i < n; i += kTopkThreads) {
    uint32_t key = 0u;
    if (pv ? pv[i] != 0 : true) {
      key = f32_sort_key(pk[static_cast<long long>(i) * key_stride]);
      ++local;
    }
    skey[i] = key;
  }
  if (local) atomicAdd(&s_nv, local);
  __syncthreads();
  const int K = min(k, s_nv);
  if (K == 0) {
    if (tid == 0) n_out[prob] = 0;
    return;
  }
  // ---- radix select: T = K-th largest key
  if (tid == 0) {
    s_prefix = 0u;
    s_need = K;
  }
  for (int pass = 3; pass >= 0; --pass) {
    if (tid < 256) hist[tid] = 0u;
    __syncthreads();
    const uint32_t prefix = s_prefix;
    const int sh = 8 * pass;
    for (int i = tid; i < n; i += kTopkThreads) {
      const uint32_t key = skey[i];
      if (key == 0u) continue;
      const bool match = (pass == 3) || ((key >> (sh + 8)) == (prefix >> (sh + 8)));
      if (match) atomicAdd(&hist[(key >> sh) & 255u], 1u);
    }
    __syncthreads();
    if (tid == 0) {
      int need = s_need, cum = 0, b = 255;
      for (; b > 0; --b) {
        if (cum + static_cast<int>(hist[b]) >= need) break;
        cum += hist[b];
      }
      s_prefix = prefix | (static_cast<uint32_t>(b) << sh);
      s_need = need - cum;
      s_eq = hist[b];
    }
    __syncthreads();
  }
  const uint32_t T = s_prefix;
  const int need = s_need;       // how many entries equal to T are taken (>= 1)
  const int above = K - need;    // entries strictly above T
  const bool ties_ordered = s_eq != need;
  for (int i = tid; i < n; i += kTopkThreads) {
    const uint32_t key = skey[i];
    if (key > T || (!ties_ordered && key == T)) {
      const int p = atomicAdd(&s_pos, 1);
      sbuf[p] = (static_cast<unsigned long long>(key) << 32) | (0xFFFFFFFFu - static_cast<uint32_t>(i));
    }
  }
  if (ties_ordered) {
    // more entries equal to T than slots: lowest indices win
    for (int base = 0; base < n; base += kTopkThreads) {
      const int i = base + tid;
      const bool flag = i < n && skey[i] == T;
      const unsigned bal = __ballot_sync(0xffffffffu, flag);
      if ((tid & 31) == 0) s_warp[tid >> 5] = __popc(bal);
      __syncthreads();
      int off = s_run;
      for (int w = 0; w < (tid >> 5); ++w) off += s_warp[w];
      off += __popc(bal & ((1u << (tid & 31)) - 1u));
      if (flag && off < need)
        sbuf[above + off] = (static_cast<unsigned long long>(T) << 32) |
                            (0xFFFFFFFFu - static_cast<uint32_t>(i));
      __syncthreads();
      if (tid == 0) {
        int tot = 0;
        for (int w = 0; w < kTopkThreads / 32; ++w) tot += s_warp[w];
        s_run += tot;
      }
      __syncthreads();
      if (s_run >= need) break;
    }
  }
  for (int i = K + tid; i < np2; i += kTopkThreads) sbuf[i] = 0ull;
  __syncthreads();
  // ---- bitonic sort, descending, on packed (key, ~index)
  for (int kk = 2; kk <= np2; kk <<= 1) {
    for (int j = kk >> 1; j > 0; j >>= 1) {
      for (int t = tid; t < (np2 >> 1); t += kTopkThreads) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        const int l = i | j;
        const unsigned long long a = sbuf[i], b = sbuf[l];
        const bool up = (i & kk) == 0;
        if (up ? (b > a) : (a > b)) {
          sbuf[i] = b;
          sbuf[l] = a;
        }
      }
      __syncthreads();
    }
  }
  int* po = order + static_cast<long long>(prob) * order_stride;
  for (int i = tid; i < K; i += kTopkThreads)
    po[i] = static_cast<int>(0xFFFFFFFFu - static_cast<uint32_t>(sbuf[i] & 0xFFFFFFFFull));
  if (tid == 0) n_out[prob] = K;
}

// Rank sort, descending, ties by ascending index.  order[prob][rank] = index for valid items;
// n_valid[prob] = number of valid items.  keys read at keys[prob*problem_stride + i*key_stride].
// grid (ceil(n/256), problems), 256 threads.
__global__ void __launch_bounds__(256)
rank_sort_desc_kernel(const float* __restrict__ keys, long long outer_stride,
                      long long inner_stride, int inner, int key_stride,
                      const unsigned char* __restrict__ valid, int n, int* __restrict__ order,
                      int* __restrict__ n_valid) {
  __shared__ float sk[256];
  __shared__ unsigned char sv[256];
  const int prob = blockIdx.y;
  const float* pk = keys + (prob / inner) * outer_stride + (prob % inner) * inner_stride;
  const unsigned char* pv = valid ? valid + static_cast<long long>(prob) * n : nullptr;
  const int i = blockIdx.x * 256 + threadIdx.x;
  const bool vi = (i < n) && (pv ? pv[i] != 0 : true);
  const float ki = (i < n) ? pk[static_cast<long long>(i) * key_stride] : 0.f;
  int rank = 0, nv = 0;
  for (int j0 = 0; j0 < n; j0 += 256) {
    const int j = j0 + threadIdx.x;
    sk[threadIdx.x] = (j < n) ? pk[static_cast<long long>(j) * key_stride] : 0.f;
    sv[threadIdx.x] = (j < n) && (pv ? pv[j] != 0 : true);
    __syncthreads();
    const int lim = min(256, n - j0);
#pragma unroll 8
    for (int t = 0; t < lim; ++t) {
      const float kj = sk[t];
      const int jj = j0 + t;
      const bool ahead = (kj > ki) || (kj == ki && jj < i);
      rank += (sv[t] && ahead) ? 1 : 0;
      nv += sv[t] ? 1 : 0;
    }
    __syncthreads();
  }
  if (vi) order[static_cast<long long>(prob) * n + rank] = i;
  if (i == 0 && n_valid) n_valid[prob] = nv;
}

// sorted[prob][k][0..3] = src[prob / inner][order[prob][k]][0..3], k < min(count, n_out)
__global__ void gather_boxes_kernel(const float* __restrict__ src, int src_stride,
                                    long long src_outer_stride, int inner,
                                    const int* __restrict__ order,
                                    int order_stride, const int* __restrict__ counts, int n_out,
                                    float* __restrict__ dst, int* __restrict__ out_counts) {
  const int prob = blockIdx.y;
  const int cnt = min(counts ? counts[prob] : n_out, n_out);
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k == 0 && out_counts) out_counts[prob] = cnt;
  if (k >= cnt) return;
  const int idx = order[static_cast<long long>(prob) * order_stride + k];
  const float* s = src + (prob / inner) * src_outer_stride + static_cast<long long>(idx) * src_stride;
  float4 v = make_float4(s[0], s[1], s[2], s[3]);
  *reinterpret_cast<float4*>(dst + (static_cast<long long>(prob) * n_out + k) * 4) = v;
}

static inline int check_launch() { return cudaGetLastError() == cudaSuccess ? MNC_OK : MNC_ERR_CUDA; }

}  // namespace mnc

using namespace mnc;

static bool nms_takes_lazy_path(int n_max, int max_keep);

extern "C" long long mnc_nms_workspace_bytes(int n_max, int problems) {
  const long long col_blocks = (n_max + 63) / 64;
  return static_cast<long long>(problems) * col_blocks * n_max * 8;
}

extern "C" int mnc_nms_sorted(const float* boxes, int box_stride, long long problem_stride,
                              const int* counts, int n_max, int problems, float thresh,
                              int max_keep, void* workspace, int* keep_out, int keep_stride,
                              int* num_out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (n_max <= 0 || problems <= 0) return MNC_ERR_ARG;
  const int col_blocks = (n_max + 63) / 64;
  if (col_blocks * 8 > 48 * 1024) return MNC_ERR_ARG;
  if (max_keep <= 0 || max_keep > n_max) max_keep = n_max;
  if (nms_takes_lazy_path(n_max, max_keep) && g_nms_lazy == 3 && max_keep <= kWideMaxKeep) {
    nms_lazy_cluster_wide_kernel<<<problems * kLazyClusterSize, kWideBlock,
                                   max_keep * (sizeof(float4) + sizeof(int)), stream>>>(
        boxes, box_stride, problem_stride, counts, n_max, thresh, max_keep, keep_out, keep_stride,
        num_out);
    return check_launch();
  }
  if (nms_takes_lazy_path(n_max, max_keep) && g_nms_lazy >= 2) {
    nms_lazy_cluster_kernel<<<problems * kLazyClusterSize, kLazyClusterThreads,
                              max_keep * (sizeof(float4) + sizeof(int)), stream>>>(
        boxes, box_stride, problem_stride, counts, n_max, thresh, max_keep, keep_out, keep_stride,
        num_out);
    return check_launch();
  }
  if (nms_takes_lazy_path(n_max, max_keep)) {
    nms_lazy_kernel<<<problems, kLazyThreads, max_keep * sizeof(float4), stream>>>(
        boxes, box_stride, problem_stride, counts, n_max, thresh, max_keep, keep_out, keep_stride,
        num_out);
    return check_launch();
  }
  dim3 grid(col_blocks, col_blocks, problems);
  nms_mask_kernel<<<grid, 128, 0, stream>>>(boxes, box_stride, problem_stride, counts, n_max,
                                            thresh, static_cast<unsigned long long*>(workspace));
  nms_scan_kernel<<<problems, 256, col_blocks * 8, stream>>>(
      static_cast<const unsigned long long*>(workspace), counts, n_max, max_keep, keep_out,
      keep_stride, num_out);
  return check_launch();
}

static bool nms_takes_lazy_path(int n_max, int max_keep) {
  if (max_keep <= 0 || max_keep > n_max) max_keep = n_max;
  return g_nms_lazy && n_max >= kLazyMinN && max_keep <= kLazyMaxKeep && max_keep * 4 <= n_max;
}

extern "C" int mnc_nms_sorted_launches(int n_max, int max_keep) {
  return nms_takes_lazy_path(n_max, max_keep) ? 1 : 2;
}

extern "C" int mnc_nms_set_lazy(int on) {
  const int prev = g_nms_lazy;
  g_nms_lazy = on < 0 ? 0 : (on > 3 ? 3 : on);
  return prev;
}

extern "C" int mnc_rank_sort_desc(const float* keys, long long outer_stride,
                                  long long inner_stride, int inner, int key_stride,
                                  const unsigned char* valid, int n, int problems, int* order,
                                  int* n_valid, void* stream_) {
  if (n <= 0 || problems <= 0 || inner <= 0) return MNC_ERR_ARG;
  if (n > 2048 && n <= 32768) {
    // large single lists (the 21546 RPN anchors): O(n log^2 n) in shared memory
    int np2 = 1;
    while (np2 < n) np2 <<= 1;
    const int smem = np2 * 6;
    static SmemGrant grant;   // always opt in: static shared memory counts against the 48 KB default
    if (!ensure_dynamic_smem(bitonic_sort_desc_kernel, smem, grant)) return MNC_ERR_CUDA;
    bitonic_sort_desc_kernel<<<problems, 1024, smem, static_cast<cudaStream_t>(stream_)>>>(
        keys, outer_stride, inner_stride, inner, key_stride, valid, n, np2, order, n_valid);
    return check_launch();
  }
  dim3 grid((n + 255) / 256, problems);
  rank_sort_desc_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream_)>>>(
      keys, outer_stride, inner_stride, inner, key_stride, valid, n, order, n_valid);
  return check_launch();
}

extern "C" int mnc_topk_sort_desc(const float* keys, long long outer_stride, long long inner_stride,
                                  int inner, int key_stride, const unsigned char* valid, int n,
                                  int problems, int k, int* order, int order_stride, int* n_out,
                                  void* stream_) {
  if (n <= 0 || problems <= 0 || inner <= 0 || k <= 0 || order_stride < (k < n ? k : n))
    return MNC_ERR_ARG;
  int np2 = 2;
  while (np2 < (k < n ? k : n)) np2 <<= 1;
  const size_t smem = static_cast<size_t>(np2) * 8 + static_cast<size_t>(n) * 4;
  if (smem > 200 * 1024) return MNC_ERR_ARG;   // callers fall back to mnc_rank_sort_desc
  static SmemGrant grant;
  if (!ensure_dynamic_smem(topk_sort_desc_kernel, static_cast<int>(smem), grant)) return MNC_ERR_CUDA;
  topk_sort_desc_kernel<<<problems, kTopkThreads, smem, static_cast<cudaStream_t>(stream_)>>>(
      keys, outer_stride, inner_stride, inner, key_stride, valid, n, k, np2, order, order_stride,
      n_out);
  return check_launch();
}

extern "C" int mnc_gather_boxes(const float* src, int src_stride, long long src_outer_stride,
                                int inner, const int* order, int order_stride, const int* counts,
                                int n_out, int problems, float* dst, int* out_counts,
                                void* stream_) {
  if (inner <= 0) return MNC_ERR_ARG;
  dim3 grid((n_out + 255) / 256, problems);
  gather_boxes_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream_)>>>(
      src, src_stride, src_outer_stride, inner, order, order_stride, counts, n_out, dst,
      out_counts);
  return check_launch();
}

// ---------------------------------------------------------------------------------------------
// Reference-compatible host entry point: same arguments and meaning as
//   void _nms(int* keep_out, int* num_out, const float* boxes_host, int boxes_num,
//             int boxes_dim, float nms_overlap_thresh, int device_id)   (lib/nms/gpu_nms.hpp:1-2)
// plus an int status instead of printing CUDA errors (nms_kernel.cu:12-19).  Buffers are
// caller-owned host memory; the call is synchronous.  Only the keep list (<= n ints) and its
// length come back over PCIe.
namespace {
struct HostScratch {
  void* dev = nullptr;
  size_t bytes = 0;
  int device = -1;
};
HostScratch g_scratch;

int ensure_scratch(size_t bytes, int device) {
  if (g_scratch.device != device || g_scratch.bytes < bytes) {
    if (g_scratch.dev) cudaFree(g_scratch.dev);
    g_scratch.dev = nullptr;
    g_scratch.bytes = 0;
    if (cudaMalloc(&g_scratch.dev, bytes) != cudaSuccess) return MNC_ERR_CUDA;
    g_scratch.bytes = bytes;
    g_scratch.device = device;
  }
  return MNC_OK;
}
}  // namespace

extern "C" int mnc_nms_host(int* keep_out, int* num_out, const float* boxes_host, int boxes_num,
                            int boxes_dim, float nms_overlap_thresh, int device_id) {
  if (boxes_num < 0 || boxes_dim < 4 || !keep_out || !num_out) return MNC_ERR_ARG;
  if (boxes_num == 0) {
    *num_out = 0;
    return MNC_OK;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return MNC_ERR_NOGPU;
  int cur = 0;
  cudaGetDevice(&cur);
  if (cur != device_id && cudaSetDevice(device_id) != cudaSuccess) return MNC_ERR_CUDA;
  const size_t box_bytes = static_cast<size_t>(boxes_num) * boxes_dim * sizeof(float);
  const size_t box_al = (box_bytes + 255) & ~static_cast<size_t>(255);
  const size_t mask_bytes = static_cast<size_t>(mnc_nms_workspace_bytes(boxes_num, 1));
  const size_t keep_bytes = (static_cast<size_t>(boxes_num) + 1) * sizeof(int);
  int rc = ensure_scratch(box_al + mask_bytes + keep_bytes + 256, device_id);
  if (rc != MNC_OK) return rc;
  char* base = static_cast<char*>(g_scratch.dev);
  float* d_boxes = reinterpret_cast<float*>(base);
  void* d_mask = base + box_al;
  int* d_keep = reinterpret_cast<int*>(base + box_al + mask_bytes);
  int* d_num = d_keep + boxes_num;
  if (cudaMemcpy(d_boxes, boxes_host, box_bytes, cudaMemcpyHostToDevice) != cudaSuccess)
    return MNC_ERR_CUDA;
  rc = mnc_nms_sorted(d_boxes, boxes_dim, 0, nullptr, boxes_num, 1, nms_overlap_thresh, boxes_num,
                      d_mask, d_keep, boxes_num, d_num, nullptr);
  if (rc != MNC_OK) return rc;
  int num = 0;
  if (cudaMemcpy(&num, d_num, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess)
    return MNC_ERR_CUDA;
  if (num > 0 &&
      cudaMemcpy(keep_out, d_keep, sizeof(int) * num, cudaMemcpyDeviceToHost) != cudaSuccess)
    return MNC_ERR_CUDA;
  *num_out = num;
  return MNC_OK;
}


// nms.gpu_nms.gpu_nms in one call (lib/nms/gpu_nms.pyx:16-31): UNSORTED dets (n, dim >= 5, score in
// column 4) in host memory -> indices of the kept rows, in score order.  The sort
// (`scores.argsort()[::-1]`, ties by ascending index), the gather, the NMS and the greedy scan all
// run on the device; the host sees one H2D of the dets and one D2H of the order + keep lists
// (the numpy sort + fancy indexing of the .pyx wrapper would otherwise dominate the drop-in).
extern "C" int mnc_gpu_nms_host(int* keep_out, int* num_out, const float* dets_host, int n, int dim,
                                float nms_overlap_thresh, int device_id) {
  if (n < 0 || dim < 5 || !keep_out || !num_out) return MNC_ERR_ARG;
  if (n == 0) {
    *num_out = 0;
    return MNC_OK;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return MNC_ERR_NOGPU;
  int cur = 0;
  cudaGetDevice(&cur);
  if (cur != device_id && cudaSetDevice(device_id) != cudaSuccess) return MNC_ERR_CUDA;
  auto al = [](size_t b) { return (b + 255) & ~static_cast<size_t>(255); };
  const size_t dets_b = al(static_cast<size_t>(n) * dim * sizeof(float));
  const size_t sorted_b = al(static_cast<size_t>(n) * 4 * sizeof(float));
  const size_t ints_b = al((static_cast<size_t>(n) + 4) * sizeof(int));
  const size_t mask_b = al(static_cast<size_t>(mnc_nms_workspace_bytes(n, 1)));
  int rc = ensure_scratch(dets_b + sorted_b + 2 * ints_b + mask_b + 256, device_id);
  if (rc != MNC_OK) return rc;
  char* base = static_cast<char*>(g_scratch.dev);
  float* d_dets = reinterpret_cast<float*>(base);
  float* d_sorted = reinterpret_cast<float*>(base + dets_b);
  int* d_order = reinterpret_cast<int*>(base + dets_b + sorted_b);       // [n] + n_valid + count
  int* d_keep = reinterpret_cast<int*>(base + dets_b + sorted_b + ints_b);  // [n] + num
  void* d_mask = base + dets_b + sorted_b + 2 * ints_b;
  if (cudaMemcpy(d_dets, dets_host, static_cast<size_t>(n) * dim * sizeof(float),
                 cudaMemcpyHostToDevice) != cudaSuccess)
    return MNC_ERR_CUDA;
  if ((rc = mnc_rank_sort_desc(d_dets + 4, 0, 0, 1, dim, nullptr, n, 1, d_order, d_order + n,
                               nullptr)) != MNC_OK)
    return rc;
  if ((rc = mnc_gather_boxes(d_dets, dim, 0, 1, d_order, n, nullptr, n, 1, d_sorted,
                             d_order + n + 1, nullptr)) != MNC_OK)
    return rc;
  if ((rc = mnc_nms_sorted(d_sorted, 4, 0, nullptr, n, 1, nms_overlap_thresh, n, d_mask, d_keep, n,
                           d_keep + n, nullptr)) != MNC_OK)
    return rc;
  int num = 0;
  if (cudaMemcpy(&num, d_keep + n, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess)
    return MNC_ERR_CUDA;
  if (num > 0) {
    // keep (positions in the sorted list) -> original row indices, on the host: two small copies
    static thread_local int* h_order = nullptr;
    static thread_local int h_cap = 0;
    if (h_cap < n) {
      free(h_order);
      h_order = static_cast<int*>(malloc(sizeof(int) * n));
      h_cap = h_order ? n : 0;
      if (!h_order) return MNC_ERR_ARG;
    }
    if (cudaMemcpy(h_order, d_order, sizeof(int) * n, cudaMemcpyDeviceToHost) != cudaSuccess ||
        cudaMemcpy(keep_out, d_keep, sizeof(int) * num, cudaMemcpyDeviceToHost) != cudaSuccess)
      return MNC_ERR_CUDA;
    for (int i = 0; i < num; ++i) keep_out[i] = h_order[keep_out[i]];
  }
  *num_out = num;
  return MNC_OK;
}
