// Host-side launch helpers shared by the .cu files.
#pragma once
#include <cuda_runtime.h>

#include "mnc_b200.h"

namespace mnc {

// The error behind the last MNC_ERR_CUDA of this host thread (per thread, like CUDA's own).
inline thread_local cudaError_t last_cuda_error = cudaSuccess;

// Status of a runtime call; a failure is recorded for mnc_last_cuda_error and taken off the
// runtime's pending error, so that the next check on this thread (torch's, say) does not repeat it.
inline int cuda_status(cudaError_t e) {
  if (e == cudaSuccess) return MNC_OK;
  last_cuda_error = e;
  cudaGetLastError();
  return MNC_ERR_CUDA;
}

inline int check_launch() { return cuda_status(cudaGetLastError()); }

inline int grid_for(long long n, int block, int cap) {
  long long g = (n + block - 1) / block;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return static_cast<int>(g);
}

// cudaFuncSetAttribute(cudaFuncAttributeMaxDynamicSharedMemorySize) applies to the CURRENT device
// only, and entry points such as mnc_nms_host(device_id) may be called for several devices from
// one process: remember, per device, the largest opt-in already granted for a kernel.
constexpr int kMaxDevices = 64;
struct SmemGrant {
  int granted[kMaxDevices] = {};
};

template <typename Kernel>
inline int ensure_dynamic_smem(Kernel kernel, int bytes, SmemGrant& g) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) dev = 0;
  if (bytes <= g.granted[dev]) return MNC_OK;
  const int rc = cuda_status(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  if (rc == MNC_OK) g.granted[dev] = bytes;
  return rc;
}

}  // namespace mnc
