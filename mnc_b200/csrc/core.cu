// Library identity and diagnostics for the mnc_b200 C-ABI.
#include <cuda_runtime.h>

#include "mnc_b200.h"
#include "launch_util.h"

extern "C" int mnc_abi_version(void) { return 1; }

extern "C" const char* mnc_last_cuda_error(void) {
  return cudaGetErrorString(mnc::last_cuda_error);
}

extern "C" int mnc_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}
