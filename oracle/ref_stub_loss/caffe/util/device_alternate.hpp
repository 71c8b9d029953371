// oracle/ref_stub_loss -- TEST INFRASTRUCTURE.  Stand-in for caffe/util/device_alternate.hpp: the
// CUDA macros are the stub common.hpp's; CUBLAS_CHECK is added.
#ifndef MNC_REF_STUB_DEVICE_ALTERNATE_HPP_
#define MNC_REF_STUB_DEVICE_ALTERNATE_HPP_
#include <cublas_v2.h>

#include "caffe/common.hpp"
#define CUBLAS_CHECK(condition) \
  do { cublasStatus_t s_ = condition; CHECK_EQ(s_, CUBLAS_STATUS_SUCCESS); } while (0)
#endif
