// oracle/ref_stub_loss -- TEST INFRASTRUCTURE.  The Caffe-runtime stand-in of oracle/ref_stub
// extended for the loss layers (oracle/loss.mk): shared_ptr, the cuBLAS handle, DCHECK.  Nothing
// here restates reference arithmetic.
#ifndef MNC_REF_STUB_LOSS_COMMON_HPP_
#define MNC_REF_STUB_LOSS_COMMON_HPP_
#include <cublas_v2.h>

#include <memory>

#include "../../ref_stub/caffe/common.hpp"

#define DCHECK_GE(a, b) ::caffe::stub::Null()
#define DCHECK_LT(a, b) ::caffe::stub::Null()

namespace caffe {
using std::shared_ptr;
class Caffe {
 public:
  static cublasHandle_t cublas_handle() {
    static cublasHandle_t h = 0;
    if (!h) cublasCreate(&h);
    return h;
  }
};
}  // namespace caffe
#endif
