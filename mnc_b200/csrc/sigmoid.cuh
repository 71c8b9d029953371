// SigmoidForward (sigmoid_layer.cu:9-14) as the reference build compiles it, shared by the loss
// layers and SigmoidLayer.
#pragma once
#include <cuda_runtime.h>

namespace mnc {

// expf of the float argument, then 1 + e and the quotient in double, rounded to float once.
__device__ __forceinline__ float ref_sigmoid(float x) {
  return static_cast<float>(__ddiv_rn(1.0, __dadd_rn(1.0, static_cast<double>(expf(-x)))));
}

}  // namespace mnc
