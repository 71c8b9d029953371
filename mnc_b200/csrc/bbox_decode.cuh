// bbox_transform_inv for one box / one delta quadruple (lib/transform/bbox_transform.py:72-97), all
// fp32, one rounding per numpy operation.  Shared by ProposalLayer's decode (proposal.cu, which
// clips the box) and the state its TRAIN phase keeps for the backward (rpn_train.cu, which tests
// the unclipped box against the image).  expf is within 2 ulp of numpy's float32 exp.
#pragma once

#include <cuda_runtime.h>

namespace mnc {

// The predicted centre and size; the box is (cx - 0.5 w, cy - 0.5 h, cx + 0.5 w, cy + 0.5 h).
__device__ __forceinline__ void decode_center(float x1, float y1, float x2, float y2, float dx,
                                              float dy, float dw, float dh, float& pred_ctr_x,
                                              float& pred_ctr_y, float& pred_w, float& pred_h) {
  const float widths = __fadd_rn(__fsub_rn(x2, x1), 1.0f);
  const float heights = __fadd_rn(__fsub_rn(y2, y1), 1.0f);
  const float ctr_x = __fadd_rn(x1, __fmul_rn(0.5f, widths));
  const float ctr_y = __fadd_rn(y1, __fmul_rn(0.5f, heights));
  pred_ctr_x = __fadd_rn(__fmul_rn(dx, widths), ctr_x);
  pred_ctr_y = __fadd_rn(__fmul_rn(dy, heights), ctr_y);
  pred_w = __fmul_rn(expf(dw), widths);
  pred_h = __fmul_rn(expf(dh), heights);
}

}  // namespace mnc
