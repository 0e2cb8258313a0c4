// One anchor of a feature map as AnchorGenerator.grid_anchors builds it (mmdet/core/anchor/anchor_generator.py:
// shifts = arange(W) * stride etc. as fp32, then base + shift, one fp32 add per coordinate), shared by the RPN's
// proposals (bags_rpn.cu) and its training targets (bags_anchor_target.cu).  No kernel.
#pragma once
#include <cuda_runtime.h>

namespace bags {

// base anchor `ba` at feature location (wx, hy) of a level with this stride
__device__ __forceinline__ float4 grid_anchor(float4 ba, int wx, int hy, int stride) {
  const float sx = static_cast<float>(wx * stride), sy = static_cast<float>(hy * stride);
  return make_float4(__fadd_rn(ba.x, sx), __fadd_rn(ba.y, sy), __fadd_rn(ba.z, sx), __fadd_rn(ba.w, sy));
}

}  // namespace bags
