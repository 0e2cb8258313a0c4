// IoU with the reference's "+1" widths (mmdet/ops/nms/src/nms_kernel.cu:13-21), shared by the class-aware NMS
// (bags_nms.cuh) and the RPN's suppression (bags_rpn.cu).  A header of its own, with no kernel, so that a translation
// unit can use it without instantiating another's kernels.
#pragma once
#include <cuda_runtime.h>

namespace bags {

__device__ __forceinline__ float iou_plus1(const float4 a, const float4 b) {
  const float left = fmaxf(a.x, b.x), right = fminf(a.z, b.z);
  const float top = fmaxf(a.y, b.y), bottom = fminf(a.w, b.w);
  const float width = fmaxf(right - left + 1.f, 0.f), height = fmaxf(bottom - top + 1.f, 0.f);
  const float inter = width * height;
  const float sa = (a.z - a.x + 1.f) * (a.w - a.y + 1.f);
  const float sb = (b.z - b.x + 1.f) * (b.w - b.y + 1.f);
  return inter / (sa + sb - inter);
}

}  // namespace bags
