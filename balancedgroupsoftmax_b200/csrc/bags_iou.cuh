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

// torch.maximum / torch.minimum / clamp: NaN in, NaN out
__device__ __forceinline__ float max_nan(float a, float b) { return (a != a || b != b) ? __int_as_float(0x7fc00000) : fmaxf(a, b); }
__device__ __forceinline__ float min_nan(float a, float b) { return (a != a || b != b) ? __int_as_float(0x7fc00000) : fminf(a, b); }

// bbox_overlaps(gt, anchors) (mmdet/core/bbox/geometry.py, mode 'iou', not aligned) for one pair in its torch op
// sequence, one rounding per op and no contraction: lt = max, rb = min, wh = ((rb - lt) + 1).clamp(min=0),
// overlap = w * h, area = ((x2 - x1) + 1) * ((y2 - y1) + 1), iou = overlap / ((area_gt + area_anchor) - overlap).
// Not iou_plus1, which restates the NMS op's compiled sequence.
__device__ __forceinline__ float area_plus1(const float4 b) {
  return __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), 1.f), __fadd_rn(__fsub_rn(b.w, b.y), 1.f));
}
__device__ __forceinline__ float iou_overlaps(const float4 g, float area_g, const float4 a, float area_a) {
  const float w = max_nan(__fadd_rn(__fsub_rn(min_nan(g.z, a.z), max_nan(g.x, a.x)), 1.f), 0.f);
  const float h = max_nan(__fadd_rn(__fsub_rn(min_nan(g.w, a.w), max_nan(g.y, a.y)), 1.f), 0.f);
  const float overlap = __fmul_rn(w, h);
  return __fdiv_rn(overlap, __fsub_rn(__fadd_rn(area_g, area_a), overlap));
}

}  // namespace bags
