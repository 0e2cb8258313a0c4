// Class-aware batched NMS for the test-time consumer of the merged BAGS scores (SURVEY.md 8f-2).
//
// The reference loops over the 1230 foreground classes in Python and calls its NMS op once per class
// (mmdet/core/post_processing/bbox_nms.py:34-54; IoU with "+1" widths and "suppress if IoU > thr" in
// mmdet/ops/nms/src/nms_kernel.cu:13-21,60; candidates pre-sorted by score, :76-78).  Here all classes are
// processed by ONE launch: one CTA per class builds the suppression bit matrix of its candidates in shared memory and
// one warp runs the greedy scan over it.  At most kNmsMaxSeg candidates per class (test-time RoI count is 1000 per
// image, configs/bags/*: rpn max_num = 1000).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "bags_iou.cuh"

namespace bags {

constexpr int kNmsMaxSeg = 1024;
constexpr int kNmsThreads = 1024;   // 32 warps: the mask rows are dealt to the warps; with 8 the loop was issue-latency bound

// No candidate list is compacted on the host.  The caller sorts every class's scores once (one batched
// device sort: order[s][i] = RoI index of the i-th best score of class s+1) and counts the scores above the threshold
// per class on the device; CTA s gathers its count[s] best boxes straight from the decoded-box tensor and suppresses.
//   boxes     [n, box_cols] fp32: box_cols == 4 (class-agnostic) or 4 * (S + 1) (per class, class 0 = background)
//   order     [S, n] int32, counts [S] int32 (clamped to n), keep [S, n] uint8 out (0 beyond counts[s])
//   overflow  set to 1 if a class has more than kNmsMaxSeg candidates (its tail is dropped; the caller raises)
__global__ void __launch_bounds__(kNmsThreads)
class_nms_dense_kernel(const float* __restrict__ boxes, int box_cols, const int* __restrict__ order,
                       const int* __restrict__ counts, int n, float iou_thr, uint8_t* __restrict__ keep,
                       int* __restrict__ overflow) {
  extern __shared__ __align__(16) uint8_t nms_smem[];
  const int s = blockIdx.x;
  int cnt = counts[s];
  cnt = cnt < n ? cnt : n;
  cnt = cnt > 0 ? cnt : 0;   // a negative count would start the zeroing loop below before this class's keep row
  if (cnt > kNmsMaxSeg) { if (threadIdx.x == 0) *overflow = 1; cnt = kNmsMaxSeg; }
  const int* ord = order + static_cast<long long>(s) * n;
  uint8_t* kp = keep + static_cast<long long>(s) * n;
  for (int i = cnt + threadIdx.x; i < n; i += kNmsThreads) kp[i] = 0;
  if (cnt <= 0) return;
  const int words = (cnt + 31) >> 5;
  float4* sbox = reinterpret_cast<float4*>(nms_smem);
  uint32_t* mask = reinterpret_cast<uint32_t*>(sbox + ((cnt + 1) & ~1));
  const int coff = (box_cols == 4) ? 0 : 4 * (s + 1);
  for (int i = threadIdx.x; i < cnt; i += kNmsThreads)
    sbox[i] = *reinterpret_cast<const float4*>(boxes + static_cast<long long>(ord[i]) * box_cols + coff);
  __syncthreads();
  // one warp per row i, lane b <-> candidate 32 w + b: consecutive lanes read consecutive boxes (a thread-per-word
  // mapping strides the float4 reads by 512 B -- a 32-way bank conflict that made this loop 12x slower) and a ballot
  // assembles the word.  Rows are dealt round-robin to the warps; only words at or right of the diagonal are needed.
  {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = warp; i < cnt; i += kNmsThreads / 32) {
      const float4 bi = sbox[i];
      uint32_t mine = 0u;                       // lane w ends up holding word w of the row (words <= 32)
      for (int w = (i >> 5); w < words; ++w) {
        const int j = (w << 5) + lane;
        const bool sup = (j > i) && (j < cnt) && (iou_plus1(bi, sbox[j < cnt ? j : i]) > iou_thr);
        const uint32_t bits = __ballot_sync(0xffffffffu, sup);
        if (lane == w) mine = bits;
      }
      if (lane < words) mask[i * words + lane] = mine;
    }
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    uint32_t removed = 0u;
    for (int i = 0; i < cnt; ++i) {
      const uint32_t word = __shfl_sync(0xffffffffu, removed, i >> 5);
      const bool alive = ((word >> (i & 31)) & 1u) == 0u;
      if (alive && lane < words) removed |= mask[i * words + lane];
      if (lane == 0) kp[i] = alive ? 1 : 0;
    }
  }
}

}  // namespace bags
