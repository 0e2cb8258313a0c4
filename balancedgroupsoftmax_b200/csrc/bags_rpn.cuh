// RPN proposal generation (RPNHead.get_bboxes, mmdet/models/anchor_heads/rpn_head.py:55-104 and
// anchor_head.py:250-276, with the NMS op of mmdet/ops/nms): every (image, level) segment of a batch selected, decoded
// and suppressed, and every image's levels merged, in four launches whatever the batch and level counts.
//
//   1. select   one 8-CTA cluster per segment.  Each CTA reads its share of the logits [B, A, H, W] in memory order,
//               computes the sigmoid in registers (1 / (1 + expf(-x)), as torch.sigmoid) and radix-selects the top
//               nms_pre of the 64-bit keys (order(score) << 32 | ~flat), flat = (h W + w) A + a, in 8-bit digits
//               with the histograms summed over the cluster through distributed shared memory.  The keys are
//               distinct, so the selection is exact and ties go to the lower flat index.  A level with at most
//               nms_pre anchors, or nms_pre <= 0, takes every anchor.  The selected keys are gathered into the
//               shared memory of the cluster's first CTA, which sorts them (score desc, flat asc), builds each anchor
//               (base anchor + (w stride, h stride), one fp32 add, as grid_anchors), decodes it with delta2bbox's
//               operation sequence (one rounding per torch op), drops boxes below min_bbox_size and writes the list.
//   2. mask     the suppression bit matrix of every segment (IoU with "+1" widths, iou_plus1; bit j of row i set when
//               j > i and IoU > nms_thr), one 64-row x 256-column tile per CTA, into L2-resident scratch.
//   3. scan     one CTA per segment: warp 0 runs the greedy scan while the other warps stage the next rows of the
//               matrix into shared memory.  The survivors keep the level's input order, as the op returns its kept
//               indices ascending: score order for a selected level, anchor order for one that was not.  The first
//               nms_post of them in that order are written out in score order.
//   4. merge    per image, each survivor's rank in (score desc, level asc, position asc) by binary search in every
//               level's list; ranks below max_num are written to [B, max_num, 5], zero rows after the image's count.
//
// The kernels are a translation unit of their own (bags_rpn.cu), linked into the same library; bags_api.cu sees this
// header's launch table and launcher only.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace bags {

constexpr int kRpnMaxLevels = 8;
constexpr int kRpnMaxImages = 32;
constexpr int kRpnMaxAnchors = 16;     // base anchors per location (scales x ratios)
constexpr int kRpnMaxCand = 4096;      // candidates per (image, level): min(nms_pre, anchors) or every anchor
constexpr int kRpnCluster = 8;         // CTAs per segment in the select launch
constexpr int kRpnSelectThreads = 512;

struct RpnLevel {
  const float* logits;    // [B, A, H, W]
  const float* deltas;    // [B, 4 A, H, W]
  int H, W, A, stride;
  int n;                  // H W A anchors
  int K;                  // candidates: n, or nms_pre when the level is selected
  int select;             // 1: top nms_pre of n
  int post;               // min(K, nms_post): survivors kept
  int tiles, tile0;       // mask tiles of one image's segment, and the first of them within the image
  int surv0;              // first survivor slot of this level within the image
  size_t cand_off, mask_off, surv_off;   // byte offsets of the level's pieces within one image's scratch
  float4 base[kRpnMaxAnchors];
};

struct RpnParams {
  RpnLevel lvl[kRpnMaxLevels];
  int img_h[kRpnMaxImages], img_w[kRpnMaxImages];
  int n_levels, B, nms_post, max_num;
  int tiles_per_img, surv_per_img;
  float nms_thr, min_bbox_size, max_ratio;
  float means[4], stds[4];
  uint8_t* scratch;
  size_t img_bytes;       // scratch bytes of one image's segments
  int* counts_scratch;    // [B, L, 2]: candidates after min_bbox_size, survivors
  float* out;             // [B, max_num, 5]
  int* counts;            // [B]
};

// scratch layout: from n_levels, B, nms_post and each level's K, fills the levels' offsets, tiles and survivor slots,
// points counts_scratch and scratch into `scratch` (may be NULL) and returns the bytes it needs
size_t rpn_layout(RpnParams& p, void* scratch);

// the four launches on `stream`; returns the first launch error
cudaError_t launch_rpn_proposals(const RpnParams& p, cudaStream_t stream);

}  // namespace bags
