// RPN training targets (anchor_target, mmdet/core/anchor/anchor_target.py, with MaxIoUAssigner of
// core/bbox/assigners/max_iou_assigner.py and the base sampler of core/bbox/samplers/base_sampler.py): every anchor of
// every image of a batch assigned, sampled and encoded in four launches after one memset, whatever the batch and gt
// counts, with no host read.
//
//   0. memset   the per-gt maxima and the per-image counters of the scratch.
//   1. gt max   per gt, the max over the image's inside anchors of bbox_overlaps(gt, anchor) (iou_overlaps), as a
//               64-bit key (order(iou) << 32 | ~anchor index) atomically maxed: NaN wins, ties go to the first anchor.
//               Each CTA holds 1024 anchors in registers and streams the image's gts through shared memory in tiles,
//               so no gt count has a cap and no [G, N] matrix exists.
//   2. assign   per inside anchor, the max over gts (first gt on ties, NaN wins) and MaxIoUAssigner's steps 2 to 4
//               with fp32 thresholds; step 4 recomputes each IoU and lets the last gt win.  Counts each image's
//               positives and negatives.
//   3. select   one 8-CTA cluster per (image, positives | negatives): radix-selects the k smallest of the 64-bit
//               sampling keys (sample_key(seed, image, n) << 32 | n) of the gallery, in 8-bit digits with the
//               histograms summed through distributed shared memory; k = min(#pos, int(num pos_fraction)) for the
//               positives and min(#neg, num - k_pos, capped by neg_pos_ub) for the negatives.
//   4. write    the dense [B, N] labels and label weights and [B, N, 4] box targets (bbox2delta's op sequence) and
//               weights, zero outside the inside anchors, and the three device totals.
//
// Anchors are numbered per image as anchor_target concatenates them: level after level, each location-major
// ((h W + w) A + a), built on the device as grid_anchors builds them (bags_anchor.cuh).  The kernels are a
// translation unit of their own (bags_anchor_target.cu); bags_api.cu sees this header's launch table only.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace bags {

constexpr int kAtMaxLevels = 8;
constexpr int kAtMaxImages = 32;
constexpr int kAtMaxAnchors = 16;      // base anchors per location
constexpr int kAtCluster = 8;          // CTAs per (image, gallery) in the select launch
constexpr int kAtSelectThreads = 512;

struct AtLevel {
  int H, W, A, stride;
  int n;                  // H W A anchors
  int off;                // first anchor of the level within an image
  float4 base[kAtMaxAnchors];
};

struct AtImage {
  int gt_off, gt_cnt;     // the image's rows of the concatenated gts
  int valid_h[kAtMaxLevels], valid_w[kAtMaxLevels];   // valid_flags: min(ceil(pad / stride), feat)
  float x_hi, y_hi;       // anchor_inside_flags: x2 < img_w + allowed_border, y2 < img_h + allowed_border (fp32)
};

struct AtParams {
  AtLevel lvl[kAtMaxLevels];
  AtImage img[kAtMaxImages];
  int n_levels, B, N;     // N anchors per image
  const float4* gts;      // [total gts] (x1, y1, x2, y2)
  int border_on;          // allowed_border >= 0: the border test applies
  float border_lo;        // x1 >= -allowed_border, y1 >= -allowed_border (fp32)
  float pos_thr, neg_lo, neg_hi, min_pos;   // fp32 thresholds; negatives are neg_lo <= max < neg_hi when neg_on
  int neg_on, assign_all;
  int num, exp_pos;       // sampler num and int(num * pos_fraction)
  double neg_pos_ub;      // < 0: no bound
  float pos_weight;       // label weight of a sampled positive
  float means[4], stds[4];
  unsigned long long seed;
  const long long* seed_step;   // optional device step counter: seed + step * 0x9E3779B97F4A7C15
  // scratch
  int* counts;                  // [B, 2] positives, negatives (zeroed by the memset)
  unsigned long long* gt_key;   // [total gts] per-gt max key (zeroed by the memset)
  unsigned long long* sel;      // [B, 2, 2] (threshold, k) of the positives and negatives
  int* assign;                  // [B, N] -2 outside, -1 ignored, 0 negative, i + 1 positive of gt i
  size_t zero_bytes;            // bytes of the memset from the scratch's start
  // outputs
  long long* labels;            // [B, N]
  float* label_weights;         // [B, N]
  float4* bbox_targets;         // [B, N]
  float4* bbox_weights;         // [B, N]
  long long* totals;            // [3] num_total_pos, num_total_neg, their sum
};

// scratch layout for p.B, p.N and `total_gts`: points p's scratch pieces into `scratch` (may be NULL) and returns the
// bytes it needs
size_t anchor_target_layout(AtParams& p, int total_gts, void* scratch);

// the memset and four launches on `stream`; returns the first launch error
cudaError_t launch_anchor_target(const AtParams& p, cudaStream_t stream);

}  // namespace bags
