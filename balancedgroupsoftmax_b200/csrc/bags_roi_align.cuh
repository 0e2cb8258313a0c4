// FPN RoI feature extractor (SingleRoIExtractor + RoIAlign, mmdet/models/roi_extractors/single_level.py and
// mmdet/ops/roi_align/src/roi_align_kernel.cu): every RoI of every image pooled from its level in one launch, and
// the gradient scattered back into every level in one more.
//
// One CTA per (RoI, channel chunk).  Thread 0 maps the RoI to its level as map_roi_levels does when torch evaluates
// it on CUDA (each elementwise op rounded to fp32, the division by the Python scalar finest_scale a multiplication by
// its fp32 reciprocal):
//   level = clamp(floor(log2f(sqrt((x2 - x1 + 1) (y2 - y1 + 1)) * fp32(1 / finest_scale) + fp32(1e-6))), 0, L - 1)
// (no mapping with one level) and reads the batch index as the reference's (int) cast does.  A NaN level, or a batch
// index outside [0, B), gives a row of zeros and no gradient.  The RoI is then pooled as ROIAlignForward<float>,
// with the rounding sequence its -O2 sm_90a build has (read from its SASS; every step is spelled out here so that
// nothing depends on how this file's arithmetic is contracted):
//   start = x1 s                      roi_w = fmaxf(fma(x2 + 1, s, -start), 0)        bin = roi_w / out_w
//   samples per bin: sample_num, or (int)ceilf(bin) when sample_num <= 0
//   sample x = (fma(pw, bin, start)) + ((ix + 0.5) bin) / sw     (the same for y)
//   x < -1 or x > W (either axis): 0.  Else x <= 0 -> 0, lo = (int)x, lo >= W - 1 -> lo = hi = W - 1, x = lo;
//   lx = x - lo, hx = 1 - lx;  val = fma(ly lx, rb, fma(ly hx, lb, fma(hy lx, rt, (hy hx) lt)))
//   out = (sum over iy, then ix, of val) / (sh sw)
// Both axes' samples are separable, so the CTA tabulates them (lo, hi, l, h, in range) once in shared memory; a RoI
// with more than kRoiAlignMaxSamples samples on an axis (adaptive sample counts on a large RoI) computes them in the
// loop instead, with the same arithmetic.
//
// Backward: the reference adds (gout w_i) / count for each of the 4 corners of every sample with atomicAdd.  Here a
// CTA lists the distinct rows and columns its samples touch (at most 2 out_h sh x 2 out_w sw, whatever the RoI's
// size), each with the (bin, weight) pairs that reach it, and computes each touched pixel of its channel chunk in
// registers from the staged gout:
//   grad[r, q] += (sum_{(ph, wy) -> r} wy sum_{(pw, wx) -> q} wx gout[ph, pw]) / count
// in a fixed order, then adds it to the level's gradient with one reduction per touched pixel.  A RoI that overflows
// the sample tables falls back to the reference's per-corner scatter.  The order of additions across RoIs is open.
//
// The kernels are a translation unit of their own (bags_roi_align.cu), linked into the same library; bags_api.cu sees
// this header's launch table and launchers only.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bags {

constexpr int kRoiAlignThreads = 256;
constexpr int kRoiAlignMaxLevels = 8;
constexpr int kRoiAlignMaxOut = 64;        // out_h, out_w <= this
constexpr int kRoiAlignMaxSamples = 128;   // per-axis sample table: out * samples per bin
constexpr int kRoiAlignStage = 4096;       // gout floats staged per backward CTA: chunk * out_h * out_w <= this

struct RoiAlignLevel {
  const float* feat;   // [B, C, H, W] (forward)
  float* grad;         // [B, C, H, W] (backward; NULL: this level takes no gradient)
  int H, W;
  float scale;         // spatial_scale as fp32
};

struct RoiAlignParams {
  RoiAlignLevel lvl[kRoiAlignMaxLevels];
  int n_levels, B, C, k, out_h, out_w, sample_num;
  int chunk;               // channels per CTA
  float inv_finest;        // fp32(1 / finest_scale)
  const float* rois_map;   // [k, 5] RoIs the levels are mapped from
  const float* rois;       // [k, 5] RoIs that are pooled
  float* out;              // forward: [k, C, out_h, out_w]
  int* levels;             // forward, optional: [k] level of each RoI, -1 for none
  const float* gout;       // backward: [k, C, out_h, out_w]
};

// one launch over every RoI and channel chunk (bags_roi_align.cu); they return cudaGetLastError() of the launch
cudaError_t launch_roi_align_fwd(const RoiAlignParams& p, cudaStream_t stream);
cudaError_t launch_roi_align_bwd(const RoiAlignParams& p, cudaStream_t stream);

}  // namespace bags
