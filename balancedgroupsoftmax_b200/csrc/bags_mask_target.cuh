// Training targets of the mask heads (FCNMaskHead.get_target -> mask_target, mmdet/core/mask/mask_target.py): each
// positive RoI's gt mask cut to its proposal box and resized to mask_h x mask_w as cv2.resize(uint8, INTER_LINEAR).
//
// One CTA per RoI, every image of the batch in one launch.  The CTA reads its box and gt index, cuts the crop by
// numpy's slice rules, builds the tap tables of both axes in shared memory and then computes each output pixel from
// the mask bytes with OpenCV's fixed-point arithmetic for 8-bit images:
//   per axis  scale = 1 / (D / S) in double; f = float((d + 0.5) * scale - 0.5); s = floor(f); f -= s
//             weights rint((1 - f) * 2048) and rint(f * 2048); taps s and s + 1 clamped to the crop
//   x axis    clamped: left of the first pixel or right of the last one the tap is that pixel with weight 2048
//   y axis    not clamped: the fraction is kept and only the row index is clamped
//   pixel     R(y) = src[y][x0] a0 + src[y][x1] a1;  out = (((b0 (R(y0) >> 4)) >> 16) + ((b1 (R(y1) >> 4)) >> 16) + 2) >> 2
// cv2 copies a crop of exactly the output size, and resizes a crop of exactly twice the output size on both axes with
// INTER_AREA, (sum of the 2 x 2 block + 2) >> 2; both are done the same way here.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bags {

constexpr int kMaskTargetThreads = 128;
constexpr int kMaskTargetMaxImages = 64;    // images per launch (the table travels as a kernel argument)
constexpr int kMaskTargetMaxSize = 256;     // mask_h, mask_w <= this (the tap tables live in static shared memory)

struct MaskTargetImage {
  const float* boxes;        // [num_pos, 4] (x1, y1, x2, y2)
  const long long* gt_inds;  // [num_pos]
  const uint8_t* masks;      // [num_gt, H, W]
  int roi_begin;             // first row of this image in the launch's output
  int num_gt, H, W;
};

struct MaskTargetParams {
  MaskTargetImage img[kMaskTargetMaxImages];
  int n_images;
  int mask_h, mask_w;
  float* out;                // [rows of this launch, mask_h, mask_w]
};

struct MaskTargetTap {
  int i0, i1;                // source indices inside the crop
  int a0, a1;                // fixed-point weights, a0 + a1 == 2048
};

__device__ __forceinline__ MaskTargetTap mask_target_tap(int d, int S, int D, bool clamp) {
  // every double and float operation spelled out: nvcc contracts nothing the CPU does not
  const double scale = __ddiv_rn(1.0, __ddiv_rn(static_cast<double>(D), static_cast<double>(S)));
  float f = __double2float_rn(__dsub_rn(__dmul_rn(static_cast<double>(d) + 0.5, scale), 0.5));
  int s = static_cast<int>(floorf(f));
  f = __fsub_rn(f, static_cast<float>(s));
  if (clamp) {
    if (s < 0) f = 0.f, s = 0;
    if (s >= S - 1) f = 0.f, s = S - 1;
  }
  MaskTargetTap t;
  t.a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
  t.a1 = __float2int_rn(__fmul_rn(f, 2048.f));
  t.i0 = min(max(s, 0), S - 1);
  t.i1 = min(max(s + 1, 0), S - 1);
  return t;
}

// numpy's float32 -> int32 cast on x86: truncation toward zero; NaN and values outside int32 give INT_MIN
__device__ __forceinline__ int np_int32(float v) {
  return (v >= -2147483648.f && v < 2147483648.f) ? static_cast<int>(v) : -2147483647 - 1;
}

// int32 sum that wraps as numpy's int32 scalars do
__device__ __forceinline__ int wrap_add(int a, int b) {
  return static_cast<int>(static_cast<unsigned>(a) + static_cast<unsigned>(b));
}

// [start, stop) of a Python slice start:stop over a dimension of n
__device__ __forceinline__ void py_slice(int start, int stop, int n, int& lo, int& hi) {
  long long a = start, b = stop;
  if (a < 0) a = a + n < 0 ? 0 : a + n;
  else if (a > n) a = n;
  if (b < 0) b = b + n < 0 ? 0 : b + n;
  else if (b > n) b = n;
  lo = static_cast<int>(a);
  hi = static_cast<int>(b > a ? b : a);
}

__global__ void __launch_bounds__(kMaskTargetThreads) bags_mask_target_kernel(const MaskTargetParams p) {
  __shared__ MaskTargetTap xt[kMaskTargetMaxSize], yt[kMaskTargetMaxSize];
  const int row = blockIdx.x, tid = threadIdx.x;
  int k = 0;
  while (k + 1 < p.n_images && p.img[k + 1].roi_begin <= row) ++k;
  const MaskTargetImage& im = p.img[k];
  const int r = row - im.roi_begin;
  const int mh = p.mask_h, mw = p.mask_w, npix = mh * mw;
  float* out = p.out + static_cast<size_t>(row) * npix;

  const long long gt = im.gt_inds[r];
  const int left = np_int32(im.boxes[4 * r + 0]), top = np_int32(im.boxes[4 * r + 1]);
  const int right = np_int32(im.boxes[4 * r + 2]), bottom = np_int32(im.boxes[4 * r + 3]);
  const int w = max(wrap_add(wrap_add(right, -left), 1), 1), h = max(wrap_add(wrap_add(bottom, -top), 1), 1);
  int x_lo, x_hi, y_lo, y_hi;
  py_slice(left, wrap_add(left, w), im.W, x_lo, x_hi);
  py_slice(top, wrap_add(top, h), im.H, y_lo, y_hi);
  const int cw = x_hi - x_lo, ch = y_hi - y_lo;
  if (gt < 0 || gt >= im.num_gt || cw == 0 || ch == 0) {   // the reference raises: a row of NaN
    for (int q = tid; q < npix; q += kMaskTargetThreads) out[q] = __int_as_float(0x7fc00000);
    return;
  }
  const uint8_t* src = im.masks + static_cast<size_t>(gt) * im.H * im.W + static_cast<size_t>(y_lo) * im.W + x_lo;
  const int W = im.W;

  if (cw == mw && ch == mh) {                      // cv2 copies
    for (int q = tid; q < npix; q += kMaskTargetThreads) out[q] = src[static_cast<size_t>(q / mw) * W + q % mw];
    return;
  }
  if (cw == 2 * mw && ch == 2 * mh) {              // cv2 takes INTER_AREA
    for (int q = tid; q < npix; q += kMaskTargetThreads) {
      const uint8_t* s = src + static_cast<size_t>(2 * (q / mw)) * W + 2 * (q % mw);
      out[q] = static_cast<float>((s[0] + s[1] + s[W] + s[W + 1] + 2) >> 2);
    }
    return;
  }
  for (int d = tid; d < mw; d += kMaskTargetThreads) xt[d] = mask_target_tap(d, cw, mw, true);
  for (int d = tid; d < mh; d += kMaskTargetThreads) yt[d] = mask_target_tap(d, ch, mh, false);
  __syncthreads();
  for (int q = tid; q < npix; q += kMaskTargetThreads) {
    const MaskTargetTap ty = yt[q / mw], tx = xt[q % mw];
    const uint8_t* r0 = src + static_cast<size_t>(ty.i0) * W;
    const uint8_t* r1 = src + static_cast<size_t>(ty.i1) * W;
    const int R0 = r0[tx.i0] * tx.a0 + r0[tx.i1] * tx.a1;
    const int R1 = r1[tx.i0] * tx.a0 + r1[tx.i1] * tx.a1;
    const int v = (((ty.a0 * (R0 >> 4)) >> 16) + ((ty.a1 * (R1 >> 4)) >> 16) + 2) >> 2;
    out[q] = static_cast<float>(min(v, 255));
  }
}

}  // namespace bags
