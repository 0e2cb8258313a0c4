// Test-time masks of the mask heads (FCNMaskHead.get_seg_masks / get_seg_masks_without, fcn_mask_head.py:125-239):
// resize each detection's probability map to its box, threshold it, paste it into an empty image and encode the image
// as COCO compressed RLE -- without materialising the image.
//
// One CTA per detection walks the candidate transition positions of its canvas in column-major order.  A transition
// (pixel i differs from pixel i-1) needs pixel i or i-1 inside the box, so only rows [top, top + h] of the box
// columns are candidates: w * (h + 1) positions, in increasing flattened order.  The CTA takes them in tiles of
// kSegmTile, compacts the tile's transitions with a block scan and turns each into its run length, its delta against
// the run two before (pycocotools' rleToString) and its 5-bit characters.  A sizing pass (out == NULL) writes each
// detection's string length; the write pass places every string at the sum of the lengths before it.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bags {

constexpr int kSegmThreads = 256;
constexpr int kSegmPer = 8;                               // consecutive candidates per thread
constexpr int kSegmTile = kSegmThreads * kSegmPer;

// cv2.resize(INTER_LINEAR) of a float32 map as OpenCV computes it with IPP (its default build): per axis the source
// coordinate (d + 0.5) * (S / D) - 0.5 in double, the fraction rounded once to float, clamped at both borders (the
// edge taps read one pixel); then a horizontal and a vertical pass of a + t * (b - a) with one fused multiply-add.
// Every operation is spelled out so that nvcc contracts nothing the CPU does not.
struct SegmTap {
  int i0, i1;
  float t;
};

__device__ __forceinline__ SegmTap segm_tap(int d, int S, double ratio) {
  const double x = __dsub_rn(__dmul_rn(static_cast<double>(d) + 0.5, ratio), 0.5);
  const double f = floor(x);
  SegmTap tap{static_cast<int>(f), 0, __double2float_rn(__dsub_rn(x, f))};
  if (tap.i0 < 0) tap.i0 = 0, tap.t = 0.f;
  if (tap.i0 >= S - 1) tap.i0 = S - 1, tap.t = 0.f;
  tap.i1 = tap.i0 + 1 < S ? tap.i0 + 1 : S - 1;
  return tap;
}

__device__ __forceinline__ float segm_lerp(float a, float b, float t) { return __fmaf_rn(t, __fsub_rn(b, a), a); }

struct SegmBox {
  const float* p;         // this detection's [mh, mw] probabilities
  int mh, mw, w, h;
  double rx, ry;          // mw / w, mh / h
  bool copy;              // dsize == ssize: cv2 copies
  double thr;
};

// thresholded resized value at box pixel (y, x)
__device__ __forceinline__ int segm_pixel(const SegmBox& b, int y, int x) {
  float v;
  if (b.copy) {
    v = __ldg(b.p + static_cast<size_t>(y) * b.mw + x);
  } else {
    const SegmTap tx = segm_tap(x, b.mw, b.rx), ty = segm_tap(y, b.mh, b.ry);
    const float* r0 = b.p + static_cast<size_t>(ty.i0) * b.mw;
    const float* r1 = b.p + static_cast<size_t>(ty.i1) * b.mw;
    const float top = segm_lerp(__ldg(r0 + tx.i0), __ldg(r0 + tx.i1), tx.t);
    const float bot = segm_lerp(__ldg(r1 + tx.i0), __ldg(r1 + tx.i1), tx.t);
    v = segm_lerp(top, bot, ty.t);
  }
  return static_cast<double>(v) > b.thr ? 1 : 0;
}

// characters of one rleToString value: 5-bit groups, low first, 0x20 = more follow, + 48
__device__ __forceinline__ int segm_chars(long long x, char* out) {
  int n = 0;
  bool more = true;
  while (more) {
    int c = static_cast<int>(x & 0x1f);
    x >>= 5;
    more = (c & 0x10) ? x != -1 : x != 0;
    if (more) c |= 0x20;
    if (out) out[n] = static_cast<char>(c + 48);
    ++n;
  }
  return n;
}

// exclusive block scan of one value per thread; *total = the sum.  Ends with a barrier.
__device__ __forceinline__ long long segm_block_scan(long long v, long long* warp_sums, long long* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += u;
  }
  if (lane == 31) warp_sums[warp] = incl;
  __syncthreads();
  long long before = 0, sum = 0;
#pragma unroll
  for (int k = 0; k < kSegmThreads / 32; ++k) {
    const long long s = warp_sums[k];
    if (k < warp) before += s;
    sum += s;
  }
  *total = sum;
  __syncthreads();
  return before + incl - v;
}

__global__ void __launch_bounds__(kSegmThreads) bags_segm_rle_kernel(
    const float* __restrict__ probs, int mh, int mw, const int4* __restrict__ boxes, int img_h, int img_w, double thr,
    long long* __restrict__ lengths, char* __restrict__ out) {
  __shared__ long long pos[3 + kSegmTile];   // [0, 3): the last three transitions before the tile (0 before any)
  __shared__ long long warp_sums[kSegmThreads / 32];
  const int d = blockIdx.x, tid = threadIdx.x;
  const int4 bx = boxes[d];
  const int left = bx.x, top = bx.y, w = bx.z, h = bx.w;
  SegmBox b;
  b.p = probs + static_cast<size_t>(d) * mh * mw;
  b.mh = mh; b.mw = mw; b.w = w; b.h = h;
  b.rx = __ddiv_rn(static_cast<double>(mw), static_cast<double>(w));
  b.ry = __ddiv_rn(static_cast<double>(mh), static_cast<double>(h));
  b.copy = (w == mw && h == mh);
  b.thr = thr;
  const long long N = static_cast<long long>(img_h) * img_w;
  const bool full_height = top == 0 && h == img_h;   // the last box row is followed by the next column's first

  char* dst = nullptr;
  if (out != nullptr) {                            // this string's offset: the lengths of the detections before it
    long long s = 0;
    for (int k = tid; k < d; k += kSegmThreads) s += lengths[k];
    long long total;
    segm_block_scan(s, warp_sums, &total);
    dst = out + total;
  }
  if (tid < 3) pos[tid] = 0;
  long long ntr = 0, nchars = 0;   // transitions and characters so far (the same in every thread)
  const long long rows = static_cast<long long>(h) + 1, ncand = static_cast<long long>(w) * rows;
  __syncthreads();

  for (long long tile = 0; tile < ncand; tile += kSegmTile) {
    // 1. this thread's kSegmPer consecutive candidates: which are transitions
    unsigned flags = 0;
    long long q = tile + static_cast<long long>(tid) * kSegmPer;
    int col = static_cast<int>(q / rows), r = static_cast<int>(q % rows);
    int prev = -1;   // the pixel before the candidate, once known
#pragma unroll 1
    for (int j = 0; j < kSegmPer && q < ncand; ++j, ++q) {
      const long long i = static_cast<long long>(left + col) * img_h + top + r;
      const bool dup = r == h && full_height && col < w - 1;   // also the next column's first candidate
      const int cur = r < h ? segm_pixel(b, r, col) : 0;
      if (prev < 0) {
        if (r > 0) prev = segm_pixel(b, r - 1, col);
        else if (full_height && col > 0) prev = segm_pixel(b, h - 1, col - 1);   // the previous column's last row
        else prev = 0;                                                         // above the box, or pixel 0
      }
      if (!dup && i < N && cur != prev) flags |= 1u << j;
      prev = cur;
      if (++r == rows) r = 0, ++col, prev = -1;
    }
    // 2. compact the tile's transition positions after the carried three
    long long ntile;
    const long long slot = segm_block_scan(__popc(flags), warp_sums, &ntile);
    {
      long long k = slot;
      long long qq = tile + static_cast<long long>(tid) * kSegmPer;
      for (int j = 0; j < kSegmPer; ++j, ++qq)
        if (flags & (1u << j)) {
          const int c = static_cast<int>(qq / rows), rr = static_cast<int>(qq % rows);
          pos[3 + k++] = static_cast<long long>(left + c) * img_h + top + rr;
        }
    }
    __syncthreads();
    // 3. each transition g closes run g - 1: its characters, as a contiguous chunk of slots per thread
    const long long chunk = (ntile + kSegmThreads - 1) / kSegmThreads;
    const long long s0 = tid * chunk < ntile ? tid * chunk : ntile;
    const long long s1 = s0 + chunk < ntile ? s0 + chunk : ntile;
    long long mine = 0;
    for (long long s = s0; s < s1; ++s) {
      long long x = pos[3 + s] - pos[2 + s];
      if (ntr + s >= 3) x -= pos[1 + s] - pos[s];
      mine += segm_chars(x, nullptr);
    }
    long long tile_chars;
    long long at = nchars + segm_block_scan(mine, warp_sums, &tile_chars);
    if (dst != nullptr)
      for (long long s = s0; s < s1; ++s) {
        long long x = pos[3 + s] - pos[2 + s];
        if (ntr + s >= 3) x -= pos[1 + s] - pos[s];
        at += segm_chars(x, dst + at);
      }
    // 4. carry the last three transitions
    long long carry = 0;
    if (tid < 3) carry = pos[3 + ntile - 3 + tid];
    __syncthreads();
    if (tid < 3) pos[tid] = carry;
    __syncthreads();
    ntr += ntile;
    nchars += tile_chars;
  }

  // the last run ends at the end of the image
  if (tid == 0) {
    long long x = N - pos[2];
    if (ntr > 2) x -= pos[1] - pos[0];
    const long long len = nchars + segm_chars(x, dst ? dst + nchars : nullptr);
    if (out == nullptr) lengths[d] = len;
  }
}

}  // namespace bags
