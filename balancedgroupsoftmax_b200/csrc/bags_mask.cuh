// Class-specific mask logits fused with their BCE loss -- conv_logits (a 1x1 conv, fcn_mask_head.py:82,102) restricted
// to the one channel mask_cross_entropy reads per RoI (pred[arange(P), labels], cross_entropy_loss.py:54-61) instead of
// the [P, classes, H, W] logits:
//
//   bags_mask_sort_kernel  one CTA: the stable per-class index of the RoIs with 0 <= label < classes (box_class_sort).
//   bags_mask_fwd_kernel   one CTA per (RoI, tile of kMaskTile pixels).  Pass 1 reads y[p, :, tile] from HBM and forms
//                          z = b[l] + sum_c W[l,c] y[p,c,q]; then the BCE-with-logits of each pixel and its gradient
//                          g = (sigmoid(z) - t) / (P H W).  Pass 2 re-reads the same tile, still in L2, for the tile's
//                          share of the backward's dW: rsum[p, tile, c] = sum_q g[p,q] y[p,c,q] (and sum_q g for db).
//                          The tile losses go to a contiguous array that the last CTA to arrive sums in a fixed order.
//   bags_mask_bwd_kernel   one CTA per work unit.  Class units: 32 columns of dW[l, :] (or db[l]) from the rsum rows of
//                          the class's RoIs, its (RoI, tile) pairs dealt to 8 warps in ascending order and the warps'
//                          partials added in warp order (zero for a class without RoIs).  RoI units: one tile of
//                          dY[p, :, q] = gout g[p,q] W[l, :] (zero for an invalid row).
// y is read from HBM once; no atomics on floats, so every output is bit-identical from run to run.
#pragma once
#include "bags_kernels.cuh"
#include "bags_box.cuh"

namespace bags {

constexpr int kMaskThreads = 256;
constexpr int kMaskTile = 64;            // pixels per CTA (BAGS_MASK_TILE in the header)
constexpr int kMaskCounterWord = 17;     // the forward's arrival counter: word 17 of the workspace's counter line

struct MaskFwdParams {
  const void* y;                         // [P, Cin, HW] bf16 or fp32
  const float* w; long long ldw;         // [classes, Cin] fp32
  const float* bias;                     // [classes] or nullptr
  const long long* labels;               // [P]
  const float* targets;                  // [P, HW]
  int P, Cin, HW, classes, tiles;
  float n;                               // P * HW, the mean's normaliser
  float* loss;                           // [1]
  float* g;                              // [P, HW]
  float* rsum;                           // [P, tiles, Cin + 1], then the tile losses [P * tiles]
  unsigned int* counter;                 // zero on entry, reset on exit
};

struct MaskBwdParams {
  const float* g; const float* rsum; const float* gout;
  const float* w; long long ldw;
  const long long* labels;
  const int* index;
  int P, Cin, HW, classes, tiles, chunks, class_units;   // chunks: 32-column slices of the Cin + 1 dW / db columns
  float* dW; long long lddw;
  float* db;
  void* dY;
};

__device__ __forceinline__ bool mask_valid(long long l, int classes) { return MaskLabelValid()(l, classes); }

// V consecutive elements of y at element offset ``off`` (V = 4: 8- (bf16) or 16-byte (fp32) aligned)
template <bool BF16, int V>
__device__ __forceinline__ void mask_load(const void* base, long long off, float* v) {
  if constexpr (V == 4) {
    const float4 f = box_load4<BF16>(base, off);
    v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
  } else if constexpr (BF16) {
    v[0] = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(base)[off]);
  } else {
    v[0] = __ldg(reinterpret_cast<const float*>(base) + off);
  }
}

__global__ void __launch_bounds__(kBoxThreads)
bags_mask_sort_kernel(const long long* labels, int P, int classes, int* index) {
  __shared__ int s_cursor[kBoxMaxClasses];
  __shared__ short s_lab[kBoxSortBatch];
  __shared__ int s_scan[kBoxThreads / 32];
  box_class_sort<MaskLabelValid>(labels, P, classes, index, s_cursor, s_lab, s_scan);
}

template <bool BF16, int V>
__global__ void __launch_bounds__(kMaskThreads, 4)
bags_mask_fwd_kernel(const MaskFwdParams p) {
  constexpr int QV = kMaskTile / V;            // threads along the tile's pixels
  constexpr int NG = kMaskThreads / QV;        // channel groups
  __shared__ float s_red[NG][kMaskTile];
  __shared__ float s_g[kMaskTile];
  __shared__ float s_warp[kMaskThreads / 32];
  __shared__ unsigned int s_last;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int pr = blockIdx.x / p.tiles, t = blockIdx.x % p.tiles;
  const int q0 = t * kMaskTile, nq = min(kMaskTile, p.HW - q0);
  const long long l = __ldg(p.labels + pr);
  const long long ybase = static_cast<long long>(pr) * p.Cin * p.HW + q0;
  float* rs = p.rsum + (static_cast<long long>(pr) * p.tiles + t) * (p.Cin + 1);
  float tile_loss = 0.f;
  if (mask_valid(l, p.classes)) {   // CTA-uniform
    // pass 1: per channel group, sum_c W[l,c] y[p,c,q] over its channels; then the groups in order
    const int qv = tid % QV, cg = tid / QV;
    const float* wl = p.w + l * p.ldw;
    float acc[V];
#pragma unroll
    for (int v = 0; v < V; ++v) acc[v] = 0.f;
    if (qv * V < nq) {   // V = 4 only when HW % 4 == 0, so the whole vector is inside the tile
#pragma unroll 4
      for (int c = cg; c < p.Cin; c += NG) {
        const float wc = __ldg(wl + c);
        float yv[V];
        mask_load<BF16, V>(p.y, ybase + static_cast<long long>(c) * p.HW + qv * V, yv);
#pragma unroll
        for (int v = 0; v < V; ++v) acc[v] = fmaf(wc, yv[v], acc[v]);
      }
    }
#pragma unroll
    for (int v = 0; v < V; ++v) s_red[cg][qv * V + v] = acc[v];
    __syncthreads();
    if (tid < kMaskTile) {
      float gq = 0.f, lq = 0.f;
      if (tid < nq) {
        float z = 0.f;
#pragma unroll 4
        for (int k = 0; k < NG; ++k) z += s_red[k][tid];
        if (p.bias != nullptr) z += __ldg(p.bias + l);
        const long long o = static_cast<long long>(pr) * p.HW + q0 + tid;
        const float tq = __ldg(p.targets + o);
        // F.binary_cross_entropy_with_logits: max(z, 0) - z t + log1p(exp(-|z|)); d/dz = sigmoid(z) - t
        const float e = expf(-fabsf(z));
        const float s = z >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
        lq = fmaxf(z, 0.f) - z * tq + log1pf(e);
        gq = (s - tq) / p.n;
        p.g[o] = gq;
      }
      s_g[tid] = gq;
      tile_loss = warp_sum(lq);          // warps 0 and 1
    }
    __syncthreads();
    // pass 2: the tile's sum_q g y per channel, one warp per channel, the tile re-read from L2
    for (int c = warp; c < p.Cin; c += kMaskThreads / 32) {
      const long long yo = ybase + static_cast<long long>(c) * p.HW;
      float v = 0.f;
      for (int q = lane; q < nq; q += 32) {
        float yv[1];
        mask_load<BF16, 1>(p.y, yo + q, yv);
        v = fmaf(s_g[q], yv[0], v);
      }
      v = warp_sum(v);
      if (lane == 0) rs[c] = v;
    }
    if (warp == kMaskThreads / 32 - 1) {
      float v = lane < nq ? s_g[lane] : 0.f;
      if (lane + 32 < nq) v += s_g[lane + 32];
      v = warp_sum(v);
      if (lane == 0) rs[p.Cin] = v;
    }
  } else {
    // an invalid row: g = 0, nothing of it reaches dW or db (the class index leaves it out)
    if (tid < nq) p.g[static_cast<long long>(pr) * p.HW + q0 + tid] = 0.f;
  }
  // the tile's loss, then the tile losses in a fixed order by the last CTA to arrive
  float* part = p.rsum + static_cast<long long>(p.P) * p.tiles * (p.Cin + 1);
  if (lane == 0 && warp < 2) s_warp[warp] = tile_loss;
  __syncthreads();
  if (tid == 0) {
    part[blockIdx.x] = mask_valid(l, p.classes) ? s_warp[0] + s_warp[1] : 0.f;
    __threadfence();
    s_last = (atomicAdd(p.counter, 1u) == gridDim.x - 1) ? 1u : 0u;
  }
  __syncthreads();
  if (s_last == 0u) return;
  __threadfence();
  float v = 0.f;
#pragma unroll 8
  for (int i = tid; i < static_cast<int>(gridDim.x); i += kMaskThreads) v += __ldcg(part + i);
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) s_warp[warp] = v;
  __syncthreads();
  if (tid == 0) {
    float total = 0.f;
    for (int w = 0; w < kMaskThreads / 32; ++w) total += s_warp[w];
    *p.loss = total / p.n;
    *p.counter = 0u;
  }
}

template <bool BF16, int V>
__global__ void __launch_bounds__(kMaskThreads, 4)
bags_mask_bwd_kernel(const MaskBwdParams p) {
  const float go = p.gout != nullptr ? __ldg(p.gout) : 1.f;
  const int tid = threadIdx.x;
  int u = blockIdx.x;
  if (u < p.class_units) {
    // class unit: 32 columns (lane = column) of one class; warp w takes the (RoI, tile) pairs j = w, w + 8, ... of the
    // class's RoIs in ascending id, then the warps' partials are added in warp order -- a fixed order for a given
    // class, so a class with many RoIs (or a class-agnostic head) is spread over 8 warps and several CTAs
    __shared__ float s_part[kMaskThreads / 32][32];
    const int warp = tid >> 5, lane = tid & 31;
    const int l = u / p.chunks;
    const int c = (u % p.chunks) * 32 + lane;
    const int lo = __ldg(p.index + l), hi = __ldg(p.index + l + 1);
    const int* rois = p.index + p.classes + 1;
    const long long row = static_cast<long long>(p.tiles) * (p.Cin + 1);
    const int pairs = (hi - lo) * p.tiles;
    float acc = 0.f;
    if (c <= p.Cin) {
#pragma unroll 4
      for (int j = warp; j < pairs; j += kMaskThreads / 32) {
        const int i = lo + j / p.tiles, t = j % p.tiles;
        acc += __ldg(p.rsum + __ldg(rois + i) * row + static_cast<long long>(t) * (p.Cin + 1) + c);
      }
    }
    s_part[warp][lane] = acc;
    __syncthreads();
    if (warp == 0 && c <= p.Cin) {
      float total = 0.f;
#pragma unroll
      for (int w = 0; w < kMaskThreads / 32; ++w) total += s_part[w][lane];
      if (c < p.Cin) {
        if (p.dW != nullptr) p.dW[l * p.lddw + c] = go * total;
      } else if (p.db != nullptr) {
        p.db[l] = go * total;
      }
    }
    return;
  }
  u -= p.class_units;
  constexpr int QV = kMaskTile / V;
  constexpr int NG = kMaskThreads / QV;
  const int pr = u / p.tiles, t = u % p.tiles;
  const int q0 = t * kMaskTile, nq = min(kMaskTile, p.HW - q0);
  const int qv = tid % QV, cg = tid / QV;
  if (qv * V >= nq) return;
  const long long l = __ldg(p.labels + pr);
  const bool valid = mask_valid(l, p.classes);
  float gq[V];
#pragma unroll
  for (int v = 0; v < V; ++v) gq[v] = valid ? go * __ldg(p.g + static_cast<long long>(pr) * p.HW + q0 + qv * V + v) : 0.f;
  const float* wl = p.w + (valid ? l : 0) * p.ldw;
  const long long base = static_cast<long long>(pr) * p.Cin * p.HW + q0 + qv * V;
#pragma unroll 4
  for (int c = cg; c < p.Cin; c += NG) {
    const float wc = valid ? __ldg(wl + c) : 0.f;
    const long long off = base + static_cast<long long>(c) * p.HW;
    if constexpr (V == 4) {
      if constexpr (BF16) {
        uint2 q;
        q.x = pack_bf16x2(gq[0] * wc, gq[1] * wc);
        q.y = pack_bf16x2(gq[2] * wc, gq[3] * wc);
        *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(p.dY) + off) = q;
      } else {
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.dY) + off) =
            make_float4(gq[0] * wc, gq[1] * wc, gq[2] * wc, gq[3] * wc);
      }
    } else if constexpr (BF16) {
      reinterpret_cast<__nv_bfloat16*>(p.dY)[off] = __float2bfloat16_rn(gq[0] * wc);
    } else {
      reinterpret_cast<float*>(p.dY)[off] = gq[0] * wc;
    }
  }
}

}  // namespace bags
