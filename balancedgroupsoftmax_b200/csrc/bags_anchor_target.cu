// Kernels of the RPN training targets: see bags_anchor_target.cuh for what they compute.
#include <cooperative_groups.h>

#include "bags_anchor.cuh"
#include "bags_anchor_target.cuh"
#include "bags_hash.cuh"
#include "bags_iou.cuh"

namespace cg = cooperative_groups;

namespace bags {

constexpr int kAtThreads = 256;        // gt max, assign and write
constexpr int kAtPer = 4;              // anchors per thread in the gt max and assign launches
constexpr int kAtSpan = kAtThreads * kAtPer;
constexpr int kAtGtTile = 256;         // gts staged in shared memory at a time

// monotone in v, NaN above every number, -0 and +0 one value (torch.max compares them equal)
__device__ __forceinline__ uint32_t iou_order(float v) {
  if (v != v) return 0xffffffffu;
  const uint32_t b = __float_as_uint(v == 0.f ? 0.f : v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float iou_of_order(uint32_t u) {
  if (u == 0xffffffffu) return __int_as_float(0x7fc00000);
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

__device__ __forceinline__ unsigned long long effective_seed(const AtParams& p) {
  return p.seed_step ? p.seed + static_cast<unsigned long long>(__ldg(p.seed_step)) * 0x9E3779B97F4A7C15ull : p.seed;
}

// the sampling key of anchor n of image img: distinct per n (the index is the low half)
__device__ __forceinline__ unsigned long long anchor_key(unsigned long long seed, int img, int n) {
  return (static_cast<unsigned long long>(sample_key(seed, img, n)) << 32) | static_cast<unsigned>(n);
}

// anchor n of an image (level after level, location-major) and whether it is an inside anchor of image `im`
__device__ __forceinline__ float4 anchor_at(const AtParams& p, const AtImage& im, int n, bool& inside) {
  int l = 0;
  while (l + 1 < p.n_levels && p.lvl[l + 1].off <= n) ++l;
  const AtLevel& L = p.lvl[l];
  const int m = n - L.off;
  const int hw = m / L.A, a = m - hw * L.A;
  const int hy = hw / L.W, wx = hw - hy * L.W;
  const float4 an = grid_anchor(L.base[a], wx, hy, L.stride);
  inside = hy < im.valid_h[l] && wx < im.valid_w[l];
  if (p.border_on)
    inside = inside && an.x >= p.border_lo && an.y >= p.border_lo && an.z < im.x_hi && an.w < im.y_hi;
  return an;
}

__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long y = __shfl_xor_sync(0xffffffffu, v, o);
    v = y > v ? y : v;
  }
  return v;
}

// ---------------------------------------------------------------------------------------------------------------
// 1. per-gt max over the inside anchors
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kAtThreads) bags_at_gt_max_kernel(const __grid_constant__ AtParams p) {
  __shared__ float4 s_gt[kAtGtTile];
  __shared__ float s_area[kAtGtTile];
  __shared__ unsigned long long s_key[kAtGtTile];
  const int img = blockIdx.y;
  const AtImage& im = p.img[img];
  const int n0 = blockIdx.x * kAtSpan + threadIdx.x;
  float4 an[kAtPer];
  float area[kAtPer];
  unsigned in = 0u;
#pragma unroll
  for (int e = 0; e < kAtPer; ++e) {
    const int n = n0 + e * kAtThreads;
    bool inside = false;
    if (n < p.N) an[e] = anchor_at(p, im, n, inside);
    area[e] = inside ? area_plus1(an[e]) : 0.f;
    in |= inside ? 1u << e : 0u;
  }
  if (!__syncthreads_or(in != 0u)) return;
  const int lane = threadIdx.x & 31;
  for (int t0 = 0; t0 < im.gt_cnt; t0 += kAtGtTile) {
    const int nt = min(kAtGtTile, im.gt_cnt - t0);
    for (int j = threadIdx.x; j < nt; j += kAtThreads) {
      const float4 g = p.gts[im.gt_off + t0 + j];
      s_gt[j] = g;
      s_area[j] = area_plus1(g);
      s_key[j] = 0ull;
    }
    __syncthreads();
    for (int j = 0; j < nt; ++j) {
      const float4 g = s_gt[j];
      const float ag = s_area[j];
      unsigned long long best = 0ull;
#pragma unroll
      for (int e = 0; e < kAtPer; ++e) {
        if ((in >> e) & 1u) {
          const unsigned long long k = (static_cast<unsigned long long>(iou_order(iou_overlaps(g, ag, an[e], area[e])))
                                        << 32) | (0xffffffffu - static_cast<unsigned>(n0 + e * kAtThreads));
          best = k > best ? k : best;
        }
      }
      best = warp_max_u64(best);
      if (lane == 0 && best != 0ull) atomicMax(&s_key[j], best);
    }
    __syncthreads();
    for (int j = threadIdx.x; j < nt; j += kAtThreads)
      if (s_key[j] != 0ull) atomicMax(&p.gt_key[im.gt_off + t0 + j], s_key[j]);
    __syncthreads();   // the tile is rewritten next
  }
}

// ---------------------------------------------------------------------------------------------------------------
// 2. assign: per-anchor max over the gts and MaxIoUAssigner's steps 2 to 4; each image's positive / negative counts
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kAtThreads) bags_at_assign_kernel(const __grid_constant__ AtParams p) {
  __shared__ float4 s_gt[kAtGtTile];
  __shared__ float s_area[kAtGtTile];
  __shared__ float s_max[kAtGtTile];   // the gt's max IoU; NaN when step 4 skips the gt
  __shared__ int s_arg[kAtGtTile];     // the gt's first anchor at that max
  __shared__ int s_cnt[2];
  const int img = blockIdx.y;
  const AtImage& im = p.img[img];
  const int n0 = blockIdx.x * kAtSpan + threadIdx.x;
  if (threadIdx.x < 2) s_cnt[threadIdx.x] = 0;
  float4 an[kAtPer];
  float area[kAtPer], best[kAtPer];
  int arg[kAtPer], last[kAtPer];
  unsigned in = 0u;
#pragma unroll
  for (int e = 0; e < kAtPer; ++e) {
    const int n = n0 + e * kAtThreads;
    bool inside = false;
    if (n < p.N) an[e] = anchor_at(p, im, n, inside);
    area[e] = inside ? area_plus1(an[e]) : 0.f;
    in |= inside ? 1u << e : 0u;
    best[e] = 0.f;
    arg[e] = 0;
    last[e] = -1;
  }
  const bool any = __syncthreads_or(in != 0u);
  if (any) {
    for (int t0 = 0; t0 < im.gt_cnt; t0 += kAtGtTile) {
      const int nt = min(kAtGtTile, im.gt_cnt - t0);
      for (int j = threadIdx.x; j < nt; j += kAtThreads) {
        const float4 g = p.gts[im.gt_off + t0 + j];
        const unsigned long long k = p.gt_key[im.gt_off + t0 + j];
        const float m = iou_of_order(static_cast<uint32_t>(k >> 32));
        s_gt[j] = g;
        s_area[j] = area_plus1(g);
        s_max[j] = m >= p.min_pos ? m : __int_as_float(0x7fc00000);
        s_arg[j] = static_cast<int>(0xffffffffu - static_cast<uint32_t>(k));
      }
      __syncthreads();
      for (int j = 0; j < nt; ++j) {
        const float4 g = s_gt[j];
        const float ag = s_area[j], gm = s_max[j];
        const int ga = s_arg[j], i = t0 + j;
#pragma unroll
        for (int e = 0; e < kAtPer; ++e) {
          if ((in >> e) & 1u) {
            const float v = iou_overlaps(g, ag, an[e], area[e]);
            if (i == 0 || (best[e] == best[e] && (v != v || v > best[e]))) {
              best[e] = v;
              arg[e] = i;
            }
            if (gm == gm && (p.assign_all ? v == gm : ga == n0 + e * kAtThreads)) last[e] = i;
          }
        }
      }
      __syncthreads();   // the tile is rewritten next
    }
  }
  int npos = 0, nneg = 0;
#pragma unroll
  for (int e = 0; e < kAtPer; ++e) {
    const int n = n0 + e * kAtThreads;
    if (n >= p.N) continue;
    int a = -2;
    if ((in >> e) & 1u) {
      const float m = best[e];
      a = -1;
      if (p.neg_on && m >= p.neg_lo && m < p.neg_hi) a = 0;
      if (m >= p.pos_thr) a = arg[e] + 1;
      if (last[e] >= 0) a = last[e] + 1;
      npos += a > 0;
      nneg += a == 0;
    }
    p.assign[static_cast<size_t>(img) * p.N + n] = a;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    npos += __shfl_xor_sync(0xffffffffu, npos, o);
    nneg += __shfl_xor_sync(0xffffffffu, nneg, o);
  }
  if ((threadIdx.x & 31) == 0 && (npos | nneg)) {
    atomicAdd(&s_cnt[0], npos);
    atomicAdd(&s_cnt[1], nneg);
  }
  __syncthreads();
  if (threadIdx.x < 2 && s_cnt[threadIdx.x]) atomicAdd(&p.counts[2 * img + threadIdx.x], s_cnt[threadIdx.x]);
}

// ---------------------------------------------------------------------------------------------------------------
// 3. select: the k smallest sampling keys of each image's positives and negatives, one cluster per gallery
// ---------------------------------------------------------------------------------------------------------------
// the sampler's k of gallery t (0 positives, 1 negatives) of an image with these counts (base_sampler.py:sample)
__device__ __forceinline__ int sample_count(const AtParams& p, int t, int npos, int nneg) {
  const int kpos = min(npos, p.exp_pos);
  if (t == 0) return kpos;
  int exp_neg = p.num - kpos;
  if (p.neg_pos_ub >= 0.0) {
    const double ub = p.neg_pos_ub * static_cast<double>(max(1, kpos));
    if (ub < static_cast<double>(exp_neg)) exp_neg = static_cast<int>(ub);
  }
  return min(nneg, max(exp_neg, 0));
}

__device__ __forceinline__ bool in_gallery(int a, int t) { return t == 0 ? a > 0 : a == 0; }

__global__ void __cluster_dims__(kAtCluster, 1, 1) __launch_bounds__(kAtSelectThreads)
bags_at_select_kernel(const __grid_constant__ AtParams p) {
  __shared__ unsigned hist[2][256];
  __shared__ unsigned tot[256];
  __shared__ unsigned s_digit, s_below, s_bucket;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = static_cast<int>(cluster.block_rank());
  const int seg = blockIdx.x / kAtCluster;
  const int img = seg >> 1, t = seg & 1;
  const int tid = threadIdx.x;
  const int npos = p.counts[2 * img], nneg = p.counts[2 * img + 1];
  const int k = sample_count(p, t, npos, nneg);
  const int count = t == 0 ? npos : nneg;
  unsigned long long thr = 0ull;
  if (k > 0 && k < count) {   // the cluster's CTAs all take this branch or none does
    const unsigned long long seed = effective_seed(p);
    const int* assign = p.assign + static_cast<size_t>(img) * p.N;
    const int chunk = (p.N + kAtCluster - 1) / kAtCluster;
    const int m0 = rank * chunk, m1 = min(p.N, m0 + chunk);
    unsigned long long prefix = 0ull;
    unsigned krem = static_cast<unsigned>(k);
    int shift = 56;
    for (int pass = 0; shift >= 0; shift -= 8, ++pass) {
      unsigned* h = hist[pass & 1];
      if (tid < 256) h[tid] = 0u;
      __syncthreads();
      for (int m = m0 + tid; m < m1; m += kAtSelectThreads) {
        if (!in_gallery(__ldg(assign + m), t)) continue;
        const unsigned long long key = anchor_key(seed, img, m);
        if (shift == 56 || (key >> (shift + 8)) == (prefix >> (shift + 8))) atomicAdd(&h[(key >> shift) & 255u], 1u);
      }
      cluster.sync();
      if (tid < 256) {
        unsigned c = 0u;
        for (int r = 0; r < kAtCluster; ++r) c += cluster.map_shared_rank(h, r)[tid];
        tot[tid] = c;
      }
      __syncthreads();
      if (tid < 32) {   // lane j: digits 8 j .. 8 j + 7, from the bottom
        unsigned s = 0u;
#pragma unroll
        for (int i = 0; i < 8; ++i) s += tot[8 * tid + i];
        unsigned x = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned y = __shfl_up_sync(0xffffffffu, x, o);
          if (tid >= o) x += y;
        }
        unsigned cum = x - s;
        if (cum < krem && krem <= x) {
          for (int i = 0; i < 8; ++i) {
            const unsigned c = tot[8 * tid + i];
            if (cum + c >= krem) {
              s_digit = 8u * tid + i;
              s_below = cum;
              s_bucket = c;
              break;
            }
            cum += c;
          }
        }
      }
      __syncthreads();
      krem -= s_below;
      prefix |= static_cast<unsigned long long>(s_digit) << shift;
      const bool done = s_bucket == krem;   // the whole bucket is taken (keys are distinct: always by the last digit)
      __syncthreads();                      // s_* are rewritten by the next pass
      if (done) break;
    }
    cluster.sync();   // no CTA leaves while another may still read its histograms
    thr = prefix | ((1ull << shift) - 1ull);   // keys <= thr are selected
  } else if (k > 0) {
    thr = ~0ull;   // the whole gallery
  }
  if (rank == 0 && tid == 0) {
    p.sel[2 * seg] = thr;
    p.sel[2 * seg + 1] = static_cast<unsigned long long>(k);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// 4. write the dense targets
// ---------------------------------------------------------------------------------------------------------------
// bbox2delta (mmdet/core/bbox/transforms.py) for one pair in torch's op sequence, then .sub_(means).div_(stds)
__device__ __forceinline__ float4 bbox2delta(const AtParams& p, float4 a, float4 g) {
  const float px = __fmul_rn(__fadd_rn(a.x, a.z), 0.5f), py = __fmul_rn(__fadd_rn(a.y, a.w), 0.5f);
  const float pw = __fadd_rn(__fsub_rn(a.z, a.x), 1.f), ph = __fadd_rn(__fsub_rn(a.w, a.y), 1.f);
  const float gx = __fmul_rn(__fadd_rn(g.x, g.z), 0.5f), gy = __fmul_rn(__fadd_rn(g.y, g.w), 0.5f);
  const float gw = __fadd_rn(__fsub_rn(g.z, g.x), 1.f), gh = __fadd_rn(__fsub_rn(g.w, g.y), 1.f);
  const float dx = __fdiv_rn(__fsub_rn(gx, px), pw), dy = __fdiv_rn(__fsub_rn(gy, py), ph);
  const float dw = logf(__fdiv_rn(gw, pw)), dh = logf(__fdiv_rn(gh, ph));
  return make_float4(__fdiv_rn(__fsub_rn(dx, p.means[0]), p.stds[0]), __fdiv_rn(__fsub_rn(dy, p.means[1]), p.stds[1]),
                     __fdiv_rn(__fsub_rn(dw, p.means[2]), p.stds[2]), __fdiv_rn(__fsub_rn(dh, p.means[3]), p.stds[3]));
}

__global__ void __launch_bounds__(kAtThreads) bags_at_write_kernel(const __grid_constant__ AtParams p) {
  const int img = blockIdx.y;
  const int n = blockIdx.x * kAtThreads + threadIdx.x;
  if (blockIdx.x == 0 && img == 0 && threadIdx.x == 0) {
    long long tp = 0, tn = 0;
    for (int b = 0; b < p.B; ++b) {
      tp += max(static_cast<long long>(p.sel[4 * b + 1]), 1ll);
      tn += max(static_cast<long long>(p.sel[4 * b + 3]), 1ll);
    }
    p.totals[0] = tp;
    p.totals[1] = tn;
    p.totals[2] = tp + tn;
  }
  if (n >= p.N) return;
  const size_t o = static_cast<size_t>(img) * p.N + n;
  const int a = p.assign[o];
  long long label = 0;
  float lw = 0.f;
  float4 tgt = make_float4(0.f, 0.f, 0.f, 0.f), bw = tgt;
  if (a >= 0) {
    const int t = a > 0 ? 0 : 1;
    const unsigned long long thr = p.sel[4 * img + 2 * t], k = p.sel[4 * img + 2 * t + 1];
    if (k > 0ull && anchor_key(effective_seed(p), img, n) <= thr) {
      lw = 1.f;
      if (a > 0) {
        bool inside;
        const float4 an = anchor_at(p, p.img[img], n, inside);
        tgt = bbox2delta(p, an, p.gts[p.img[img].gt_off + a - 1]);
        bw = make_float4(1.f, 1.f, 1.f, 1.f);
        label = 1;
        lw = p.pos_weight;
      }
    }
  }
  p.labels[o] = label;
  p.label_weights[o] = lw;
  p.bbox_targets[o] = tgt;
  p.bbox_weights[o] = bw;
}

static size_t align256(size_t x) { return (x + 255) & ~static_cast<size_t>(255); }

size_t anchor_target_layout(AtParams& p, int total_gts, void* scratch) {
  uint8_t* s = static_cast<uint8_t*>(scratch);
  size_t off = 0;
  auto take = [&](size_t bytes) -> void* {
    void* q = s ? s + off : nullptr;
    off += align256(bytes);
    return q;
  };
  p.counts = static_cast<int*>(take(static_cast<size_t>(p.B) * 2 * sizeof(int)));
  p.gt_key = static_cast<unsigned long long*>(take(static_cast<size_t>(total_gts) * 8));
  p.zero_bytes = off;
  p.sel = static_cast<unsigned long long*>(take(static_cast<size_t>(p.B) * 4 * 8));
  p.assign = static_cast<int*>(take(static_cast<size_t>(p.B) * p.N * sizeof(int)));
  return off;
}

cudaError_t launch_anchor_target(const AtParams& p, cudaStream_t stream) {
  cudaError_t e = cudaMemsetAsync(p.counts, 0, p.zero_bytes, stream);
  if (e != cudaSuccess) return e;
  const dim3 grid((p.N + kAtSpan - 1) / kAtSpan, p.B);
  bags_at_gt_max_kernel<<<grid, kAtThreads, 0, stream>>>(p);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  bags_at_assign_kernel<<<grid, kAtThreads, 0, stream>>>(p);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  bags_at_select_kernel<<<p.B * 2 * kAtCluster, kAtSelectThreads, 0, stream>>>(p);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  bags_at_write_kernel<<<dim3((p.N + kAtThreads - 1) / kAtThreads, p.B), kAtThreads, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace bags
