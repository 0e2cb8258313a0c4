// Kernels of the RPN proposal generation: see bags_rpn.cuh for what they compute.
#include <cooperative_groups.h>

#include "bags_anchor.cuh"
#include "bags_iou.cuh"
#include "bags_rpn.cuh"

namespace cg = cooperative_groups;

namespace bags {

// torch's addcmul(px, 1, pw, dx) on CUDA rounds px + pw * dx once (an fma), not twice as px + pw * dx in two torch
// ops would; tests/test_gpu_rpn.py pins this against torch.
constexpr bool kAddcmulFused = true;

constexpr int kRpnMaskThreads = 256;   // one 64-row x 256-column tile: thread = (row, column word)
constexpr int kRpnScanThreads = 256;   // warp 0 scans, warps 1..7 stage rows
constexpr int kRpnScanRows = 32;       // rows per staged chunk
constexpr int kRpnMergeThreads = 256;
constexpr int kRpnWords = kRpnMaxCand / 64;

__device__ __forceinline__ uint32_t score_order(float s) {   // monotone in s; NaN above every number
  const uint32_t b = __float_as_uint(s);
  return s != s ? 0xffffffffu : ((b & 0x80000000u) ? ~b : (b | 0x80000000u));
}

__device__ __forceinline__ float sigmoid_ref(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }

__device__ __forceinline__ float clamp_nan(float v, float lo, float hi) {   // torch.clamp: NaN passes through
  return v != v ? v : fminf(fmaxf(v, lo), hi);
}

__device__ __forceinline__ uint8_t* img_scratch(const RpnParams& p, int img) {
  return p.scratch + static_cast<size_t>(img) * p.img_bytes;
}

// candidate list of one segment: boxes [K], scores [K], flat indices [K]
struct RpnCand {
  float4* box;
  float* score;
  int* flat;
};

__device__ __forceinline__ RpnCand cand_of(const RpnParams& p, int img, const RpnLevel& L) {
  uint8_t* base = img_scratch(p, img) + L.cand_off;
  RpnCand c;
  c.box = reinterpret_cast<float4*>(base);
  c.score = reinterpret_cast<float*>(base + 16 * static_cast<size_t>(L.K));
  c.flat = reinterpret_cast<int*>(base + 20 * static_cast<size_t>(L.K));
  return c;
}

__device__ __forceinline__ float4* surv_box(const RpnParams& p, int img, const RpnLevel& L) {
  return reinterpret_cast<float4*>(img_scratch(p, img) + L.surv_off);
}
__device__ __forceinline__ float* surv_score(const RpnParams& p, int img, const RpnLevel& L) {
  return reinterpret_cast<float*>(img_scratch(p, img) + L.surv_off + 16 * static_cast<size_t>(L.post));
}

// 64-bit selection key of memory position m of a level: (score order, ~flat index), flat = (h W + w) A + a
__device__ __forceinline__ unsigned long long select_key(const float* logits, int m, int HW, int A) {
  const int a = m / HW, hw = m - a * HW;
  const uint32_t flat = static_cast<uint32_t>(hw) * static_cast<uint32_t>(A) + static_cast<uint32_t>(a);
  return (static_cast<unsigned long long>(score_order(sigmoid_ref(__ldg(logits + m)))) << 32) |
         static_cast<unsigned long long>(0xffffffffu - flat);
}

// delta2bbox (mmdet/core/bbox/transforms.py:34-111) on one anchor, one rounding per torch op
__device__ __forceinline__ float4 decode(const RpnParams& p, float4 an, float d0, float d1, float d2, float d3,
                                         float max_w, float max_h) {
  const float dx = __fadd_rn(__fmul_rn(d0, p.stds[0]), p.means[0]);
  const float dy = __fadd_rn(__fmul_rn(d1, p.stds[1]), p.means[1]);
  const float dw = clamp_nan(__fadd_rn(__fmul_rn(d2, p.stds[2]), p.means[2]), -p.max_ratio, p.max_ratio);
  const float dh = clamp_nan(__fadd_rn(__fmul_rn(d3, p.stds[3]), p.means[3]), -p.max_ratio, p.max_ratio);
  const float px = __fmul_rn(__fadd_rn(an.x, an.z), 0.5f), py = __fmul_rn(__fadd_rn(an.y, an.w), 0.5f);
  const float pw = __fadd_rn(__fsub_rn(an.z, an.x), 1.f), ph = __fadd_rn(__fsub_rn(an.w, an.y), 1.f);
  const float gw = __fmul_rn(pw, expf(dw)), gh = __fmul_rn(ph, expf(dh));
  const float gx = kAddcmulFused ? __fmaf_rn(pw, dx, px) : __fadd_rn(px, __fmul_rn(pw, dx));
  const float gy = kAddcmulFused ? __fmaf_rn(ph, dy, py) : __fadd_rn(py, __fmul_rn(ph, dy));
  const float hw_ = __fmul_rn(gw, 0.5f), hh = __fmul_rn(gh, 0.5f);
  float4 b;
  b.x = clamp_nan(__fadd_rn(__fsub_rn(gx, hw_), 0.5f), 0.f, max_w);
  b.y = clamp_nan(__fadd_rn(__fsub_rn(gy, hh), 0.5f), 0.f, max_h);
  b.z = clamp_nan(__fsub_rn(__fadd_rn(gx, hw_), 0.5f), 0.f, max_w);
  b.w = clamp_nan(__fsub_rn(__fadd_rn(gy, hh), 0.5f), 0.f, max_h);
  return b;
}

// exclusive prefix of `v` over the block (warp shuffles + one shared slot per warp); `total` gets the block's sum
template <int kThreads>
__device__ __forceinline__ int block_exclusive_scan(int v, int* warp_sums, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  int before = 0;
  total = 0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) {
    const int s = warp_sums[w];
    before += w < warp ? s : 0;
    total += s;
  }
  __syncthreads();
  return before + x - v;
}

// ---------------------------------------------------------------------------------------------------------------
// 1. select, sort, decode: one cluster per (image, level)
// ---------------------------------------------------------------------------------------------------------------
__global__ void __cluster_dims__(kRpnCluster, 1, 1) __launch_bounds__(kRpnSelectThreads)
bags_rpn_select_kernel(const __grid_constant__ RpnParams p) {
  __shared__ unsigned long long keys[kRpnMaxCand];   // the segment's selected keys (rank 0)
  __shared__ unsigned hist[2][256];
  __shared__ unsigned tot[256];
  __shared__ int warp_sums[kRpnSelectThreads / 32];
  __shared__ int s_count;
  __shared__ unsigned s_digit, s_above, s_bucket;

  cg::cluster_group cluster = cg::this_cluster();
  const int rank = static_cast<int>(cluster.block_rank());
  const int seg = blockIdx.x / kRpnCluster;
  const int img = seg / p.n_levels, l = seg - img * p.n_levels;
  const RpnLevel& L = p.lvl[l];
  const int tid = threadIdx.x;
  const int n = L.n, K = L.K, HW = L.H * L.W, A = L.A;
  const float* logits = L.logits + static_cast<size_t>(img) * n;
  const int chunk = (n + kRpnCluster - 1) / kRpnCluster;
  const int m0 = rank * chunk, m1 = min(n, m0 + chunk);

  if (tid == 0) s_count = 0;
  cluster.sync();   // every CTA of the cluster runs and rank 0's counter is zero before any remote access

  unsigned long long thr = 0ull;   // keys >= thr are selected
  if (L.select) {
    unsigned long long prefix = 0ull;
    unsigned krem = static_cast<unsigned>(K);
    for (int shift = 56, pass = 0; shift >= 0; shift -= 8, ++pass) {
      unsigned* h = hist[pass & 1];
      if (tid < 256) h[tid] = 0u;
      __syncthreads();
      for (int m = m0 + tid; m < m1; m += kRpnSelectThreads) {
        const unsigned long long key = select_key(logits, m, HW, A);
        if (shift == 56 || (key >> (shift + 8)) == (prefix >> (shift + 8)))
          atomicAdd(&h[(key >> shift) & 255u], 1u);
      }
      cluster.sync();
      if (tid < 256) {
        unsigned c = 0u;
        for (int r = 0; r < kRpnCluster; ++r) c += cluster.map_shared_rank(h, r)[tid];
        tot[tid] = c;
      }
      __syncthreads();
      if (tid < 32) {   // lane j: digits 255 - 8 j .. 248 - 8 j, from the top
        unsigned s = 0u;
#pragma unroll
        for (int i = 0; i < 8; ++i) s += tot[255 - 8 * tid - i];
        unsigned x = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned y = __shfl_up_sync(0xffffffffu, x, o);
          if (tid >= o) x += y;
        }
        unsigned cum = x - s;
        if (cum < krem && krem <= x) {
          for (int i = 0; i < 8; ++i) {
            const unsigned c = tot[255 - 8 * tid - i];
            if (cum + c >= krem) {
              s_digit = 255u - 8u * tid - i;
              s_above = cum;
              s_bucket = c;
              break;
            }
            cum += c;
          }
        }
      }
      __syncthreads();
      krem -= s_above;
      prefix |= static_cast<unsigned long long>(s_digit) << shift;
      const bool done = s_bucket == krem;   // the whole bucket is taken (keys are distinct: always by the last digit)
      __syncthreads();                      // s_* are rewritten by the next pass
      if (done) break;
    }
    thr = prefix;
  }
  unsigned long long* keys0 = cluster.map_shared_rank(keys, 0);
  int* count0 = cluster.map_shared_rank(&s_count, 0);
  for (int m = m0 + tid; m < m1; m += kRpnSelectThreads) {
    const unsigned long long key = select_key(logits, m, HW, A);
    if (key >= thr) keys0[atomicAdd(count0, 1)] = key;
  }
  cluster.sync();
  if (rank != 0) return;

  // rank 0: sort (score desc, flat asc) -- the keys are distinct; zero keys pad to a power of two and sort last
  int P = 1;
  while (P < K) P <<= 1;
  for (int i = K + tid; i < P; i += kRpnSelectThreads) keys[i] = 0ull;
  __syncthreads();
  for (int k = 2; k <= P; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < P; i += kRpnSelectThreads) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = keys[i], b = keys[ixj];
          if (((i & k) == 0) ? (a < b) : (a > b)) {
            keys[i] = b;
            keys[ixj] = a;
          }
        }
      }
      __syncthreads();
    }
  }

  // decode each candidate; min_bbox_size drops boxes in order (stable compaction over contiguous runs)
  constexpr int kPer = kRpnMaxCand / kRpnSelectThreads;
  const int per = (K + kRpnSelectThreads - 1) / kRpnSelectThreads;
  const int i0 = tid * per;
  const float* deltas = L.deltas + static_cast<size_t>(img) * 4 * n;
  const float max_w = static_cast<float>(p.img_w[img] - 1), max_h = static_cast<float>(p.img_h[img] - 1);
  float4 box[kPer];
  float score[kPer];
  int flat[kPer];
  unsigned ok = 0u;
  int nv = 0;
#pragma unroll
  for (int e = 0; e < kPer; ++e) {
    const int i = i0 + e;
    if (e < per && i < K) {
      const uint32_t f = 0xffffffffu - static_cast<uint32_t>(keys[i]);
      const int a = static_cast<int>(f % static_cast<uint32_t>(A)), hw = static_cast<int>(f / static_cast<uint32_t>(A));
      const int hy = hw / L.W, wx = hw - hy * L.W;
      const float4 an = grid_anchor(L.base[a], wx, hy, L.stride);
      const float* d = deltas + static_cast<size_t>(4 * a) * HW + hw;
      box[e] = decode(p, an, __ldg(d), __ldg(d + HW), __ldg(d + 2 * HW), __ldg(d + 3 * HW), max_w, max_h);
      score[e] = sigmoid_ref(__ldg(logits + static_cast<size_t>(a) * HW + hw));
      flat[e] = static_cast<int>(f);
      bool keep = true;
      if (p.min_bbox_size > 0.f) {
        const float w = __fadd_rn(__fsub_rn(box[e].z, box[e].x), 1.f);
        const float h = __fadd_rn(__fsub_rn(box[e].w, box[e].y), 1.f);
        keep = (w >= p.min_bbox_size) && (h >= p.min_bbox_size);
      }
      if (keep) {
        ok |= 1u << e;
        ++nv;
      }
    }
  }
  int total;
  int o = block_exclusive_scan<kRpnSelectThreads>(nv, warp_sums, total);
  const RpnCand c = cand_of(p, img, L);
#pragma unroll
  for (int e = 0; e < kPer; ++e) {
    if ((ok >> e) & 1u) {
      c.box[o] = box[e];
      c.score[o] = score[e];
      c.flat[o] = flat[e];
      ++o;
    }
  }
  if (tid == 0) p.counts_scratch[2 * seg] = total;
}

// ---------------------------------------------------------------------------------------------------------------
// 2. suppression bit matrix: bit j of mask[i][j / 64] set when j > i and IoU(i, j) > nms_thr
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kRpnMaskThreads) bags_rpn_mask_kernel(const __grid_constant__ RpnParams p) {
  __shared__ float4 rows[64];
  __shared__ float4 cols[256];
  const int img = blockIdx.x / p.tiles_per_img;
  const int t = blockIdx.x - img * p.tiles_per_img;
  int l = 0;
  while (l + 1 < p.n_levels && p.lvl[l + 1].tile0 <= t) ++l;
  const RpnLevel& L = p.lvl[l];
  const int seg = img * p.n_levels + l;
  const int words_k = (L.K + 63) >> 6;
  const int groups = (words_k + 3) >> 2;
  const int lt = t - L.tile0;
  const int rb = lt / groups, cgp = lt - rb * groups;
  const int cnt = p.counts_scratch[2 * seg];
  if (cgp * 4 + 3 < rb || rb * 64 >= cnt) return;   // below the diagonal, or past the candidates
  const RpnCand c = cand_of(p, img, L);
  const int tid = threadIdx.x;
  if (tid < 64 && rb * 64 + tid < cnt) rows[tid] = c.box[rb * 64 + tid];
  const int cbase = cgp * 256;
  if (cbase + tid < cnt) cols[tid] = c.box[cbase + tid];
  __syncthreads();
  const int r = tid & 63, cw = cgp * 4 + (tid >> 6);
  const int row = rb * 64 + r;
  const int words = (cnt + 63) >> 6;
  if (row >= cnt || cw < rb || cw >= words) return;
  const float4 bi = rows[r];
  unsigned long long bits = 0ull;
  const int j0 = cw * 64;
  const int jend = min(64, cnt - j0);
  for (int b = 0; b < jend; ++b) {
    const int j = j0 + b;
    if (j > row && iou_plus1(bi, cols[j - cbase]) > p.nms_thr) bits |= 1ull << b;
  }
  unsigned long long* mask = reinterpret_cast<unsigned long long*>(img_scratch(p, img) + L.mask_off);
  mask[static_cast<size_t>(row) * words_k + cw] = bits;
}

// ---------------------------------------------------------------------------------------------------------------
// 3. greedy scan, positions in the level's input order, first nms_post survivors
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kRpnScanThreads) bags_rpn_scan_kernel(const __grid_constant__ RpnParams p) {
  __shared__ unsigned long long buf[2][kRpnScanRows][kRpnWords];
  __shared__ unsigned long long kbits[kRpnWords];   // kept, by sorted position (selected) or flat index (not)
  __shared__ int wpre[kRpnWords];
  __shared__ int warp_sums[kRpnScanThreads / 32];
  const int seg = blockIdx.x;
  const int img = seg / p.n_levels, l = seg - img * p.n_levels;
  const RpnLevel& L = p.lvl[l];
  const int cnt = p.counts_scratch[2 * seg];
  const int words = (cnt + 63) >> 6, words_k = (L.K + 63) >> 6;
  const unsigned long long* mask =
      reinterpret_cast<const unsigned long long*>(img_scratch(p, img) + L.mask_off);
  const RpnCand c = cand_of(p, img, L);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int chunks = (cnt + kRpnScanRows - 1) / kRpnScanRows;

  auto stage = [&](int ch, int t0, int nt) {
    for (int idx = t0; idx < kRpnScanRows * kRpnWords; idx += nt) {
      const int r = idx / kRpnWords, w = idx - r * kRpnWords;
      const int row = ch * kRpnScanRows + r;
      if (row < cnt && w >= (row >> 6) && w < words) buf[ch & 1][r][w] = mask[static_cast<size_t>(row) * words_k + w];
    }
  };
  if (tid < kRpnWords) kbits[tid] = 0ull;
  if (chunks > 0) stage(0, tid, kRpnScanThreads);
  __syncthreads();
  unsigned long long rem0 = 0ull, rem1 = 0ull, kp0 = 0ull, kp1 = 0ull;   // lane holds words lane and lane + 32
  for (int ch = 0; ch < chunks; ++ch) {
    if (warp == 0) {
      const int rend = min(kRpnScanRows, cnt - ch * kRpnScanRows);
      for (int r = 0; r < rend; ++r) {
        const int i = ch * kRpnScanRows + r, wi = i >> 6;
        const unsigned long long word = __shfl_sync(0xffffffffu, wi >= 32 ? rem1 : rem0, wi & 31);
        if (((word >> (i & 63)) & 1ull) == 0ull) {
          const unsigned long long* rowp = buf[ch & 1][r];
          if (lane >= wi && lane < words) rem0 |= rowp[lane];
          if (lane + 32 >= wi && lane + 32 < words) rem1 |= rowp[lane + 32];
          if (lane == (wi & 31)) {
            if (wi >= 32) kp1 |= 1ull << (i & 63);
            else kp0 |= 1ull << (i & 63);
          }
        }
      }
    } else if (ch + 1 < chunks) {
      stage(ch + 1, tid - 32, kRpnScanThreads - 32);
    }
    __syncthreads();
  }
  if (!L.select) {   // survivors in anchor order: re-index the kept bits by flat index (< n <= kRpnMaxCand)
    __shared__ unsigned long long sorted_bits[kRpnWords];
    if (warp == 0) {
      sorted_bits[lane] = kp0;
      sorted_bits[lane + 32] = kp1;
    }
    __syncthreads();
    for (int i = tid; i < cnt; i += kRpnScanThreads)
      if ((sorted_bits[i >> 6] >> (i & 63)) & 1ull) {
        const int f = c.flat[i];
        atomicOr(&kbits[f >> 6], 1ull << (f & 63));
      }
  } else if (warp == 0) {
    kbits[lane] = kp0;
    kbits[lane + 32] = kp1;
  }
  __syncthreads();
  if (warp == 0) {   // exclusive popcount prefix over the 64 words
    const int a = __popcll(kbits[2 * lane]), b = __popcll(kbits[2 * lane + 1]);
    int x = a + b;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    wpre[2 * lane] = x - a - b;
    wpre[2 * lane + 1] = x - b;
  }
  __syncthreads();
  // candidate i (sorted order) survives when kept and its position in the input order is below nms_post
  const int per = (cnt + kRpnScanThreads - 1) / kRpnScanThreads;
  const int i0 = tid * per, i1 = min(cnt, i0 + per);
  auto survives = [&](int i) -> bool {
    const int x = L.select ? i : c.flat[i];
    if (!L.select && !((kbits[x >> 6] >> (x & 63)) & 1ull)) return false;
    if (L.select && !((kbits[i >> 6] >> (i & 63)) & 1ull)) return false;
    const int pos = wpre[x >> 6] + __popcll(kbits[x >> 6] & ((1ull << (x & 63)) - 1ull));
    return pos < p.nms_post;
  };
  int nv = 0;
  for (int i = i0; i < i1; ++i) nv += survives(i) ? 1 : 0;
  int total;
  int o = block_exclusive_scan<kRpnScanThreads>(nv, warp_sums, total);
  float4* sb = surv_box(p, img, L);
  float* ss = surv_score(p, img, L);
  for (int i = i0; i < i1; ++i)
    if (survives(i)) {
      sb[o] = c.box[i];
      ss[o] = c.score[i];
      ++o;
    }
  if (tid == 0) p.counts_scratch[2 * seg + 1] = total;
}

// ---------------------------------------------------------------------------------------------------------------
// 4. merge: rank of every survivor of an image by (score desc, level asc, position asc)
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int count_above(const float* s, int n, uint32_t key, bool or_equal) {
  int lo = 0, hi = n;   // s is sorted by score_order, descending
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const uint32_t k = score_order(s[mid]);
    if (k > key || (or_equal && k == key)) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(kRpnMergeThreads) bags_rpn_merge_kernel(const __grid_constant__ RpnParams p) {
  __shared__ int sc[kRpnMaxLevels];
  const int img = blockIdx.y;
  const int t = blockIdx.x * kRpnMergeThreads + threadIdx.x;
  if (threadIdx.x < p.n_levels) sc[threadIdx.x] = p.counts_scratch[2 * (img * p.n_levels + threadIdx.x) + 1];
  __syncthreads();
  int total = 0;
  for (int l = 0; l < p.n_levels; ++l) total += sc[l];
  const int count = min(p.max_num, total);
  float* out = p.out + static_cast<size_t>(img) * p.max_num * 5;
  if (t < p.surv_per_img) {
    int l = 0;
    while (l + 1 < p.n_levels && p.lvl[l + 1].surv0 <= t) ++l;
    const int i = t - p.lvl[l].surv0;
    if (i < sc[l]) {
      const float* s = surv_score(p, img, p.lvl[l]);
      const float score = s[i];
      const uint32_t key = score_order(score);
      int rank = i;
      for (int m = 0; m < p.n_levels; ++m)
        if (m != l) rank += count_above(surv_score(p, img, p.lvl[m]), sc[m], key, m < l);
      if (rank < p.max_num) {
        const float4 b = surv_box(p, img, p.lvl[l])[i];
        float* o = out + static_cast<size_t>(rank) * 5;
        o[0] = b.x;
        o[1] = b.y;
        o[2] = b.z;
        o[3] = b.w;
        o[4] = score;
      }
    }
  }
  if (t < p.max_num && t >= count) {
    float* o = out + static_cast<size_t>(t) * 5;
    o[0] = o[1] = o[2] = o[3] = o[4] = 0.f;
  }
  if (t == 0) p.counts[img] = count;
}

static size_t align256(size_t x) { return (x + 255) & ~static_cast<size_t>(255); }

size_t rpn_layout(RpnParams& p, void* scratch) {
  size_t off = 0;
  int tiles = 0, surv = 0;
  for (int l = 0; l < p.n_levels; ++l) {
    RpnLevel& L = p.lvl[l];
    const size_t K = static_cast<size_t>(L.K), words = (K + 63) / 64;
    L.post = L.K < p.nms_post ? L.K : p.nms_post;
    L.cand_off = off;
    off += align256(24 * K);
    L.mask_off = off;
    off += align256(K * words * 8);
    L.surv_off = off;
    off += align256(20 * static_cast<size_t>(L.post));
    L.tile0 = tiles;
    L.tiles = static_cast<int>(words * ((words + 3) / 4));
    tiles += L.tiles;
    L.surv0 = surv;
    surv += L.post;
  }
  p.img_bytes = off;
  p.tiles_per_img = tiles;
  p.surv_per_img = surv;
  const size_t head = align256(static_cast<size_t>(p.B) * p.n_levels * 2 * sizeof(int));
  p.counts_scratch = static_cast<int*>(scratch);
  p.scratch = scratch ? static_cast<uint8_t*>(scratch) + head : nullptr;
  return head + static_cast<size_t>(p.B) * off;
}

cudaError_t launch_rpn_proposals(const RpnParams& p, cudaStream_t stream) {
  const int segs = p.B * p.n_levels;
  bags_rpn_select_kernel<<<segs * kRpnCluster, kRpnSelectThreads, 0, stream>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  if (p.tiles_per_img > 0) {
    bags_rpn_mask_kernel<<<p.B * p.tiles_per_img, kRpnMaskThreads, 0, stream>>>(p);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
  }
  bags_rpn_scan_kernel<<<segs, kRpnScanThreads, 0, stream>>>(p);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  const int span = p.surv_per_img > p.max_num ? p.surv_per_img : p.max_num;
  bags_rpn_merge_kernel<<<dim3((span + kRpnMergeThreads - 1) / kRpnMergeThreads, p.B), kRpnMergeThreads, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace bags
