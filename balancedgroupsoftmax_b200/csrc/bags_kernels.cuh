// HBM-bound kernels of the BAGS head (everything that is not the fc_cls contraction):
//
//   group_ce_kernel      per-bin log-softmax / NLL over logit slices, per-bin loss,
//                        and the un-scaled logit gradient dz~ ("grad in forward")
//                        reference: gs_bbox_head_with0.py:91-112,134-171 ;
//                                   losses/cross_entropy_loss.py:9-19 ; losses/utils.py:26-53
//   sample_others_kernel device replacement of _sample_others (gs_bbox_head_with0.py:63-89):
//                        exact-k uniform subset of the "others" rows, no host sync
//   mask_avg_kernel      avg_g = max(sum_n w_g[n], 1)   (gs_bbox_head_with0.py:109)
//   merge_scores_kernel  test-time score merge (gs_bbox_head_with0.py:239-273)
//   cast kernels         fp32 -> bf16 operand staging
#pragma once
#include "bags_ptx.cuh"

namespace bags {

constexpr int kMaxG = 8;

struct GroupTable {
  int G;
  int start[kMaxG];
  int len[kMaxG];
};

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

// ----------------------------------------------------------------------------
// grouped softmax cross-entropy, forward + logit gradient
// ----------------------------------------------------------------------------
// One warp per RoI row, the row staged in shared memory (coalesced 16 B loads),
// then per bin: max -> exp/sum (exp written back to smem) -> loss; finally one
// vectorised pass writes dz~ = w/avg * (softmax - onehot) for every column.
//
//   z        [N, ldz] fp32 logits (ldz % 4 == 0, 16 B aligned rows)
//   labels   [N] int64 in [0, classes)
//   l2b      [G, classes] int32 : label -> in-bin label (0 = "others")
//   wmask    [G, N] uint8 0/1 sample weights, or nullptr (all ones)
//   avg      [G] fp32 normalisers (device), or nullptr (=> N)
//   loss     [G] fp32 out : sum_n w*(lse - z_t) / avg
//   lse      [N, G] fp32 out (optional)
//   dz       [N, ldd] bf16 (DZ_F32 = false) or fp32 (true), optional
//   colsum   [C] fp32, += sum_n dz~[n, c]  (optional; caller zeroes)
//   part     [gridDim.x, kMaxG] fp32 scratch ; counter: 1 uint32 (zero on entry, reset on exit)
template <int NV, bool DZ_F32, bool WF = false>   // WF: wmask points at fp32 weights (reweight head variant)
__global__ void __launch_bounds__(256)
group_ce_kernel(const float* __restrict__ z, long long ldz, const long long* __restrict__ labels,
                const int* __restrict__ l2b, int classes, GroupTable gt,
                const uint8_t* __restrict__ wmask, const float* __restrict__ avg, int N, int C,
                float* __restrict__ loss, float* __restrict__ lse, void* __restrict__ dz,
                long long ldd, float* __restrict__ colsum, float* __restrict__ part,
                unsigned int* __restrict__ counter) {
  extern __shared__ __align__(16) float smem_rows[];  // [8 warps][NV*128]
  __shared__ float s_scale[8][kMaxG];   // coef / sum   per (warp, bin) for the current row
  __shared__ float s_coef[8][kMaxG];    // w / avg
  __shared__ int s_tcol[8][kMaxG];      // absolute target column
  __shared__ float s_lacc[8][kMaxG];    // per-warp loss accumulators
  __shared__ float s_inv_avg[kMaxG];
  __shared__ bool s_last;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* row = smem_rows + warp * (NV * 128);
  const int nchunks = C >> 2;  // float4 chunks (C % 4 == 0 checked on host)

  if (threadIdx.x < kMaxG) {
    const int g = threadIdx.x;
    s_inv_avg[g] = (g < gt.G) ? 1.0f / (avg != nullptr ? __ldg(avg + g) : fmaxf((float)N, 1.0f)) : 0.f;
  }
  if (lane < kMaxG) s_lacc[warp][lane] = 0.f;

  // Row-invariant map: bin of float4 chunk (lane + 32 j); -1 = no bin, -2 = straddles a boundary.
  int gidx[NV];
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int c0 = 4 * (lane + 32 * j);
    int g0 = -1, g3 = -1;
    for (int g = 0; g < gt.G; ++g) {
      if (c0 >= gt.start[g] && c0 < gt.start[g] + gt.len[g]) g0 = g;
      if (c0 + 3 >= gt.start[g] && c0 + 3 < gt.start[g] + gt.len[g]) g3 = g;
    }
    gidx[j] = (g0 == g3) ? g0 : -2;
  }
  float csum[NV][4];
#pragma unroll
  for (int j = 0; j < NV; ++j) { csum[j][0] = csum[j][1] = csum[j][2] = csum[j][3] = 0.f; }
  __syncthreads();

  for (int n = blockIdx.x * 8 + warp; n < N; n += gridDim.x * 8) {
    // ---- stage the row (coalesced 16 B loads) ----
    const float4* zr = reinterpret_cast<const float4*>(z + (long long)n * ldz);
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int c = lane + 32 * j;
      if (c < nchunks) reinterpret_cast<float4*>(row)[c] = ldg_stream_f4(zr + c);
    }
    __syncwarp();
    const long long lab = __ldg(labels + n);
    const bool lab_ok = (lab >= 0 && lab < classes);

    for (int g = 0; g < gt.G; ++g) {
      const int s = gt.start[g], len = gt.len[g];
      int t = lab_ok ? __ldg(l2b + g * classes + (int)lab) : 0;
      t = (t >= 0 && t < len) ? t : 0;
      const float w = (wmask != nullptr) ? (WF ? __ldg(reinterpret_cast<const float*>(wmask) + (long long)g * N + n)
                                               : (float)__ldg(wmask + (long long)g * N + n))
                                         : 1.0f;
      // pass 1: max
      float m = -INFINITY;
#pragma unroll 4
      for (int i = lane; i < len; i += 32) m = fmaxf(m, row[s + i]);
      m = warp_max(m);
      const float zt = row[s + t];  // broadcast read, before pass 2 overwrites
      __syncwarp();
      // pass 2: e = exp(v - m) kept in smem, sum
      const float mb = m * kLog2e;
      float sum = 0.f;
#pragma unroll 4
      for (int i = lane; i < len; i += 32) {
        const float e = exp2f(fmaf(row[s + i], kLog2e, -mb));
        row[s + i] = e;
        sum += e;
      }
      sum = warp_sum(sum);
      const float lse_v = m + logf(sum);
      if (lane == 0) {
        if (lse != nullptr) lse[(long long)n * gt.G + g] = lse_v;
        s_lacc[warp][g] += w * (lse_v - zt);
        const float coef = w * s_inv_avg[g];
        s_coef[warp][g] = coef;
        s_scale[warp][g] = coef / sum;
        s_tcol[warp][g] = s + t;
      }
    }
    __syncwarp();

    // ---- pass 3: dz~ = w/avg * (softmax - onehot) for the whole row, vectorised ----
    if (dz != nullptr || colsum != nullptr) {
#pragma unroll
      for (int j = 0; j < NV; ++j) {
        const int c = lane + 32 * j;
        if (c < nchunks) {
          const float4 e4 = reinterpret_cast<const float4*>(row)[c];
          const float e[4] = {e4.x, e4.y, e4.z, e4.w};
          float d[4];
          const int gj = gidx[j];
          if (gj >= 0) {
            const float sc = s_scale[warp][gj], cf = s_coef[warp][gj];
            const int tq = s_tcol[warp][gj] - 4 * c;
#pragma unroll
            for (int q = 0; q < 4; ++q) d[q] = e[q] * sc - (q == tq ? cf : 0.f);
          } else {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const int col = 4 * c + q;
              float v = 0.f;
              if (gj == -2) {
                for (int g = 0; g < gt.G; ++g)
                  if (col >= gt.start[g] && col < gt.start[g] + gt.len[g])
                    v = e[q] * s_scale[warp][g] - (col == s_tcol[warp][g] ? s_coef[warp][g] : 0.f);
              }
              d[q] = v;
            }
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) csum[j][q] += d[q];
          if (dz != nullptr) {
            if (DZ_F32) {
              *reinterpret_cast<float4*>(reinterpret_cast<float*>(dz) + (long long)n * ldd + 4 * c) =
                  make_float4(d[0], d[1], d[2], d[3]);
            } else {
              uint2 o;
              o.x = pack_bf16x2(d[0], d[1]);
              o.y = pack_bf16x2(d[2], d[3]);
              *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(dz) + (long long)n * ldd + 4 * c) = o;
            }
          }
        }
      }
    }
    __syncwarp();
  }

  // ---- bias-gradient column sums: warp registers -> CTA reduction in smem (the row staging
  //      buffers are free now) -> ONE global reduction per column per CTA ----
  if (colsum != nullptr) {
    __syncthreads();
    float* red = smem_rows;  // [8][NV*128] : warp w owns its slice, no conflicts
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int c = lane + 32 * j;
      if (c < nchunks)
        reinterpret_cast<float4*>(red + warp * (NV * 128))[c] = make_float4(csum[j][0], csum[j][1], csum[j][2], csum[j][3]);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < nchunks; c += 256) {
      float4 a = reinterpret_cast<const float4*>(red)[c];
#pragma unroll
      for (int w = 1; w < 8; ++w) {
        const float4 b = reinterpret_cast<const float4*>(red + w * (NV * 128))[c];
        a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
      }
      red_add_v4_f32(colsum + 4 * c, a.x, a.y, a.z, a.w);
    }
  }

  // ---- per-bin loss: fixed-order two-level reduction (reproducible for a fixed grid) ----
  __syncthreads();
  if (threadIdx.x < kMaxG) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += s_lacc[w][threadIdx.x];
    part[blockIdx.x * kMaxG + threadIdx.x] = s;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int done = atomicAdd(counter, 1u);
    s_last = (done == gridDim.x - 1);
  }
  __syncthreads();
  if (s_last) {
    __threadfence();
    if (warp < gt.G) {
      const int g = warp;
      float s = 0.f;
      for (int b = lane; b < (int)gridDim.x; b += 32) s += __ldcg(part + b * kMaxG + g);
      s = warp_sum(s);
      if (lane == 0) loss[g] = s * s_inv_avg[g];
    }
    if (threadIdx.x == 0) *counter = 0u;
  }
}

// ----------------------------------------------------------------------------
// "others" sampler  (device replacement of np.random.choice on the host)
// ----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t mix32(uint32_t x) {  // murmur3 finaliser
  x ^= x >> 16; x *= 0x85ebca6bu; x ^= x >> 13; x *= 0xc2b2ae35u; x ^= x >> 16;
  return x;
}
__device__ __forceinline__ uint32_t sample_key(unsigned long long seed, int g, int n) {
  uint32_t h = mix32(static_cast<uint32_t>(seed) ^ 0x9e3779b9u);
  h = mix32(h ^ static_cast<uint32_t>(seed >> 32));
  h = mix32(h ^ (static_cast<uint32_t>(g) * 0x632be5abu + 0x7f4a7c15u));
  h = mix32(h ^ static_cast<uint32_t>(n));
  return h;
}

// One CTA (1024 threads) per bin.  Bin 0: all ones.  Bin g>=1:
//   F = #rows with in-bin label > 0 ; k = int(F * ratio) ; O = N - F
//   F == 0 -> w = 0 ; k >= O -> w = 1 ; else in-bin rows + the k "others" rows with
//   the smallest (random key, row index) pairs  (a uniform k-subset).
//   avg_g = max(sum w, 1).
// Rows are read from global memory ONCE: thread t keeps rows t, t+1024, ... (EPT of them) in
// registers as (is_other, key); N > 1024*EPT uses the EPT = 0 instantiation, which re-reads.
template <int EPT>
__global__ void __launch_bounds__(1024)
sample_others_kernel(const long long* __restrict__ labels, const int* __restrict__ l2b, int classes,
                     int G, int N, double ratio, unsigned long long seed,
                     uint8_t* __restrict__ wmask, float* __restrict__ avg,
                     const unsigned long long* __restrict__ seed_step = nullptr) {
  pdl_trigger();   // the fused forward's GEMM mainloop does not depend on the masks: let it start now
  // optional device-resident step counter (CUDA-graph replays: the by-value seed is frozen at capture time, the
  // counter is advanced by the caller between replays, by a kernel that is NOT this kernel's stream predecessor)
  if (seed_step != nullptr) seed += __ldg(seed_step) * 0x9E3779B97F4A7C15ull;
  const int g = blockIdx.x;
  const int tid = threadIdx.x;
  __shared__ int s_hist[256];
  __shared__ int s_warp[32];
  __shared__ int s_F;
  __shared__ uint32_t s_prefix;
  __shared__ int s_need;
  __shared__ int s_base;
  uint8_t* w = wmask + (long long)g * N;

  // PDL: all reads / selection work may overlap the previous kernel in the stream; pdl_wait() before the first
  // write guarantees that kernel (and, transitively, everything before it) no longer uses the output buffers.
  if (g == 0) {
    pdl_wait();
    for (int n = tid; n < N; n += 1024) w[n] = 1;
    if (tid == 0) avg[0] = fmaxf((float)N, 1.0f);
    return;
  }
  const int* map = l2b + g * classes;
  auto in_bin = [&](int n) -> bool {
    const long long lab = __ldg(labels + n);
    return (lab >= 0 && lab < classes) ? (__ldg(map + lab) > 0) : false;
  };
  constexpr int R = EPT > 0 ? EPT : 1;
  bool r_fg[R];
  uint32_t r_key[R];
  // ---- count in-bin rows (and cache them) ----
  int cnt = 0;
  if (EPT > 0) {
#pragma unroll
    for (int e = 0; e < R; ++e) {
      const int n = tid + e * 1024;
      r_fg[e] = (n < N) ? in_bin(n) : true;  // out-of-range slots behave like kept rows: never sampled
      r_key[e] = sample_key(seed, g, n);
      cnt += (n < N && r_fg[e]) ? 1 : 0;
    }
  } else {
    for (int n = tid; n < N; n += 1024) cnt += in_bin(n) ? 1 : 0;
  }
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  if ((tid & 31) == 0) s_warp[tid >> 5] = cnt;
  __syncthreads();
  if (tid < 32) {
    int v = s_warp[tid];
    v = __reduce_add_sync(0xffffffffu, v);
    if (tid == 0) s_F = v;
  }
  __syncthreads();
  const int F = s_F;
  const int O = N - F;
  const long long k_ll = (long long)((double)F * ratio);  // Python int(): truncation
  int mode;  // 0: zeros, 1: ones, 2: in-bin only, 3: sample
  if (F == 0) mode = 0;
  else if (k_ll >= (long long)O) mode = 1;
  else if (k_ll == 0) mode = 2;
  else mode = 3;
  const int k = (int)(k_ll < (long long)O ? k_ll : 0);
  if (mode != 3) pdl_wait();
  if (tid == 0 && mode != 3)
    avg[g] = (mode == 0) ? 1.0f : (mode == 1) ? fmaxf((float)N, 1.0f) : fmaxf((float)(F + k), 1.0f);
  if (mode != 3) {
    if (EPT > 0) {
#pragma unroll
      for (int e = 0; e < R; ++e) {
        const int n = tid + e * 1024;
        if (n < N) w[n] = (mode == 1) ? 1 : (mode == 0) ? 0 : (r_fg[e] ? 1 : 0);
      }
    } else {
      for (int n = tid; n < N; n += 1024) w[n] = (mode == 1) ? 1 : (mode == 0) ? 0 : (in_bin(n) ? 1 : 0);
    }
    return;
  }
  // ---- radix select: the k-th smallest key among "others" ----
  // after the loop: keys < prefix are all selected; `need` rows with key == prefix remain.
  uint32_t prefix = 0, mask = 0;
  int need = k;
  for (int shift = 24; shift >= 0; shift -= 8) {
    if (tid < 256) s_hist[tid] = 0;
    __syncthreads();
    if (EPT > 0) {
#pragma unroll
      for (int e = 0; e < R; ++e)
        if (!r_fg[e] && (r_key[e] & mask) == prefix) atomicAdd(&s_hist[(r_key[e] >> shift) & 255u], 1);
    } else {
      for (int n = tid; n < N; n += 1024) {
        if (!in_bin(n)) {
          const uint32_t key = sample_key(seed, g, n);
          if ((key & mask) == prefix) atomicAdd(&s_hist[(key >> shift) & 255u], 1);
        }
      }
    }
    __syncthreads();
    if (tid < 32) {
      // 256 bins -> 32 lanes x 8 bins: lane-local sums, warp inclusive scan, then the owning lane
      // walks its 8 bins.  Finds digit d with  count(< d) < need <= count(<= d).
      int c[8];
      int ls = 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) { c[i] = s_hist[tid * 8 + i]; ls += c[i]; }
      int incl = ls;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (tid >= o) incl += t;
      }
      const int excl = incl - ls;
      if (excl < need && need <= incl) {
        int acc = excl, d = tid * 8;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          if (acc + c[i] >= need) { d = tid * 8 + i; break; }
          acc += c[i];
        }
        s_prefix = prefix | (static_cast<uint32_t>(d) << shift);
        s_need = need - acc;
      }
    }
    __syncthreads();
    prefix = s_prefix;
    need = s_need;
    mask |= (0xFFu << shift);
  }
  // ---- write weights; ties on the threshold key broken by ascending row index ----
  pdl_wait();
  if (tid == 0) { s_base = 0; avg[g] = fmaxf((float)(F + k), 1.0f); }
  __syncthreads();
  const int rounds = (N + 1023) / 1024;
  for (int e = 0; e < rounds; ++e) {
    const int n = e * 1024 + tid;
    bool other = false, tie = false;
    uint32_t key = 0;
    if (n < N) {
      bool fg = true;
      if (EPT > 0) {
#pragma unroll
        for (int q = 0; q < R; ++q)
          if (q == e) { fg = r_fg[q]; key = r_key[q]; }
      } else {
        fg = in_bin(n);
        key = sample_key(seed, g, n);
      }
      other = !fg;
      tie = other && (key == prefix);
    }
    // block-wide exclusive rank of `tie` in row order
    const unsigned bal = __ballot_sync(0xffffffffu, tie);
    const int wrank = __popc(bal & ((1u << (tid & 31)) - 1u));
    if ((tid & 31) == 0) s_warp[tid >> 5] = __popc(bal);
    __syncthreads();
    const int cw = s_warp[tid & 31];
    const int woff = __reduce_add_sync(0xffffffffu, ((tid & 31) < (tid >> 5)) ? cw : 0);  // warps before mine
    const int tot = __reduce_add_sync(0xffffffffu, cw);
    const int rank = s_base + woff + wrank;
    if (n < N) {
      uint8_t wv;
      if (!other) wv = 1;
      else if (key < prefix) wv = 1;
      else if (tie && rank < need) wv = 1;
      else wv = 0;
      w[n] = wv;
    }
    __syncthreads();
    if (tid == 0) s_base += tot;
    __syncthreads();
  }
}

// Reweight head variant (gs_bbox_head_with0_reweight.py:57-85,101-109): the sampled 0/1 weight of every RoI is
// multiplied by a per-class weight looked up with the RoI's in-bin label (bin 0 keeps plain ones), and the
// normaliser becomes max(sum of the products, 1).  One CTA per bin.
//   cls_weight [G, wstride] fp32: row g holds the len_g weights of bin g (index 0 = "others"); row 0 is unused
__global__ void __launch_bounds__(256)
reweight_kernel(const long long* __restrict__ labels, const int* __restrict__ l2b, int classes, int N,
                const uint8_t* __restrict__ wmask, const float* __restrict__ cls_weight, int wstride,
                float* __restrict__ wfloat, float* __restrict__ avg) {
  const int g = blockIdx.x;
  __shared__ float s_part[8];
  float acc = 0.f;
  for (int n = threadIdx.x; n < N; n += 256) {
    float w = (wmask != nullptr) ? static_cast<float>(wmask[(long long)g * N + n]) : 1.0f;
    if (g > 0) {
      const long long lab = labels[n];
      int t = (lab >= 0 && lab < classes) ? l2b[g * classes + (int)lab] : 0;
      t = (t >= 0 && t < wstride) ? t : 0;
      w *= cls_weight[(long long)g * wstride + t];
    }
    wfloat[(long long)g * N + n] = w;
    acc += w;
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += s_part[i];
    avg[g] = fmaxf(t, 1.0f);
  }
}

// avg_g = max(sum_n w_g[n], 1) for caller-provided masks (parity mode)
__global__ void __launch_bounds__(256)
mask_avg_kernel(const uint8_t* __restrict__ wmask, int N, float* __restrict__ avg) {
  pdl_trigger();
  const int g = blockIdx.x;
  __shared__ int s_w[8];
  int c = 0;
  for (int n = threadIdx.x; n < N; n += 256) c += wmask[(long long)g * N + n];
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int i = 0; i < 8; ++i) t += s_w[i];
    pdl_wait();
    avg[g] = fmaxf((float)t, 1.0f);
  }
}

// ----------------------------------------------------------------------------
// test-time score merge
// ----------------------------------------------------------------------------
//   p_g = softmax(z[:, slice_g]) ; score[:,0] = p_0[:,0]
//   score[:, cls] = p_0[:,1] * p_g[:, j]  for the (g>=1, j>=1) column that maps to cls.
//   cls2col [classes] int32: logit column feeding class `cls` (cls2col[0] = start_0), -1 => 0.
template <int NV>
__global__ void __launch_bounds__(256)
merge_scores_kernel(const float* __restrict__ z, long long ldz, GroupTable gt,
                    const int* __restrict__ cls2col, int N, int C, int classes,
                    float* __restrict__ scores, long long lds) {
  extern __shared__ __align__(16) float smem_rows[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* row = smem_rows + warp * (NV * 128);
  const int nchunks = C >> 2;
  for (int n = blockIdx.x * 8 + warp; n < N; n += gridDim.x * 8) {
    const float4* zr = reinterpret_cast<const float4*>(z + (long long)n * ldz);
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int c = lane + 32 * j;
      if (c < nchunks) reinterpret_cast<float4*>(row)[c] = ldg_stream_f4(zr + c);
    }
    __syncwarp();
    float inv_sum[kMaxG];
#pragma unroll
    for (int g = 0; g < kMaxG; ++g) {
      inv_sum[g] = 0.f;
      if (g < gt.G) {
        const int s = gt.start[g], len = gt.len[g];
        float m = -INFINITY;
        for (int i = lane; i < len; i += 32) m = fmaxf(m, row[s + i]);
        m = warp_max(m);
        __syncwarp();
        float sum = 0.f;
        for (int i = lane; i < len; i += 32) {
          const float e = expf(row[s + i] - m);
          row[s + i] = e;
          sum += e;
        }
        sum = warp_sum(sum);
        inv_sum[g] = 1.0f / sum;
      }
    }
    __syncwarp();
    const float pfg = (gt.len[0] > 1) ? row[gt.start[0] + 1] * inv_sum[0] : 0.f;
    float* out = scores + (long long)n * lds;
    for (int cls = lane; cls < classes; cls += 32) {
      const int col = __ldg(cls2col + cls);
      float v = 0.f;
      if (col >= 0 && col < C) {
        float is = 0.f;
        int gsel = -1;
#pragma unroll
        for (int g = 0; g < kMaxG; ++g)
          if (g < gt.G && col >= gt.start[g] && col < gt.start[g] + gt.len[g]) { is = inv_sum[g]; gsel = g; }
        const float p = row[col] * is;
        v = (gsel == 0) ? p : pfg * p;
      }
      out[cls] = v;
    }
    __syncwarp();
  }
}

// ----------------------------------------------------------------------------
// backward preparation: everything the two backward GEMMs need that is not a GEMM, in ONE launch that the
// dW GEMM's mainloop overlaps (programmatic dependent launch):
//   (1) dW = 0                      (the dW GEMM reduces its split-K partials into it)
//   (2) W' = diag(gout[bin(row)]) W  (B operand of the dX GEMM when per-bin upstream gradients are given)
//   (3) colpart[t, c] = sum over row group t of dz[n, c]   (bias-gradient partials; the dW epilogue adds
//       the groups and applies gout)
// ----------------------------------------------------------------------------
struct BwdPrepParams {
  float* dW; long long lddw; int C, K;
  const void* w; void* wscr; long long ldw; const float* gout; GroupTable gt;
  const void* dz; long long ldd; int N; float* colpart; int ctiles;
  int z_ctas, s_ctas, c_ctas;   // CTA ranges of the three jobs (0 = job disabled)
  int skip_scale_if_uniform;    // the consumer reads W itself and scales its output when all gout[g] are equal
  long long* timing;            // debug timeline rows [0, 2048), one per CTA: start, wait returned, end; or nullptr
};

// all per-bin upstream gradients equal?  (then diag(gout) W == gout[0] W: no scaled copy of W is needed)
__device__ __forceinline__ bool gout_uniform(const float* gout, int G, float& g0) {
  g0 = __ldg(gout);
  bool u = true;
  for (int g = 1; g < G; ++g) u = u && (__ldg(gout + g) == g0);
  return u;
}

// One job of the backward preparation, executed by 256 threads (`tid` in [0,256)).  `b` indexes the job like a CTA
// of bwd_prep_kernel would; `s_part` is 2 KB of shared memory; BAR_ID < 0 synchronises with __syncthreads(),
// otherwise with the named barrier BAR_ID over 256 threads (used from inside the merged backward kernel).
template <bool F32, int BAR_ID>
__device__ __forceinline__ void bwd_prep_job(const BwdPrepParams& p, int b, int tid, float (*s_part)[64]) {
  if (b < p.z_ctas) {
    // ---- (1) zero dW ----
    const int vec_per_row = p.K >> 2;
    const long long total = static_cast<long long>(p.C) * vec_per_row;
    for (long long i = b * 256ll + tid; i < total; i += p.z_ctas * 256ll) {
      const int r = static_cast<int>(i / vec_per_row), c = static_cast<int>(i - static_cast<long long>(r) * vec_per_row);
      reinterpret_cast<float4*>(p.dW + static_cast<long long>(r) * p.lddw)[c] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  } else if (b < p.z_ctas + p.s_ctas) {
    // ---- (2) row-scaled copy of W: flat index space, four independent 16-byte loads in flight per thread ----
    constexpr int V = F32 ? 4 : 8;
    if (p.skip_scale_if_uniform) {
      float g0;
      if (gout_uniform(p.gout, p.gt.G, g0)) return;
    }
    const int vec_per_row = p.K / V;
    const long long total = static_cast<long long>(p.C) * vec_per_row;
    const long long stride = static_cast<long long>(p.s_ctas) * 256;
    const char* wsrc = reinterpret_cast<const char*>(p.w);
    char* wdst = reinterpret_cast<char*>(p.wscr);
    const long long row_bytes = p.ldw * (F32 ? 4 : 2);
    for (long long i0 = static_cast<long long>(b - p.z_ctas) * 256 + tid; i0 < total; i0 += 4 * stride) {
      uint4 raw[4];
      int rr[4], cc[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const long long i = i0 + u * stride;
        rr[u] = -1;
        if (i < total) {
          rr[u] = static_cast<int>(i / vec_per_row);
          cc[u] = static_cast<int>(i - static_cast<long long>(rr[u]) * vec_per_row);
          raw[u] = __ldg(reinterpret_cast<const uint4*>(wsrc + rr[u] * row_bytes) + cc[u]);
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (rr[u] < 0) continue;
        float sc = 0.f;
#pragma unroll
        for (int g = 0; g < kMaxG; ++g)
          if (g < p.gt.G && rr[u] >= p.gt.start[g] && rr[u] < p.gt.start[g] + p.gt.len[g]) sc = __ldg(p.gout + g);
        uint4 o;
        if (F32) {
          o.x = __float_as_uint(__uint_as_float(raw[u].x) * sc); o.y = __float_as_uint(__uint_as_float(raw[u].y) * sc);
          o.z = __float_as_uint(__uint_as_float(raw[u].z) * sc); o.w = __float_as_uint(__uint_as_float(raw[u].w) * sc);
        } else {
          const uint32_t in[4] = {raw[u].x, raw[u].y, raw[u].z, raw[u].w};
          uint32_t q4[4];
#pragma unroll
          for (int q = 0; q < 4; ++q)
            q4[q] = pack_bf16x2(__uint_as_float(in[q] << 16) * sc, __uint_as_float(in[q] & 0xffff0000u) * sc);
          o = make_uint4(q4[0], q4[1], q4[2], q4[3]);
        }
        reinterpret_cast<uint4*>(wdst + rr[u] * row_bytes)[cc[u]] = o;
      }
    }
  } else if (b < p.z_ctas + p.s_ctas + p.c_ctas) {
    // ---- (3) column sums of dz over one row group, one 64-column strip per job.  Thread t owns 8 columns
    // (t % 8) of rows (t / 8) + 32 i: 16-byte loads, 8 of them in flight per thread; padded columns of dz exist
    // up to ldd, columns beyond that read as zero.  bf16 rows have ldd % 8 == 0; fp32 rows only ldd % 4 == 0, so
    // an fp32 thread whose 8 columns straddle ldd reads the leading group of 4 alone ----
    const int ci = b - p.z_ctas - p.s_ctas;
    const int nstrips = (p.C + 63) / 64;
    const int strip = ci % nstrips, rg = ci / nstrips;
    const int rows_per_group = (p.N + p.ctiles - 1) / p.ctiles;
    const int r0 = rg * rows_per_group;
    const int r1 = (r0 + rows_per_group < p.N) ? r0 + rows_per_group : p.N;
    const int cgp = tid & 7, rl = tid >> 3;
    const int col = strip * 64 + cgp * 8;
    float acc[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[q] = 0.f;
    const bool second4 = col + 8 <= p.ldd;   // (F32: the upper 16 bytes of the thread's 8 columns)
    if (second4 || (F32 && col + 4 <= p.ldd)) {
      for (int rb = r0 + rl; rb < r1; rb += 32 * 8) {
        uint4 v[8], v2[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int r = rb + 32 * u;
          v[u] = make_uint4(0u, 0u, 0u, 0u);
          v2[u] = make_uint4(0u, 0u, 0u, 0u);
          if (r < r1) {
            if (F32) {
              const uint4* src = reinterpret_cast<const uint4*>(reinterpret_cast<const float*>(p.dz) + static_cast<long long>(r) * p.ldd + col);
              v[u] = __ldcg(src);
              if (second4) v2[u] = __ldcg(src + 1);
            } else {
              v[u] = __ldcg(reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.dz) + static_cast<long long>(r) * p.ldd + col));
            }
          }
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          if (F32) {
            acc[0] += __uint_as_float(v[u].x); acc[1] += __uint_as_float(v[u].y);
            acc[2] += __uint_as_float(v[u].z); acc[3] += __uint_as_float(v[u].w);
            acc[4] += __uint_as_float(v2[u].x); acc[5] += __uint_as_float(v2[u].y);
            acc[6] += __uint_as_float(v2[u].z); acc[7] += __uint_as_float(v2[u].w);
          } else {
            const uint32_t in[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              acc[2 * q] += __uint_as_float(in[q] << 16);
              acc[2 * q + 1] += __uint_as_float(in[q] & 0xffff0000u);
            }
          }
        }
      }
    }
    // 32 row-lanes per column: fold lanes l and l ^ 8, 16 (rows 1, 2 apart within the warp), then 8 warps via smem
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], 8);
      acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], 16);
    }
    const int warp = tid >> 5, lane = tid & 31;
    if (lane < 8) {
#pragma unroll
      for (int q = 0; q < 8; ++q) s_part[warp][lane * 8 + q] = acc[q];
    }
    if (BAR_ID < 0) __syncthreads();
    else asm volatile("bar.sync %0, 256;" ::"r"(BAR_ID) : "memory");
    if (tid < 64) {
      float t = 0.f;
#pragma unroll
      for (int w8 = 0; w8 < 8; ++w8) t += s_part[w8][tid];
      const int c = strip * 64 + tid;
      if (c < p.C) p.colpart[static_cast<long long>(rg) * p.C + c] = t;
    }
  }
}

template <bool F32>
__global__ void __launch_bounds__(256)
bwd_prep_kernel(const BwdPrepParams p) {
  __shared__ float s_part[8][64];
  long long* const tl = (p.timing != nullptr && threadIdx.x == 0 && blockIdx.x < 2048) ? p.timing + blockIdx.x * 8ll
                                                                                        : nullptr;
  if (tl != nullptr) tl[0] = global_timer_ns();
  pdl_wait();      // dz comes from the forward kernel; nothing before it may still be running either
  pdl_trigger();   // from here on the backward GEMMs may start: their mainloops only read dz, x and W
  if (tl != nullptr) tl[1] = global_timer_ns();
  bwd_prep_job<F32, -1>(p, blockIdx.x, threadIdx.x, s_part);
  if (tl != nullptr) tl[2] = global_timer_ns();
}

// ----------------------------------------------------------------------------
// fp32 -> bf16 staging (rows x cols, independent leading dims; cols % 4 == 0 fast path)
// ----------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
cast_bf16_kernel(const float* __restrict__ src, long long lds, __nv_bfloat16* __restrict__ dst,
                 long long ldd, int rows, int cols) {
  const int cv = cols >> 2;
  const long long total = (long long)rows * cv;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += gridDim.x * 256ll) {
    const int r = (int)(i / cv), c = (int)(i - (long long)r * cv);
    const float4 v = __ldg(reinterpret_cast<const float4*>(src + (long long)r * lds) + c);
    uint2 o;
    o.x = pack_bf16x2(v.x, v.y);
    o.y = pack_bf16x2(v.z, v.w);
    *reinterpret_cast<uint2*>(dst + (long long)r * ldd + 4 * c) = o;
  }
}

// Second pass of a split-K forward layer: out = act(ws + bias) in the output dtype (ws: fp32 sums of the split-K GEMM).
template <bool OUT_BF16>
__global__ void __launch_bounds__(256)
bias_act_store_kernel(const float* __restrict__ ws, long long ldws, const float* __restrict__ bias, void* __restrict__ out,
                      long long ldo, int rows, int cols, int relu) {
  const int qpr = (cols + 3) >> 2;   // float4 groups per row (the last may be partial)
  const long long quads = static_cast<long long>(rows) * qpr;
  for (long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; q < quads;
       q += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(q / qpr), c = static_cast<int>(q % qpr) * 4;
    const float4 v4 = *reinterpret_cast<const float4*>(ws + static_cast<long long>(r) * ldws + c);   // ldws % 4 == 0, padded
    float v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (bias != nullptr && c + e < cols) v[e] += __ldg(bias + c + e);
      if (relu) v[e] = fmaxf(v[e], 0.f);
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (c + e >= cols) break;
      if (OUT_BF16) reinterpret_cast<__nv_bfloat16*>(out)[static_cast<long long>(r) * ldo + c + e] = __float2bfloat16_rn(v[e]);
      else          reinterpret_cast<float*>(out)[static_cast<long long>(r) * ldo + c + e] = v[e];
    }
  }
}

// Backward of y = act(x W^T + b) up to the two contractions (shared FCs / fc_reg of the head's trunk,
// convfc_bbox_head.py:138-143,167): g = (y > 0 ? dy : 0) for a ReLU layer (y == nullptr: g = dy), cast to the GEMM
// operand dtype with a padded leading dimension.  HBM-bound elementwise pass: reads dy (+ y), writes g.
template <typename TDY, typename TY, bool OUT_BF16>
__global__ void __launch_bounds__(256)
act_bwd_kernel(const TDY* __restrict__ dy, long long lddy, const TY* __restrict__ y, long long ldy,
               void* __restrict__ g, long long ldg, int rows, int cols) {
  const long long quads = static_cast<long long>(rows) * (cols / 4);
  for (long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; q < quads;
       q += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(q / (cols / 4)), c = static_cast<int>(q % (cols / 4)) * 4;
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] = static_cast<float>(dy[static_cast<long long>(r) * lddy + c + e]);
    if (y != nullptr) {
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (!(static_cast<float>(y[static_cast<long long>(r) * ldy + c + e]) > 0.f)) v[e] = 0.f;
    }
    if (OUT_BF16) {
      uint2 o;
      o.x = pack_bf16x2(v[0], v[1]);
      o.y = pack_bf16x2(v[2], v[3]);
      *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(g) + static_cast<long long>(r) * ldg + c) = o;
    } else {
      *reinterpret_cast<float4*>(reinterpret_cast<float*>(g) + static_cast<long long>(r) * ldg + c) =
          make_float4(v[0], v[1], v[2], v[3]);
    }
  }
}

}  // namespace bags
