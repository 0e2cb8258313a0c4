// Kernels of the FPN RoI feature extractor: see bags_roi_align.cuh for what they compute.
#include "bags_roi_align.cuh"

namespace bags {

// one sample of one axis: corner indices, weights of lo (h) and hi (l), and whether it lies in [-1, size]
struct RoiAxis {
  int lo, hi;
  float l, h;
  int valid;
};

struct RoiHead {
  int level, batch, sh, sw, H, W;
  float start_h, start_w, bin_h, bin_w;
  const float* feat;
  float* grad;
};

__device__ __forceinline__ RoiAxis roi_axis(float start, float bin, int p, int i, int s, int size) {
  const float c = __fadd_rn(__fmaf_rn(static_cast<float>(p), bin, start),
                            __fdiv_rn(__fmul_rn(__fadd_rn(static_cast<float>(i), 0.5f), bin), static_cast<float>(s)));
  RoiAxis a;
  a.valid = !(c < -1.f || c > static_cast<float>(size));
  float v = c <= 0.f ? 0.f : c;
  a.lo = __float2int_rz(v);
  if (a.lo >= size - 1) {
    a.hi = a.lo = size - 1;
    v = static_cast<float>(a.lo);
  } else {
    a.hi = a.lo + 1;
  }
  a.l = __fsub_rn(v, static_cast<float>(a.lo));
  a.h = __fsub_rn(1.f, a.l);
  return a;
}

__device__ __forceinline__ int roi_level(const float* r, int n_levels, float inv_finest) {
  if (n_levels == 1) return 0;
  const float w = __fadd_rn(__fsub_rn(r[3], r[1]), 1.f);
  const float h = __fadd_rn(__fsub_rn(r[4], r[2]), 1.f);
  const float s = __fsqrt_rn(__fmul_rn(w, h));
  const float t = floorf(log2f(__fadd_rn(__fmul_rn(s, inv_finest), static_cast<float>(1e-6))));
  if (t != t) return -1;
  return t <= 0.f ? 0 : (t >= static_cast<float>(n_levels - 1) ? n_levels - 1 : static_cast<int>(t));
}

// the RoI's level, batch, start, bin size and samples per bin (level -1: the RoI gets a zero row / no gradient)
__device__ __forceinline__ RoiHead roi_head(const RoiAlignParams& p, int roi) {
  RoiHead hd{};
  hd.level = roi_level(p.rois_map + 5 * static_cast<size_t>(roi), p.n_levels, p.inv_finest);
  const float* r = p.rois + 5 * static_cast<size_t>(roi);
  hd.batch = __float2int_rz(r[0]);
  if (hd.level < 0) return hd;
  const RoiAlignLevel& L = p.lvl[hd.level];
  hd.H = L.H;
  hd.W = L.W;
  hd.feat = L.feat;
  hd.grad = L.grad;
  hd.start_w = __fmul_rn(r[1], L.scale);
  hd.start_h = __fmul_rn(r[2], L.scale);
  const float roi_w = fmaxf(__fmaf_rn(__fadd_rn(r[3], 1.f), L.scale, -hd.start_w), 0.f);
  const float roi_h = fmaxf(__fmaf_rn(__fadd_rn(r[4], 1.f), L.scale, -hd.start_h), 0.f);
  hd.bin_h = __fdiv_rn(roi_h, static_cast<float>(p.out_h));
  hd.bin_w = __fdiv_rn(roi_w, static_cast<float>(p.out_w));
  hd.sh = p.sample_num > 0 ? p.sample_num : __float2int_rz(ceilf(hd.bin_h));
  hd.sw = p.sample_num > 0 ? p.sample_num : __float2int_rz(ceilf(hd.bin_w));
  return hd;
}

__device__ __forceinline__ float roi_bilinear(const float* f, int W, const RoiAxis& y, const RoiAxis& x) {
  const float w1 = __fmul_rn(y.h, x.h), w2 = __fmul_rn(y.h, x.l), w3 = __fmul_rn(y.l, x.h), w4 = __fmul_rn(y.l, x.l);
  float v = __fmul_rn(w1, f[y.lo * W + x.lo]);
  v = __fmaf_rn(w2, f[y.lo * W + x.hi], v);
  v = __fmaf_rn(w3, f[y.hi * W + x.lo], v);
  return __fmaf_rn(w4, f[y.hi * W + x.hi], v);
}

// out[c, bin] for the chunk's channels; TAB: the samples come from the shared tables
template <bool TAB>
__device__ __forceinline__ void roi_pool_chunk(const RoiAlignParams& p, const RoiHead& hd, const RoiAxis* ys,
                                               const RoiAxis* xs, const float* fb, float* out, int nc) {
  const int ow = p.out_w, nbin = p.out_h * ow, sh = hd.sh, sw = hd.sw, W = hd.W;
  const size_t plane = static_cast<size_t>(hd.H) * W;
  const float cnt = static_cast<float>(sh * sw);
  for (int idx = threadIdx.x; idx < nc * nbin; idx += kRoiAlignThreads) {
    const int c = idx / nbin, bin = idx - c * nbin, ph = bin / ow, pw = bin - ph * ow;
    const float* f = fb + c * plane;
    float acc = 0.f;
    for (int iy = 0; iy < sh; ++iy) {
      const RoiAxis y = TAB ? ys[ph * sh + iy] : roi_axis(hd.start_h, hd.bin_h, ph, iy, sh, hd.H);
      for (int ix = 0; ix < sw; ++ix) {
        const RoiAxis x = TAB ? xs[pw * sw + ix] : roi_axis(hd.start_w, hd.bin_w, pw, ix, sw, W);
        acc = __fadd_rn(acc, (y.valid && x.valid) ? roi_bilinear(f, W, y, x) : 0.f);
      }
    }
    out[idx] = __fdiv_rn(acc, cnt);
  }
}

__device__ __forceinline__ bool roi_tabulated(const RoiAlignParams& p, const RoiHead& hd) {
  return static_cast<long long>(p.out_h) * hd.sh <= kRoiAlignMaxSamples &&
         static_cast<long long>(p.out_w) * hd.sw <= kRoiAlignMaxSamples;
}

__device__ __forceinline__ void roi_fill_tables(const RoiAlignParams& p, const RoiHead& hd, RoiAxis* ys, RoiAxis* xs) {
  const int ny = p.out_h * hd.sh, nx = p.out_w * hd.sw;
  for (int t = threadIdx.x; t < ny; t += kRoiAlignThreads)
    ys[t] = roi_axis(hd.start_h, hd.bin_h, t / hd.sh, t % hd.sh, hd.sh, hd.H);
  for (int t = threadIdx.x; t < nx; t += kRoiAlignThreads)
    xs[t] = roi_axis(hd.start_w, hd.bin_w, t / hd.sw, t % hd.sw, hd.sw, hd.W);
}

__global__ void __launch_bounds__(kRoiAlignThreads) bags_roi_align_fwd_kernel(const RoiAlignParams p) {
  __shared__ RoiAxis ys[kRoiAlignMaxSamples], xs[kRoiAlignMaxSamples];
  __shared__ RoiHead hd;
  const int roi = blockIdx.x, c0 = blockIdx.y * p.chunk, nc = min(p.chunk, p.C - c0);
  const int nbin = p.out_h * p.out_w;
  if (threadIdx.x == 0) {
    hd = roi_head(p, roi);
    if (p.levels && blockIdx.y == 0) p.levels[roi] = hd.level;
    if (hd.batch < 0 || hd.batch >= p.B) hd.level = -1;
  }
  __syncthreads();
  float* out = p.out + (static_cast<size_t>(roi) * p.C + c0) * nbin;
  if (hd.level < 0) {
    for (int i = threadIdx.x; i < nc * nbin; i += kRoiAlignThreads) out[i] = 0.f;
    return;
  }
  const float* fb = hd.feat + (static_cast<size_t>(hd.batch) * p.C + c0) * hd.H * hd.W;
  if (roi_tabulated(p, hd)) {
    roi_fill_tables(p, hd, ys, xs);
    __syncthreads();
    roi_pool_chunk<true>(p, hd, ys, xs, fb, out, nc);
  } else {
    roi_pool_chunk<false>(p, hd, ys, xs, fb, out, nc);
  }
}

// The distinct indices one axis's samples touch, ascending, each with the (bin, weight) pairs that reach it:
// slot 2t is sample t's lo corner (weight h), slot 2t + 1 its hi corner (weight l); samples outside [-1, size] touch
// nothing.  ent_* hold the pairs ordered by (index, slot); index d's pairs are ent[off[d], off[d + 1]).
struct RoiTouch {
  int less[2 * kRoiAlignMaxSamples];     // per slot: valid slots with a smaller index, or -1 for an invalid slot
  int first[2 * kRoiAlignMaxSamples];    // per slot: 1 when no earlier valid slot has its index
  int ent_bin[2 * kRoiAlignMaxSamples];
  float ent_w[2 * kRoiAlignMaxSamples];
  int val[2 * kRoiAlignMaxSamples];
  int off[2 * kRoiAlignMaxSamples + 1];
  int n;                                 // distinct indices
};

__device__ __forceinline__ int touch_index(const RoiAxis* a, int s) { return (s & 1) ? a[s >> 1].hi : a[s >> 1].lo; }

// phase 1 (after the tables are filled): per-slot counts
__device__ __forceinline__ void roi_touch_count(const RoiAxis* a, int n, int per_bin, RoiTouch& t) {
  for (int s = threadIdx.x; s < 2 * n; s += kRoiAlignThreads) {
    if (!a[s >> 1].valid) {
      t.less[s] = -1;
      t.first[s] = 0;
      continue;
    }
    const int v = touch_index(a, s);
    int less = 0, before = 0;
    for (int j = 0; j < 2 * n; ++j) {
      if (!a[j >> 1].valid) continue;
      const int u = touch_index(a, j);
      less += u < v;
      before += (u == v) & (j < s);
    }
    t.less[s] = less;
    t.first[s] = before == 0;
    t.ent_bin[less + before] = (s >> 1) / per_bin;
    t.ent_w[less + before] = (s & 1) ? a[s >> 1].l : a[s >> 1].h;
  }
}

// phase 2: the distinct indices and their offsets
__device__ __forceinline__ void roi_touch_index(const RoiAxis* a, int n, RoiTouch& t) {
  int nvalid = 0, nd = 0;
  for (int s = threadIdx.x; s < 2 * n; s += kRoiAlignThreads) {
    if (!t.first[s]) continue;
    const int v = touch_index(a, s);
    int d = 0;
    for (int j = 0; j < 2 * n; ++j) d += t.first[j] && touch_index(a, j) < v;
    t.val[d] = v;
    t.off[d] = t.less[s];
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < 2 * n; ++s) {
      nvalid += t.less[s] >= 0;
      nd += t.first[s];
    }
    t.n = nd;
    t.off[nd] = nvalid;
  }
}

__global__ void __launch_bounds__(kRoiAlignThreads) bags_roi_align_bwd_kernel(const RoiAlignParams p) {
  __shared__ RoiAxis ys[kRoiAlignMaxSamples], xs[kRoiAlignMaxSamples];
  __shared__ RoiTouch ty, tx;
  __shared__ float sg[kRoiAlignStage];
  __shared__ RoiHead hd;
  const int roi = blockIdx.x, c0 = blockIdx.y * p.chunk, nc = min(p.chunk, p.C - c0);
  const int ow = p.out_w, nbin = p.out_h * ow;
  if (threadIdx.x == 0) {
    hd = roi_head(p, roi);
    if (hd.batch < 0 || hd.batch >= p.B || (hd.level >= 0 && hd.grad == nullptr)) hd.level = -1;
  }
  __syncthreads();
  if (hd.level < 0) return;
  const int H = hd.H, W = hd.W, sh = hd.sh, sw = hd.sw;
  const float cnt = static_cast<float>(sh * sw);
  float* gb = hd.grad + (static_cast<size_t>(hd.batch) * p.C + c0) * H * W;
  const float* go = p.gout + (static_cast<size_t>(roi) * p.C + c0) * nbin;

  if (!roi_tabulated(p, hd)) {   // the reference's scatter: 4 corners per sample
    for (int idx = threadIdx.x; idx < nc * nbin; idx += kRoiAlignThreads) {
      const int c = idx / nbin, bin = idx - c * nbin, ph = bin / ow, pw = bin - ph * ow;
      const float g = go[idx];
      float* f = gb + static_cast<size_t>(c) * H * W;
      for (int iy = 0; iy < sh; ++iy) {
        const RoiAxis y = roi_axis(hd.start_h, hd.bin_h, ph, iy, sh, H);
        if (!y.valid) continue;
        for (int ix = 0; ix < sw; ++ix) {
          const RoiAxis x = roi_axis(hd.start_w, hd.bin_w, pw, ix, sw, W);
          if (!x.valid) continue;
          atomicAdd(f + y.lo * W + x.lo, __fdiv_rn(__fmul_rn(g, __fmul_rn(y.h, x.h)), cnt));
          atomicAdd(f + y.lo * W + x.hi, __fdiv_rn(__fmul_rn(g, __fmul_rn(y.h, x.l)), cnt));
          atomicAdd(f + y.hi * W + x.lo, __fdiv_rn(__fmul_rn(g, __fmul_rn(y.l, x.h)), cnt));
          atomicAdd(f + y.hi * W + x.hi, __fdiv_rn(__fmul_rn(g, __fmul_rn(y.l, x.l)), cnt));
        }
      }
    }
    return;
  }

  const int ny = p.out_h * sh, nx = ow * sw;
  roi_fill_tables(p, hd, ys, xs);
  for (int i = threadIdx.x; i < nc * nbin; i += kRoiAlignThreads) sg[i] = go[i];
  __syncthreads();
  roi_touch_count(ys, ny, sh, ty);
  roi_touch_count(xs, nx, sw, tx);
  __syncthreads();
  roi_touch_index(ys, ny, ty);
  roi_touch_index(xs, nx, tx);
  __syncthreads();
  const int nr = ty.n, nq = tx.n, npix = nr * nq;
  for (int idx = threadIdx.x; idx < nc * npix; idx += kRoiAlignThreads) {
    const int c = idx / npix, rem = idx - c * npix, r = rem / nq, q = rem - r * nq;
    const float* g = sg + c * nbin;
    float acc = 0.f;
    for (int e = ty.off[r]; e < ty.off[r + 1]; ++e) {
      const float* gr = g + ty.ent_bin[e] * ow;
      float s = 0.f;
      for (int f = tx.off[q]; f < tx.off[q + 1]; ++f) s = __fmaf_rn(tx.ent_w[f], gr[tx.ent_bin[f]], s);
      acc = __fmaf_rn(ty.ent_w[e], s, acc);
    }
    if (acc != 0.f)
      atomicAdd(gb + (static_cast<size_t>(c) * H + ty.val[r]) * W + tx.val[q], __fdiv_rn(acc, cnt));
  }
}

cudaError_t launch_roi_align_fwd(const RoiAlignParams& p, cudaStream_t stream) {
  bags_roi_align_fwd_kernel<<<dim3(p.k, (p.C + p.chunk - 1) / p.chunk), kRoiAlignThreads, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_roi_align_bwd(const RoiAlignParams& p, cudaStream_t stream) {
  bags_roi_align_bwd_kernel<<<dim3(p.k, (p.C + p.chunk - 1) / p.chunk), kRoiAlignThreads, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace bags
