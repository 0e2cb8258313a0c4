// Class-specific box regression fused with its SmoothL1 loss -- fc_reg restricted to the four columns a positive RoI's
// loss reads (bbox_head.py:118-128, smooth_l1_loss.py) instead of the [N, 4 * classes] GEMM:
//
//   bags_box_fwd_kernel  one warp per RoI: pred[n, j] = x[n] . W[4l + j] + b[4l + j] in fp32 for a positive RoI
//                        (0 < l = labels[n] < classes), SmoothL1 and its gradient g = w sl1'(d) / avg; every other
//                        row gets g = 0.  The loss is summed rows-in-order per warp, warps-in-order per CTA, and the
//                        CTA partials in a fixed tree by the last CTA to arrive.  The grid's last CTA builds the
//                        backward's class index meanwhile: a stable counting sort of the positives by class.
//   bags_box_bwd_kernel  one CTA per work unit.  Class units: dW rows 4c..4c+3 over one K slice (zero for a class
//                        without positives) and db, summing the class's positives in ascending RoI order.  RoI
//                        units: one K slice of dX[n] = g[n] W[4l..4l+3] (zero for a non-positive RoI).  No atomics:
//                        every output is bit-identical from run to run.
#pragma once
#include "bags_kernels.cuh"

namespace bags {

constexpr int kBoxThreads = 256;          // forward: 8 warps, one RoI per warp and step
constexpr int kBoxMaxClasses = 8192;      // the sort CTA keeps one int32 cursor per class in shared memory
constexpr int kBoxSortBatch = 4096;       // labels staged per batch of the stable placement (int16 each)
constexpr int kBoxBwdThreads = 128;       // backward: 4 consecutive k per thread
constexpr int kBoxSlice = 4 * kBoxBwdThreads;
constexpr int kBoxCounterWord = 16;       // the forward's arrival counter: word 16 of the workspace's counter line

struct BoxFwdParams {
  const void* x; long long ldx;           // [N, K] bf16 or fp32
  const float* w; long long ldw;          // [4 * classes, K] fp32
  const float* bias;                      // [4 * classes] or nullptr
  const long long* labels;                // [N]
  const float* targets; const float* weights;   // [N, 4]
  float beta, avg;
  int N, K, classes;
  float* loss;                            // [1]
  float* g;                               // [N, 4]
  float* pred;                            // [N, 4] or nullptr
  int* index;                             // [classes + 1] offsets, then [N] RoI ids sorted by class
  float* part;                            // [gridDim.x] CTA partials
  unsigned int* counter;                  // zero on entry, reset on exit
};

struct BoxBwdParams {
  const float* g; const float* gout;
  const void* x; long long ldx;
  const float* w; long long ldw;
  const long long* labels;
  const int* index;
  int N, K, classes, kslices, class_units;
  float* dW; long long lddw;
  float* db;
  void* dX; long long lddx;
};

template <bool BF16>
__device__ __forceinline__ float4 box_load4(const void* base, long long off) {
  if constexpr (BF16) {
    const uint2 u = __ldg(reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(base) + off));
    return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u), __uint_as_float(u.y << 16),
                       __uint_as_float(u.y & 0xffff0000u));
  } else {
    return __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + off));
  }
}

__device__ __forceinline__ bool box_positive(long long l, int classes) { return l > 0 && l < classes; }

// The label rules of the class index: a box loss reads the RoIs with 0 < l < classes, a mask loss every 0 <= l <
// classes (class-agnostic mask heads pass label 0 to their one channel).
struct BoxPositive {
  __device__ __forceinline__ bool operator()(long long l, int classes) const { return box_positive(l, classes); }
};
struct MaskLabelValid {
  __device__ __forceinline__ bool operator()(long long l, int classes) const { return l >= 0 && l < classes; }
};

// The class index of the RoIs whose label passes ``Valid``: offsets[c] = #such RoIs of classes < c (offsets[classes]
// = all of them) and, after the offsets, those RoIs ordered by class and, inside a class, by ascending RoI id.  Run by
// one CTA of kBoxThreads.
template <class Valid>
__device__ __forceinline__ void box_class_sort(const long long* labels, int N, int classes, int* index, int* s_cursor,
                                               short* s_lab, int* s_scan) {
  const Valid valid;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  int* offsets = index;
  int* rois = index + classes + 1;
  for (int c = tid; c < classes; c += kBoxThreads) s_cursor[c] = 0;
  __syncthreads();
  for (int n = tid; n < N; n += kBoxThreads) {
    const long long l = __ldg(labels + n);
    if (valid(l, classes)) atomicAdd(s_cursor + l, 1);
  }
  __syncthreads();
  // exclusive scan: thread t owns the contiguous class run [t * per, (t + 1) * per)
  const int per = (classes + kBoxThreads - 1) / kBoxThreads;
  const int lo = min(tid * per, classes), hi = min(lo + per, classes);
  int own = 0;
  for (int c = lo; c < hi; ++c) own += s_cursor[c];
  int incl = own;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) s_scan[warp] = incl;
  __syncthreads();
  int run = incl - own;
  for (int w = 0; w < warp; ++w) run += s_scan[w];
  __syncthreads();
  for (int c = lo; c < hi; ++c) {
    const int cnt = s_cursor[c];
    offsets[c] = run;
    s_cursor[c] = run;
    run += cnt;
  }
  if (tid == kBoxThreads - 1) offsets[classes] = run;
  __syncthreads();
  // stable placement: one warp walks the RoIs in order, 32 at a time; lanes with the same class take consecutive
  // slots in lane order
  for (int base = 0; base < N; base += kBoxSortBatch) {
    const int m = min(kBoxSortBatch, N - base);
    for (int i = tid; i < m; i += kBoxThreads) {
      const long long l = __ldg(labels + base + i);
      s_lab[i] = valid(l, classes) ? static_cast<short>(l) : static_cast<short>(-1);
    }
    __syncthreads();
    if (warp == 0) {
      for (int i0 = 0; i0 < m; i0 += 32) {
        const int i = i0 + lane;
        const int l = i < m ? s_lab[i] : -1;
        const unsigned peers = __match_any_sync(0xffffffffu, l);
        int cur = 0;
        if (l >= 0) {
          cur = s_cursor[l];
          rois[cur + __popc(peers & ((1u << lane) - 1u))] = base + i;
        }
        __syncwarp();
        if (l >= 0 && lane == 31 - __clz(peers)) s_cursor[l] = cur + __popc(peers);
        __syncwarp();
      }
    }
    __syncthreads();
  }
}

template <bool BF16>
__global__ void __launch_bounds__(kBoxThreads)
bags_box_fwd_kernel(const BoxFwdParams p) {
  __shared__ int s_cursor[kBoxMaxClasses];
  __shared__ short s_lab[kBoxSortBatch];
  __shared__ int s_scan[kBoxThreads / 32];
  __shared__ float s_warp[kBoxThreads / 32];
  __shared__ unsigned int s_last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float mine = 0.f;   // lane 0: this warp's rows, in ascending order
  if (blockIdx.x == gridDim.x - 1) {
    box_class_sort<BoxPositive>(p.labels, p.N, p.classes, p.index, s_cursor, s_lab, s_scan);
  } else {
    const int stride = (gridDim.x - 1) * (kBoxThreads / 32);
    const float inv_avg = 1.f / p.avg;
    for (int n = blockIdx.x * (kBoxThreads / 32) + warp; n < p.N; n += stride) {
      const long long l = __ldg(p.labels + n);
      float4 gv = make_float4(0.f, 0.f, 0.f, 0.f), pv = gv;
      if (box_positive(l, p.classes)) {   // warp-uniform
        const float* w0 = p.w + 4 * l * p.ldw;
        const long long xo = static_cast<long long>(n) * p.ldx;
        float a[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 2
        for (int k = 4 * lane; k < p.K; k += 128) {
          const float4 xv = box_load4<BF16>(p.x, xo + k);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float4 r = __ldg(reinterpret_cast<const float4*>(w0 + j * p.ldw + k));
            a[j] = fmaf(xv.x, r.x, a[j]);
            a[j] = fmaf(xv.y, r.y, a[j]);
            a[j] = fmaf(xv.z, r.z, a[j]);
            a[j] = fmaf(xv.w, r.w, a[j]);
          }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) a[j] = warp_sum(a[j]);
        if (lane == 0) {
          const float4 t = __ldg(reinterpret_cast<const float4*>(p.targets) + n);
          const float4 wt = __ldg(reinterpret_cast<const float4*>(p.weights) + n);
          const float tj[4] = {t.x, t.y, t.z, t.w}, wj[4] = {wt.x, wt.y, wt.z, wt.w};
          float pj[4], gj[4], row = 0.f;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            pj[j] = a[j] + (p.bias != nullptr ? __ldg(p.bias + 4 * l + j) : 0.f);
            const float d = pj[j] - tj[j];
            const float ad = fabsf(d);
            // torch.where(diff < beta, 0.5 * diff * diff / beta, diff - 0.5 * beta) and the gradient autograd gives
            // it: d / beta inside (abs'(0) = 0), sign(d) from |d| == beta on
            const bool quad = ad < p.beta;
            row += wj[j] * (quad ? 0.5f * ad * ad / p.beta : ad - 0.5f * p.beta);
            gj[j] = (wj[j] * inv_avg) * (quad ? d / p.beta : copysignf(1.f, d));
          }
          mine += row;
          gv = make_float4(gj[0], gj[1], gj[2], gj[3]);
          pv = make_float4(pj[0], pj[1], pj[2], pj[3]);
        }
      }
      if (lane == 0) {
        reinterpret_cast<float4*>(p.g)[n] = gv;
        if (p.pred != nullptr) reinterpret_cast<float4*>(p.pred)[n] = pv;
      }
    }
  }
  // loss: warps in order, then CTA partials in a fixed order by the last CTA to arrive
  if (lane == 0) s_warp[warp] = mine;
  __syncthreads();
  if (threadIdx.x == 0) {
    float cta = 0.f;
    for (int w = 0; w < kBoxThreads / 32; ++w) cta += s_warp[w];
    p.part[blockIdx.x] = cta;
    __threadfence();
    s_last = (atomicAdd(p.counter, 1u) == gridDim.x - 1) ? 1u : 0u;
  }
  __syncthreads();
  if (s_last == 0u) return;
  __threadfence();
  float v = 0.f;
  for (int i = threadIdx.x; i < static_cast<int>(gridDim.x); i += kBoxThreads) v += __ldcg(p.part + i);
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) s_warp[warp] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    float total = 0.f;
    for (int w = 0; w < kBoxThreads / 32; ++w) total += s_warp[w];
    *p.loss = p.N > 0 ? total / p.avg : 0.f;
    *p.counter = 0u;
  }
}

template <bool BF16>
__global__ void __launch_bounds__(kBoxBwdThreads)
bags_box_bwd_kernel(const BoxBwdParams p) {
  const float go = p.gout != nullptr ? __ldg(p.gout) : 1.f;
  const float4* g4 = reinterpret_cast<const float4*>(p.g);
  int u = blockIdx.x;
  if (u < p.class_units) {
    const int c = p.dW != nullptr ? u / p.kslices : u;
    const int s = p.dW != nullptr ? u % p.kslices : 0;
    const int lo = __ldg(p.index + c), hi = __ldg(p.index + c + 1);
    const int* rois = p.index + p.classes + 1;
    if (p.dW != nullptr) {
      const int k = s * kBoxSlice + 4 * threadIdx.x;
      if (k < p.K) {
        float4 a[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) a[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int i = lo; i < hi; ++i) {
          const int n = __ldg(rois + i);
          const float4 gv = __ldg(g4 + n);
          const float4 xv = box_load4<BF16>(p.x, static_cast<long long>(n) * p.ldx + k);
          const float gj[4] = {gv.x * go, gv.y * go, gv.z * go, gv.w * go};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            a[j].x = fmaf(gj[j], xv.x, a[j].x);
            a[j].y = fmaf(gj[j], xv.y, a[j].y);
            a[j].z = fmaf(gj[j], xv.z, a[j].z);
            a[j].w = fmaf(gj[j], xv.w, a[j].w);
          }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j)
          *reinterpret_cast<float4*>(p.dW + (4LL * c + j) * p.lddw + k) = a[j];
      }
    }
    if (p.db != nullptr && s == 0 && threadIdx.x < 4) {
      float acc = 0.f;
      for (int i = lo; i < hi; ++i) acc += __ldg(p.g + 4LL * __ldg(rois + i) + threadIdx.x) * go;
      p.db[4 * c + threadIdx.x] = acc;
    }
    return;
  }
  u -= p.class_units;
  const int n = u / p.kslices;
  const int k = (u % p.kslices) * kBoxSlice + 4 * threadIdx.x;
  if (k >= p.K) return;
  const long long l = __ldg(p.labels + n);
  float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
  if (box_positive(l, p.classes)) {
    const float4 gv = __ldg(g4 + n);
    const float gj[4] = {gv.x * go, gv.y * go, gv.z * go, gv.w * go};
    const float* w0 = p.w + 4 * l * p.ldw + k;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float4 r = __ldg(reinterpret_cast<const float4*>(w0 + j * p.ldw));
      o.x = fmaf(gj[j], r.x, o.x);
      o.y = fmaf(gj[j], r.y, o.y);
      o.z = fmaf(gj[j], r.z, o.z);
      o.w = fmaf(gj[j], r.w, o.w);
    }
  }
  const long long off = static_cast<long long>(n) * p.lddx + k;
  if constexpr (BF16) {
    uint2 q;
    q.x = pack_bf16x2(o.x, o.y);
    q.y = pack_bf16x2(o.z, o.w);
    *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(p.dX) + off) = q;
  } else {
    *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.dX) + off) = o;
  }
}

}  // namespace bags
