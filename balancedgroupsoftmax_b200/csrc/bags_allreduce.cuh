// Gradient exchange of the fc_cls bucket over NVLink peer memory (sm_90a, NVSwitch).
//
// Replaces the reference's NCCL all-reduce + div of the flattened gradients
// (mmdet/core/utils/dist_utils.py:9-41: _allreduce_coalesced -> dist.all_reduce, tensor.div_(world_size),
// copy back) by ONE kernel working directly on the ranks' gradient buckets, which live in symmetric
// (peer-mapped) memory:
//
//   barrier (all ranks' local dW / db are complete)            epoch flag words in the peers' buffers, sys scope
//   two-shot exchange: rank r owns vectors [r*chunk, (r+1)*chunk)
//       NVLS   : multimem.ld_reduce.add.v4.f32 on the multicast address (the switch sums the N copies)
//                -> * scale -> multimem.st.v4.f32 (the switch broadcasts to the N copies)
//       peer   : ld.relaxed.sys.v4 from each rank's copy in rank order -> * scale -> st to each rank's copy
//   barrier (every rank's slice has landed everywhere)
//
// Each element is reduced by exactly one rank in a fixed order, so all ranks end with bit-identical buckets.
// 5.07 MB per head: 2 * (N-1)/N * 5.07 MB cross each GPU's links plus two flag round trips.
//
// Flags (inside every rank's bucket allocation, zeroed once by the caller):
//   slot[b][r]  written by rank r's block b with an EPOCH number (fire and forget: st.relaxed.sys at the first barrier,
//               st.release.sys at the second), polled locally by this rank's block b (ld.relaxed.sys until it
//               reaches the expected epoch, then one ld.acquire.sys);
//   epoch[b]    this rank's block b's own count of barriers so far (all ranks run the same launches, so they agree);
//   status      set to 1 when a wait timed out (bounded in time; the kernel then traps -- see rank_barrier).
// Epochs only grow, so nothing is reset and CUDA-graph replays need no host work; a sender may be one barrier ahead
// of a slow receiver, hence the >= comparison (on the wrapped difference).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "bags_ptx.cuh"

namespace bags {

constexpr int kMaxRanks = 16;
// Small blocks with few registers: an exchange block fits on an SM next to a GEMM CTA of this library (48-55 K
// registers), so an exchange launched on a side stream really overlaps the next step's kernels.
constexpr int kArMaxBlocks = 320;
constexpr int kArThreads = 256;

struct AllReduceParams {
  float* peer[kMaxRanks];   // this process's mapping of every rank's bucket (peer[rank] is the local one)
  float* mc;                // multicast mapping of the bucket (NVLS) or nullptr
  long long flag_off;       // byte offset of the flag words inside the bucket allocation
  long long count;          // floats to reduce (multiple of 4), starting at the bucket base
  int rank, world;
  float scale;              // 1/world for the mean (dist_utils.py:23), 1 for a sum
  long long timeout_ns;     // how long a rank barrier waits for a missing peer before it gives up
  int trap_on_timeout;      // 1: a peer that never arrives kills the kernel (__trap: sticky error, the process fails
                            //    loudly -- NCCL would hang); 0 (construction-time self test only): set the status word,
                            //    skip the exchange and let the host fall back to NCCL
  long long* timing;        // debug timeline [grid][8] (%globaltimer) or nullptr
};

__device__ __forceinline__ void st_release_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_relaxed_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ float4 ld_relaxed_sys_f4(const float* p) {
  float4 v;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_sys_f4(float* p, const float4 v) {
  asm volatile("st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
               ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float4 multimem_ld_reduce_f4(const float* mc) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(mc) : "memory");
  return v;
}
__device__ __forceinline__ void multimem_st_f4(float* mc, const float4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
               ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// Block-level barrier across ranks: block b of every rank meets block b of every other rank.
// Thread t < world publishes `epoch` in rank t's slot for (block, this rank) and polls its own slot for (block, t).
// Preceded / followed by __syncthreads() so that the release store / acquire fence of the signalling threads order
// the whole block's accesses (PTX memory model: cumulativity through the CTA barrier).
// A rank that never shows up does not hang the device for ever: after `timeout_ns` (default 30 s, generous against
// checkpoint / evaluation hooks and data-loader stalls on some ranks) the block records the failure in the status word and
// TRAPS -- the process dies with a sticky CUDA error instead of training on un-averaged gradients.  Only the
// construction-time self test runs in the soft mode (status word, no exchange, host falls back to NCCL).
__device__ __forceinline__ uint32_t* ar_flags(const AllReduceParams& p, int rank) {
  return reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(p.peer[rank]) + p.flag_off);
}
// The FIRST barrier's flag store is relaxed: the data it publishes was written by the preceding kernel and is in L2,
// the point of coherence peers read through, so no system-scope release is needed.  The second one releases this
// block's peer stores.  Polling is relaxed, with one acquire load once the epoch has arrived.
__device__ __forceinline__ bool rank_barrier(const AllReduceParams& p, uint32_t epoch, int* s_fail, bool first = false) {
  __syncthreads();
  if (threadIdx.x < static_cast<unsigned>(p.world)) {
    const int t = static_cast<int>(threadIdx.x);
    uint32_t* theirs = ar_flags(p, t) + blockIdx.x * p.world + p.rank;
    uint32_t* mine = ar_flags(p, p.rank) + blockIdx.x * p.world + t;
    uint32_t spins = 0;
    long long t0 = 0;
    bool ok = true;
    // the clock is only consulted every 1024 probes: the common case (peers arrive within microseconds) never reads it
    auto expired = [&]() -> bool {
      if ((++spins & 1023u) != 0u) return false;
      const long long now = global_timer_ns();
      if (t0 == 0) { t0 = now; return false; }
      return now - t0 > p.timeout_ns;
    };
    if (first) st_relaxed_sys_u32(theirs, epoch);
    else       st_release_sys_u32(theirs, epoch);
    while (static_cast<int32_t>(ld_relaxed_sys_u32(mine) - epoch) < 0) {
      if (expired()) { ok = false; break; }
    }
    if (ok) {
      (void)ld_acquire_sys_u32(mine);
    } else {
      *s_fail = 1;
      atomicExch(ar_flags(p, p.rank) + kArMaxBlocks * p.world + kArMaxBlocks, 1u);
      if (p.trap_on_timeout) {
        // Never hand un-averaged gradients back to a host that proceeds as if they were exchanged
        // (the reference's NCCL call would simply wait here): fail the whole process, loudly.
        printf("bags_grad_allreduce: rank %d block %d waited %lld ms for rank %d (epoch %u) -- aborting\n", p.rank,
               (int)blockIdx.x, p.timeout_ns / 1000000, t, epoch);
        __trap();
      }
    }
  }
  __syncthreads();
  return *s_fail == 0;
}

template <bool MULTIMEM>
__global__ void __launch_bounds__(kArThreads, 6)
bags_grad_allreduce_kernel(const AllReduceParams p) {
  if (threadIdx.x == 0) stamp(p.timing, 0);
  pdl_trigger();   // the next kernel of the stream (next step's sampler / forward) may start launching
  pdl_wait();      // the local gradients come from the preceding backward kernel
  if (threadIdx.x == 0) stamp(p.timing, 1);
  __shared__ int s_fail;
  if (threadIdx.x == 0) s_fail = 0;
  // this block's barrier count so far (same on every rank); two more after this launch -- on EVERY exit path, so a
  // soft-failed exchange (self test) leaves the epochs of all ranks consistent
  uint32_t* my_epoch = ar_flags(p, p.rank) + kArMaxBlocks * p.world + blockIdx.x;
  const uint32_t epoch = *my_epoch;
  if (!rank_barrier(p, epoch + 1u, &s_fail, true)) {
    if (threadIdx.x == 0) *my_epoch = epoch + 2u;
    return;
  }
  if (threadIdx.x == 0) stamp(p.timing, 2);

  const long long vecs = p.count >> 2;
  const long long chunk = (vecs + p.world - 1) / p.world;
  const long long v0 = chunk * p.rank;
  const long long v1 = (v0 + chunk < vecs) ? (v0 + chunk) : vecs;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  constexpr int UNROLL = 4;   // loads in flight per thread: one NVLink round trip is ~2 us
  for (long long v = v0 + static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; v < v1; v += stride * UNROLL) {
    float4 acc[UNROLL];
    if (MULTIMEM) {
#pragma unroll
      for (int u = 0; u < UNROLL; ++u)
        if (v + u * stride < v1) acc[u] = multimem_ld_reduce_f4(p.mc + 4 * (v + u * stride));
    } else {
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int r = 0; r < p.world; ++r) {
        float4 t[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u)
          if (v + u * stride < v1) t[u] = ld_relaxed_sys_f4(p.peer[r] + 4 * (v + u * stride));
#pragma unroll
        for (int u = 0; u < UNROLL; ++u)
          if (v + u * stride < v1) { acc[u].x += t[u].x; acc[u].y += t[u].y; acc[u].z += t[u].z; acc[u].w += t[u].w; }
      }
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      if (v + u * stride >= v1) continue;
      const float4 o = make_float4(acc[u].x * p.scale, acc[u].y * p.scale, acc[u].z * p.scale, acc[u].w * p.scale);
      if (MULTIMEM) {
        multimem_st_f4(p.mc + 4 * (v + u * stride), o);
      } else {
        for (int r = 0; r < p.world; ++r) st_relaxed_sys_f4(p.peer[r] + 4 * (v + u * stride), o);
      }
    }
  }
  if (threadIdx.x == 0) stamp(p.timing, 3);
  rank_barrier(p, epoch + 2u, &s_fail);
  if (threadIdx.x == 0) { *my_epoch = epoch + 2u; stamp(p.timing, 4); }
}

}  // namespace bags
