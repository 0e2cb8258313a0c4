// Thin inline-PTX wrappers for the sm_90a features the BAGS kernels use:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (fences, groups, shared-memory descriptors),
// setmaxnreg and a few cache-hinted global accesses.  No CUTLASS/CuTe dependency.
//
// The wgmma descriptor bit layout follows the PTX ISA "matrix descriptor" table for
// wgmma.mma_async (the fields CUTLASS names GMMA::DescriptorIterator / GmmaDescriptor).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace bags {

// ----------------------------------------------------------------------------
// generic helpers
// ----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "elect.sync _|P1, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P1;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// Programmatic dependent launch: a kernel launched with the programmatic-stream-serialization attribute may
// start while its predecessor is still running; pdl_wait() blocks until the predecessor grid has completed and
// its writes are visible.  pdl_trigger() in the predecessor lets dependents start launching early.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ long long global_timer_ns() {
  long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ int sm_id() {
  int r;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(r));
  return r;
}
// Debug timeline (test hook): slot layout per CTA is 8 x int64; a null pointer disables it.
__device__ __forceinline__ void stamp(long long* timing, int slot) {
  if (timing != nullptr) timing[blockIdx.x * 8 + slot] = global_timer_ns();
}
// further banks of 8 slots per CTA, stored after the first bank of the whole grid
__device__ __forceinline__ void stamp_bank(long long* timing, int bank, int slot) {
  if (timing != nullptr) timing[(bank * gridDim.x + blockIdx.x) * 8 + slot] = global_timer_ns();
}
// second bank of 8 slots per CTA, stored after the first bank of the whole grid
__device__ __forceinline__ void stamp2(long long* timing, int slot) {
  if (timing != nullptr) timing[(gridDim.x + blockIdx.x) * 8 + slot] = global_timer_ns();
}

// ----------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P1;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}

// Bounded wait: a broken pipeline must never hang the GPU.  After ~2^28
// failed probes (seconds) the kernel traps.
#ifndef BAGS_WAIT_LIMIT
#define BAGS_WAIT_LIMIT (1u << 28)
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  // (no printf here: a call inside the mainloop makes ptxas serialise the wgmma pipeline)
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > BAGS_WAIT_LIMIT) __trap();
  }
}

// ----------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
// 2-D tiled load global -> shared::cta, completion on an mbarrier (tx bytes).
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar,
                                            int32_t c_inner, int32_t c_outer) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)),
        "r"(c_inner), "r"(c_outer)
      : "memory");
}


// expect `bytes` more transaction bytes on `bar` without arriving (the arrivals come from other threads)
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}

// ----------------------------------------------------------------------------
// wgmma : fences, groups, descriptors
// ----------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// Shared-memory matrix descriptor (64 bit), 128-byte swizzle (the layout TMA SWIZZLE_128B writes):
//   [ 0,14) start address >> 4      [16,30) leading-dim byte offset >> 4
//   [32,46) stride-dim byte offset >> 4      [49,52) base offset (0: tiles are 1024 B aligned)
//   [62,64) swizzle mode (1 = 128B)
// K-major: rows of 128 B, 8-row atoms SBO = 1024 B apart (LBO unused); a K step of 32 B advances the start address.
// MN-major (bf16 only): 64-element MN slabs LBO apart, 8-row K groups SBO = 1024 B apart; a K step of 16 rows
// advances the start address by 2048 B.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// 2-D tiled store shared::cta -> global (bulk async group); out-of-bounds parts of the box are clipped.
__device__ __forceinline__ void tma_store_2d(const void* tmap, const void* smem_src, int32_t c_inner,
                                             int32_t c_outer) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(smem_src)), "r"(c_inner), "r"(c_outer)
               : "memory");
}
// same, but global += smem (fp32 add performed by the TMA unit at L2)
__device__ __forceinline__ void tma_reduce_add_2d(const void* tmap, const void* smem_src, int32_t c_inner,
                                                  int32_t c_outer) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(smem_src)), "r"(c_inner), "r"(c_outer)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ----------------------------------------------------------------------------
// global memory helpers
// ----------------------------------------------------------------------------
__device__ __forceinline__ float4 ldg_stream_f4(const float4* p) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p));
  return v;
}
__device__ __forceinline__ void red_add_f32(float* p, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
__device__ __forceinline__ void red_add_v4_f32(float* p, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c),
               "f"(d)
               : "memory");
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

}  // namespace bags
