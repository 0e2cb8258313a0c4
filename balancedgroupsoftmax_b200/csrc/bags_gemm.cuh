// Persistent, warp-specialised wgmma GEMM for sm_90a.
//
//   D[M,N] (+)= A[M,K] * B[N,K]^T       fp32 accumulation in registers
//
// A and B are each either "K-major" (contraction index contiguous in HBM, i.e.
// a row-major [rows,K] matrix) or "MN-major" (row-major [K,rows]: contraction
// index strided).  That covers the three contractions of the BAGS head without
// any transposed copies in HBM:
//
//   forward  z  = X  W^T  : A = X   [N_roi,K]  K-major , B = W   [C,K]      K-major   (bags_gemm_kernel)
//   backward dX = dz W    : A = dz  [N_roi,C]  K-major , B = W   [C,K]      MN-major  (bags_bwd_merged_kernel)
//   backward dW = dz^T X  : A = dz  [N_roi,C]  MN-major, B = X   [N_roi,K]  MN-major  (bags_bwd_merged_kernel)
//
// Pipeline (one CTA per SM, 384 threads = 3 warpgroups):
//   warpgroup 0   : producer.  TMA (cp.async.bulk.tensor, 128B swizzle, mbarrier tx) for every bf16 operand and
//                   every K-major fp32 operand.  wgmma reads tf32 operands K-major only, so an MN-major fp32
//                   operand is transposed on the way in: the 128 producer threads load it with coalesced 16-byte
//                   reads and write it into the K-major swizzled layout.
//   warpgroups 1,2: consumers.  Each owns 64 rows of the 128 x BLOCK_N tile (wgmma m64nNk16 / k8, accumulators in
//                   registers) and runs its own epilogue straight from the accumulator fragments.
// smem ring of STAGES {A tile, B tile}.
#pragma once
#include "bags_ptx.cuh"
#include "bags_kernels.cuh"
#include "bags_wgmma.cuh"

namespace bags {

enum EpiMode : int {
  EPI_STORE_F32 = 0,   // out fp32 = act(acc + bias[n])          act = ReLU when GemmParams::relu, else identity
  EPI_STORE_BF16 = 1,  // out bf16 = act(acc + bias[n])
  EPI_RED_F32 = 2,     // out fp32 += rowscale(m) * acc   (split-K via red.global)
};

constexpr int kMaxGroups = 8;

struct GemmParams {
  int M, N, K;         // logical problem
  int num_m_tiles, num_n_tiles, num_splits;
  int kblocks_total;   // ceil(K / BLOCK_K)
  void* out;           // [M, ldo]
  long long ldo;       // elements
  const float* bias;   // [N] or nullptr                    (EPI_STORE_F32 / EPI_STORE_BF16)
  int relu;            // 1: max(., 0) after the bias         (EPI_STORE_F32 / EPI_STORE_BF16; the shared-FC trunk,
                       //    convfc_bbox_head.py:138-143)
  // EPI_RED_F32: per-row scale = gscale[group(m)], groups = [gstart, gstart+glen)
  const float* gscale; // device [G] or nullptr (=> 1.0)
  int G;
  int gstart[kMaxGroups];
  int glen[kMaxGroups];
  const float* colsum_in;  // optional [colsum_tiles, M]: db_out[m] = rowscale(m) * sum_t colsum_in[t, m]
  int colsum_tiles;
  float* colsum_out;       // written by the (n_tile==0, split==0) unit
  // MN-major fp32 operands (loaded without TMA): base pointer, leading dimension (elements), extents
  const float* a_ptr; long long lda; int a_rows, a_k;
  const float* b_ptr; long long ldb; int b_rows, b_k;
};

template <int BLOCK_N, bool A_MN, bool B_MN, int EPI, bool TF32, int STAGES>
struct GemmCfg {
  static constexpr int BLOCK_M = 128;
  static constexpr int ELT = TF32 ? 4 : 2;
  static constexpr int BLOCK_K = 128 / ELT;          // 64 bf16 / 32 tf32 : one 128B swizzle row
  static constexpr int K_STEPS = 4;                  // wgmma k16 (bf16) / k8 (tf32): 32 B of K each
  static constexpr int A_BYTES = BLOCK_M * 128;      // 16 KB
  static constexpr int B_BYTES = BLOCK_N * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int SLAB = 128 / ELT;             // MN elements per 128B (MN-major slab width)
  static constexpr bool A_MANUAL = A_MN && TF32;     // transposed by the producer threads
  static constexpr bool B_MANUAL = B_MN && TF32;
  static constexpr bool ANY_MANUAL = A_MANUAL || B_MANUAL;
  static constexpr int TMA_BYTES = (A_MANUAL ? 0 : A_BYTES) + (B_MANUAL ? 0 : B_BYTES);
  // TMA boxes per stage
  static constexpr int A_BOXES = A_MN ? BLOCK_M / SLAB : 1;
  static constexpr int A_BOX_BYTES = A_BYTES / A_BOXES;
  static constexpr int B_BOXES = B_MN ? BLOCK_N / SLAB : 1;
  static constexpr int B_BOX_BYTES = B_BYTES / B_BOXES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= 232448, "exceeds 227 KB of shared memory");
  static_assert(BLOCK_N == 256, "the consumers issue m64n256 MMAs");
  static constexpr int NUM_THREADS = 384;
  static constexpr int STAGES_ = STAGES;
  static constexpr int BLOCK_N_ = BLOCK_N;
};

__device__ __forceinline__ float row_group_scale(const GemmParams& p, int m) {
  if (p.gscale == nullptr) return 1.0f;
  float s = 0.0f;
#pragma unroll
  for (int g = 0; g < kMaxGroups; ++g) {
    if (g < p.G && m >= p.gstart[g] && m < p.gstart[g] + p.glen[g]) s = __ldg(p.gscale + g);
  }
  return s;
}

// Transposing load of one fp32 tile stored MN-major in HBM ([k][row], row contiguous) into the K-major 128B-swizzled
// layout wgmma reads: tile element (r, k) goes to r * 128 + (((k >> 2) ^ (r & 7)) << 4) + (k & 3) * 4.
// A warp covers 8 row quads x 4 k per step: 128-byte coalesced reads, 4-way bank conflicts on the scattered stores.
// Rows / k outside the matrix are zero (like the TMA's out-of-bounds fill).
template <int ROWS>
__device__ __forceinline__ void load_tile_transposed(uint8_t* dst, const float* src, long long ld, int rows, int kdim,
                                                     int r0, int k0, int tid) {
  constexpr int STEPS = (ROWS / 32) * 8;   // warp steps of (8 quads x 4 k)
  const int lane = tid & 31, wid = tid >> 5;
#pragma unroll 4
  for (int s = wid; s < STEPS; s += 4) {
    const int r = ((s % (ROWS / 32)) * 8 + (lane & 7)) * 4;
    const int k = (s / (ROWS / 32)) * 4 + (lane >> 3);
    const int gr = r0 + r, gk = k0 + k;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (gk < kdim) {
      const float* g = src + static_cast<long long>(gk) * ld + gr;
      if (gr + 3 < rows) {
        const float4 q = __ldg(reinterpret_cast<const float4*>(g));
        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
      } else {
#pragma unroll
        for (int e = 0; e < 4; ++e) if (gr + e < rows) v[e] = __ldg(g + e);
      }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int rr = r + e;
      *reinterpret_cast<float*>(dst + rr * 128 + (((k >> 2) ^ (rr & 7)) << 4) + (k & 3) * 4) = v[e];
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Pieces shared by the GEMM kernel and the merged backward kernel.  Every problem a kernel runs has the same stage
// layout (128 x 256 tiles of 128-byte rows), so one shared-memory ring and one set of barriers serve all of them.
// ---------------------------------------------------------------------------------------------------------------------
struct Pipe {
  uint8_t* smem_a;
  uint8_t* smem_b;
  uint64_t* full_bar;
  uint64_t* empty_bar;
  int stage;
  uint32_t phase;
};

// balanced k-block range of split `split`
__device__ __forceinline__ void split_range(const GemmParams& p, int split, int& kb0, int& kb1) {
  const int base = p.kblocks_total / p.num_splits, rem = p.kblocks_total % p.num_splits;
  kb0 = split * base + (split < rem ? split : rem);
  kb1 = kb0 + base + (split < rem ? 1 : 0);
}

// Producer side of one unit: k-blocks [kb0, kb1) of the tile at (m0, n0).  Thread 0 issues the TMA loads; with an
// MN-major fp32 operand all 128 producer threads take part (b_ptr: the B matrix that operand path reads).
template <class Cfg, bool A_MN, bool B_MN>
__device__ __forceinline__ void produce_unit(const CUtensorMap* tmap_a, const CUtensorMap* tmap_b, const GemmParams& p,
                                             const float* b_ptr, int m0, int n0, int kb0, int kb1, Pipe& pp, int tid) {
  constexpr int STAGES = Cfg::STAGES_;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&pp.empty_bar[pp.stage], pp.phase ^ 1u);
    const int k0 = kb * Cfg::BLOCK_K;
    uint8_t* sa = pp.smem_a + pp.stage * Cfg::A_BYTES;
    uint8_t* sb = pp.smem_b + pp.stage * Cfg::B_BYTES;
    uint64_t* fb = &pp.full_bar[pp.stage];
    if (tid == 0 && Cfg::TMA_BYTES > 0) {
      if (Cfg::ANY_MANUAL) mbar_expect_tx(fb, Cfg::TMA_BYTES);
      else                 mbar_arrive_expect_tx(fb, Cfg::TMA_BYTES);
      if (!Cfg::A_MANUAL) {
#pragma unroll
        for (int i = 0; i < Cfg::A_BOXES; ++i) {
          if (A_MN) tma_load_2d(sa + i * Cfg::A_BOX_BYTES, tmap_a, fb, m0 + i * Cfg::SLAB, k0);
          else      tma_load_2d(sa + i * Cfg::A_BOX_BYTES, tmap_a, fb, k0, m0);
        }
      }
      if (!Cfg::B_MANUAL) {
#pragma unroll
        for (int i = 0; i < Cfg::B_BOXES; ++i) {
          if (B_MN) tma_load_2d(sb + i * Cfg::B_BOX_BYTES, tmap_b, fb, n0 + i * Cfg::SLAB, k0);
          else      tma_load_2d(sb + i * Cfg::B_BOX_BYTES, tmap_b, fb, k0, n0);
        }
      }
    }
    if (Cfg::ANY_MANUAL) {
      if (Cfg::A_MANUAL) load_tile_transposed<Cfg::BLOCK_M>(sa, p.a_ptr, p.lda, p.a_rows, p.a_k, m0, k0, tid);
      if (Cfg::B_MANUAL) load_tile_transposed<Cfg::BLOCK_N_>(sb, b_ptr, p.ldb, p.b_rows, p.b_k, n0, k0, tid);
      fence_proxy_async_smem();   // generic-proxy stores -> visible to the wgmma (async proxy) reads
      mbar_arrive(fb);
    }
    if (++pp.stage == STAGES) { pp.stage = 0; pp.phase ^= 1u; }
  }
}

// Consumer side of one unit: the mainloop of warpgroup `cw` (rows 64 cw .. 64 cw + 63 of the tile).  One k-block of
// wgmma stays in flight: after committing k-block kb the warpgroup waits for kb - 1 only and releases that stage, so
// the tensor pipe does not drain between k-blocks.  The unit ends with everything complete and every stage it used
// released; pp.stage / pp.phase then name the next unit's first stage, as on the producer's side.
template <class Cfg, bool A_MN, bool B_MN, bool TF32>
__device__ __forceinline__ void consume_unit(float (&acc)[128], int cw, int kb0, int kb1, Pipe& pp, int lane) {
  constexpr int STAGES = Cfg::STAGES_;
  // K-major: 8-row atoms 1024 B apart, K step 32 B.  MN-major (bf16): slabs of 64 elements, K step 16 rows = 2048 B.
  constexpr bool A_T = A_MN && !TF32, B_T = B_MN && !TF32;
  constexpr uint32_t A_LBO = A_T ? Cfg::BLOCK_K * 128 : 16, B_LBO = B_T ? Cfg::BLOCK_K * 128 : 16;
  constexpr uint32_t A_KSTEP = A_T ? 2048 : 32, B_KSTEP = B_T ? 2048 : 32;
  // this warpgroup's 64 A rows: the second MN slab (MN-major) / rows 64..127 (K-major) -- 8 KB either way
  const uint32_t a_off = cw * 8192;
  int prev = 0;   // stage of k-block kb - 1
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&pp.full_bar[pp.stage], pp.phase);
    const uint32_t sa = smem_u32(pp.smem_a + pp.stage * Cfg::A_BYTES) + a_off;
    const uint32_t sb = smem_u32(pp.smem_b + pp.stage * Cfg::B_BYTES);
    fence_regs(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < Cfg::K_STEPS; ++k) {
      const uint64_t adesc = make_smem_desc(sa + k * A_KSTEP, A_LBO, 1024);
      const uint64_t bdesc = make_smem_desc(sb + k * B_KSTEP, B_LBO, 1024);
      const uint32_t accum = (kb > kb0 || k > 0) ? 1u : 0u;
      if (TF32) wgmma_tf32_n256(acc, adesc, bdesc, accum);
      else      wgmma_bf16_n256<A_T ? 1 : 0, B_T ? 1 : 0>(acc, adesc, bdesc, accum);
    }
    wgmma_commit();
    // keep this k-block's MMAs in flight; the previous k-block's are complete, so its stage can be refilled
    wgmma_wait<1>();
    fence_regs(acc);
    if (kb > kb0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&pp.empty_bar[prev]);
    }
    prev = pp.stage;
    if (++pp.stage == STAGES) { pp.stage = 0; pp.phase ^= 1u; }
  }
  wgmma_wait<0>();
  fence_regs(acc);
  if (kb1 > kb0) {
    __syncwarp();
    if (lane == 0) mbar_arrive(&pp.empty_bar[prev]);   // the last k-block's stage
  }
}

// Epilogue from the fragments: thread holds rows r and r + 8, column pairs 8j + 2 (lane & 3).
// EPI_STORE_*: out = act(oscale * acc + bias);  EPI_RED_F32: out += rowscale(m) * acc.
template <int BLOCK_N, int EPI>
__device__ __forceinline__ void epilogue_unit(const float (&acc)[128], const GemmParams& p, int m_tile, int n_tile,
                                              int split, int cw, int warp, int lane, float oscale) {
  const bool pair_ok = ((p.ldo & 1) == 0) && ((reinterpret_cast<uintptr_t>(p.out) & 7) == 0);
  const int r_a = m_tile * 128 + cw * 64 + warp * 16 + (lane >> 2);
  const int c_base = n_tile * BLOCK_N + 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = r_a + 8 * h;
    if (m >= p.M) continue;
    float scale = oscale;
    if (EPI == EPI_RED_F32) {
      scale = row_group_scale(p, m);
      if (p.colsum_out != nullptr && n_tile == 0 && split == 0 && (lane & 3) == 0) {
        float cs = 0.f;
        for (int tt = 0; tt < p.colsum_tiles; ++tt) cs += __ldg(p.colsum_in + static_cast<long long>(tt) * p.M + m);
        p.colsum_out[m] = scale * cs;
      }
    }
    uint8_t* orow = reinterpret_cast<uint8_t*>(p.out) + static_cast<long long>(m) * p.ldo * (EPI == EPI_STORE_BF16 ? 2 : 4);
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      const int n = c_base + 8 * j;
      if (n >= p.N) continue;
      float v0 = acc[4 * j + 2 * h] * scale, v1 = acc[4 * j + 2 * h + 1] * scale;
      const bool two = n + 1 < p.N;
      if (EPI == EPI_RED_F32) {
        float* o = reinterpret_cast<float*>(orow) + n;
        if (two && pair_ok) {
          asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(o), "f"(v0), "f"(v1) : "memory");
        } else {
          red_add_f32(o, v0);
          if (two) red_add_f32(o + 1, v1);
        }
      } else {
        if (p.bias != nullptr) { v0 += __ldg(p.bias + n); if (two) v1 += __ldg(p.bias + n + 1); }
        if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
        if (EPI == EPI_STORE_BF16) {
          __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(orow) + n;
          if (two && pair_ok) *reinterpret_cast<uint32_t*>(o) = pack_bf16x2(v0, v1);
          else { o[0] = __float2bfloat16_rn(v0); if (two) o[1] = __float2bfloat16_rn(v1); }
        } else {
          float* o = reinterpret_cast<float*>(orow) + n;
          if (two && pair_ok) *reinterpret_cast<float2*>(o) = make_float2(v0, v1);
          else { o[0] = v0; if (two) o[1] = v1; }
        }
      }
    }
  }
}

__device__ __forceinline__ Pipe setup_pipe(uint8_t* smem_raw, int stages, int a_bytes, int stage_bytes, bool manual) {
  // 1024-byte alignment is required by the 128B swizzle atoms.
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  Pipe pp;
  pp.smem_a = smem;
  pp.smem_b = smem + stages * a_bytes;
  pp.full_bar = reinterpret_cast<uint64_t*>(smem + stages * stage_bytes);
  pp.empty_bar = pp.full_bar + stages;
  pp.stage = 0;
  pp.phase = 0;
  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(&pp.full_bar[s], manual ? 128 : 1);
      mbar_init(&pp.empty_bar[s], 8);   // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  return pp;
}

// The forward GEMM: both operands K-major, so every load is a TMA load issued by producer thread 0.
template <int BLOCK_N, int EPI, bool TF32, int STAGES>
__global__ void __launch_bounds__(384, 1)
bags_gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const GemmParams p) {
  using Cfg = GemmCfg<BLOCK_N, false, false, EPI, TF32, STAGES>;
  extern __shared__ uint8_t smem_raw[];
  const int wg = threadIdx.x >> 7;
  const int tid = threadIdx.x & 127;
  pdl_trigger();   // a dependent kernel may begin its own prologue
  if (threadIdx.x == 0) { tma_prefetch_desc(&tmap_a); tma_prefetch_desc(&tmap_b); }
  Pipe pp = setup_pipe(smem_raw, STAGES, Cfg::A_BYTES, Cfg::STAGE_BYTES, false);

  const int units_per_split = p.num_m_tiles * p.num_n_tiles;
  const int num_units = units_per_split * p.num_splits;
  if (wg == 0) {
    // ===================== producer =====================
    setmaxnreg_dec<40>();
    if (tid == 0) {
      for (int u = blockIdx.x; u < num_units; u += gridDim.x) {
        const int split = u / units_per_split;
        const int t = u - split * units_per_split;
        const int m_tile = t / p.num_n_tiles, n_tile = t - m_tile * p.num_n_tiles;
        int kb0, kb1;
        split_range(p, split, kb0, kb1);
        produce_unit<Cfg, false, false>(&tmap_a, &tmap_b, p, nullptr, m_tile * 128, n_tile * BLOCK_N, kb0, kb1, pp, tid);
      }
    }
  } else {
    // ===================== consumers =====================
    setmaxnreg_inc<232>();
    const int cw = wg - 1, warp = tid >> 5, lane = tid & 31;
    float acc[128];
    for (int u = blockIdx.x; u < num_units; u += gridDim.x) {
      const int split = u / units_per_split;
      const int t = u - split * units_per_split;
      const int m_tile = t / p.num_n_tiles, n_tile = t - m_tile * p.num_n_tiles;
      int kb0, kb1;
      split_range(p, split, kb0, kb1);
      consume_unit<Cfg, false, false, TF32>(acc, cw, kb0, kb1, pp, lane);
      epilogue_unit<BLOCK_N, EPI>(acc, p, m_tile, n_tile, split, cw, warp, lane, 1.0f);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Merged backward: the contractions of the BAGS head's backward in ONE persistent launch.
//
//   dW units : dW[C,K]  += gout(bin(c)) * dz^T x       (A = dz MN-major, B = x MN-major, split-K, red.add)
//   dX units : dX[N,K]   = dz W'                       (A = dz K-major,  B = W' MN-major, plain stores)
//
// The units form one work list (dW first: their split-K partials are the longer tail), dealt round-robin to the
// CTAs, so the SMs that finish their dW share early take dX tiles instead of idling at a kernel boundary.  A request
// for only dW or only dX leaves the other list empty (dx_units = 0 / dw_units = 0).  When the
// bins tile [0, C) and all gout[g] are equal (the reference's setting) the dX units read W itself and scale their
// output by gout[0]: the preparation kernel then skips the scaled copy W' (it makes the same device-side decision).
// With gaps between the bins W' is always built, since its gap rows are 0 while W's are not.
//
// Programmatic dependent launch: the preparation kernel (when it runs) triggers only after its own griddepcontrol.wait,
// so at this kernel's start dz (the forward's output) and x are complete, and W was never written on the device side.
// Each access waits only for what it reads:
//   - the producer's dW units (dz^T, x): no wait, unless no preparation kernel ran (inputs_ready = 0);
//   - the producer's dX units (dz, W or W'): a wait before the first load of W' (wprime_prepared and gout not
//     uniform); none when they read W itself;
//   - the consumers: a wait before their first epilogue, since dW may still be being zeroed and db's column-sum
//     partials are the preparation kernel's;
//   - gout is read before any wait: the preparation kernel does not write it, and it is nullptr when none ran.
// So the mainloop of the first units runs under the preparation kernel's tail.
// ---------------------------------------------------------------------------------------------------------------------
struct BwdMergedParams {
  GemmParams dw;     // tile counts, splits and epilogue fields of the dW problem
  GemmParams dx;     // ... of the dX problem (b_ptr: W')
  int dw_units, dx_units;
  const float* w;    // W (B of the dX units when gout is uniform)
  const float* gout; // [G] per-bin upstream gradients of the dX units, or nullptr (dX reads b_ptr unscaled)
  int G;
  int uniform_ok;    // the bins tile [0, C): a uniform gout may take the W shortcut
  int inputs_ready;     // a preparation kernel ran between the forward and this launch: dz and x are complete at launch
  int wprime_prepared;  // dx.b_ptr is W', written by that preparation kernel (else it is W)
  int dx_tma;           // bf16 dX with K and its row stride multiples of 8: stored through t_dx (dx_epilogue_tma)
  // optional debug timeline (bags_debug_set_timing), two rows of 8 int64 per CTA, or nullptr.  Row 0, %globaltimer
  // of the first consumer thread: CTA start, griddepcontrol.wait returned, then for each of the first three units
  // the end of its mainloop and the end of its epilogue.  Row 1: slots 0-2 the k-blocks of those units (negative
  // for a dX unit), slot 7 the producer's first load.
  long long* timing;
};

template <bool TF32>
using BwdDwCfg = GemmCfg<256, true, true, EPI_RED_F32, TF32, 4>;
template <bool TF32>
using BwdDxCfg = GemmCfg<256, false, true, TF32 ? EPI_STORE_F32 : EPI_STORE_BF16, TF32, 4>;

// The bf16 dX tile leaves through shared memory and TMA stores: each consumer warpgroup stages its 64 x 256 rows in
// two halves of 64 x 128 (two 128B-swizzled boxes of 64 columns, 16 KB), after the ring and its barriers.
constexpr int kDxStageBytes = 2 * 16384;
template <bool TF32>
constexpr int bwd_merged_smem_bytes() {
  return 4 * BwdDwCfg<TF32>::STAGE_BYTES + 1024 /*align slack*/ + 1024 /*barriers*/ + kDxStageBytes;
}
static_assert(bwd_merged_smem_bytes<false>() <= 232448, "exceeds 227 KB of shared memory");

// bf16 dX epilogue of warpgroup `cw` through its 16 KB staging buffer `stg`: the same values as epilogue_unit's
// (bf16 of scale * acc), written with one TMA store per 64 x 64 box instead of 8-row scattered 4-byte stores.
// The tensor map spans [N, K] with K % 8 == 0, so the clipped boxes at the edges never write past column K.
// Thread 0 of the warpgroup issues the stores and, before the buffer is refilled, waits until they have read it.
__device__ __forceinline__ void dx_epilogue_tma(const float (&acc)[128], const CUtensorMap* tmap, uint8_t* stg,
                                                int M, int N, int m0, int n0, int cw, int warp, int lane, int tid,
                                                float scale) {
  const int rw = m0 + 64 * cw;   // first row of this warpgroup
#pragma unroll
  for (int hc = 0; hc < 2; ++hc) {
    if (tid == 0) tma_store_wait_read<0>();   // the previous half's (or unit's) stores have read the buffer
    asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      const int j = 16 * hc + jj;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = warp * 16 + (lane >> 2) + 8 * h;
        *reinterpret_cast<uint32_t*>(stg + (jj >> 3) * 8192 + r * 128 + (((jj & 7) ^ (r & 7)) << 4) + 4 * (lane & 3)) =
            pack_bf16x2(acc[4 * j + 2 * h] * scale, acc[4 * j + 2 * h + 1] * scale);
      }
    }
    fence_proxy_async_smem();   // the staged half is read by the TMA (async proxy)
    asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");
    if (tid == 0 && rw < M) {
#pragma unroll
      for (int b = 0; b < 2; ++b)
        if (n0 + 128 * hc + 64 * b < N) tma_store_2d(tmap, stg + b * 8192, n0 + 128 * hc + 64 * b, rw);
      tma_store_commit();
    }
  }
}

template <bool TF32>
__global__ void __launch_bounds__(384, 1)
bags_bwd_merged_kernel(const __grid_constant__ CUtensorMap t_dzT, const __grid_constant__ CUtensorMap t_xT,
                       const __grid_constant__ CUtensorMap t_dz, const __grid_constant__ CUtensorMap t_w,
                       const __grid_constant__ CUtensorMap t_wp, const __grid_constant__ CUtensorMap t_dx,
                       const BwdMergedParams p) {
  using CW = BwdDwCfg<TF32>;
  using CX = BwdDxCfg<TF32>;
  static_assert(CW::STAGE_BYTES == CX::STAGE_BYTES && CW::A_BYTES == CX::A_BYTES, "one ring serves both problems");
  static_assert(CW::ANY_MANUAL == CX::ANY_MANUAL, "one barrier arrival count serves both problems");
  extern __shared__ uint8_t smem_raw[];
  const int wg = threadIdx.x >> 7;
  const int tid = threadIdx.x & 127;
  // debug timeline: row 0 belongs to the first consumer thread, row 1 slot 7 to the producer thread
  long long* const tl = (p.timing != nullptr && (threadIdx.x == 128 || threadIdx.x == 0))
                            ? p.timing + blockIdx.x * 16ll + (threadIdx.x == 0 ? 8 : 0) : nullptr;
  if (tl != nullptr && threadIdx.x == 128) tl[0] = global_timer_ns();
  pdl_trigger();
  Pipe pp = setup_pipe(smem_raw, 4, CW::A_BYTES, CW::STAGE_BYTES, CW::ANY_MANUAL);
  uint8_t* const stg = reinterpret_cast<uint8_t*>(pp.full_bar) + 1024;   // dX staging (1024-byte aligned)
  // gout is never written by the preparation kernel, and without one it is nullptr here (see inputs_ready)
  float g0 = 1.0f;
  const bool uniform = p.uniform_ok && p.gout != nullptr && gout_uniform(p.gout, p.G, g0);
  const float* xb = uniform ? p.w : p.dx.b_ptr;
  const CUtensorMap* txb = uniform ? &t_w : &t_wp;
  const float xscale = uniform ? g0 : 1.0f;

  const int dw_per_split = p.dw.num_m_tiles * p.dw.num_n_tiles;
  const int num_units = p.dw_units + p.dx_units;
  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (CW::ANY_MANUAL || tid == 0) {
      // dz and x: ready at launch when the preparation kernel ran (it triggers only after its own wait); W' is the
      // preparation kernel's output, W itself is not
      bool waited = false;
      if (!p.inputs_ready) { pdl_wait(); waited = true; }
      const bool wait_dx = !uniform && p.wprime_prepared;
      if (tl != nullptr) tl[7] = global_timer_ns();
      for (int u = blockIdx.x; u < num_units; u += gridDim.x) {
        if (u < p.dw_units) {
          const int split = u / dw_per_split, t = u - split * dw_per_split;
          const int m_tile = t / p.dw.num_n_tiles, n_tile = t - m_tile * p.dw.num_n_tiles;
          int kb0, kb1;
          split_range(p.dw, split, kb0, kb1);
          produce_unit<CW, true, true>(&t_dzT, &t_xT, p.dw, p.dw.b_ptr, m_tile * 128, n_tile * 256, kb0, kb1, pp, tid);
        } else {
          const int t = u - p.dw_units;
          const int m_tile = t / p.dx.num_n_tiles, n_tile = t - m_tile * p.dx.num_n_tiles;
          if (wait_dx && !waited) { pdl_wait(); waited = true; }
          produce_unit<CX, false, true>(&t_dz, txb, p.dx, xb, m_tile * 128, n_tile * 256, 0, p.dx.kblocks_total, pp, tid);
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int cw = wg - 1, warp = tid >> 5, lane = tid & 31;
    // first epilogue: dW may still be being zeroed, and db's column-sum partials come from the preparation kernel
    auto epilogue_wait = [&]() {
      pdl_wait();
      if (tl != nullptr) tl[1] = global_timer_ns();
    };
    float acc[128];
    int i = 0;   // the CTA's unit count (timeline slots)
    for (int u = blockIdx.x; u < num_units; u += gridDim.x, ++i) {
      if (u < p.dw_units) {
        const int split = u / dw_per_split, t = u - split * dw_per_split;
        const int m_tile = t / p.dw.num_n_tiles, n_tile = t - m_tile * p.dw.num_n_tiles;
        int kb0, kb1;
        split_range(p.dw, split, kb0, kb1);
        consume_unit<CW, true, true, TF32>(acc, cw, kb0, kb1, pp, lane);
        if (tl != nullptr && i < 3) { tl[2 + 2 * i] = global_timer_ns(); tl[8 + i] = kb1 - kb0; }
        if (i == 0) epilogue_wait();
        epilogue_unit<256, EPI_RED_F32>(acc, p.dw, m_tile, n_tile, split, cw, warp, lane, 1.0f);
      } else {
        const int t = u - p.dw_units;
        const int m_tile = t / p.dx.num_n_tiles, n_tile = t - m_tile * p.dx.num_n_tiles;
        consume_unit<CX, false, true, TF32>(acc, cw, 0, p.dx.kblocks_total, pp, lane);
        if (tl != nullptr && i < 3) { tl[2 + 2 * i] = global_timer_ns(); tl[8 + i] = -p.dx.kblocks_total; }
        if (i == 0) epilogue_wait();
        if (!TF32 && p.dx_tma)
          dx_epilogue_tma(acc, &t_dx, stg + cw * (kDxStageBytes / 2), p.dx.M, p.dx.N, m_tile * 128, n_tile * 256, cw,
                          warp, lane, tid, xscale);
        else
          epilogue_unit<256, TF32 ? EPI_STORE_F32 : EPI_STORE_BF16>(acc, p.dx, m_tile, n_tile, 0, cw, warp, lane, xscale);
      }
      if (tl != nullptr && i < 3) tl[3 + 2 * i] = global_timer_ns();
    }
    if (!TF32 && p.dx_tma && tid == 0) tma_store_wait_all();   // the staging buffer stays valid until the stores end
  }
}

}  // namespace bags
