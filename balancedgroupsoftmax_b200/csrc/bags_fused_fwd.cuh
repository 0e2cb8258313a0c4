// Fused BAGS forward for sm_90a:  fc_cls GEMM  ->  grouped softmax-CE  ->  dz~  in ONE kernel.
//
//   z = x W^T + b  is accumulated in registers and never written to HBM.
//
// A group of 4 CTAs owns a 128-row tile of RoIs at a time; CTA r of the group holds logit columns [320r, 320r+320) of
// those rows.  The grid is persistent: 4 * groups CTAs, CTA 4i + r is rank r of group i, and group i walks the row
// tiles i, i + groups, ...  The host sizes the grid so that every CTA is resident at once (a cooperative launch, which
// fails instead of hanging when the grid cannot be co-resident), because the four CTAs of a group wait for each other.
// The group is not a hardware cluster on purpose: a cluster must sit inside one GPC, and with one CTA per SM (shared
// memory) only 30 four-CTA clusters -- 120 of the 132 SMs of an H100 SXM -- fit at once, so the 32 row tiles of 4096
// RoIs ran in two waves.  Without the cluster, the same 128 CTAs run in one wave.  The four CTAs of a row tile
// exchange their softmax partials through L2 instead of distributed shared memory (about 5 KB per CTA at 5 bins).
// The CTA is two warpgroups and nothing else: each owns 64 rows and keeps its 64 x 320 fp32 accumulators in registers
// (two wgmma m64n160 per K step).  Thread 0 also issues the TMA loads, and every thread loads a share of the per-row
// labels / weights.  The CTA has no producer warp on purpose: a ninth warp puts three warps on one SM sub-partition,
// whose 16K registers then cap every thread of the kernel at 168, too few for the 160 accumulators -- ptxas spills
// and serialises the wgmma.  With eight warps each thread may use 255 registers, and the mainloop keeps one k-block
// of MMAs in flight while it waits for the next stage.
// In the wgmma fragment a row is held by the four lanes of a quad (80 columns each), so row reductions are a walk
// over the thread's own columns plus two quad shuffles.  Bins are contiguous column ranges, so every walk keeps a
// running (bin, value) pair and touches shared memory only where the bin changes.  A thread holds two columns of
// each 8-column chunk, and a CTA's 320 columns hold at most G + 1 bin changes, so the bin is resolved per chunk: a
// chunk inside the running bin is walked without any lookup, only the few others element by element.
//
//   accumulators := bias before the first MMA (the epilogue never adds it)
//   pass A  : per row and bin, the max m over this CTA's columns
//   pass B  : z := e = exp(z - m) in place, sum e; z[target] is kept for the loss
//   exchange: every CTA stores its (max, sum) per row and bin to the group's slot in global memory and counts its
//             arrival on the group's counter (and zeroes its share of the optional `clear` buffer while it waits);
//             once all four have arrived, each reads the four partials back (L2) and combines them into the lse,
//             loss_bin += w/avg * (lse - z[target]) where the target column is this CTA's
//   pass C  : dz~ = e * exp(m - lse) * w/avg - onehot * w/avg -> operand dtype -> the idle pipeline stages -> TMA
//             stores to HBM ; column sums of dz~ (bias gradient) from the staged tile.  One exponential per logit.
//
// reference semantics: gs_bbox_head_with0.py:91-112 (labels/weights), :134-171 (slices + CE),
// cross_entropy_loss.py:9-19, losses/utils.py:26-53 (sum / avg_factor).
//
// Preconditions (checked on the host, otherwise the unfused path runs): C <= 1280, G <= 6, bins
// tile [0, C) contiguously.  The kernel itself takes any C: every column >= C is masked (bias preload, bins, column
// sums), the W tensor map zero-fills its rows >= C, and dz is stored for columns < C and rows < N only.
//
// The same kernel is the plain softmax-CE head (bags_ce_fwd, reweight_bbox_head.py / bbox_head.py:97-129): one bin
// (0, C), l2b == nullptr (the label is the target column), fp32 per-RoI weights, and optionally the top-1 accuracy,
// counted where the loss is formed (z[target] == row max) and reduced with the loss partials.
#pragma once
#include "bags_kernels.cuh"
#include "bags_ptx.cuh"
#include "bags_wgmma.cuh"

namespace bags {

struct FusedFwdParams {
  int N, C, K, kblocks;
  GroupTable gt;
  const float* bias;        // [C] or nullptr
  const long long* labels;  // [N]
  const int* l2b;           // [G, classes], or nullptr: the label is the target column (one bin (0, C), plain CE)
  int classes;
  const uint8_t* wmask;     // [G, N] 0/1 bytes (or fp32 weights when the kernel is instantiated with WF) or nullptr (all ones)
  const float* avg;         // [G] or nullptr (N)
  float* loss;              // [G]
  // optional top-1 accuracy of bin 0 (nullptr: none): acc[0] = acc_scale * #{rows : z[target] == row max}
  float* acc;
  float acc_scale;          // 100 / N
  float* lse;               // [N, G] or nullptr
  float* colsum;            // [row tiles, C] per-row-tile column sums of dz (plain stores) or nullptr
  float* part;              // [gridDim.x, kMaxG]
  unsigned int* counter;
  // softmax-partial exchange of the CTA groups (per-stream workspace, zeroed once): per group two slots (tile
  // parity) of [4 ranks][MAXG][128] (max, sum), and an arrival counter every kFusedCounterStride words
  float2* xch;
  unsigned int* xch_counter;
  void* dz;                 // [N, ldd] operand dtype, or nullptr (loss only)
  long long ldd;
  int want_dz;
  // dz columns [0, dz_tma_cols) leave through TMA stores (the extent of tmap_dz, 0: none), [dz_tma_cols, C) through
  // plain stores.  At the right edge of a tensor a TMA store writes whole 16-byte pieces, so the map ends at the last
  // 16-byte boundary at or before C, and the padding columns [C, ldd) stay untouched.
  int dz_tma_cols;
  // optional: a buffer the kernel sets to zero while its CTAs wait for their peers' softmax partials (the caller's dW:
  // the backward's split-K red.add then needs no zeroing job)
  float4* clear;
  long long clear_vecs;
  // optional debug timeline (bags_debug_set_timing), [gridDim.x][8] %globaltimer stamps of thread 0, or nullptr:
  // 0 start, 1 end of the mainloop, 2 after pass A, 3 after pass B, 4 exchange wait done, 5 end of pass C, 6 end of
  // the CTA.  Slots 1-5 are those of the CTA's last row tile.
  long long* timing;
};

template <bool TF32>
struct FusedCfg {
  static constexpr int BLOCK_M = 128;
  static constexpr int BLOCK_N = 320;
  static constexpr int HALF_N = 160;
  static constexpr int STAGES = 3;
  static constexpr int ELT = TF32 ? 4 : 2;
  static constexpr int BLOCK_K = 128 / ELT;
  static constexpr int K_STEPS = 4;
  static constexpr int A_BYTES = BLOCK_M * 128;
  static constexpr int B_BYTES = BLOCK_N * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int RANKS = 4;                                    // CTAs per row tile (C <= 4 * BLOCK_N)
  static constexpr int NUM_THREADS = 256;
  static constexpr int MAXG = 6;
  static constexpr int ROW_BYTES = 5 * MAXG * BLOCK_M * 4;          // tcol, coef, max, scale, z[target] per (bin, row)
  static constexpr int PART_BYTES = MAXG * 2 * 256 * 4;             // per-thread running partials
  static constexpr int MISC_BYTES = 2 * BLOCK_N * 4 /*bias, bin*/ + 64 /*loss*/ + 256 /*barriers*/;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + ROW_BYTES + PART_BYTES + MISC_BYTES + 1024;
  static_assert(SMEM_BYTES <= 232448, "fused forward exceeds shared memory");
  // dz of the tile is staged in the (then idle) pipeline stages as 128-byte-wide column boxes of 128 rows, 128B
  // swizzled, and written by TMA stores
  static constexpr int BOX_COLS = 128 / ELT;
  static constexpr int BOX_BYTES = BLOCK_M * 128;
  static constexpr int BOXES = BLOCK_N / BOX_COLS;
  static_assert(BOXES * BOX_BYTES <= STAGES * STAGE_BYTES, "the dz tile does not fit the pipeline stages");
  static constexpr int CHUNKS = BLOCK_N / 8;   // 8-column chunks of the tile: a thread holds 2 columns of each
  static constexpr int SLOT_ELEMS = RANKS * MAXG * BLOCK_M;          // float2 per exchange slot
  static_assert(MAXG < kMaxG, "the last per-CTA partial slot carries the accuracy count");
};

// Exchange workspace of the fused forward (the caller's per-stream workspace): at most kFusedMaxGroups CTA groups,
// one arrival counter per 128-byte line, two exchange slots per group.
constexpr int kFusedMaxGroups = 64;
constexpr int kFusedCounterStride = 32;
constexpr size_t kFusedXchCounterBytes = static_cast<size_t>(kFusedMaxGroups) * kFusedCounterStride * 4;
constexpr size_t kFusedXchSlotBytes = static_cast<size_t>(FusedCfg<false>::SLOT_ELEMS) * 8;
constexpr size_t kFusedXchBytes = kFusedXchCounterBytes + static_cast<size_t>(kFusedMaxGroups) * 2 * kFusedXchSlotBytes;

__device__ __forceinline__ unsigned int atom_add_release_gpu(unsigned int* addr, unsigned int v) {
  unsigned int old;
  asm volatile("atom.add.release.gpu.u32 %0, [%1], %2;" : "=r"(old) : "l"(addr), "r"(v) : "memory");
  return old;
}
__device__ __forceinline__ unsigned int ld_acquire_gpu(const unsigned int* addr) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(addr) : "memory");
  return v;
}

// WF = true: p.wmask points at fp32 per-(bin, RoI) weights instead of 0/1 bytes (the reweight head variant,
// gs_bbox_head_with0_reweight.py:57-85)
// tmap_dz: dz [N, C] in the operand dtype (row stride ldd), boxes of BOX_COLS x 128, 128B swizzle; unused without dz
template <bool TF32, bool WF = false>
__global__ void __launch_bounds__(FusedCfg<TF32>::NUM_THREADS, 1)
bags_fwd_fused_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                      const __grid_constant__ CUtensorMap tmap_dz, const FusedFwdParams p) {
  using Cfg = FusedCfg<TF32>;
  constexpr int BLOCK_M = Cfg::BLOCK_M, BLOCK_N = Cfg::BLOCK_N, BLOCK_K = Cfg::BLOCK_K, STAGES = Cfg::STAGES;
  constexpr int MAXG = Cfg::MAXG, HALF_N = Cfg::HALF_N, RANKS = Cfg::RANKS;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // 1 KB aligned
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * Cfg::A_BYTES;
  int* s_tcol = reinterpret_cast<int*>(smem + STAGES * Cfg::STAGE_BYTES);           // [MAXG][128]
  float* s_coef = reinterpret_cast<float*>(s_tcol + MAXG * BLOCK_M);                 // [MAXG][128] w / avg
  float* s_mrow = s_coef + MAXG * BLOCK_M;                                           // [MAXG][128] CTA row max
  float* s_scale = s_mrow + MAXG * BLOCK_M;                                          // [MAXG][128] exp(max - lse) w / avg
  float* s_zt = s_scale + MAXG * BLOCK_M;                                            // [MAXG][128] z[target column]
  float* s_part = s_zt + MAXG * BLOCK_M;                                             // [MAXG][2][256]
  float* s_bias = s_part + MAXG * 2 * 256;                                           // [320]
  int* s_colbin = reinterpret_cast<int*>(s_bias + BLOCK_N);                          // [320] bin or -1
  float* s_loss = reinterpret_cast<float*>(s_colbin + BLOCK_N);                      // [16]
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_loss + 16);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  __shared__ int s_gs[kMaxG], s_ge[kMaxG];
  // per quad lane q: bit J set = chunk J takes the per-element path of the walks (see below)
  __shared__ unsigned long long s_slow[4];
  static_assert(Cfg::CHUNKS <= 64, "one bit per chunk");

  const int tid = threadIdx.x, wg = tid >> 7;   // warpgroup: rows [64 wg, 64 wg + 64) of the tile
  const int rank = static_cast<int>(blockIdx.x) % RANKS, group = static_cast<int>(blockIdx.x) / RANKS;
  const int groups = static_cast<int>(gridDim.x) / RANKS;
  const int row_tiles = (p.N + BLOCK_M - 1) / BLOCK_M;
  const int n0 = rank * BLOCK_N;   // first logit column of this CTA
  const int G = p.gt.G;
  unsigned int* xch_counter = p.xch_counter + group * kFusedCounterStride;

  if (threadIdx.x == 0) {
    stamp(p.timing, 0);
    tma_prefetch_desc(&tmap_x);
    tma_prefetch_desc(&tmap_w);
    if (p.want_dz && p.dz_tma_cols > 0) tma_prefetch_desc(&tmap_dz);
#pragma unroll
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], Cfg::NUM_THREADS); }
    fence_mbar_init();
  }
  if (threadIdx.x < 16) s_loss[threadIdx.x] = 0.f;
  if (threadIdx.x < 4) s_slow[threadIdx.x] = 0ull;
  if (threadIdx.x < kMaxG) {
    int gs = 0, ge = 0;
#pragma unroll
    for (int i = 0; i < kMaxG; ++i)
      if (i == static_cast<int>(threadIdx.x)) { gs = p.gt.start[i]; ge = p.gt.start[i] + p.gt.len[i]; }
    s_gs[threadIdx.x] = gs;
    s_ge[threadIdx.x] = ge;
  }
  for (int c = threadIdx.x; c < BLOCK_N; c += Cfg::NUM_THREADS) {
    const int col = n0 + c;
    int b = -1;
#pragma unroll
    for (int i = 0; i < MAXG; ++i)
      if (i < G && col < p.C && col >= p.gt.start[i] && col < p.gt.start[i] + p.gt.len[i]) b = i;
    s_colbin[c] = b;
    s_bias[c] = (p.bias != nullptr && col < p.C) ? __ldg(p.bias + col) : 0.f;
  }
  // The walks below go over the thread's two columns 8J + 2q, 8J + 2q + 1 of every 8-column chunk J in column order,
  // keeping a running bin.  Chunk J is "slow" for quad lane q unless both columns lie in a bin (< C) and in the same
  // bin as the lane's last column of chunk J - 1 -- then the running bin is already theirs, and the walk needs no
  // bin lookup there.  Bins are contiguous, so a CTA has at most G + 1 bin changes plus the chunks at or past C.
  __syncthreads();   // s_colbin; s_slow is zero
  if (threadIdx.x < 4 * Cfg::CHUNKS) {
    const int qq = threadIdx.x & 3, J = threadIdx.x >> 2, c = 8 * J + 2 * qq;
    const int b0 = s_colbin[c], b1 = s_colbin[c + 1], bp = J > 0 ? s_colbin[c - 7] : -1;
    if (b0 < 0 || b1 != b0 || bp != b0) atomicOr(&s_slow[qq], 1ull << J);
  }
  __syncthreads();

  const int warp = (tid >> 5) & 3, lane = tid & 31, q = lane & 3;
  const int row_l0 = wg * 64 + warp * 16 + (lane >> 2);   // rows row_l0 and row_l0 + 8 of the tile
  // ===================== the group's row tiles: row_tile = group + tile_i * groups =====================
  // The k-blocks of all tiles are numbered in one sequence (it = tile_i * kblocks + kb): k-block `it` uses stage
  // it % STAGES in phase (it / STAGES) & 1, and every k-block releases its stage once, so the barriers simply
  // continue from one tile to the next.
  for (int row_tile = group, tile_i = 0; row_tile < row_tiles; row_tile += groups, ++tile_i) {
  const int m0 = row_tile * BLOCK_M;
  const int it0 = tile_i * p.kblocks;

  // TMA producer (thread 0): k-block kb of this tile goes to stage (it0 + kb) % STAGES
  auto issue = [&](int kb) {
    const int stage = (it0 + kb) % STAGES;
    mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
    const int k0 = kb * BLOCK_K;
    uint8_t* sa = smem_a + stage * Cfg::A_BYTES;
    uint8_t* sb = smem_b + stage * Cfg::B_BYTES;
    tma_load_2d(sa, &tmap_x, &full_bar[stage], k0, m0);
    tma_load_2d(sb, &tmap_w, &full_bar[stage], k0, n0);
    tma_load_2d(sb + HALF_N * 128, &tmap_w, &full_bar[stage], k0, n0 + HALF_N);
  };
  // the previous tile's dz left the stages through TMA stores, which must have read them before they are refilled
  if (tid == 0 && tile_i > 0) tma_store_wait_read<0>();
  for (int kb = 0; kb < STAGES && kb < p.kblocks; ++kb) {
    const int it = it0 + kb;
    // the stage is free once the previous tile's k-block it - STAGES has released it (all threads wait: see below)
    if (it >= STAGES) mbar_wait(&empty_bar[it % STAGES], static_cast<uint32_t>((it - STAGES) / STAGES) & 1u);
    if (tid == 0) issue(kb);
  }

  // ---- row information, part 1: the target column of every (row, bin) while the first stages load.  Labels and the
  // label -> bin-label table are not produced by the preceding kernel, so they are read before griddepcontrol.wait.
  // Thread t handles row t % 128 and bins t / 128, t / 128 + 2, t / 128 + 4. ----
  static_assert(Cfg::NUM_THREADS == 2 * BLOCK_M && MAXG == 6, "row information: two threads per row, three bins each");
  const int info_row = tid & (BLOCK_M - 1), info_g0 = tid / BLOCK_M;
  const bool info_ok = m0 + info_row < p.N;
  {
    const long long lab = info_ok ? __ldg(p.labels + m0 + info_row) : -1;
    const bool lab_ok = info_ok && lab >= 0 && lab < p.classes;
    for (int g = info_g0; g < G; g += 2) {
      int t = !lab_ok ? 0 : (p.l2b != nullptr ? __ldg(p.l2b + g * p.classes + static_cast<int>(lab)) : static_cast<int>(lab));
      t = (t >= 0 && t < s_ge[g] - s_gs[g]) ? t : 0;
      s_tcol[g * BLOCK_M + info_row] = s_gs[g] + t;
    }
  }

  // ===================== mainloop =====================
  float acc0[80], acc1[80];
#pragma unroll
  for (int j = 0; j < HALF_N / 8; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const float b0 = s_bias[8 * j + 2 * q + e], b1 = s_bias[HALF_N + 8 * j + 2 * q + e];
      acc0[4 * j + e] = b0; acc0[4 * j + 2 + e] = b0;
      acc1[4 * j + e] = b1; acc1[4 * j + 2 + e] = b1;
    }
  }
  {
    const uint32_t a_off = wg * 8192;   // this warpgroup's 64 rows of the A tile
    for (int kb = 0; kb < p.kblocks; ++kb) {
      const int stage = (it0 + kb) % STAGES;
      mbar_wait(&full_bar[stage], static_cast<uint32_t>((it0 + kb) / STAGES) & 1u);
      const uint32_t sa = smem_u32(smem_a + stage * Cfg::A_BYTES) + a_off;
      const uint32_t sb = smem_u32(smem_b + stage * Cfg::B_BYTES);
      fence_regs(acc0);
      fence_regs(acc1);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < Cfg::K_STEPS; ++k) {
        const uint64_t adesc = make_smem_desc(sa + k * 32, 16, 1024);
        const uint64_t bdesc0 = make_smem_desc(sb + k * 32, 16, 1024);
        const uint64_t bdesc1 = make_smem_desc(sb + HALF_N * 128 + k * 32, 16, 1024);
        if (TF32) { wgmma_tf32_n160(acc0, adesc, bdesc0, 1u); wgmma_tf32_n160(acc1, adesc, bdesc1, 1u); }
        else      { wgmma_bf16_n160<0, 0>(acc0, adesc, bdesc0, 1u); wgmma_bf16_n160<0, 0>(acc1, adesc, bdesc1, 1u); }
      }
      wgmma_commit();
      // keep this k-block's MMAs in flight; the previous k-block's are complete, so its stage can be refilled
      wgmma_wait<1>();
      fence_regs(acc0);
      fence_regs(acc1);
      if (kb > 0) {
        const int prev = it0 + kb - 1;
        // every thread arrives and waits, only the TMA issue is thread 0's: with the barrier wait inside a branch
        // that one thread takes, ptxas serialises the wgmma (C7518)
        mbar_arrive(&empty_bar[prev % STAGES]);
        if (kb - 1 + STAGES < p.kblocks) {   // once the whole CTA is done with the stage, refill it
          mbar_wait(&empty_bar[prev % STAGES], static_cast<uint32_t>(prev / STAGES) & 1u);
          if (tid == 0) issue(kb - 1 + STAGES);
        }
      }
    }
    wgmma_wait<0>();
    fence_regs(acc0);
    fence_regs(acc1);
    mbar_arrive(&empty_bar[(it0 + p.kblocks - 1) % STAGES]);   // the last k-block's stage, for the next tile
  }
  if (tid == 0) stamp(p.timing, 1);
  pdl_wait();   // every global write below comes after the predecessor grid

  // ---- row information, part 2: w / avg.  Masks and avg come from the preceding sampler kernel (programmatic
  // dependent launch), so they are read after the wait; they are stored after pass A, which hides the latency ----
  float info_coef[MAXG / 2];
#pragma unroll
  for (int i = 0; i < MAXG / 2; ++i) {
    const int g = info_g0 + 2 * i, row = m0 + info_row;
    float w = 0.f, inv_avg = 0.f;
    if (g < G) {
      if (info_ok)
        w = (p.wmask != nullptr)
                ? (WF ? __ldg(reinterpret_cast<const float*>(p.wmask) + static_cast<long long>(g) * p.N + row)
                      : static_cast<float>(__ldg(p.wmask + static_cast<long long>(g) * p.N + row)))
                : 1.0f;
      inv_avg = 1.0f / (p.avg != nullptr ? __ldg(p.avg + g) : fmaxf(static_cast<float>(p.N), 1.0f));
    }
    info_coef[i] = w * inv_avg;
  }

  // Walk the thread's 2 x 160 elements in column order, one 8-column chunk at a time:
  // F(accumulators, j, J, c): rows row_l0 / row_l0 + 8 x local columns c, c + 1 of chunk J are acc[4j], acc[4j + 1] /
  // acc[4j + 2], acc[4j + 3].  A chunk whose bit in `slow` is clear lies in the running bin (see s_slow): the walk
  // takes it without a bin lookup; the others go element by element through s_colbin.  (Computing the bin from the
  // kernel parameters instead costs more registers than the kernel has: ptxas spills.)
  const unsigned long long slow = s_slow[q];
#define BAGS_CHUNKS(F)                                                                                       \
  do {                                                                                                       \
    _Pragma("unroll") for (int j = 0; j < HALF_N / 8; ++j) F(acc0, j, j, 8 * j + 2 * q);                     \
    _Pragma("unroll") for (int j = 0; j < HALF_N / 8; ++j) F(acc1, j, HALF_N / 8 + j, HALF_N + 8 * j + 2 * q); \
  } while (0)
#define BAGS_IS_SLOW(J) (((slow >> (J)) & 1ull) != 0ull)
  // per-thread partials of (bin, row slot) -> s_part; the running pair is flushed where the bin changes
#define BAGS_PART(g, rr) s_part[((g) * 2 + (rr)) * 256 + tid]

  // ---- pass A: per-bin max over this thread's columns, then over the quad ----
#pragma unroll
  for (int g = 0; g < MAXG; ++g) BAGS_PART(g, 0) = BAGS_PART(g, 1) = -INFINITY;
  {
    int gc = -1;
    float mc[2] = {-INFINITY, -INFINITY};
    auto stepA = [&](float z0, float z1, int c) {
      const int b = s_colbin[c];
      if (b != gc) {
        if (gc >= 0) { BAGS_PART(gc, 0) = mc[0]; BAGS_PART(gc, 1) = mc[1]; }
        gc = b; mc[0] = mc[1] = -INFINITY;
      }
      mc[0] = fmaxf(mc[0], z0);
      mc[1] = fmaxf(mc[1], z1);
    };
    auto chunkA = [&](float (&a)[80], int j, int J, int c) {
      if (BAGS_IS_SLOW(J)) {
        stepA(a[4 * j], a[4 * j + 2], c);
        stepA(a[4 * j + 1], a[4 * j + 3], c + 1);
      } else {
        mc[0] = fmaxf(fmaxf(mc[0], a[4 * j]), a[4 * j + 1]);
        mc[1] = fmaxf(fmaxf(mc[1], a[4 * j + 2]), a[4 * j + 3]);
      }
    };
    BAGS_CHUNKS(chunkA);
    if (gc >= 0) { BAGS_PART(gc, 0) = mc[0]; BAGS_PART(gc, 1) = mc[1]; }
  }
  for (int g = 0; g < G; ++g) {
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      float m = BAGS_PART(g, rr);
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
      if (q == 0) s_mrow[g * BLOCK_M + row_l0 + 8 * rr] = m;
    }
  }
#pragma unroll
  for (int i = 0; i < MAXG / 2; ++i)
    if (info_g0 + 2 * i < G) s_coef[(info_g0 + 2 * i) * BLOCK_M + info_row] = info_coef[i];
  __syncthreads();   // s_tcol / s_coef of every row; s_mrow of the quad
  if (tid == 0) stamp(p.timing, 2);

  // ---- pass B: z := e = exp(z - max) in place, per-bin sum of e; z[target] for the loss ----
#pragma unroll
  for (int g = 0; g < MAXG; ++g) BAGS_PART(g, 0) = BAGS_PART(g, 1) = 0.f;
  {
    int gc = -1;
    float mb[2] = {0.f, 0.f}, sc[2] = {0.f, 0.f}, zt[2] = {0.f, 0.f};
    int tc[2] = {-1, -1};
    // z[target] is picked into a register on the way and stored where the bin ends, by the lane that holds the
    // target column (the target lies inside its bin)
    auto flushB = [&]() {
      if (gc >= 0) {
        BAGS_PART(gc, 0) = sc[0]; BAGS_PART(gc, 1) = sc[1];
#pragma unroll
        for (int rr = 0; rr < 2; ++rr)
          if (tc[rr] >= 0 && tc[rr] < BLOCK_N && ((tc[rr] >> 1) & 3) == q) s_zt[gc * BLOCK_M + row_l0 + 8 * rr] = zt[rr];
      }
    };
    auto expB = [&](float& z0, float& z1, int c) {
      zt[0] = (c == tc[0]) ? z0 : zt[0];
      zt[1] = (c == tc[1]) ? z1 : zt[1];
      z0 = exp2f(fmaf(z0, kLog2e, -mb[0]));
      z1 = exp2f(fmaf(z1, kLog2e, -mb[1]));
      sc[0] += z0;
      sc[1] += z1;
    };
    auto stepB = [&](float& z0, float& z1, int c) {
      const int b = s_colbin[c];
      if (b != gc) {
        flushB();
        gc = b; sc[0] = sc[1] = 0.f;
        if (b >= 0) {
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            mb[rr] = s_mrow[b * BLOCK_M + row_l0 + 8 * rr] * kLog2e;
            tc[rr] = s_tcol[b * BLOCK_M + row_l0 + 8 * rr] - n0;   // local column of the target
          }
        }
      }
      if (b >= 0) expB(z0, z1, c);
    };
    auto chunkB = [&](float (&a)[80], int j, int J, int c) {
      if (BAGS_IS_SLOW(J)) {
        stepB(a[4 * j], a[4 * j + 2], c);
        stepB(a[4 * j + 1], a[4 * j + 3], c + 1);
      } else {
        expB(a[4 * j], a[4 * j + 2], c);
        expB(a[4 * j + 1], a[4 * j + 3], c + 1);
      }
    };
    BAGS_CHUNKS(chunkB);
    flushB();
  }

  // ---- exchange: publish (max, sum) of every (row, bin) to the group's slot of this tile's parity ----
  // Two slots suffice: a CTA writes the slot of its tile i + 2 only after it has seen all four arrivals of tile i + 1,
  // and a peer arrives for tile i + 1 only after it has read its partials of tile i.
  float2* xch = p.xch + static_cast<size_t>(group * 2 + (tile_i & 1)) * Cfg::SLOT_ELEMS;   // [4 ranks][MAXG][128]
  {
    float2* mine = xch + rank * MAXG * BLOCK_M;
    for (int g = 0; g < G; ++g) {
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        float s = BAGS_PART(g, rr);
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        if (q == 0) {
          const int row_l = row_l0 + 8 * rr;
          mine[g * BLOCK_M + row_l] = make_float2(s_mrow[g * BLOCK_M + row_l], s);
        }
      }
    }
  }
#undef BAGS_PART
  __syncthreads();   // this CTA's partials are stored (and s_zt is complete)
  unsigned int xch_target = 0;
  if (tid == 0) {
    stamp(p.timing, 3);
    // Arrival counters are never reset: every tile adds four arrivals, so a tile's four arrivals are the ones that
    // take the counter to the next multiple of 4 -- across tiles, launches and graph replays on one stream.
    __threadfence();
    xch_target = (atom_add_release_gpu(xch_counter, 1u) & ~3u) + 4u;
  }
  // The optional buffer clear (a write: only after the wait -- the buffer may still be in use by an earlier kernel) is
  // issued while the peers' partials are awaited.
  if (tile_i == 0 && p.clear != nullptr) {
    const long long stride = static_cast<long long>(gridDim.x) * Cfg::NUM_THREADS;
    const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long i = static_cast<long long>(blockIdx.x) * Cfg::NUM_THREADS + tid; i < p.clear_vecs; i += stride)
      p.clear[i] = zero4;
  }
  if (tid == 0) {
    uint32_t spins = 0, ns = 32;
    while (static_cast<int>(ld_acquire_gpu(xch_counter) - xch_target) < 0) {
      if (++spins > BAGS_WAIT_LIMIT) __trap();
      __nanosleep(ns);
      ns = ns < 256 ? 2 * ns : 256;
    }
    stamp(p.timing, 4);
  }
  __syncthreads();   // all four CTAs' partials are visible (read through L2 below)
  // PDL INVARIANT: every CTA triggers once it runs -- here, after its first exchange -- and a dependent grid is launched
  // only after all CTAs of this grid have triggered, i.e. are resident.  So a dependent can never hold an SM that a CTA
  // of this grid still needs to become resident, which the waits on the group's peers rely on.  (Triggering here
  // rather than at the start of the kernel made the 4096-RoI benchmark step about 3 % faster on an H100 80GB HBM3 at
  // 400 W.)  Dependents guard their first dependent access with griddepcontrol.wait.
  if (tile_i == 0) pdl_trigger();
  {
    // The quad's 2 x G (row, bin) pairs k = 2 g + rr are spread over its four lanes (lane q: k = q, q + 4, q + 8), and
    // every lane issues all its L2 loads before it uses any.
    constexpr int PAIRS = 2 * MAXG / 4;
    float2 v[PAIRS][RANKS];
#pragma unroll
    for (int i = 0; i < PAIRS; ++i) {
      const int k = q + 4 * i, g = k >> 1, row_l = row_l0 + 8 * (k & 1);
#pragma unroll
      for (int s = 0; s < RANKS; ++s)
        v[i][s] = g < G ? __ldcg(&xch[(s * MAXG + g) * BLOCK_M + row_l]) : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int i = 0; i < PAIRS; ++i) {
      const int k = q + 4 * i, g = k >> 1, row_l = row_l0 + 8 * (k & 1), row = m0 + row_l;
      if (g < G) {
        const float M = fmaxf(fmaxf(v[i][0].x, v[i][1].x), fmaxf(v[i][2].x, v[i][3].x));
        float S = 0.f;
#pragma unroll
        for (int s = 0; s < RANKS; ++s)
          S += (v[i][s].x == -INFINITY) ? 0.f : v[i][s].y * exp2f((v[i][s].x - M) * kLog2e);
        const float lse_v = M + logf(S);
        const float cf = s_coef[g * BLOCK_M + row_l];
        s_scale[g * BLOCK_M + row_l] = exp2f((s_mrow[g * BLOCK_M + row_l] - lse_v) * kLog2e) * cf;
        const int tcol = s_tcol[g * BLOCK_M + row_l];
        if (tcol >= n0 && tcol < n0 + BLOCK_N) {
          const float zt = s_zt[g * BLOCK_M + row_l];
          if (cf != 0.f) atomicAdd(&s_loss[g], cf * (lse_v - zt));
          // top-1 accuracy (a comparison, not an argmax: a tie with the row max counts as correct); the count rides
          // the spare last slot of the per-CTA loss partials
          if (p.acc != nullptr && g == 0 && row < p.N && zt == M) atomicAdd(&s_loss[kMaxG - 1], 1.f);
        }
        if (p.lse != nullptr && row < p.N && s_gs[g] >= n0 && s_gs[g] < n0 + BLOCK_N)
          p.lse[static_cast<long long>(row) * G + g] = lse_v;
      }
    }
  }
  __syncwarp();   // s_scale of the quad
  // ---- pass C: dz -> the staged tile (operand dtype, the pipeline stages) -> TMA stores; column sums ----
  // Column c of the tile is column c % BOX_COLS of box c / BOX_COLS; a box row is 128 bytes whose 16-byte pieces are
  // swizzled with the row (piece ^ row % 8), as TMA SWIZZLE_128B expects.  Both rows of the thread have row % 8 =
  // lane / 4.  Columns >= C and rows >= N are staged like the others and never stored.
  if (p.want_dz) {
    constexpr int ELT = Cfg::ELT, BOX_BYTES = Cfg::BOX_BYTES;
    const int r8 = lane >> 2;
    uint8_t* const stg = smem + row_l0 * 128 + (TF32 ? 8 * (q & 1) : 4 * q);
    // stg: the thread's row and byte within a 16-byte piece; stage_off(J): box and swizzled piece of chunk J
    const uint32_t swz = TF32 ? static_cast<uint32_t>(((q >> 1) ^ r8) << 4) : static_cast<uint32_t>(r8 << 4);
    auto stage_off = [&](int J) -> uint32_t {
      return TF32 ? (J / 4) * BOX_BYTES + ((static_cast<uint32_t>(J % 4) << 5) ^ swz)
                  : (J / 8) * BOX_BYTES + ((static_cast<uint32_t>(J % 8) << 4) ^ swz);
    };
    int gc = -1;
    float sc[2] = {0.f, 0.f}, cf[2] = {0.f, 0.f};
    int tc[2] = {-1, -1};
    auto dzC = [&](float e, int rr, int c) {
      float v = e * sc[rr];
      if (c == tc[rr]) v -= cf[rr];
      return v;
    };
    auto stepC = [&](float e0, float e1, int c, float& d0, float& d1) {   // rows 0/1 x column c
      const int b = s_colbin[c];
      if (b != gc) {
        gc = b;
        if (b >= 0) {
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            sc[rr] = s_scale[b * BLOCK_M + row_l0 + 8 * rr];
            cf[rr] = s_coef[b * BLOCK_M + row_l0 + 8 * rr];
            tc[rr] = s_tcol[b * BLOCK_M + row_l0 + 8 * rr] - n0;
          }
        }
      }
      d0 = b >= 0 ? dzC(e0, 0, c) : 0.f;
      d1 = b >= 0 ? dzC(e1, 1, c) : 0.f;
    };
    auto chunkC = [&](float (&a)[80], int j, int J, int c) {
      float d[2][2];
      if (BAGS_IS_SLOW(J)) {
        stepC(a[4 * j], a[4 * j + 2], c, d[0][0], d[1][0]);
        stepC(a[4 * j + 1], a[4 * j + 3], c + 1, d[0][1], d[1][1]);
      } else {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          d[0][e] = dzC(a[4 * j + e], 0, c + e);
          d[1][e] = dzC(a[4 * j + 2 + e], 1, c + e);
        }
      }
      const uint32_t off = stage_off(J);
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        if (TF32) *reinterpret_cast<float2*>(stg + off + rr * 1024) = make_float2(d[rr][0], d[rr][1]);
        else      *reinterpret_cast<uint32_t*>(stg + off + rr * 1024) = pack_bf16x2(d[rr][0], d[rr][1]);
      }
    };
    BAGS_CHUNKS(chunkC);
    fence_proxy_async_smem();   // the staged tile is read by the TMA (async proxy)
    __syncthreads();
    if (tid == 0) {
#pragma unroll 1
      for (int bx = 0; bx < Cfg::BOXES; ++bx)
        if (n0 + bx * Cfg::BOX_COLS < p.dz_tma_cols)
          tma_store_2d(&tmap_dz, smem + bx * BOX_BYTES, n0 + bx * Cfg::BOX_COLS, m0);
      tma_store_commit();
    }
    // the last few columns [dz_tma_cols, C) (at most 16 bytes of a row, all in one CTA) take plain stores
    const int tail0 = max(p.dz_tma_cols, n0) - n0, tail = min(p.C, n0 + BLOCK_N) - n0 - tail0;
    if (tail > 0) {
      for (int i = tid; i < BLOCK_M * 8; i += Cfg::NUM_THREADS) {
        const int r = i >> 3, c = tail0 + (i & 7);
        if ((i & 7) < tail && m0 + r < p.N) {
          const int byte = (c % Cfg::BOX_COLS) * ELT;
          const uint8_t* a = smem + (c / Cfg::BOX_COLS) * BOX_BYTES + r * 128 + ((((byte >> 4) ^ r) & 7) << 4) + (byte & 15);
          uint8_t* dst = static_cast<uint8_t*>(p.dz) + (static_cast<long long>(m0 + r) * p.ldd + n0 + c) * ELT;
          if (TF32) *reinterpret_cast<float*>(dst) = *reinterpret_cast<const float*>(a);
          else      *reinterpret_cast<uint16_t*>(dst) = *reinterpret_cast<const uint16_t*>(a);
        }
      }
    }
    if (p.colsum != nullptr) {   // optional per-row-tile bias-gradient partials: the stored (rounded) values, in row order
      for (int c = tid; c < BLOCK_N; c += Cfg::NUM_THREADS) {
        if (n0 + c >= p.C) continue;
        const int byte = (c % Cfg::BOX_COLS) * ELT;
        const uint8_t* col = smem + (c / Cfg::BOX_COLS) * BOX_BYTES + (byte & 15);
        const int piece = byte >> 4;
        float s = 0.f;
#pragma unroll 8
        for (int r = 0; r < BLOCK_M; ++r) {
          const uint8_t* a = col + r * 128 + ((piece ^ (r & 7)) << 4);
          s += TF32 ? *reinterpret_cast<const float*>(a) : __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(a));
        }
        p.colsum[static_cast<long long>(row_tile) * p.C + n0 + c] = s;
      }
    }
  }
#undef BAGS_CHUNKS
#undef BAGS_IS_SLOW
  __syncthreads();   // the staged tile and the tile's shared row information are no longer read
  if (tid == 0) stamp(p.timing, 5);
  }   // row tiles
  if (tid < 32) {
    // ---- loss bookkeeping: per-CTA partials, the last CTA of the grid sums them in a fixed order ----
    unsigned int last = 0;
    if (lane == 0) {
      float4* dst = reinterpret_cast<float4*>(p.part + static_cast<size_t>(blockIdx.x) * kMaxG);
      dst[0] = make_float4(s_loss[0], s_loss[1], s_loss[2], s_loss[3]);
      dst[1] = make_float4(s_loss[4], s_loss[5], s_loss[6], s_loss[7]);
      last = (atom_add_release_gpu(p.counter, 1u) == gridDim.x - 1) ? 1u : 0u;   // release: the partials first
    }
    last = __shfl_sync(0xffffffffu, last, 0);
    if (last) {
      __threadfence();
      float accl[kMaxG];
#pragma unroll
      for (int g = 0; g < kMaxG; ++g) accl[g] = 0.f;
      for (int b = lane; b < static_cast<int>(gridDim.x); b += 32) {
        const float4* src = reinterpret_cast<const float4*>(p.part + static_cast<size_t>(b) * kMaxG);
        const float4 u = __ldcg(src), w = __ldcg(src + 1);
        accl[0] += u.x; accl[1] += u.y; accl[2] += u.z; accl[3] += u.w;
        accl[4] += w.x; accl[5] += w.y; accl[6] += w.z; accl[7] += w.w;
      }
#pragma unroll
      for (int g = 0; g < kMaxG; ++g) {
        const float t = warp_sum(accl[g]);
        if (lane == 0 && g < G) p.loss[g] = t;   // already divided by avg (coef = w/avg)
        if (lane == 0 && g == kMaxG - 1 && p.acc != nullptr) p.acc[0] = t * p.acc_scale;   // exact count (< 2^24)
      }
      if (lane == 0) *p.counter = 0u;
    }
  }
  if (tid == 0) {
    tma_store_wait_all();   // the dz stores have read the stages and are complete
    stamp(p.timing, 6);
  }
}

}  // namespace bags
