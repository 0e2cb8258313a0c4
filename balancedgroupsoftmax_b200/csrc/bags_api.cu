// C-ABI entry points of libbags_b200.so (see include/bags_b200.h).
// Host side only: argument validation, TMA descriptor encoding, kernel launches.
// No torch, no allocations, no device synchronisation.
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <utility>

#include "../../include/bags_b200.h"
#include "bags_gemm.cuh"
#include "bags_fused_fwd.cuh"
#include "bags_kernels.cuh"
#include "bags_allreduce.cuh"
#include "bags_nms.cuh"

using namespace bags;

// ----------------------------------------------------------------------------
// error handling
// ----------------------------------------------------------------------------
static thread_local std::string g_last_error;

static int fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return code;
}

#define BAGS_CUDA(expr)                                                                   \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess)                                                                \
      return fail(BAGS_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),  \
                  __FILE__, __LINE__);                                                    \
  } while (0)

#define BAGS_REQUIRE(cond, ...)                              \
  do {                                                       \
    if (!(cond)) return fail(BAGS_ERR_INVALID, __VA_ARGS__); \
  } while (0)

extern "C" int bags_abi_version(void) { return BAGS_ABI_VERSION; }
extern "C" const char* bags_last_error(void) { return g_last_error.c_str(); }

// ----------------------------------------------------------------------------
// per-process device info (SM count, arch check) and driver entry point
// ----------------------------------------------------------------------------
struct DeviceInfo {
  int num_sms = 0;
  int cc_major = 0;
};
static std::mutex g_mutex;
static DeviceInfo g_dev[64];
static bool g_dev_ok[64] = {false};

// test hook: device buffer [ctas][8] int64 that the next launches stamp with %globaltimer values
static long long* g_timing = nullptr;
extern "C" int bags_debug_set_timing(void* dev_ptr) {
  g_timing = reinterpret_cast<long long*>(dev_ptr);
  return BAGS_OK;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode = nullptr;

static int device_info(DeviceInfo& out) {
  int dev = 0;
  BAGS_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) return fail(BAGS_ERR_INVALID, "device index %d out of range", dev);
  std::lock_guard<std::mutex> lk(g_mutex);
  if (!g_dev_ok[dev]) {
    DeviceInfo d;
    BAGS_CUDA(cudaDeviceGetAttribute(&d.num_sms, cudaDevAttrMultiProcessorCount, dev));
    BAGS_CUDA(cudaDeviceGetAttribute(&d.cc_major, cudaDevAttrComputeCapabilityMajor, dev));
    g_dev[dev] = d;
    g_dev_ok[dev] = true;
  }
  out = g_dev[dev];
  if (out.cc_major != 9)
    return fail(BAGS_ERR_ARCH, "libbags_b200 is built for sm_90a (H100); found compute capability %d.x",
                out.cc_major);
  if (g_encode == nullptr) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    BAGS_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    if (fn == nullptr || qres != cudaDriverEntryPointSuccess)
      return fail(BAGS_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
    g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  }
  return BAGS_OK;
}

// 2-D row-major tensor [outer, inner] (inner contiguous), 128B-swizzled boxes.
static int make_tmap(CUtensorMap* tm, const void* ptr, int dtype, long long inner, long long outer,
                     long long ld_elems, int box_inner, int box_outer, bool atom32 = false, bool swz64 = false) {
  const int elt = (dtype == BAGS_DTYPE_BF16) ? 2 : 4;
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0)
    return fail(BAGS_ERR_INVALID, "operand pointer %p is not 16-byte aligned", ptr);
  if (((ld_elems * elt) & 15) != 0)
    return fail(BAGS_ERR_INVALID, "operand row stride %lld bytes is not a multiple of 16", ld_elems * elt);
  if (box_inner * elt != (swz64 ? 64 : 128)) return fail(BAGS_ERR_INVALID, "internal: box inner must span the swizzle width");
  cuuint64_t gdim[2] = {static_cast<cuuint64_t>(inner), static_cast<cuuint64_t>(outer)};
  cuuint64_t gstr[1] = {static_cast<cuuint64_t>(ld_elems * elt)};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(box_inner), static_cast<cuuint32_t>(box_outer)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(tm, dtype == BAGS_DTYPE_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32,
                        2, const_cast<void*>(ptr), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        swz64 ? CU_TENSOR_MAP_SWIZZLE_64B : (atom32 ? CU_TENSOR_MAP_SWIZZLE_128B_ATOM_32B : CU_TENSOR_MAP_SWIZZLE_128B),
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(BAGS_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d (inner=%lld outer=%lld ld=%lld box=%dx%d)",
                (int)r, inner, outer, ld_elems, box_inner, box_outer);
  return BAGS_OK;
}

static int make_group_table(GroupTable& gt, const int32_t* slices_host, int G, int C) {
  BAGS_REQUIRE(slices_host != nullptr, "slices_host is NULL");
  BAGS_REQUIRE(G >= 1 && G <= kMaxG, "G=%d outside [1,%d]", G, kMaxG);
  gt.G = G;
  int prev_end = 0;
  for (int g = 0; g < kMaxG; ++g) {
    gt.start[g] = 0;
    gt.len[g] = 0;
    if (g < G) {
      const int s = slices_host[2 * g], l = slices_host[2 * g + 1];
      BAGS_REQUIRE(s >= prev_end && l >= 1 && s + l <= C,
                   "pred_slice row %d = (%d,%d) is not an ascending, in-range slice of %d logits", g, s, l, C);
      gt.start[g] = s;
      gt.len[g] = l;
      prev_end = s + l;
    }
  }
  return BAGS_OK;
}

// Tuning / experiment switches come from the environment.  They are read ONCE per name (no getenv on the per-call path);
// bags_reload_env() drops the cache (tests flip switches inside one process).
struct EnvEntry { const char* name; bool set; int value; };
static EnvEntry g_env[96];
static int g_env_n = 0;
static std::mutex g_env_mutex;
static int env_int(const char* name, int dflt) {
  std::lock_guard<std::mutex> lk(g_env_mutex);
  for (int i = 0; i < g_env_n; ++i)
    if (g_env[i].name == name || strcmp(g_env[i].name, name) == 0) return g_env[i].set ? g_env[i].value : dflt;
  const char* v = getenv(name);
  EnvEntry e{name, v && *v, (v && *v) ? atoi(v) : 0};
  if (g_env_n < 96) g_env[g_env_n++] = e;
  return e.set ? e.value : dflt;
}
extern "C" int bags_reload_env(void) {
  std::lock_guard<std::mutex> lk(g_env_mutex);
  g_env_n = 0;
  return BAGS_OK;
}

// Kernel launch.  pdl: with the programmatic-stream-serialization attribute (PDL; BAGS_PDL=0 turns it off), so the
// kernel may begin while its predecessor in the stream is still running; every kernel of this library guards its
// first access to predecessor-produced data (and its first write) with griddepcontrol.wait, so stream semantics are
// preserved.  cooperative: the runtime guarantees that all CTAs of the grid are resident at once, and fails the launch
// when they cannot be (for kernels whose CTAs wait for each other).
template <typename... KArgs, typename... Args>
static cudaError_t launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl,
                          bool cooperative, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  unsigned n = 0;
  if (pdl && env_int("BAGS_PDL", 1)) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n++].val.programmaticStreamSerializationAllowed = 1;
  }
  if (cooperative) {
    attr[n].id = cudaLaunchAttributeCooperative;
    attr[n++].val.cooperative = 1;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// ----------------------------------------------------------------------------
// GEMM launcher
// ----------------------------------------------------------------------------
struct GemmArgs {
  const void* a; long long lda; bool a_mn;
  const void* b; long long ldb; bool b_mn;
  int M, N, K;
  int dtype;
  int splits;
  GemmParams p;  // epilogue fields pre-filled (out, ldo, bias, gscale, ...)
};

template <int BLOCK_N, bool A_MN, bool B_MN, int EPI, bool TF32, int STAGES>
static int launch_gemm(const GemmArgs& ga, const DeviceInfo& di, cudaStream_t stream, bool pdl = false) {
  using Cfg = GemmCfg<BLOCK_N, A_MN, B_MN, EPI, TF32, STAGES>;
  auto kernel = bags_gemm_kernel<BLOCK_N, A_MN, B_MN, EPI, TF32, STAGES>;
  CUtensorMap ta, tb;
  int rc;
  // A (an MN-major fp32 operand is read without TMA: the tensor map is still encoded, which validates alignment)
  if (A_MN) rc = make_tmap(&ta, ga.a, ga.dtype, ga.M, ga.K, ga.lda, Cfg::SLAB, Cfg::BLOCK_K);
  else      rc = make_tmap(&ta, ga.a, ga.dtype, ga.K, ga.M, ga.lda, Cfg::BLOCK_K, Cfg::BLOCK_M);
  if (rc) return rc;
  if (B_MN) rc = make_tmap(&tb, ga.b, ga.dtype, ga.N, ga.K, ga.ldb, Cfg::SLAB, Cfg::BLOCK_K);
  else      rc = make_tmap(&tb, ga.b, ga.dtype, ga.K, ga.N, ga.ldb, Cfg::BLOCK_K, BLOCK_N);
  if (rc) return rc;

  GemmParams p = ga.p;
  p.a_ptr = static_cast<const float*>(ga.a); p.lda = ga.lda; p.a_rows = ga.M; p.a_k = ga.K;
  p.b_ptr = static_cast<const float*>(ga.b); p.ldb = ga.ldb; p.b_rows = ga.N; p.b_k = ga.K;
  p.M = ga.M; p.N = ga.N; p.K = ga.K;
  p.num_m_tiles = (ga.M + Cfg::BLOCK_M - 1) / Cfg::BLOCK_M;
  p.num_n_tiles = (ga.N + BLOCK_N - 1) / BLOCK_N;
  p.kblocks_total = (ga.K + Cfg::BLOCK_K - 1) / Cfg::BLOCK_K;
  int splits = ga.splits < 1 ? 1 : ga.splits;
  if (splits > p.kblocks_total) splits = p.kblocks_total;
  if (EPI != EPI_RED_F32) splits = 1;
  p.num_splits = splits;
  const int units = p.num_m_tiles * p.num_n_tiles * splits;
  if (units == 0) return BAGS_OK;
  const int grid = units < di.num_sms ? units : di.num_sms;

  BAGS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
  BAGS_CUDA(launch(kernel, dim3(grid), dim3(Cfg::NUM_THREADS), Cfg::SMEM_BYTES, stream, pdl, false, ta, tb, p));
  return BAGS_OK;
}

static int pick_splits(int tiles, int kblocks, int num_sms) {
  int s = num_sms / (tiles > 0 ? tiles : 1);
  if (s < 1) s = 1;
  if (s > kblocks) s = kblocks;
  return s;
}

// ----------------------------------------------------------------------------
// public entry points
// ----------------------------------------------------------------------------
// workspace: loss counter (256 B) and per-CTA loss partials of up to 4096 CTAs, then the fused forward's exchange
// (arrival counters and slots of its CTA groups)
static constexpr size_t kLossWorkspaceBytes = 256 + 4096 * kMaxG * sizeof(float);
extern "C" size_t bags_workspace_bytes(void) { return kLossWorkspaceBytes + kFusedXchBytes; }

// y = act(x W^T + b): the head's shared FCs (ReLU), fc_reg and fc_cls (identity) on the same wgmma pipeline
// (convfc_bbox_head.py:138-143,166-167: nn.Linear + ReLU through cuBLAS / ATen in the reference)
extern "C" int bags_linear_act_fwd(const void* x, long long ldx, const void* w, long long ldw, const float* bias,
                                   void* out, long long ldo, int N, int K, int C, int dtype, int out_dtype, int relu,
                                   void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  BAGS_REQUIRE(N >= 0 && K >= 1 && C >= 1, "bags_linear_act_fwd: bad shape N=%d K=%d C=%d", N, K, C);
  BAGS_REQUIRE(N == 0 || (x && w && out), "bags_linear_act_fwd: NULL operand");
  BAGS_REQUIRE(dtype == BAGS_DTYPE_F32 || dtype == BAGS_DTYPE_BF16, "bags_linear_act_fwd: bad dtype %d", dtype);
  BAGS_REQUIRE(out_dtype == BAGS_DTYPE_F32 || (out_dtype == BAGS_DTYPE_BF16 && dtype == BAGS_DTYPE_BF16),
               "bags_linear_act_fwd: output dtype %d not available for operand dtype %d", out_dtype, dtype);
  BAGS_REQUIRE(ldx >= K && ldw >= K && ldo >= C, "bags_linear_act_fwd: leading dimension smaller than row");
  if (N == 0) return BAGS_OK;
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  if (out_dtype == BAGS_DTYPE_F32) {
    BAGS_REQUIRE(bias == nullptr || (reinterpret_cast<uintptr_t>(bias) & 15) == 0,
                 "bags_linear_act_fwd: bias must be 16-byte aligned");
    BAGS_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0, "bags_linear_act_fwd: out must be 16-byte aligned");
  }
  GemmArgs ga{};
  ga.a = x; ga.lda = ldx; ga.a_mn = false;
  ga.b = w; ga.ldb = ldw; ga.b_mn = false;
  ga.M = N; ga.N = C; ga.K = K; ga.dtype = dtype; ga.splits = 1;
  ga.p.out = out; ga.p.ldo = ldo; ga.p.bias = bias; ga.p.relu = relu ? 1 : 0;
  if (dtype == BAGS_DTYPE_BF16)
    return out_dtype == BAGS_DTYPE_BF16 ? launch_gemm<256, false, false, EPI_STORE_BF16, false, 4>(ga, di, stream)
                                        : launch_gemm<256, false, false, EPI_STORE_F32, false, 4>(ga, di, stream);
  return launch_gemm<256, false, false, EPI_STORE_F32, true, 4>(ga, di, stream);
}

// Split-K factor worth using for a forward layer (1 = the single-pass kernel): few output tiles and a long contraction --
// shared_fcs.0 at 2 x 512 RoIs is 8 x 4 tiles of 128 x 256 with K = 12544, i.e. 32 busy SMs out of 132 without it.
extern "C" int bags_linear_act_splits(int N, int K, int C, int dtype) {
  DeviceInfo di;
  if (device_info(di)) return 1;
  const int tiles = ((N + 127) / 128) * ((C + 255) / 256);
  const int kblocks = (K + (dtype == BAGS_DTYPE_BF16 ? 63 : 31)) / (dtype == BAGS_DTYPE_BF16 ? 64 : 32);
  if (tiles <= 0 || tiles * 2 > di.num_sms || kblocks < 16) return 1;
  int s = di.num_sms / tiles;
  if (s > kblocks / 4) s = kblocks / 4;
  return s < 2 ? 1 : (s > 16 ? 16 : s);
}

// Two-pass forward for such layers: split-K GEMM with red.add into a zeroed fp32 workspace [N, ldws], then
// out = act(ws + bias) in the output dtype.
extern "C" int bags_linear_act_fwd_splitk(const void* x, long long ldx, const void* w, long long ldw, const float* bias,
                                          void* out, long long ldo, int N, int K, int C, int dtype, int out_dtype, int relu,
                                          float* ws, long long ldws, int splits, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  BAGS_REQUIRE(N >= 0 && K >= 1 && C >= 1, "bags_linear_act_fwd_splitk: bad shape N=%d K=%d C=%d", N, K, C);
  BAGS_REQUIRE(N == 0 || (x && w && out && ws), "bags_linear_act_fwd_splitk: NULL operand");
  BAGS_REQUIRE(dtype == BAGS_DTYPE_F32 || dtype == BAGS_DTYPE_BF16, "bags_linear_act_fwd_splitk: bad dtype %d", dtype);
  BAGS_REQUIRE(out_dtype == BAGS_DTYPE_F32 || out_dtype == BAGS_DTYPE_BF16, "bags_linear_act_fwd_splitk: bad output dtype");
  BAGS_REQUIRE(ldx >= K && ldw >= K && ldo >= C && ldws >= C && (ldws % 4) == 0 && splits >= 2,
               "bags_linear_act_fwd_splitk: bad leading dimension / split count");
  BAGS_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "bags_linear_act_fwd_splitk: workspace must be 16-byte aligned");
  if (N == 0) return BAGS_OK;
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  BAGS_CUDA(cudaMemsetAsync(ws, 0, sizeof(float) * static_cast<size_t>(N) * static_cast<size_t>(ldws), stream));
  GemmArgs ga{};
  ga.a = x; ga.lda = ldx; ga.a_mn = false;
  ga.b = w; ga.ldb = ldw; ga.b_mn = false;
  ga.M = N; ga.N = C; ga.K = K; ga.dtype = dtype; ga.splits = splits;
  ga.p.out = ws; ga.p.ldo = ldws;
  int rc = (dtype == BAGS_DTYPE_BF16) ? launch_gemm<256, false, false, EPI_RED_F32, false, 4>(ga, di, stream)
                                      : launch_gemm<256, false, false, EPI_RED_F32, true, 4>(ga, di, stream);
  if (rc) return rc;
  const long long quads = static_cast<long long>(N) * ((C + 3) / 4);
  long long grid = (quads + 255) / 256;
  if (grid > 132 * 8) grid = 132 * 8;
  if (out_dtype == BAGS_DTYPE_BF16)
    bias_act_store_kernel<true><<<static_cast<unsigned>(grid), 256, 0, stream>>>(ws, ldws, bias, out, ldo, N, C, relu ? 1 : 0);
  else
    bias_act_store_kernel<false><<<static_cast<unsigned>(grid), 256, 0, stream>>>(ws, ldws, bias, out, ldo, N, C, relu ? 1 : 0);
  BAGS_CUDA(cudaGetLastError());
  return BAGS_OK;
}

// g = (y > 0 ? dy : 0) in the operand dtype of the backward contractions (y == NULL: g = dy, i.e. a cast)
extern "C" int bags_act_bwd(const void* dy, long long lddy, int dy_dtype, const void* y, long long ldy, int y_dtype,
                            void* g, long long ldg, int g_dtype, int rows, int cols, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  BAGS_REQUIRE(rows >= 0 && cols >= 0 && (cols % 4) == 0, "bags_act_bwd: cols must be a multiple of 4");
  if (rows == 0 || cols == 0) return BAGS_OK;
  BAGS_REQUIRE(dy && g, "bags_act_bwd: NULL argument");
  BAGS_REQUIRE(lddy >= cols && ldg >= cols && (ldg % 4) == 0 && (y == nullptr || ldy >= cols), "bags_act_bwd: bad leading dimension");
  BAGS_REQUIRE((reinterpret_cast<uintptr_t>(g) & 15) == 0, "bags_act_bwd: g must be 16-byte aligned");
  const bool f_dy = dy_dtype == BAGS_DTYPE_F32, f_y = y_dtype == BAGS_DTYPE_F32, f_g = g_dtype == BAGS_DTYPE_F32;
  const long long quads = static_cast<long long>(rows) * (cols / 4);
  long long grid = (quads + 255) / 256;
  if (grid > 132 * 8) grid = 132 * 8;
  const dim3 gr(static_cast<unsigned>(grid)), bl(256);
  typedef __nv_bfloat16 bf;
#define BAGS_ACT(TDY, TY, OB) act_bwd_kernel<TDY, TY, OB><<<gr, bl, 0, stream>>>(                                   \
      static_cast<const TDY*>(dy), lddy, static_cast<const TY*>(y), ldy, g, ldg, rows, cols)
  if (f_dy && f_y && f_g) BAGS_ACT(float, float, false);
  else if (f_dy && f_y) BAGS_ACT(float, float, true);
  else if (f_dy && f_g) BAGS_ACT(float, bf, false);
  else if (f_dy) BAGS_ACT(float, bf, true);
  else if (f_y && f_g) BAGS_ACT(bf, float, false);
  else if (f_y) BAGS_ACT(bf, float, true);
  else if (f_g) BAGS_ACT(bf, bf, false);
  else BAGS_ACT(bf, bf, true);
#undef BAGS_ACT
  BAGS_CUDA(cudaGetLastError());
  return BAGS_OK;
}

extern "C" int bags_sample_others(const int64_t* labels, const int32_t* label2bin, int N, int G,
                                  int classes, double ratio, uint64_t seed, const uint64_t* seed_step,
                                  uint8_t* wmask, float* avg, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  BAGS_REQUIRE(labels && label2bin && wmask && avg, "bags_sample_others: NULL argument");
  BAGS_REQUIRE(G >= 1 && G <= kMaxG && classes >= 1 && N >= 0, "bags_sample_others: bad shape");
  BAGS_REQUIRE(ratio >= 0.0, "bags_sample_others: negative ratio");
  const long long* lab = reinterpret_cast<const long long*>(labels);
  const unsigned long long sd = static_cast<unsigned long long>(seed);
  const unsigned long long* st = reinterpret_cast<const unsigned long long*>(seed_step);
  auto kernel = N <= 4096 ? sample_others_kernel<4> : N <= 16384 ? sample_others_kernel<16> : sample_others_kernel<0>;
  BAGS_CUDA(launch(kernel, dim3(G), dim3(1024), 0, stream, true, false, lab, label2bin, classes, G, N, ratio, sd, wmask, avg, st));
  return BAGS_OK;
}

extern "C" int bags_mask_avg(const uint8_t* wmask, int N, int G, float* avg, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  BAGS_REQUIRE(wmask && avg, "bags_mask_avg: NULL argument");
  BAGS_REQUIRE(G >= 1 && G <= kMaxG && N >= 0, "bags_mask_avg: bad shape");
  mask_avg_kernel<<<G, 256, 0, stream>>>(wmask, N, avg);
  BAGS_CUDA(cudaGetLastError());
  return BAGS_OK;
}

template <int NV>
static int launch_group_ce(const float* logits, long long ldz, const int64_t* labels,
                           const int32_t* label2bin, const GroupTable& gt, const uint8_t* wmask, bool wf,
                           const float* avg, int N, int C, int classes, float* loss, float* lse,
                           void* dz, long long ldd, int dz_dtype, float* colsum, void* workspace,
                           int num_sms, cudaStream_t stream) {
  const int smem = 8 * NV * 128 * (int)sizeof(float);
  // persistent CTAs (2 per SM: 126 regs x 256 threads): every CTA walks several row octets so the
  // bias-gradient column sums are reduced in registers/smem and hit global atomics once per CTA
  int per_sm = (200 * 1024) / (smem + 2048);
  if (per_sm > 2) per_sm = 2;
  if (per_sm < 1) per_sm = 1;
  int grid = (N + 7) / 8;
  if (grid > num_sms * per_sm) grid = num_sms * per_sm;
  if (grid > 4096) grid = 4096;
  if (grid < 1) grid = 1;
  unsigned int* counter = reinterpret_cast<unsigned int*>(workspace);
  float* part = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 256);
  const long long* lab = reinterpret_cast<const long long*>(labels);
  const bool dz_f32 = dz_dtype == BAGS_DTYPE_F32;
  auto k = wf ? (dz_f32 ? group_ce_kernel<NV, true, true> : group_ce_kernel<NV, false, true>)
              : (dz_f32 ? group_ce_kernel<NV, true> : group_ce_kernel<NV, false>);
  BAGS_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  k<<<grid, 256, smem, stream>>>(logits, ldz, lab, label2bin, classes, gt, wmask, avg, N, C, loss, lse, dz, ldd,
                                 colsum, part, counter);
  BAGS_CUDA(cudaGetLastError());
  return BAGS_OK;
}

extern "C" int bags_group_ce(const float* logits, long long ldz, const int64_t* labels,
                             const int32_t* label2bin, const int32_t* slices_host, const void* weights,
                             int weights_dtype, const float* avg, int N, int C, int G, int classes, float* loss,
                             float* lse, void* dz, long long ldd, int dz_dtype, float* colsum, void* workspace,
                             size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  BAGS_REQUIRE(label2bin && loss && workspace && (N == 0 || (logits && labels)), "bags_group_ce: NULL argument");
  BAGS_REQUIRE(weights_dtype == BAGS_WEIGHTS_U8 || weights_dtype == BAGS_WEIGHTS_F32,
               "bags_group_ce: bad weights dtype %d", weights_dtype);
  BAGS_REQUIRE(workspace_bytes >= bags_workspace_bytes(), "bags_group_ce: workspace too small (%zu < %zu)",
               workspace_bytes, bags_workspace_bytes());
  BAGS_REQUIRE(N >= 0 && C >= 4 && (C % 4) == 0 && C <= 4096, "bags_group_ce: C=%d must be a multiple of 4 in [4,4096]", C);
  BAGS_REQUIRE((ldz % 4) == 0 && ldz >= C, "bags_group_ce: ldz=%lld must be a multiple of 4 and >= C", ldz);
  BAGS_REQUIRE((reinterpret_cast<uintptr_t>(logits) & 15) == 0, "bags_group_ce: logits not 16-byte aligned");
  if (N == 0) dz = nullptr;
  BAGS_REQUIRE(dz_dtype == BAGS_DTYPE_F32 || dz_dtype == BAGS_DTYPE_BF16, "bags_group_ce: bad dz dtype");
  if (dz != nullptr) {
    BAGS_REQUIRE(ldd >= C && (ldd % 8) == 0, "bags_group_ce: ldd=%lld must be a multiple of 8 and >= C", ldd);
    BAGS_REQUIRE((reinterpret_cast<uintptr_t>(dz) & 15) == 0, "bags_group_ce: dz not 16-byte aligned");
  }
  if (colsum != nullptr)
    BAGS_REQUIRE((reinterpret_cast<uintptr_t>(colsum) & 15) == 0, "bags_group_ce: colsum not 16-byte aligned");
  GroupTable gt;
  if (int rc = make_group_table(gt, slices_host, G, C)) return rc;
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  if (colsum != nullptr) BAGS_CUDA(cudaMemsetAsync(colsum, 0, sizeof(float) * C, stream));
  if (N == 0) {
    BAGS_CUDA(cudaMemsetAsync(loss, 0, sizeof(float) * G, stream));
    return BAGS_OK;
  }
  const uint8_t* wmask = static_cast<const uint8_t*>(weights);
  const bool wf = weights_dtype == BAGS_WEIGHTS_F32;
  const int nv = (C / 4 + 31) / 32;
  if (nv <= 10)
    return launch_group_ce<10>(logits, ldz, labels, label2bin, gt, wmask, wf, avg, N, C, classes, loss, lse, dz, ldd,
                               dz_dtype, colsum, workspace, di.num_sms, stream);
  if (nv <= 16)
    return launch_group_ce<16>(logits, ldz, labels, label2bin, gt, wmask, wf, avg, N, C, classes, loss, lse, dz, ldd,
                               dz_dtype, colsum, workspace, di.num_sms, stream);
  return launch_group_ce<32>(logits, ldz, labels, label2bin, gt, wmask, wf, avg, N, C, classes, loss, lse, dz, ldd,
                             dz_dtype, colsum, workspace, di.num_sms, stream);
}


// ----------------------------------------------------------------------------
// fused forward (GEMM + grouped softmax-CE in one kernel)
// ----------------------------------------------------------------------------
static bool fused_eligible(const int32_t* slices_host, int G, int C) {
  if (slices_host == nullptr || G < 1 || G > FusedCfg<false>::MAXG || C > 4 * FusedCfg<false>::BLOCK_N || (C % 4) != 0)
    return false;
  int end = 0;
  for (int g = 0; g < G; ++g) {   // bins must tile [0, C) contiguously
    if (slices_host[2 * g] != end || slices_host[2 * g + 1] < 1) return false;
    end += slices_host[2 * g + 1];
  }
  return end == C;
}

extern "C" int bags_fused_eligible(const int32_t* slices_host, int G, int C) {
  return fused_eligible(slices_host, G, C) ? 1 : 0;
}

template <bool TF32>
static int launch_fused_fwd(const void* x, long long ldx, const void* w, long long ldw, const FusedFwdParams& p0,
                            void* dz, long long ldd, int num_sms, cudaStream_t stream, bool wf) {
  using Cfg = FusedCfg<TF32>;
  const int dtype = TF32 ? BAGS_DTYPE_F32 : BAGS_DTYPE_BF16;
  CUtensorMap tx, tw;
  int rc = make_tmap(&tx, x, dtype, p0.K, p0.N, ldx, Cfg::BLOCK_K, Cfg::BLOCK_M);
  if (rc) return rc;
  rc = make_tmap(&tw, w, dtype, p0.K, p0.C, ldw, Cfg::BLOCK_K, Cfg::HALF_N);
  if (rc) return rc;
  if (dz != nullptr && (reinterpret_cast<uintptr_t>(dz) & 15) != 0)
    return fail(BAGS_ERR_INVALID, "bags_fwd: dz must be 16-byte aligned");
  // dz [N, C] with row stride ldd: the kernel stages each tile's dz in shared memory and stores it with TMA in boxes
  // of 128 bytes x 128 rows.  A TMA store writes whole 16-byte pieces at the tensor's right edge, so the map spans the
  // columns up to the last 16-byte boundary at or before C; the kernel writes the rest, and the padding columns
  // [C, ldd) stay untouched.
  const int dz_tma_cols = p0.C & ~(16 / Cfg::ELT - 1);
  CUtensorMap tdz{};
  if (dz != nullptr && dz_tma_cols > 0) {
    rc = make_tmap(&tdz, dz, dtype, dz_tma_cols, p0.N, ldd, Cfg::BOX_COLS, Cfg::BLOCK_M);
    if (rc) return rc;
  }
  FusedFwdParams p = p0;
  p.dz = dz;
  p.ldd = ldd;
  p.dz_tma_cols = dz != nullptr ? dz_tma_cols : 0;
  p.kblocks = (p.K + Cfg::BLOCK_K - 1) / Cfg::BLOCK_K;
  p.want_dz = dz != nullptr ? 1 : 0;
  p.timing = g_timing;   // rows [0, grid) (grid <= 4 * kFusedMaxGroups); the gradient exchange stamps from row 4096
  auto kernel = wf ? bags_fwd_fused_kernel<TF32, true> : bags_fwd_fused_kernel<TF32, false>;
  BAGS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
  // persistent grid of CTA groups, all resident at once: the four CTAs of a group wait for each other's softmax
  // partials.  At 4096 RoIs on 132 SMs this is 32 groups, i.e. 128 CTAs in one wave.
  int per_sm = 0;
  BAGS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, Cfg::NUM_THREADS, Cfg::SMEM_BYTES));
  const int row_tiles = (p.N + Cfg::BLOCK_M - 1) / Cfg::BLOCK_M;
  int groups = num_sms * per_sm / Cfg::RANKS;
  if (groups > row_tiles) groups = row_tiles;
  if (groups > kFusedMaxGroups) groups = kFusedMaxGroups;
  if (groups < 1)
    return fail(BAGS_ERR_CUDA, "bags_fwd: the fused kernel cannot keep %d CTAs resident (%d SMs, %d CTA(s) per SM)",
                Cfg::RANKS, num_sms, per_sm);
  const int grid = Cfg::RANKS * groups;
  // PDL INVARIANT (also the sampler's): this kernel reads x, W, bias, labels and label2bin BEFORE its
  // griddepcontrol.wait (only the sampler's masks / avg and every global write come after it).  That is correct as long as those tensors are not
  // produced by the immediately preceding kernel of the stream with an early launch_dependents trigger -- true for torch
  // kernels (they never trigger early) and for this library's own chain (the predecessor is the sampler / the previous
  // step's backward or exchange, none of which writes them).  A future producer that triggers early must be followed by
  // a non-PDL launch (BAGS_PDL=0) or move these reads behind the wait.
  // The cooperative launch fails (BAGS_ERR_CUDA) rather than hangs when the grid cannot be co-resident, e.g. on a part
  // with fewer SMs than the device query reported or under an MPS limit.  Every CTA triggers its dependents only while
  // it runs (after its first exchange), so a dependent grid cannot take an SM that a not yet resident CTA of this grid
  // needs.
  BAGS_CUDA(launch(kernel, dim3(grid), dim3(Cfg::NUM_THREADS), Cfg::SMEM_BYTES, stream, true, true, tx, tw, tdz, p));
  return BAGS_OK;
}

extern "C" int bags_fwd(const void* x, long long ldx, const void* w, long long ldw,
                        const float* bias, const int64_t* labels, const int32_t* label2bin,
                        const int32_t* slices_host, const void* weights, int weights_dtype, const float* avg,
                        int N, int K, int C, int G, int classes, int dtype, float* logits, long long ldz,
                        float* loss, float* lse, void* dz, long long ldd, float* colsum,
                        int colsum_tiles, void* workspace, size_t workspace_bytes, void* clear, size_t clear_bytes,
                        void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  BAGS_REQUIRE(weights_dtype == BAGS_WEIGHTS_U8 || weights_dtype == BAGS_WEIGHTS_F32,
               "bags_fwd: bad weights dtype %d", weights_dtype);
  if (clear != nullptr) {
    BAGS_REQUIRE((reinterpret_cast<uintptr_t>(clear) & 15) == 0 && (clear_bytes % 16) == 0,
                 "bags_fwd: the buffer to clear must be 16-byte aligned and a multiple of 16 bytes");
    if (logits != nullptr || N == 0) {   // not the fused kernel: a plain memset
      BAGS_CUDA(cudaMemsetAsync(clear, 0, clear_bytes, stream));
      clear = nullptr;
    }
  }
  if (colsum != nullptr)
    BAGS_REQUIRE(colsum_tiles >= 1 && (logits != nullptr || colsum_tiles == (N + 127) / 128 || N == 0),
                 "bags_fwd: colsum must hold ceil(N/128) = %d row tiles of C floats (got %d)", (N + 127) / 128, colsum_tiles);
  if (logits != nullptr) {
    // caller wants materialised logits: GEMM with fp32 store, then the stand-alone grouped CE (tile 0 holds
    // the column sums, the other tiles are zero)
    if (colsum != nullptr && colsum_tiles > 1)
      BAGS_CUDA(cudaMemsetAsync(colsum, 0, sizeof(float) * C * colsum_tiles, stream));
    if (int rc = bags_linear_act_fwd(x, ldx, w, ldw, bias, logits, ldz, N, K, C, dtype, BAGS_DTYPE_F32, 0, stream_))
      return rc;
    return bags_group_ce(logits, ldz, labels, label2bin, slices_host, weights, weights_dtype, avg, N, C, G, classes,
                         loss, lse, dz, ldd, dtype, colsum, workspace, workspace_bytes, stream_);
  }
  // fused path: logits stay in registers
  BAGS_REQUIRE(fused_eligible(slices_host, G, C),
               "bags_fwd: logits == NULL requests the fused kernel, but this bin table / C=%d / G=%d is not eligible "
               "(see bags_fused_eligible); pass a logits workspace", C, G);
  BAGS_REQUIRE(dtype == BAGS_DTYPE_F32 || dtype == BAGS_DTYPE_BF16, "bags_fwd: bad dtype %d", dtype);
  BAGS_REQUIRE(label2bin && loss && workspace && (N == 0 || (x && w && labels)), "bags_fwd: NULL argument");
  BAGS_REQUIRE(workspace_bytes >= bags_workspace_bytes(), "bags_fwd: workspace too small");
  BAGS_REQUIRE(N >= 0 && K >= 1, "bags_fwd: bad shape");
  if (dz != nullptr) BAGS_REQUIRE(ldd >= C && (ldd % 8) == 0, "bags_fwd: ldd=%lld must be a multiple of 8 and >= C", ldd);
  GroupTable gt;
  if (int rc = make_group_table(gt, slices_host, G, C)) return rc;
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  if (N == 0) {
    BAGS_CUDA(cudaMemsetAsync(loss, 0, sizeof(float) * G, stream));
    if (colsum != nullptr) BAGS_CUDA(cudaMemsetAsync(colsum, 0, sizeof(float) * C * colsum_tiles, stream));
    return BAGS_OK;
  }
  if (bias != nullptr) BAGS_REQUIRE((reinterpret_cast<uintptr_t>(bias) & 15) == 0, "bags_fwd: bias must be 16-byte aligned");
  FusedFwdParams p{};
  p.N = N; p.C = C; p.K = K; p.gt = gt; p.bias = bias;
  p.labels = reinterpret_cast<const long long*>(labels);
  p.l2b = label2bin; p.classes = classes; p.wmask = static_cast<const uint8_t*>(weights); p.avg = avg;
  p.loss = loss; p.lse = lse; p.colsum = colsum;
  p.counter = reinterpret_cast<unsigned int*>(workspace);
  p.part = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 256);
  p.xch_counter = reinterpret_cast<unsigned int*>(reinterpret_cast<char*>(workspace) + kLossWorkspaceBytes);
  p.xch = reinterpret_cast<float2*>(reinterpret_cast<char*>(workspace) + kLossWorkspaceBytes + kFusedXchCounterBytes);
  p.clear = reinterpret_cast<float4*>(clear);
  p.clear_vecs = static_cast<long long>(clear_bytes / 16);
  const bool wf = weights_dtype == BAGS_WEIGHTS_F32;
  return dtype == BAGS_DTYPE_BF16 ? launch_fused_fwd<false>(x, ldx, w, ldw, p, dz, ldd, di.num_sms, stream, wf)
                                  : launch_fused_fwd<true>(x, ldx, w, ldw, p, dz, ldd, di.num_sms, stream, wf);
}

// fc_cls + plain softmax CE over all C logits (ReweightBBoxHead, BBoxHead.loss): the fused kernel with one bin (0, C),
// the label as the target column (l2b == nullptr) and fp32 per-RoI weights.  Unlike bags_fwd, C need not be a
// multiple of 4 (1231 LVIS classes): the kernel reads the bias and writes the column sums with scalar accesses and
// stores dz in pairs of even columns, which only needs ldd % 8 == 0.
extern "C" int bags_ce_fwd(const void* x, long long ldx, const void* w, long long ldw, const float* bias,
                           const int64_t* labels, const float* weights, const float* avg, int N, int K, int C,
                           int dtype, float* loss, float* acc, void* dz, long long ldd, float* colsum,
                           int colsum_tiles, void* workspace, size_t workspace_bytes, void* clear, size_t clear_bytes,
                           void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  constexpr int kMaxC = FusedCfg<false>::RANKS * FusedCfg<false>::BLOCK_N;
  BAGS_REQUIRE(dtype == BAGS_DTYPE_F32 || dtype == BAGS_DTYPE_BF16, "bags_ce_fwd: bad dtype %d", dtype);
  BAGS_REQUIRE(N >= 0 && K >= 1 && C >= 1 && C <= kMaxC, "bags_ce_fwd: bad shape N=%d K=%d C=%d (1 <= C <= %d)", N, K,
               C, kMaxC);
  BAGS_REQUIRE(loss && workspace && (N == 0 || (x && w && labels)), "bags_ce_fwd: NULL argument");
  BAGS_REQUIRE(workspace_bytes >= bags_workspace_bytes(), "bags_ce_fwd: workspace too small (%zu < %zu)",
               workspace_bytes, bags_workspace_bytes());
  BAGS_REQUIRE(acc == nullptr || N <= (1 << 24),
               "bags_ce_fwd: N=%d: the accuracy count is exact up to 2^24 rows only", N);
  if (dz != nullptr) BAGS_REQUIRE(ldd >= C && (ldd % 8) == 0, "bags_ce_fwd: ldd=%lld must be a multiple of 8 and >= C", ldd);
  if (colsum != nullptr)
    BAGS_REQUIRE(colsum_tiles == (N + 127) / 128 || (N == 0 && colsum_tiles >= 1),
                 "bags_ce_fwd: colsum must hold ceil(N/128) = %d row tiles of C floats (got %d)", (N + 127) / 128,
                 colsum_tiles);
  if (clear != nullptr)
    BAGS_REQUIRE((reinterpret_cast<uintptr_t>(clear) & 15) == 0 && (clear_bytes % 16) == 0,
                 "bags_ce_fwd: the buffer to clear must be 16-byte aligned and a multiple of 16 bytes");
  const int32_t slices[2] = {0, C};
  GroupTable gt;
  if (int rc = make_group_table(gt, slices, 1, C)) return rc;
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  if (N == 0) {
    BAGS_CUDA(cudaMemsetAsync(loss, 0, sizeof(float), stream));
    if (acc != nullptr) BAGS_CUDA(cudaMemsetAsync(acc, 0, sizeof(float), stream));
    if (colsum != nullptr) BAGS_CUDA(cudaMemsetAsync(colsum, 0, sizeof(float) * C * colsum_tiles, stream));
    if (clear != nullptr) BAGS_CUDA(cudaMemsetAsync(clear, 0, clear_bytes, stream));
    return BAGS_OK;
  }
  FusedFwdParams p{};
  p.N = N; p.C = C; p.K = K; p.gt = gt; p.bias = bias;
  p.labels = reinterpret_cast<const long long*>(labels);
  p.l2b = nullptr; p.classes = C;
  p.wmask = reinterpret_cast<const uint8_t*>(weights); p.avg = avg;
  p.loss = loss; p.acc = acc; p.acc_scale = static_cast<float>(100.0 / N);   // accuracy.py: correct * (100.0 / N)
  p.lse = nullptr; p.colsum = colsum;
  p.counter = reinterpret_cast<unsigned int*>(workspace);
  p.part = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 256);
  p.xch_counter = reinterpret_cast<unsigned int*>(reinterpret_cast<char*>(workspace) + kLossWorkspaceBytes);
  p.xch = reinterpret_cast<float2*>(reinterpret_cast<char*>(workspace) + kLossWorkspaceBytes + kFusedXchCounterBytes);
  p.clear = reinterpret_cast<float4*>(clear);
  p.clear_vecs = static_cast<long long>(clear_bytes / 16);
  return dtype == BAGS_DTYPE_BF16 ? launch_fused_fwd<false>(x, ldx, w, ldw, p, dz, ldd, di.num_sms, stream, true)
                                  : launch_fused_fwd<true>(x, ldx, w, ldw, p, dz, ldd, di.num_sms, stream, true);
}

extern "C" int bags_reweight(const int64_t* labels, const int32_t* label2bin, const uint8_t* wmask,
                             const float* cls_weight, int wstride, int N, int G, int classes, float* wfloat,
                             float* avg, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  BAGS_REQUIRE(label2bin && cls_weight && wfloat && avg && (N == 0 || labels), "bags_reweight: NULL argument");
  BAGS_REQUIRE(G >= 1 && G <= kMaxG && classes >= 1 && N >= 0 && wstride >= 1, "bags_reweight: bad shape");
  reweight_kernel<<<G, 256, 0, stream>>>(reinterpret_cast<const long long*>(labels), label2bin, classes, N, wmask,
                                         cls_weight, wstride, wfloat, avg);
  BAGS_CUDA(cudaGetLastError());
  return BAGS_OK;
}

__global__ void __launch_bounds__(256)
scale_colsum_kernel(const float* __restrict__ colsum, int tiles, float* __restrict__ db, int C, GroupTable gt,
                    const float* __restrict__ gout) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= C) return;
  float s = (gout == nullptr) ? 1.f : 0.f;
  if (gout != nullptr)
    for (int g = 0; g < gt.G; ++g)
      if (c >= gt.start[g] && c < gt.start[g] + gt.len[g]) s = __ldg(gout + g);
  float cs = 0.f;
  for (int t = 0; t < tiles; ++t) cs += colsum[(long long)t * C + c];
  db[c] = s * cs;
}


template <bool TF32>
static int launch_bwd_merged(const void* dz, long long ldd, const void* x, long long ldx, const void* w, const void* wb,
                             long long ldw, const BwdMergedParams& bp, const DeviceInfo& di, cudaStream_t stream) {
  using CW = BwdDwCfg<TF32>;
  using CX = BwdDxCfg<TF32>;
  const int dtype = TF32 ? BAGS_DTYPE_F32 : BAGS_DTYPE_BF16;
  const int C = bp.dw.M, K = bp.dw.N, N = bp.dw.K;
  CUtensorMap t_dzT, t_xT, t_dz, t_w, t_wp;
  int rc;
  if ((rc = make_tmap(&t_dzT, dz, dtype, C, N, ldd, CW::SLAB, CW::BLOCK_K))) return rc;   // dW: A = dz^T
  if ((rc = make_tmap(&t_xT, x, dtype, K, N, ldx, CW::SLAB, CW::BLOCK_K))) return rc;     // dW: B = x^T
  if ((rc = make_tmap(&t_dz, dz, dtype, C, N, ldd, CX::BLOCK_K, CX::BLOCK_M))) return rc;  // dX: A = dz
  if ((rc = make_tmap(&t_w, w, dtype, K, C, ldw, CX::SLAB, CX::BLOCK_K))) return rc;      // dX: B = W^T
  if ((rc = make_tmap(&t_wp, wb, dtype, K, C, ldw, CX::SLAB, CX::BLOCK_K))) return rc;    // dX: B = W'^T
  auto kernel = bags_bwd_merged_kernel<TF32>;
  BAGS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CW::SMEM_BYTES));
  const int units = bp.dw_units + bp.dx_units;
  const int grid = units < di.num_sms ? units : di.num_sms;
  BAGS_CUDA(launch(kernel, dim3(grid), dim3(CW::NUM_THREADS), CW::SMEM_BYTES, stream, true, false, t_dzT, t_xT, t_dz, t_w, t_wp, bp));
  return BAGS_OK;
}

static constexpr int kColsumTiles = 8;   // row groups of the bias-gradient partial sums made by bwd_prep

// bytes of the gout-scaled copy W' at the start of wscratch; the bias-gradient partials follow it
static size_t wprime_bytes(int C, long long ldw, int dtype) {
  const size_t elt = (dtype == BAGS_DTYPE_BF16) ? 2 : 4;
  return (static_cast<size_t>(C) * static_cast<size_t>(ldw) * elt + 255) & ~static_cast<size_t>(255);
}

extern "C" size_t bags_bwd_scratch_bytes(int C, long long ldw, int dtype) {
  return wprime_bytes(C, ldw, dtype) + static_cast<size_t>(kColsumTiles) * C * sizeof(float);
}

extern "C" int bags_bwd(const void* dz, long long ldd, const void* x, long long ldx, const void* w,
                        long long ldw, const float* gout, const int32_t* slices_host,
                        const float* colsum, int colsum_tiles, float* dW, long long lddw, float* db, void* dX,
                        long long lddx, void* wscratch, size_t wscratch_bytes, int N, int K, int C, int G,
                        int dtype, int flags, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bool prezeroed = (flags & BAGS_BWD_DW_PREZEROED) != 0;   // the caller (bags_fwd's clear hook) zeroed dW
  BAGS_REQUIRE(dz != nullptr || N == 0, "bags_bwd: dz is NULL");
  BAGS_REQUIRE(dtype == BAGS_DTYPE_F32 || dtype == BAGS_DTYPE_BF16, "bags_bwd: bad dtype %d", dtype);
  BAGS_REQUIRE(N >= 0 && K >= 1 && C >= 1, "bags_bwd: bad shape");
  GroupTable gt;
  if (int rc = make_group_table(gt, slices_host, G, C)) return rc;
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  const bool bf = dtype == BAGS_DTYPE_BF16;
  const int vecw = bf ? 8 : 4;

  const bool want_scale = (dX != nullptr && N > 0 && gout != nullptr);
  const bool want_colpart = (db != nullptr && colsum == nullptr && N > 0);
  if (db != nullptr && colsum == nullptr && N == 0) {   // no rows: zero bias gradient
    BAGS_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * C, stream));
    db = nullptr;
  }
  if (want_scale || want_colpart) {
    BAGS_REQUIRE(wscratch != nullptr && wscratch_bytes >= bags_bwd_scratch_bytes(C, ldw, dtype),
                 "bags_bwd: wscratch must provide bags_bwd_scratch_bytes() = %zu bytes (got %zu)",
                 bags_bwd_scratch_bytes(C, ldw, dtype), wscratch_bytes);
    BAGS_REQUIRE((reinterpret_cast<uintptr_t>(wscratch) & 255) == 0, "bags_bwd: wscratch must be 256-byte aligned");
  }
  float* colpart = (wscratch == nullptr) ? nullptr
                   : reinterpret_cast<float*>(reinterpret_cast<char*>(wscratch) + wprime_bytes(C, ldw, dtype));
  if (dW != nullptr)
    BAGS_REQUIRE((x != nullptr || N == 0) && lddw >= K && (lddw % 4) == 0 && (K % 4) == 0 &&
                     (reinterpret_cast<uintptr_t>(dW) & 15) == 0,
                 "bags_bwd: dW must be 16-byte aligned with K and lddw multiples of 4");
  if (want_scale)
    BAGS_REQUIRE(w != nullptr && (K % vecw) == 0 && (ldw % vecw) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0,
                 "bags_bwd: w must be 16-byte aligned with K and ldw multiples of %d", vecw);
  if (want_colpart)
    BAGS_REQUIRE(((ldd * (bf ? 2 : 4)) % 16) == 0 && (reinterpret_cast<uintptr_t>(dz) & 15) == 0,
                 "bags_bwd: dz rows must be 16-byte aligned");

  // ---- preparation (one small kernel): zero dW, W' = gout-scaled W, bias-gradient partial column sums; then both
  // contractions in one merged launch, or the one requested as a plain split-K dW (red.add) / dX GEMM ----
  // both contractions requested: one merged persistent launch after the preparation kernel (see bags_bwd_merged_kernel)
  const bool merged = dW != nullptr && dX != nullptr && N > 0 && env_int("BAGS_BWD_MERGED", 1);
  BwdPrepParams pp{};
  bool prep_launched = false;
  if (dW != nullptr || want_scale || want_colpart) {
    pp.dW = dW; pp.lddw = lddw; pp.C = C; pp.K = K;
    pp.w = w; pp.wscr = wscratch; pp.ldw = ldw; pp.gout = gout; pp.gt = gt;
    pp.dz = dz; pp.ldd = ldd; pp.N = N; pp.colpart = colpart; pp.ctiles = kColsumTiles;
    pp.z_ctas = (dW != nullptr && !prezeroed) ? di.num_sms : 0;
    pp.s_ctas = want_scale ? di.num_sms : 0;
    pp.c_ctas = want_colpart ? ((C + 63) / 64) * kColsumTiles : 0;
    pp.skip_scale_if_uniform = merged ? 1 : 0;   // the merged kernel reads W itself when all gout[g] are equal
    const int grid = pp.z_ctas + pp.s_ctas + pp.c_ctas;
    if (grid > 0) {
      BAGS_CUDA(launch(bf ? bwd_prep_kernel<false> : bwd_prep_kernel<true>, dim3(grid), dim3(256), 0, stream, true, false, pp));
      prep_launched = true;
    }
  }
  const float* cs_in = (colsum != nullptr) ? colsum : colpart;
  const int cs_tiles = (colsum != nullptr) ? colsum_tiles : kColsumTiles;
  if (db != nullptr) BAGS_REQUIRE(cs_in != nullptr && cs_tiles >= 1, "bags_bwd: db requested but no column sums available");

  if (merged) {
    BAGS_REQUIRE(w != nullptr && x != nullptr, "bags_bwd: w / x is NULL but dW and dX requested");
    BAGS_REQUIRE((reinterpret_cast<uintptr_t>(dX) & 15) == 0, "bags_bwd: dX not 16-byte aligned");
    const int bk = bf ? 64 : 32;
    BwdMergedParams bp{};
    GemmParams& pw = bp.dw;
    pw.M = C; pw.N = K; pw.K = N;
    pw.num_m_tiles = (C + 127) / 128; pw.num_n_tiles = (K + 255) / 256; pw.kblocks_total = (N + bk - 1) / bk;
    GemmParams& px = bp.dx;
    px.M = N; px.N = K; px.K = C;
    px.num_m_tiles = (N + 127) / 128; px.num_n_tiles = (K + 255) / 256; px.kblocks_total = (C + bk - 1) / bk;
    px.num_splits = 1;
    // split-K factor of the dW units: fewest (rounds of the work list over the SMs x longest unit), in k-blocks
    const int dw_tiles = pw.num_m_tiles * pw.num_n_tiles, dx_units = px.num_m_tiles * px.num_n_tiles;
    int splits = 1;
    long best = -1;
    for (int sp = 1; sp <= 16 && sp <= pw.kblocks_total; ++sp) {
      const long rounds = (dw_tiles * sp + dx_units + di.num_sms - 1) / di.num_sms;
      const int dwk = (pw.kblocks_total + sp - 1) / sp;
      const long cost = rounds * (dwk > px.kblocks_total ? dwk : px.kblocks_total);
      if (best < 0 || cost < best) { best = cost; splits = sp; }
    }
    splits = env_int("BAGS_DW_SPLITS", splits);
    if (splits < 1) splits = 1;
    if (splits > pw.kblocks_total) splits = pw.kblocks_total;
    pw.num_splits = splits;
    pw.out = dW; pw.ldo = lddw;
    pw.gscale = gout; pw.G = (gout != nullptr) ? gt.G : 0;
    for (int g = 0; g < kMaxGroups; ++g) { pw.gstart[g] = gt.start[g]; pw.glen[g] = gt.len[g]; }
    pw.colsum_in = (db != nullptr) ? cs_in : nullptr;
    pw.colsum_tiles = cs_tiles;
    pw.colsum_out = db;
    pw.a_ptr = static_cast<const float*>(dz); pw.lda = ldd; pw.a_rows = C; pw.a_k = N;
    pw.b_ptr = static_cast<const float*>(x); pw.ldb = ldx; pw.b_rows = K; pw.b_k = N;
    const void* wb = want_scale ? wscratch : w;
    px.out = dX; px.ldo = lddx;
    px.b_ptr = static_cast<const float*>(wb); px.ldb = ldw; px.b_rows = K; px.b_k = C;
    bp.dw_units = pw.num_m_tiles * pw.num_n_tiles * splits;
    bp.dx_units = px.num_m_tiles * px.num_n_tiles;
    bp.w = static_cast<const float*>(w);
    bp.gout = gout;
    bp.G = gt.G;
    return bf ? launch_bwd_merged<false>(dz, ldd, x, ldx, w, wb, ldw, bp, di, stream)
              : launch_bwd_merged<true>(dz, ldd, x, ldx, w, wb, ldw, bp, di, stream);
  }

  if (dW != nullptr && N > 0) {
    GemmArgs ga{};
    ga.a = dz; ga.lda = ldd; ga.a_mn = true;   // A = dz^T : [C, N_roi], stored [N_roi, C]
    ga.b = x;  ga.ldb = ldx; ga.b_mn = true;   // B = x^T  : [K, N_roi], stored [N_roi, K]
    ga.M = C; ga.N = K; ga.K = N; ga.dtype = dtype;
    const int tiles = ((C + 127) / 128) * ((K + 255) / 256);
    const int kblocks = (N + (bf ? 63 : 31)) / (bf ? 64 : 32);
    ga.splits = env_int("BAGS_DW_SPLITS", pick_splits(tiles, kblocks, di.num_sms));
    ga.p.out = dW; ga.p.ldo = lddw; ga.p.bias = nullptr;
    ga.p.gscale = gout; ga.p.G = (gout != nullptr) ? gt.G : 0;
    for (int g = 0; g < kMaxGroups; ++g) { ga.p.gstart[g] = gt.start[g]; ga.p.glen[g] = gt.len[g]; }
    ga.p.colsum_in = (db != nullptr) ? cs_in : nullptr;
    ga.p.colsum_tiles = cs_tiles;
    ga.p.colsum_out = (db != nullptr) ? db : nullptr;
    ga.p.pdl_wait_epilogue = 1;   // dW zeroing + column-sum partials come from bwd_prep; the mainloop overlaps it
    ga.p.pdl_wait_producer = prep_launched ? 0 : 1;   // no preparation kernel in between: dz comes from the preceding kernel
    int rc = bf ? launch_gemm<256, true, true, EPI_RED_F32, false, 4>(ga, di, stream, true)
                : launch_gemm<256, true, true, EPI_RED_F32, true, 4>(ga, di, stream, true);
    if (rc) return rc;
  } else if (db != nullptr) {
    scale_colsum_kernel<<<(C + 255) / 256, 256, 0, stream>>>(cs_in, cs_tiles, db, C, gt, gout);
    BAGS_CUDA(cudaGetLastError());
  }

  if (dX != nullptr && N > 0) {
    BAGS_REQUIRE(w != nullptr, "bags_bwd: w is NULL but dX requested");
    BAGS_REQUIRE((reinterpret_cast<uintptr_t>(dX) & 15) == 0, "bags_bwd: dX not 16-byte aligned");
    GemmArgs ga{};
    ga.a = dz; ga.lda = ldd; ga.a_mn = false;                 // A = dz : [N_roi, C]
    ga.b = want_scale ? wscratch : w; ga.ldb = ldw; ga.b_mn = true;   // B = W'^T: [K, C], stored [C, K]
    ga.M = N; ga.N = K; ga.K = C; ga.dtype = dtype; ga.splits = 1;
    ga.p.out = dX; ga.p.ldo = lddx; ga.p.bias = nullptr; ga.p.gscale = nullptr; ga.p.G = 0;
    ga.p.colsum_in = nullptr; ga.p.colsum_out = nullptr;
    ga.p.pdl_wait_producer = 1;   // W' is produced by bwd_prep (two kernels back; the chain of waits covers it)
    int rc = bf ? launch_gemm<256, false, true, EPI_STORE_BF16, false, 4>(ga, di, stream, true)
                : launch_gemm<256, false, true, EPI_STORE_F32, true, 4>(ga, di, stream, true);
    if (rc) return rc;
  }
  return BAGS_OK;
}

// ----------------------------------------------------------------------------
// gradient exchange over NVLink peer memory (one kernel; see bags_allreduce.cuh)
// ----------------------------------------------------------------------------
extern "C" size_t bags_grad_allreduce_flag_bytes(int world) {
  if (world < 1) world = 1;
  // slots [kArMaxBlocks][world] + epochs [kArMaxBlocks] + one status word, padded to 64 bytes
  return (static_cast<size_t>(kArMaxBlocks) * static_cast<size_t>(world) + kArMaxBlocks + 16) * sizeof(uint32_t);
}

extern "C" long long bags_grad_allreduce_status_offset(int world) {
  if (world < 1) world = 1;
  return (static_cast<long long>(kArMaxBlocks) * world + kArMaxBlocks) * static_cast<long long>(sizeof(uint32_t));
}

extern "C" int bags_grad_allreduce(void* const* peer_bufs_host, void* mc_buf, long long flag_off_bytes,
                                   long long count, int rank, int world, float scale, int max_blocks,
                                   void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  BAGS_REQUIRE(peer_bufs_host != nullptr, "bags_grad_allreduce: peer_bufs_host is NULL");
  BAGS_REQUIRE(world >= 1 && world <= kMaxRanks && rank >= 0 && rank < world,
               "bags_grad_allreduce: bad rank %d / world %d (max %d ranks)", rank, world, kMaxRanks);
  BAGS_REQUIRE(count >= 0 && (count % 4) == 0, "bags_grad_allreduce: count=%lld must be a multiple of 4 floats", count);
  BAGS_REQUIRE(flag_off_bytes >= count * 4 && (flag_off_bytes % 16) == 0,
               "bags_grad_allreduce: the flag words must follow the data (flag_off_bytes=%lld, data bytes=%lld)",
               flag_off_bytes, count * 4);
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  AllReduceParams p{};
  for (int r = 0; r < world; ++r) {
    BAGS_REQUIRE(peer_bufs_host[r] != nullptr && (reinterpret_cast<uintptr_t>(peer_bufs_host[r]) & 15) == 0,
                 "bags_grad_allreduce: peer buffer %d is NULL or not 16-byte aligned", r);
    p.peer[r] = static_cast<float*>(peer_bufs_host[r]);
  }
  BAGS_REQUIRE((reinterpret_cast<uintptr_t>(mc_buf) & 15) == 0, "bags_grad_allreduce: multicast buffer not 16-byte aligned");
  p.mc = static_cast<float*>(mc_buf);
  p.flag_off = flag_off_bytes;
  p.count = count;
  p.rank = rank; p.world = world; p.scale = scale;
  // max_blocks < 0: soft-failure mode of the construction-time self test (grid = default)
  p.trap_on_timeout = (max_blocks < 0) ? 0 : 1;
  if (max_blocks < 0) max_blocks = 0;
  p.timeout_ns = 1000000LL * env_int("BAGS_AR_TIMEOUT_MS", p.trap_on_timeout ? 30000 : 3000);
  p.timing = g_timing ? g_timing + 4096 * 8 : nullptr;   // rows [4096, ..): after the forward's and the backward's
  p.mode = env_int("BAGS_AR_MODE", 3);   // relaxed first-barrier store + relaxed polling: -3..4 us per exchange
  if (count == 0) return BAGS_OK;
  // enough threads to keep one vector per thread and unroll slot in flight, at most kArMaxBlocks blocks;
  // every rank must launch the same grid: it depends only on (count, world, max_blocks) and the environment
  int threads = env_int("BAGS_AR_THREADS", 256);
  if (threads != 128 && threads != 256) threads = 256;
  if (max_blocks > kArMaxBlocks) max_blocks = kArMaxBlocks;
  const long long per_rank = (count / 4 + world - 1) / world;
  long long blocks = (per_rank + static_cast<long long>(threads) * 4 - 1) / (static_cast<long long>(threads) * 4);
  if (blocks < 1) blocks = 1;
  const bool mm = p.mc != nullptr && !env_int("BAGS_AR_NO_MULTIMEM", 0);
  // Default grid: one block per SM on the multimem path (the exchange runs inside the step, where a small grid leaves
  // the switch bandwidth unused); the plain peer path keeps one vector per thread in flight.
  if (max_blocks <= 0) max_blocks = env_int("BAGS_AR_MAX_BLOCKS", mm ? di.num_sms : kArMaxBlocks);
  if (max_blocks <= 0 || max_blocks > kArMaxBlocks) max_blocks = kArMaxBlocks;
  if (blocks > max_blocks) blocks = max_blocks;
  const bool epoch = env_int("BAGS_AR_EPOCH", 1) != 0;
  const dim3 grid(static_cast<unsigned>(blocks)), block(static_cast<unsigned>(threads));
  auto kernel = mm ? (epoch ? bags_grad_allreduce_kernel<true, true> : bags_grad_allreduce_kernel<true, false>)
                  : (epoch ? bags_grad_allreduce_kernel<false, true> : bags_grad_allreduce_kernel<false, false>);
  BAGS_CUDA(launch(kernel, grid, block, 0, stream, true, false, p));
  return BAGS_OK;
}

// ----------------------------------------------------------------------------
// class-aware batched NMS (see bags_nms.cuh)
// ----------------------------------------------------------------------------
extern "C" int bags_class_nms_dense(const float* boxes, int box_cols, const int32_t* order, const int32_t* counts,
                                    int num_classes_fg, int n, float iou_thr, uint8_t* keep, int32_t* overflow,
                                    void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  BAGS_REQUIRE(num_classes_fg >= 0 && n >= 0, "bags_class_nms_dense: bad sizes");
  if (num_classes_fg == 0 || n == 0) return BAGS_OK;
  BAGS_REQUIRE(boxes && order && counts && keep && overflow, "bags_class_nms_dense: NULL argument");
  BAGS_REQUIRE(box_cols == 4 || box_cols == 4 * (num_classes_fg + 1),
               "bags_class_nms_dense: boxes must have 4 or 4 * (classes incl. background) = %d columns (got %d)",
               4 * (num_classes_fg + 1), box_cols);
  BAGS_REQUIRE((reinterpret_cast<uintptr_t>(boxes) & 15) == 0, "bags_class_nms_dense: boxes must be 16-byte aligned");
  const int seg = n < kNmsMaxSeg ? n : kNmsMaxSeg;
  const int words = (seg + 31) / 32;
  const size_t smem = static_cast<size_t>((seg + 1) & ~1) * sizeof(float4) + static_cast<size_t>(seg) * words * sizeof(uint32_t);
  BAGS_CUDA(cudaFuncSetAttribute(class_nms_dense_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  class_nms_dense_kernel<<<num_classes_fg, kNmsThreads, smem, stream>>>(boxes, box_cols, order, counts, n, iou_thr, keep, overflow);
  BAGS_CUDA(cudaGetLastError());
  return BAGS_OK;
}

// test hook: a kernel of `blocks` x `threads` that only waits `micros` microseconds (stands in for a latency-bound
// collective when probing how side-stream work co-schedules with the GEMM kernels)
__global__ void bags_debug_spin_kernel(long long ns) {
  const long long t0 = global_timer_ns();
  while (global_timer_ns() - t0 < ns) __nanosleep(200);
}
extern "C" int bags_debug_spin(int blocks, int threads, int micros, void* stream_) {
  BAGS_REQUIRE(blocks >= 1 && threads >= 32 && threads <= 1024 && micros >= 0, "bags_debug_spin: bad arguments");
  bags_debug_spin_kernel<<<blocks, threads, 0, static_cast<cudaStream_t>(stream_)>>>(1000LL * micros);
  BAGS_CUDA(cudaGetLastError());
  return BAGS_OK;
}

extern "C" int bags_merge_scores(const float* logits, long long ldz, const int32_t* slices_host,
                                 const int32_t* cls2col, int N, int C, int G, int classes,
                                 float* scores, long long lds, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  BAGS_REQUIRE(cls2col && (N == 0 || (logits && scores)), "bags_merge_scores: NULL argument");
  BAGS_REQUIRE(N >= 0 && C >= 4 && (C % 4) == 0 && C <= 4096, "bags_merge_scores: C=%d must be a multiple of 4 in [4,4096]", C);
  BAGS_REQUIRE((ldz % 4) == 0 && ldz >= C && lds >= classes, "bags_merge_scores: bad leading dimension");
  BAGS_REQUIRE((reinterpret_cast<uintptr_t>(logits) & 15) == 0, "bags_merge_scores: logits not 16-byte aligned");
  GroupTable gt;
  if (int rc = make_group_table(gt, slices_host, G, C)) return rc;
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  if (N == 0) return BAGS_OK;
  const int nv = (C / 4 + 31) / 32;
  int grid = (N + 7) / 8;
  if (grid > di.num_sms * 4) grid = di.num_sms * 4;
#define BAGS_LAUNCH_MERGE(NV)                                                                              \
  do {                                                                                                     \
    const int smem = 8 * NV * 128 * (int)sizeof(float);                                                    \
    auto k = merge_scores_kernel<NV>;                                                                      \
    BAGS_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));               \
    k<<<grid, 256, smem, stream>>>(logits, ldz, gt, cls2col, N, C, classes, scores, lds);                  \
  } while (0)
  if (nv <= 10) BAGS_LAUNCH_MERGE(10);
  else if (nv <= 16) BAGS_LAUNCH_MERGE(16);
  else BAGS_LAUNCH_MERGE(32);
#undef BAGS_LAUNCH_MERGE
  BAGS_CUDA(cudaGetLastError());
  return BAGS_OK;
}

extern "C" int bags_cast_bf16(const float* src, long long lds, void* dst, long long ldd, int rows,
                              int cols, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  BAGS_REQUIRE(src && dst, "bags_cast_bf16: NULL argument");
  BAGS_REQUIRE(rows >= 0 && cols >= 0 && (cols % 4) == 0 && (lds % 4) == 0 && (ldd % 4) == 0,
               "bags_cast_bf16: cols and leading dims must be multiples of 4");
  if (rows == 0 || cols == 0) return BAGS_OK;
  const long long total = (long long)rows * (cols / 4);
  long long grid = (total + 255) / 256;
  if (grid > 132 * 8) grid = 132 * 8;
  cast_bf16_kernel<<<(int)grid, 256, 0, stream>>>(src, lds, reinterpret_cast<__nv_bfloat16*>(dst), ldd, rows, cols);
  BAGS_CUDA(cudaGetLastError());
  return BAGS_OK;
}

extern "C" int bags_gemm_probe(const void* a, long long lda, int a_mn, const void* b, long long ldb,
                               int b_mn, void* out, long long ldo, int M, int N, int K, int dtype,
                               int block_n, int splits, int epi, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  BAGS_REQUIRE(a && b && out, "bags_gemm_probe: NULL argument");
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  GemmArgs ga{};
  ga.a = a; ga.lda = lda; ga.a_mn = a_mn != 0;
  ga.b = b; ga.ldb = ldb; ga.b_mn = b_mn != 0;
  ga.M = M; ga.N = N; ga.K = K; ga.dtype = dtype; ga.splits = splits;
  ga.p.out = out; ga.p.ldo = ldo; ga.p.bias = nullptr; ga.p.gscale = nullptr; ga.p.G = 0;
  ga.p.colsum_in = nullptr; ga.p.colsum_out = nullptr;
  const bool bf = dtype == BAGS_DTYPE_BF16;
  BAGS_REQUIRE(bf || dtype == BAGS_DTYPE_F32, "bags_gemm_probe: bad dtype");
  // the instantiations the product uses
  if (!a_mn && !b_mn && epi == 0 && block_n == 256)
    return bf ? launch_gemm<256, false, false, EPI_STORE_F32, false, 4>(ga, di, stream)
              : launch_gemm<256, false, false, EPI_STORE_F32, true, 4>(ga, di, stream);
  if (!a_mn && b_mn && block_n == 256 && ((bf && epi == 1) || (!bf && epi == 0)))
    return bf ? launch_gemm<256, false, true, EPI_STORE_BF16, false, 4>(ga, di, stream)
              : launch_gemm<256, false, true, EPI_STORE_F32, true, 4>(ga, di, stream);
  if (a_mn && b_mn && block_n == 256 && epi == 2)
    return bf ? launch_gemm<256, true, true, EPI_RED_F32, false, 4>(ga, di, stream)
              : launch_gemm<256, true, true, EPI_RED_F32, true, 4>(ga, di, stream);
  return fail(BAGS_ERR_INVALID, "bags_gemm_probe: configuration a_mn=%d b_mn=%d block_n=%d epi=%d dtype=%d not instantiated",
              a_mn, b_mn, block_n, epi, dtype);
}
