// C-ABI entry points of libbags_b200.so (see include/bags_b200.h).
// Host side only: argument validation, TMA descriptor encoding, kernel launches.
// No torch, no allocations, no device synchronisation.
#include <cuda.h>
#include <cuda_runtime.h>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "../../include/bags_b200.h"
#include "bags_gemm.cuh"
#include "bags_fused_fwd.cuh"
#include "bags_kernels.cuh"
#include "bags_allreduce.cuh"
#include "bags_nms.cuh"
#include "bags_box.cuh"
#include "bags_mask.cuh"
#include "bags_segm.cuh"
#include "bags_mask_target.cuh"

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

// test hook: device buffer [rows][8] int64 that the next launches stamp with %globaltimer values (row ranges: see
// bags_debug_set_timing in bags_b200.h)
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
// forward GEMM launcher: out[M, N] = A[M, K] B[N, K]^T, both operands K-major
// ----------------------------------------------------------------------------
struct GemmArgs {
  const void* a; long long lda;
  const void* b; long long ldb;
  int M, N, K;
  int dtype;
  int splits;
  GemmParams p;  // epilogue fields pre-filled (out, ldo, bias, relu)
};

template <int BLOCK_N, int EPI, bool TF32, int STAGES>
static int launch_gemm(const GemmArgs& ga, const DeviceInfo& di, cudaStream_t stream) {
  using Cfg = GemmCfg<BLOCK_N, false, false, EPI, TF32, STAGES>;
  auto kernel = bags_gemm_kernel<BLOCK_N, EPI, TF32, STAGES>;
  CUtensorMap ta, tb;
  int rc;
  if ((rc = make_tmap(&ta, ga.a, ga.dtype, ga.K, ga.M, ga.lda, Cfg::BLOCK_K, Cfg::BLOCK_M))) return rc;
  if ((rc = make_tmap(&tb, ga.b, ga.dtype, ga.K, ga.N, ga.ldb, Cfg::BLOCK_K, BLOCK_N))) return rc;

  GemmParams p = ga.p;
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
  BAGS_CUDA(launch(kernel, dim3(grid), dim3(Cfg::NUM_THREADS), Cfg::SMEM_BYTES, stream, false, false, ta, tb, p));
  return BAGS_OK;
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
  ga.a = x; ga.lda = ldx;
  ga.b = w; ga.ldb = ldw;
  ga.M = N; ga.N = C; ga.K = K; ga.dtype = dtype; ga.splits = 1;
  ga.p.out = out; ga.p.ldo = ldo; ga.p.bias = bias; ga.p.relu = relu ? 1 : 0;
  if (dtype == BAGS_DTYPE_BF16)
    return out_dtype == BAGS_DTYPE_BF16 ? launch_gemm<256, EPI_STORE_BF16, false, 4>(ga, di, stream)
                                        : launch_gemm<256, EPI_STORE_F32, false, 4>(ga, di, stream);
  return launch_gemm<256, EPI_STORE_F32, true, 4>(ga, di, stream);
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
  ga.a = x; ga.lda = ldx;
  ga.b = w; ga.ldb = ldw;
  ga.M = N; ga.N = C; ga.K = K; ga.dtype = dtype; ga.splits = splits;
  ga.p.out = ws; ga.p.ldo = ldws;
  int rc = (dtype == BAGS_DTYPE_BF16) ? launch_gemm<256, EPI_RED_F32, false, 4>(ga, di, stream)
                                      : launch_gemm<256, EPI_RED_F32, true, 4>(ga, di, stream);
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
  BAGS_REQUIRE(label2bin && avg && (N == 0 || (labels && wmask)), "bags_sample_others: NULL argument");
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
  BAGS_REQUIRE(avg && (N == 0 || wmask), "bags_mask_avg: NULL argument");
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
// the bins tile [0, C) contiguously: every logit column lies in a bin
static bool bins_tile(const int32_t* slices_host, int G, int C) {
  int end = 0;
  for (int g = 0; g < G; ++g) {
    if (slices_host[2 * g] != end || slices_host[2 * g + 1] < 1) return false;
    end += slices_host[2 * g + 1];
  }
  return end == C;
}

static bool fused_eligible(const int32_t* slices_host, int G, int C) {
  if (slices_host == nullptr || G < 1 || G > FusedCfg<false>::MAXG || C > 4 * FusedCfg<false>::BLOCK_N || (C % 4) != 0)
    return false;
  return bins_tile(slices_host, G, C);
}

extern "C" int bags_fused_eligible(const int32_t* slices_host, int G, int C) {
  return fused_eligible(slices_host, G, C) ? 1 : 0;
}

static bool aligned(const void* ptr, int bytes) { return (reinterpret_cast<uintptr_t>(ptr) % bytes) == 0; }

// the buffer a forward sets to zero (typically the caller's dW): 16-byte aligned, a multiple of 16 bytes
static int check_clear(const char* who, const void* clear, size_t clear_bytes) {
  BAGS_REQUIRE(clear == nullptr || (aligned(clear, 16) && (clear_bytes % 16) == 0),
               "%s: the buffer to clear must be 16-byte aligned and a multiple of 16 bytes", who);
  return BAGS_OK;
}

// The fused kernel's loss variants: the softmax CE with 0/1 byte weights (bags_fwd with the sampler's masks) or with
// fp32 weights (bags_fwd with BAGS_WEIGHTS_F32, bags_ce_fwd), and the sigmoid focal loss (bags_focal_fwd, fp32 weights).
enum class FusedLoss { kCeMask, kCeWeighted, kFocal };

template <bool TF32>
static int launch_fused_fwd(const char* who, FusedLoss loss, const void* x, long long ldx, const void* w, long long ldw,
                            const FusedFwdParams& p0, void* dz, long long ldd, int num_sms, cudaStream_t stream) {
  using Cfg = FusedCfg<TF32>;
  const int dtype = TF32 ? BAGS_DTYPE_F32 : BAGS_DTYPE_BF16;
  CUtensorMap tx, tw;
  int rc = make_tmap(&tx, x, dtype, p0.K, p0.N, ldx, Cfg::BLOCK_K, Cfg::BLOCK_M);
  if (rc) return rc;
  rc = make_tmap(&tw, w, dtype, p0.K, p0.C, ldw, Cfg::BLOCK_K, Cfg::HALF_N);
  if (rc) return rc;
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
  auto kernel = loss == FusedLoss::kFocal       ? bags_focal_fwd_kernel<TF32>
                : loss == FusedLoss::kCeWeighted ? bags_fwd_fused_kernel<TF32, true>
                                                 : bags_fwd_fused_kernel<TF32, false>;
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
    return fail(BAGS_ERR_CUDA, "%s: the fused kernel cannot keep %d CTAs resident (%d SMs, %d CTA(s) per SM)", who,
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

// The fused route of bags_fwd, bags_ce_fwd and bags_focal_fwd: the argument rules they share, the outputs of N == 0,
// the per-stream workspace and the launch.  The caller has checked its own arguments and filled p's N, C, K and loss
// fields (bias, labels, l2b, classes, wmask, avg, loss, acc, lse, colsum and the focal parameters); slices_host / G is
// its bin table.  Every argument check comes before device_info(), so a bad argument is reported without a GPU.
static int fused_fwd(const char* who, FusedLoss loss, const void* x, long long ldx, const void* w, long long ldw,
                     int dtype, FusedFwdParams p, const int32_t* slices_host, int G, void* dz, long long ldd,
                     int colsum_tiles, void* workspace, size_t workspace_bytes, void* clear, size_t clear_bytes,
                     cudaStream_t stream) {
  const int N = p.N, C = p.C;
  BAGS_REQUIRE(dtype == BAGS_DTYPE_F32 || dtype == BAGS_DTYPE_BF16, "%s: bad dtype %d", who, dtype);
  BAGS_REQUIRE(N >= 0 && p.K >= 1, "%s: bad shape N=%d K=%d", who, N, p.K);
  BAGS_REQUIRE(p.loss && workspace && (N == 0 || (x && w)), "%s: NULL argument", who);
  BAGS_REQUIRE(workspace_bytes >= bags_workspace_bytes(), "%s: workspace too small (%zu < %zu)", who, workspace_bytes,
               bags_workspace_bytes());
  BAGS_REQUIRE(p.acc == nullptr || N <= (1 << 24), "%s: N=%d: the accuracy count is exact up to 2^24 rows only", who, N);
  if (dz != nullptr) BAGS_REQUIRE(ldd >= C && (ldd % 8) == 0, "%s: ldd=%lld must be a multiple of 8 and >= C", who, ldd);
  BAGS_REQUIRE(dz == nullptr || N == 0 || aligned(dz, 16), "%s: dz must be 16-byte aligned", who);
  if (p.colsum != nullptr)
    BAGS_REQUIRE(colsum_tiles == (N + 127) / 128 || (N == 0 && colsum_tiles >= 1),
                 "%s: colsum must hold ceil(N/128) = %d row tiles of C floats (got %d)", who, (N + 127) / 128,
                 colsum_tiles);
  if (N > 0) {
    // the operands' TMA maps: rows of K elements at a row stride of ldx / ldw elements
    const int elt = dtype == BAGS_DTYPE_BF16 ? 2 : 4;
    BAGS_REQUIRE(ldx >= p.K && ldw >= p.K, "%s: ldx=%lld and ldw=%lld must be >= K=%d", who, ldx, ldw, p.K);
    BAGS_REQUIRE(aligned(x, 16) && aligned(w, 16), "%s: x and W must be 16-byte aligned", who);
    BAGS_REQUIRE((ldx * elt) % 16 == 0 && (ldw * elt) % 16 == 0,
                 "%s: the row strides of x and W (%lld, %lld bytes) must be multiples of 16 bytes", who, ldx * elt,
                 ldw * elt);
  }
  if (int rc = check_clear(who, clear, clear_bytes)) return rc;
  if (int rc = make_group_table(p.gt, slices_host, G, C)) return rc;
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  if (N == 0) {
    BAGS_CUDA(cudaMemsetAsync(p.loss, 0, sizeof(float) * G, stream));
    if (p.acc != nullptr) BAGS_CUDA(cudaMemsetAsync(p.acc, 0, sizeof(float), stream));
    if (p.colsum != nullptr) BAGS_CUDA(cudaMemsetAsync(p.colsum, 0, sizeof(float) * C * colsum_tiles, stream));
    if (clear != nullptr) BAGS_CUDA(cudaMemsetAsync(clear, 0, clear_bytes, stream));
    return BAGS_OK;
  }
  p.acc_scale = static_cast<float>(100.0 / N);   // accuracy.py: correct * (100.0 / N)
  p.counter = reinterpret_cast<unsigned int*>(workspace);
  p.part = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 256);
  p.xch_counter = reinterpret_cast<unsigned int*>(reinterpret_cast<char*>(workspace) + kLossWorkspaceBytes);
  p.xch = reinterpret_cast<float2*>(reinterpret_cast<char*>(workspace) + kLossWorkspaceBytes + kFusedXchCounterBytes);
  p.clear = reinterpret_cast<float4*>(clear);
  p.clear_vecs = static_cast<long long>(clear_bytes / 16);
  auto launch_for_dtype = dtype == BAGS_DTYPE_BF16 ? launch_fused_fwd<false> : launch_fused_fwd<true>;
  return launch_for_dtype(who, loss, x, ldx, w, ldw, p, dz, ldd, di.num_sms, stream);
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
  if (logits != nullptr) {
    // caller wants materialised logits: GEMM with fp32 store, then the stand-alone grouped CE (tile 0 holds
    // the column sums, the other tiles are zero); `clear` is a plain memset
    BAGS_REQUIRE(colsum == nullptr || colsum_tiles >= 1, "bags_fwd: colsum must hold at least one row tile (got %d)",
                 colsum_tiles);
    if (int rc = check_clear("bags_fwd", clear, clear_bytes)) return rc;
    if (clear != nullptr) BAGS_CUDA(cudaMemsetAsync(clear, 0, clear_bytes, stream));
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
  BAGS_REQUIRE(label2bin && (N == 0 || labels), "bags_fwd: NULL argument");
  BAGS_REQUIRE(N == 0 || bias == nullptr || aligned(bias, 16), "bags_fwd: bias must be 16-byte aligned");
  FusedFwdParams p{};
  p.N = N; p.C = C; p.K = K; p.bias = bias;
  p.labels = reinterpret_cast<const long long*>(labels);
  p.l2b = label2bin; p.classes = classes; p.wmask = static_cast<const uint8_t*>(weights); p.avg = avg;
  p.loss = loss; p.lse = lse; p.colsum = colsum;
  return fused_fwd("bags_fwd", weights_dtype == BAGS_WEIGHTS_F32 ? FusedLoss::kCeWeighted : FusedLoss::kCeMask, x, ldx,
                   w, ldw, dtype, p, slices_host, G, dz, ldd, colsum_tiles, workspace, workspace_bytes, clear,
                   clear_bytes, stream);
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
  constexpr int kMaxC = FusedCfg<false>::RANKS * FusedCfg<false>::BLOCK_N;
  BAGS_REQUIRE(C >= 1 && C <= kMaxC, "bags_ce_fwd: bad shape C=%d (1 <= C <= %d)", C, kMaxC);
  BAGS_REQUIRE(N == 0 || labels, "bags_ce_fwd: NULL argument");
  FusedFwdParams p{};
  p.N = N; p.C = C; p.K = K; p.bias = bias;
  p.labels = reinterpret_cast<const long long*>(labels);
  p.l2b = nullptr; p.classes = C;
  p.wmask = reinterpret_cast<const uint8_t*>(weights); p.avg = avg;
  p.loss = loss; p.acc = acc; p.colsum = colsum;
  const int32_t slices[2] = {0, C};
  return fused_fwd("bags_ce_fwd", FusedLoss::kCeWeighted, x, ldx, w, ldw, dtype, p, slices, 1, dz, ldd, colsum_tiles,
                   workspace, workspace_bytes, clear, clear_bytes, static_cast<cudaStream_t>(stream_));
}

// fc_cls + the sigmoid focal loss over all C logits (FocalLoss, focal_loss.py:29-88 with sigmoid_focal_loss_cuda.cu:23-96):
// the fused kernel's focal variant with one bin (0, C) and fp32 per-RoI weights.  Argument rules as bags_ce_fwd, plus
// non-NULL targets, the labels when acc is asked for, and a finite norm > 0.
extern "C" int bags_focal_fwd(const void* x, long long ldx, const void* w, long long ldw, const float* bias,
                              const int64_t* targets, const int64_t* labels, const float* weights, float norm,
                              float gamma, float alpha, int N, int K, int C, int dtype, float* loss, float* acc,
                              void* dz, long long ldd, float* colsum, int colsum_tiles, void* workspace,
                              size_t workspace_bytes, void* clear, size_t clear_bytes, void* stream_) {
  constexpr int kMaxC = FusedCfg<false>::RANKS * FusedCfg<false>::BLOCK_N;
  BAGS_REQUIRE(C >= 1 && C <= kMaxC, "bags_focal_fwd: bad shape C=%d (1 <= C <= %d)", C, kMaxC);
  BAGS_REQUIRE((N == 0 || targets) && (acc == nullptr || N == 0 || labels), "bags_focal_fwd: NULL argument");
  BAGS_REQUIRE(norm > 0.f && std::isfinite(norm), "bags_focal_fwd: norm=%g must be positive and finite",
               static_cast<double>(norm));
  FusedFwdParams p{};
  p.N = N; p.C = C; p.K = K; p.bias = bias;
  p.labels = reinterpret_cast<const long long*>(labels);
  p.targets = reinterpret_cast<const long long*>(targets);
  p.l2b = nullptr; p.classes = C;
  p.wmask = reinterpret_cast<const uint8_t*>(weights);
  p.norm = norm; p.gamma = gamma; p.alpha = alpha;
  p.loss = loss; p.acc = acc; p.colsum = colsum;
  const int32_t slices[2] = {0, C};
  return fused_fwd("bags_focal_fwd", FusedLoss::kFocal, x, ldx, w, ldw, dtype, p, slices, 1, dz, ldd, colsum_tiles,
                   workspace, workspace_bytes, clear, clear_bytes, static_cast<cudaStream_t>(stream_));
}

// ----------------------------------------------------------------------------
// class-specific box regression + SmoothL1 (bbox_head.py:118-128, smooth_l1_loss.py)
// ----------------------------------------------------------------------------
// x rows are read 4 elements at a time (8 bytes bf16, 16 bytes fp32), W rows as float4
static int check_box_operands(const char* who, const void* x, long long ldx, int dtype, const float* w, long long ldw,
                              int K, int classes) {
  BAGS_REQUIRE(dtype == BAGS_DTYPE_F32 || dtype == BAGS_DTYPE_BF16, "%s: bad dtype %d", who, dtype);
  BAGS_REQUIRE(K >= 4 && (K % 4) == 0, "%s: K=%d must be a positive multiple of 4", who, K);
  BAGS_REQUIRE(classes >= 1 && classes <= kBoxMaxClasses, "%s: classes=%d outside [1,%d]", who, classes, kBoxMaxClasses);
  if (x != nullptr)
    BAGS_REQUIRE(aligned(x, dtype == BAGS_DTYPE_BF16 ? 8 : 16) && ldx >= K && (ldx % 4) == 0,
                 "%s: x rows must be %d-byte aligned with ldx >= K and ldx %% 4 == 0 (ldx=%lld)", who,
                 dtype == BAGS_DTYPE_BF16 ? 8 : 16, ldx);
  if (w != nullptr)
    BAGS_REQUIRE(aligned(w, 16) && ldw >= K && (ldw % 4) == 0,
                 "%s: W rows must be 16-byte aligned with ldw >= K and ldw %% 4 == 0 (ldw=%lld)", who, ldw);
  return BAGS_OK;
}

extern "C" int bags_box_fwd(const void* x, long long ldx, int dtype, const float* w, long long ldw, const float* bias,
                            const int64_t* labels, const float* targets, const float* weights, float beta, float avg,
                            int N, int K, int classes, float* loss, float* g, float* pred, int32_t* index,
                            void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  BAGS_REQUIRE(N >= 0, "bags_box_fwd: bad shape N=%d", N);
  BAGS_REQUIRE(loss && index && workspace && w && (N == 0 || (x && labels && targets && weights && g)),
               "bags_box_fwd: NULL argument");
  if (int rc = check_box_operands("bags_box_fwd", x, ldx, dtype, w, ldw, K, classes)) return rc;
  BAGS_REQUIRE(beta > 0.f && std::isfinite(beta), "bags_box_fwd: beta=%g must be positive and finite",
               static_cast<double>(beta));
  BAGS_REQUIRE(N == 0 || (avg > 0.f && std::isfinite(avg)), "bags_box_fwd: avg=%g must be positive and finite",
               static_cast<double>(avg));
  BAGS_REQUIRE(aligned(targets, 16) && aligned(weights, 16) && aligned(g, 16) && aligned(pred, 16),
               "bags_box_fwd: targets, weights, g and pred must be 16-byte aligned [N, 4] arrays");
  BAGS_REQUIRE(workspace_bytes >= bags_workspace_bytes(), "bags_box_fwd: workspace too small (%zu < %zu)",
               workspace_bytes, bags_workspace_bytes());
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  BoxFwdParams p{};
  p.x = x; p.ldx = ldx; p.w = w; p.ldw = ldw; p.bias = bias;
  p.labels = reinterpret_cast<const long long*>(labels);
  p.targets = targets; p.weights = weights;
  p.beta = beta; p.avg = N > 0 ? avg : 1.f;
  p.N = N; p.K = K; p.classes = classes;
  p.loss = loss; p.g = g; p.pred = pred; p.index = index;
  p.counter = reinterpret_cast<unsigned int*>(workspace) + kBoxCounterWord;
  p.part = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 256);
  // one warp per RoI; the grid depends only on N and the SM count, so the loss's summation order does too
  int workers = (N + kBoxThreads / 32 - 1) / (kBoxThreads / 32);
  if (workers > 4 * di.num_sms) workers = 4 * di.num_sms;
  if (workers < 1) workers = 1;
  const dim3 grid(workers + 1);   // + the class-sort CTA
  if (dtype == BAGS_DTYPE_BF16) bags_box_fwd_kernel<true><<<grid, kBoxThreads, 0, stream>>>(p);
  else                          bags_box_fwd_kernel<false><<<grid, kBoxThreads, 0, stream>>>(p);
  BAGS_CUDA(cudaGetLastError());
  return BAGS_OK;
}

extern "C" int bags_box_bwd(const float* g, const float* gout, const void* x, long long ldx, int dtype, const float* w,
                            long long ldw, const int64_t* labels, const int32_t* index, int N, int K, int classes,
                            float* dW, long long lddw, float* db, void* dX, long long lddx, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  BAGS_REQUIRE(N >= 0, "bags_box_bwd: bad shape N=%d", N);
  BAGS_REQUIRE(index && (N == 0 || g) && (dW == nullptr || N == 0 || x) && (dX == nullptr || (w && (N == 0 || labels))),
               "bags_box_bwd: NULL argument");
  if (int rc = check_box_operands("bags_box_bwd", dW != nullptr ? x : nullptr, ldx, dtype, dX != nullptr ? w : nullptr,
                                  ldw, K, classes))
    return rc;
  BAGS_REQUIRE(aligned(g, 16), "bags_box_bwd: g must be a 16-byte aligned [N, 4] array");
  if (dW != nullptr)
    BAGS_REQUIRE(aligned(dW, 16) && lddw >= K && (lddw % 4) == 0,
                 "bags_box_bwd: dW rows must be 16-byte aligned with lddw >= K and lddw %% 4 == 0 (lddw=%lld)", lddw);
  if (dX != nullptr)
    BAGS_REQUIRE(aligned(dX, dtype == BAGS_DTYPE_BF16 ? 8 : 16) && lddx >= K && (lddx % 4) == 0,
                 "bags_box_bwd: dX rows must be aligned like x with lddx >= K and lddx %% 4 == 0 (lddx=%lld)", lddx);
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  BoxBwdParams p{};
  p.g = g; p.gout = gout; p.x = x; p.ldx = ldx; p.w = w; p.ldw = ldw;
  p.labels = reinterpret_cast<const long long*>(labels);
  p.index = index;
  p.N = N; p.K = K; p.classes = classes;
  p.kslices = (K + kBoxSlice - 1) / kBoxSlice;
  p.dW = dW; p.lddw = lddw; p.db = db; p.dX = dX; p.lddx = lddx;
  // work list: class units (dW rows, db) first, then RoI units (dX rows)
  const long long class_units = (dW != nullptr) ? 1LL * classes * p.kslices : (db != nullptr ? classes : 0);
  const long long roi_units = (dX != nullptr) ? 1LL * N * p.kslices : 0;
  BAGS_REQUIRE(class_units + roi_units < (1LL << 31), "bags_box_bwd: N=%d K=%d is too large", N, K);
  p.class_units = static_cast<int>(class_units);
  if (class_units + roi_units == 0) return BAGS_OK;
  const dim3 grid(static_cast<unsigned>(class_units + roi_units));
  if (dtype == BAGS_DTYPE_BF16) bags_box_bwd_kernel<true><<<grid, kBoxBwdThreads, 0, stream>>>(p);
  else                          bags_box_bwd_kernel<false><<<grid, kBoxBwdThreads, 0, stream>>>(p);
  BAGS_CUDA(cudaGetLastError());
  return BAGS_OK;
}

// ----------------------------------------------------------------------------
// class-specific mask logits + mask_cross_entropy (fcn_mask_head.py:82,102,114-123, cross_entropy_loss.py:54-61)
// ----------------------------------------------------------------------------
static int check_mask_shape(const char* who, int dtype, long long ldw, int P, int Cin, int HW, int classes) {
  BAGS_REQUIRE(P >= 0 && Cin >= 1 && HW >= 1, "%s: bad shape P=%d Cin=%d HW=%d", who, P, Cin, HW);
  BAGS_REQUIRE(dtype == BAGS_DTYPE_F32 || dtype == BAGS_DTYPE_BF16, "%s: bad dtype %d", who, dtype);
  BAGS_REQUIRE(classes >= 1 && classes <= kBoxMaxClasses, "%s: classes=%d outside [1,%d]", who, classes, kBoxMaxClasses);
  BAGS_REQUIRE(ldw >= Cin, "%s: ldw=%lld must be >= Cin=%d", who, ldw, Cin);
  const long long tiles = (HW + kMaskTile - 1) / kMaskTile;
  BAGS_REQUIRE(tiles * P < (1LL << 30), "%s: P=%d HW=%d is too large", who, P, HW);
  return BAGS_OK;
}

static long long mask_rsum_floats(int P, int Cin, int HW) {
  const long long tiles = (HW + kMaskTile - 1) / kMaskTile;
  return static_cast<long long>(P) * tiles * (Cin + 2LL);
}

// four pixels per thread when every (RoI, channel) row starts on a 4-element boundary
static bool mask_vec4(const void* y, int dtype, int HW) {
  return (HW % 4) == 0 && aligned(y, dtype == BAGS_DTYPE_BF16 ? 8 : 16);
}

extern "C" int bags_mask_fwd(const void* y, int dtype, const float* w, long long ldw, const float* bias,
                             const int64_t* labels, const float* targets, int P, int Cin, int HW, int classes,
                             float* loss, float* g, float* rsum, size_t rsum_floats, int32_t* index, void* workspace,
                             size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = check_mask_shape("bags_mask_fwd", dtype, ldw, P, Cin, HW, classes)) return rc;
  BAGS_REQUIRE(loss && index && workspace && (P == 0 || (y && w && labels && targets && g && rsum)),
               "bags_mask_fwd: NULL argument");
  BAGS_REQUIRE(static_cast<long long>(rsum_floats) >= mask_rsum_floats(P, Cin, HW),
               "bags_mask_fwd: rsum too small (%zu < %lld floats)", rsum_floats, mask_rsum_floats(P, Cin, HW));
  BAGS_REQUIRE(workspace_bytes >= bags_workspace_bytes(), "bags_mask_fwd: workspace too small (%zu < %zu)",
               workspace_bytes, bags_workspace_bytes());
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  // the class index, also for P == 0 (all offsets zero)
  bags_mask_sort_kernel<<<1, kBoxThreads, 0, stream>>>(reinterpret_cast<const long long*>(labels), P, classes, index);
  BAGS_CUDA(cudaGetLastError());
  if (P == 0) {
    BAGS_CUDA(cudaMemsetAsync(loss, 0, sizeof(float), stream));
    return BAGS_OK;
  }
  MaskFwdParams p{};
  p.y = y; p.w = w; p.ldw = ldw; p.bias = bias;
  p.labels = reinterpret_cast<const long long*>(labels);
  p.targets = targets;
  p.P = P; p.Cin = Cin; p.HW = HW; p.classes = classes;
  p.tiles = (HW + kMaskTile - 1) / kMaskTile;
  p.n = static_cast<float>(static_cast<double>(P) * HW);
  p.loss = loss; p.g = g; p.rsum = rsum;
  p.counter = reinterpret_cast<unsigned int*>(workspace) + kMaskCounterWord;
  // one CTA per (RoI, pixel tile): the grid depends only on the shape, so the loss's summation order does too
  const dim3 grid(static_cast<unsigned>(P * p.tiles));
  const bool v4 = mask_vec4(y, dtype, HW);
  if (dtype == BAGS_DTYPE_BF16) {
    if (v4) bags_mask_fwd_kernel<true, 4><<<grid, kMaskThreads, 0, stream>>>(p);
    else    bags_mask_fwd_kernel<true, 1><<<grid, kMaskThreads, 0, stream>>>(p);
  } else {
    if (v4) bags_mask_fwd_kernel<false, 4><<<grid, kMaskThreads, 0, stream>>>(p);
    else    bags_mask_fwd_kernel<false, 1><<<grid, kMaskThreads, 0, stream>>>(p);
  }
  BAGS_CUDA(cudaGetLastError());
  return BAGS_OK;
}

extern "C" int bags_mask_bwd(const float* g, const float* rsum, const float* gout, int dtype, const float* w,
                             long long ldw, const int64_t* labels, const int32_t* index, int P, int Cin, int HW,
                             int classes, float* dW, long long lddw, float* db, void* dY, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = check_mask_shape("bags_mask_bwd", dtype, ldw, P, Cin, HW, classes)) return rc;
  BAGS_REQUIRE(index && ((dW == nullptr && db == nullptr) || P == 0 || rsum) &&
               (dY == nullptr || P == 0 || (g && w && labels)),
               "bags_mask_bwd: NULL argument");
  if (dW != nullptr) BAGS_REQUIRE(lddw >= Cin, "bags_mask_bwd: lddw=%lld must be >= Cin=%d", lddw, Cin);
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  MaskBwdParams p{};
  p.g = g; p.rsum = rsum; p.gout = gout; p.w = w; p.ldw = ldw;
  p.labels = reinterpret_cast<const long long*>(labels);
  p.index = index;
  p.P = P; p.Cin = Cin; p.HW = HW; p.classes = classes;
  p.tiles = (HW + kMaskTile - 1) / kMaskTile;
  p.dW = dW; p.lddw = lddw; p.db = db; p.dY = dY;
  p.chunks = (Cin + 1 + 31) / 32;
  // work list: class units (32 columns of dW and db per class) first, then (RoI, pixel tile) units (dY)
  const long long class_units = (dW != nullptr || db != nullptr) ? 1LL * classes * p.chunks : 0;
  const long long roi_units = (dY != nullptr) ? 1LL * P * p.tiles : 0;
  BAGS_REQUIRE(class_units + roi_units < (1LL << 31), "bags_mask_bwd: P=%d Cin=%d HW=%d is too large", P, Cin, HW);
  p.class_units = static_cast<int>(class_units);
  if (class_units + roi_units == 0) return BAGS_OK;
  const dim3 grid(static_cast<unsigned>(class_units + roi_units));
  const bool v4 = dY != nullptr && mask_vec4(dY, dtype, HW);
  if (dtype == BAGS_DTYPE_BF16) {
    if (v4) bags_mask_bwd_kernel<true, 4><<<grid, kMaskThreads, 0, stream>>>(p);
    else    bags_mask_bwd_kernel<true, 1><<<grid, kMaskThreads, 0, stream>>>(p);
  } else {
    if (v4) bags_mask_bwd_kernel<false, 4><<<grid, kMaskThreads, 0, stream>>>(p);
    else    bags_mask_bwd_kernel<false, 1><<<grid, kMaskThreads, 0, stream>>>(p);
  }
  BAGS_CUDA(cudaGetLastError());
  return BAGS_OK;
}

// test-time label-channel logits (fcn_mask_head.py:125-181 and htc.py:403-421 read one channel per detection)
extern "C" int bags_mask_logits(const void* y, int dtype, const float* w, long long ldw, const float* bias,
                                const int64_t* channels, int n, int Cin, int HW, int classes, void* out,
                                void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = check_mask_shape("bags_mask_logits", dtype, ldw, n, Cin, HW, classes)) return rc;
  BAGS_REQUIRE(n == 0 || (y && w && channels && out), "bags_mask_logits: NULL argument");
  if (n == 0) return BAGS_OK;
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  MaskLogitsParams p{};
  p.y = y; p.w = w; p.ldw = ldw; p.bias = bias;
  p.channels = reinterpret_cast<const long long*>(channels);
  p.Cin = Cin; p.HW = HW; p.classes = classes;
  p.tiles = (HW + kMaskTile - 1) / kMaskTile;
  p.out = out;
  const dim3 grid(static_cast<unsigned>(n * p.tiles));
  const bool v4 = mask_vec4(y, dtype, HW);
  if (dtype == BAGS_DTYPE_BF16) {
    if (v4) bags_mask_logits_kernel<true, 4><<<grid, kMaskThreads, 0, stream>>>(p);
    else    bags_mask_logits_kernel<true, 1><<<grid, kMaskThreads, 0, stream>>>(p);
  } else {
    if (v4) bags_mask_logits_kernel<false, 4><<<grid, kMaskThreads, 0, stream>>>(p);
    else    bags_mask_logits_kernel<false, 1><<<grid, kMaskThreads, 0, stream>>>(p);
  }
  BAGS_CUDA(cudaGetLastError());
  return BAGS_OK;
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


// Split-K factor of the merged backward's dW units.  The kernel deals its work list (dW units split-major, then the
// dX units) round-robin to min(units, SMs) CTAs, and a CTA runs its units back to back, so the backward ends with the
// CTA that holds the most work.  The cost of a split factor is exactly that: the largest sum over one CTA's units of
// (k-blocks + kUnitOverheadKb), where the overhead stands for a unit's epilogue and pipeline fill.  Ties go to fewer
// splits (less split-K red.add traffic).  A pure function of the shape and the SM count.
static constexpr int kUnitOverheadKb = 2;
static int merged_dw_splits(int dw_tiles, int dw_kblocks, int dx_units, int dx_kblocks, int num_sms) {
  // the walk over the work list is O(16 units); a training loop asks for the same shape every step
  thread_local int memo_key[5] = {-1, -1, -1, -1, -1}, memo_splits = 1;
  const int key[5] = {dw_tiles, dw_kblocks, dx_units, dx_kblocks, num_sms};
  if (std::memcmp(key, memo_key, sizeof(key)) == 0) return memo_splits;
  int splits = 1;
  long long best = -1;
  std::vector<long long> load;
  for (int sp = 1; sp <= 16 && sp <= dw_kblocks; ++sp) {
    const int units = dw_tiles * sp + dx_units;
    const int ctas = units < num_sms ? units : num_sms;
    load.assign(ctas, 0);
    const int base = dw_kblocks / sp, rem = dw_kblocks % sp;
    for (int u = 0; u < units; ++u) {
      const int kb = u < dw_tiles * sp ? base + (u / dw_tiles < rem ? 1 : 0) : dx_kblocks;
      load[u % ctas] += kb + kUnitOverheadKb;
    }
    long long cost = 0;
    for (long long l : load) cost = l > cost ? l : cost;
    if (best < 0 || cost < best) { best = cost; splits = sp; }
  }
  std::memcpy(memo_key, key, sizeof(key));
  memo_splits = splits;
  return splits;
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

// One launch of bags_bwd_merged_kernel over the problems asked for through p.dw.out and p.dx.out:
//   dW[C, K] += rowscale(c) * dz^T x   split-K reduce-add, `splits` partials (< 1: merged_dw_splits)
//   dX[N, K]  = dz wb                  wb = W' (the preparation kernel's scaled copy) or W
// The caller fills the epilogue fields of p.dw (out, ldo, gscale, groups, colsum) and p.dx (out, ldo), and gout, G,
// uniform_ok, inputs_ready and wprime_prepared; this fills the shapes, tilings and operands.  Only the tensor maps of
// the problems present are encoded (the others stay zero), so x is not read without dW, nor w and wb without dX.
template <bool TF32>
static int launch_bwd_merged(const void* dz, long long ldd, const void* x, long long ldx, const void* w, const void* wb,
                             long long ldw, int N, int K, int C, int splits, BwdMergedParams p, const DeviceInfo& di,
                             cudaStream_t stream) {
  using CW = BwdDwCfg<TF32>;
  using CX = BwdDxCfg<TF32>;
  const int dtype = TF32 ? BAGS_DTYPE_F32 : BAGS_DTYPE_BF16;
  CUtensorMap t_dzT{}, t_xT{}, t_dz{}, t_w{}, t_wp{}, t_dx{};
  int rc;
  GemmParams& px = p.dx;
  if (px.out != nullptr) {
    px.M = N; px.N = K; px.K = C;
    px.num_m_tiles = (N + CX::BLOCK_M - 1) / CX::BLOCK_M;
    px.num_n_tiles = (K + CX::BLOCK_N_ - 1) / CX::BLOCK_N_;
    px.kblocks_total = (C + CX::BLOCK_K - 1) / CX::BLOCK_K;
    px.num_splits = 1;
    px.b_ptr = static_cast<const float*>(wb); px.ldb = ldw; px.b_rows = K; px.b_k = C;
    p.w = static_cast<const float*>(w);
    p.dx_units = px.num_m_tiles * px.num_n_tiles;
    // TMA-stored bf16 dX: a store box writes whole 16-byte pieces at the right edge, so K must end on one
    p.dx_tma = (!TF32 && (K % 8) == 0 && (px.ldo % 8) == 0) ? 1 : 0;
    if ((rc = make_tmap(&t_dz, dz, dtype, C, N, ldd, CX::BLOCK_K, CX::BLOCK_M))) return rc;   // A = dz
    if ((rc = make_tmap(&t_w, w, dtype, K, C, ldw, CX::SLAB, CX::BLOCK_K))) return rc;       // B = W^T
    if ((rc = make_tmap(&t_wp, wb, dtype, K, C, ldw, CX::SLAB, CX::BLOCK_K))) return rc;     // B = W'^T
    if (p.dx_tma && (rc = make_tmap(&t_dx, px.out, dtype, K, N, px.ldo, 64, 64))) return rc;  // dX store boxes
  }
  GemmParams& pw = p.dw;
  if (pw.out != nullptr) {
    pw.M = C; pw.N = K; pw.K = N;
    pw.num_m_tiles = (C + CW::BLOCK_M - 1) / CW::BLOCK_M;
    pw.num_n_tiles = (K + CW::BLOCK_N_ - 1) / CW::BLOCK_N_;
    pw.kblocks_total = (N + CW::BLOCK_K - 1) / CW::BLOCK_K;
    const int dw_tiles = pw.num_m_tiles * pw.num_n_tiles;
    if (splits < 1) splits = merged_dw_splits(dw_tiles, pw.kblocks_total, p.dx_units, px.kblocks_total, di.num_sms);
    if (splits > pw.kblocks_total) splits = pw.kblocks_total;
    pw.num_splits = splits;
    pw.a_ptr = static_cast<const float*>(dz); pw.lda = ldd; pw.a_rows = C; pw.a_k = N;
    pw.b_ptr = static_cast<const float*>(x); pw.ldb = ldx; pw.b_rows = K; pw.b_k = N;
    p.dw_units = dw_tiles * splits;
    if ((rc = make_tmap(&t_dzT, dz, dtype, C, N, ldd, CW::SLAB, CW::BLOCK_K))) return rc;   // A = dz^T
    if ((rc = make_tmap(&t_xT, x, dtype, K, N, ldx, CW::SLAB, CW::BLOCK_K))) return rc;     // B = x^T
  }
  p.timing = g_timing ? g_timing + 1024 * 8 : nullptr;   // rows [1024, 1024 + 2 grid)
  const int units = p.dw_units + p.dx_units;
  if (units == 0) return BAGS_OK;
  auto kernel = bags_bwd_merged_kernel<TF32>;
  constexpr int smem = bwd_merged_smem_bytes<TF32>();
  BAGS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int grid = units < di.num_sms ? units : di.num_sms;
  BAGS_CUDA(launch(kernel, dim3(grid), dim3(CW::NUM_THREADS), smem, stream, true, false, t_dzT, t_xT, t_dz, t_w, t_wp,
                   t_dx, p));
  return BAGS_OK;
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
  const bool bf = dtype == BAGS_DTYPE_BF16;
  const int vecw = bf ? 8 : 4;

  const bool want_scale = (dX != nullptr && N > 0 && gout != nullptr);
  const bool want_colpart = (db != nullptr && colsum == nullptr && N > 0);
  if (want_scale || want_colpart) {
    BAGS_REQUIRE(wscratch != nullptr && wscratch_bytes >= bags_bwd_scratch_bytes(C, ldw, dtype),
                 "bags_bwd: wscratch must provide bags_bwd_scratch_bytes() = %zu bytes (got %zu)",
                 bags_bwd_scratch_bytes(C, ldw, dtype), wscratch_bytes);
    BAGS_REQUIRE((reinterpret_cast<uintptr_t>(wscratch) & 255) == 0, "bags_bwd: wscratch must be 256-byte aligned");
  }
  if (dW != nullptr) {
    BAGS_REQUIRE(x != nullptr || N == 0, "bags_bwd: x is NULL but dW requested");
    BAGS_REQUIRE(lddw >= K && (lddw % 4) == 0 && (K % 4) == 0 && (reinterpret_cast<uintptr_t>(dW) & 15) == 0,
                 "bags_bwd: dW must be 16-byte aligned with K and lddw multiples of 4");
  }
  if (dX != nullptr && N > 0) {
    BAGS_REQUIRE(w != nullptr, "bags_bwd: w is NULL but dX requested");
    BAGS_REQUIRE((reinterpret_cast<uintptr_t>(dX) & 15) == 0, "bags_bwd: dX not 16-byte aligned");
  }
  if (want_scale)
    BAGS_REQUIRE((K % vecw) == 0 && (ldw % vecw) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0,
                 "bags_bwd: w must be 16-byte aligned with K and ldw multiples of %d", vecw);
  if (want_colpart)
    BAGS_REQUIRE(((ldd * (bf ? 2 : 4)) % 16) == 0 && (reinterpret_cast<uintptr_t>(dz) & 15) == 0,
                 "bags_bwd: dz rows must be 16-byte aligned");
  BAGS_REQUIRE(db == nullptr || colsum == nullptr || colsum_tiles >= 1,
               "bags_bwd: db requested from colsum with colsum_tiles = %d < 1", colsum_tiles);
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;

  if (db != nullptr && colsum == nullptr && N == 0) {   // no rows: zero bias gradient
    BAGS_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * C, stream));
    db = nullptr;
  }
  float* colpart = (wscratch == nullptr) ? nullptr
                   : reinterpret_cast<float*>(reinterpret_cast<char*>(wscratch) + wprime_bytes(C, ldw, dtype));

  // ---- preparation (one small kernel): zero dW, W' = gout-scaled W, bias-gradient partial column sums; then the
  // requested contractions in one merged launch (see bags_bwd_merged_kernel) ----
  // a dz column outside every bin is scaled by 0 when gout is given: the merged kernel's uniform-gout shortcut (dz W,
  // output scaled by gout[0]) would scale it by gout[0], so it is taken only when the bins tile [0, C)
  const bool no_gaps = bins_tile(slices_host, G, C);
  BwdPrepParams pp{};
  bool prep_launched = false;
  if (dW != nullptr || want_scale || want_colpart) {
    pp.dW = dW; pp.lddw = lddw; pp.C = C; pp.K = K;
    pp.w = w; pp.wscr = wscratch; pp.ldw = ldw; pp.gout = gout; pp.gt = gt;
    pp.dz = dz; pp.ldd = ldd; pp.N = N; pp.colpart = colpart; pp.ctiles = kColsumTiles;
    pp.z_ctas = (dW != nullptr && !prezeroed) ? di.num_sms : 0;
    pp.s_ctas = want_scale ? di.num_sms : 0;
    pp.c_ctas = want_colpart ? ((C + 63) / 64) * kColsumTiles : 0;
    pp.skip_scale_if_uniform = no_gaps ? 1 : 0;   // the merged kernel reads W itself (see bp.uniform_ok)
    pp.timing = g_timing ? g_timing + 2048 * 8 : nullptr;       // rows [2048, 4096)
    const int grid = pp.z_ctas + pp.s_ctas + pp.c_ctas;
    if (grid > 0) {
      BAGS_CUDA(launch(bf ? bwd_prep_kernel<false> : bwd_prep_kernel<true>, dim3(grid), dim3(256), 0, stream, true, false, pp));
      prep_launched = true;
    }
  }
  const float* cs_in = (colsum != nullptr) ? colsum : colpart;
  const int cs_tiles = (colsum != nullptr) ? colsum_tiles : kColsumTiles;
  if (db != nullptr && !(dW != nullptr && N > 0)) {   // (with dW units, their epilogue writes db)
    scale_colsum_kernel<<<(C + 255) / 256, 256, 0, stream>>>(cs_in, cs_tiles, db, C, gt, gout);
    BAGS_CUDA(cudaGetLastError());
  }
  if (N == 0 || (dW == nullptr && dX == nullptr)) return BAGS_OK;

  BwdMergedParams bp{};
  if (dW != nullptr) {
    GemmParams& pw = bp.dw;
    pw.out = dW; pw.ldo = lddw;
    pw.gscale = gout; pw.G = (gout != nullptr) ? gt.G : 0;
    for (int g = 0; g < kMaxGroups; ++g) { pw.gstart[g] = gt.start[g]; pw.glen[g] = gt.len[g]; }
    pw.colsum_in = (db != nullptr) ? cs_in : nullptr;
    pw.colsum_tiles = cs_tiles;
    pw.colsum_out = db;
  }
  bp.dx.out = dX; bp.dx.ldo = lddx;
  bp.gout = (dX != nullptr) ? gout : nullptr;
  bp.G = gt.G;
  bp.uniform_ok = no_gaps ? 1 : 0;
  bp.inputs_ready = prep_launched ? 1 : 0;
  bp.wprime_prepared = want_scale ? 1 : 0;
  const void* wb = want_scale ? wscratch : w;
  const int splits = env_int("BAGS_DW_SPLITS", 0);   // a forced dW split count; unset: merged_dw_splits
  return bf ? launch_bwd_merged<false>(dz, ldd, x, ldx, w, wb, ldw, N, K, C, splits, bp, di, stream)
            : launch_bwd_merged<true>(dz, ldd, x, ldx, w, wb, ldw, N, K, C, splits, bp, di, stream);
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
  if (count == 0) return BAGS_OK;
  // enough blocks to keep one vector per thread and unroll slot in flight, at most kArMaxBlocks;
  // every rank must launch the same grid: it depends only on (count, world, max_blocks) and the transport
  const long long per_rank = (count / 4 + world - 1) / world;
  long long blocks = (per_rank + kArThreads * 4LL - 1) / (kArThreads * 4LL);
  if (blocks < 1) blocks = 1;
  const bool mm = p.mc != nullptr && !env_int("BAGS_AR_NO_MULTIMEM", 0);
  // Default grid: one block per SM on the multimem path (the exchange runs inside the step, where a small grid leaves
  // the switch bandwidth unused); the plain peer path keeps one vector per thread in flight.
  if (max_blocks <= 0) max_blocks = mm ? di.num_sms : kArMaxBlocks;
  if (max_blocks > kArMaxBlocks) max_blocks = kArMaxBlocks;
  if (blocks > max_blocks) blocks = max_blocks;
  const dim3 grid(static_cast<unsigned>(blocks)), block(kArThreads);
  auto kernel = mm ? bags_grad_allreduce_kernel<true> : bags_grad_allreduce_kernel<false>;
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

// ----------------------------------------------------------------------------
// test-time masks as COCO RLE (see bags_segm.cuh)
// ----------------------------------------------------------------------------
extern "C" int bags_segm_rle(const float* probs, int n, int mask_h, int mask_w, const int32_t* boxes_host,
                             int32_t* boxes, int img_h, int img_w, double thr, int64_t* lengths, char* out,
                             void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  BAGS_REQUIRE(n >= 0, "bags_segm_rle: n = %d < 0", n);
  BAGS_REQUIRE(mask_h >= 2 && mask_w >= 2, "bags_segm_rle: mask size %d x %d: at least 2 x 2 (OpenCV resizes one-row "
               "and one-column maps by other arithmetic)", mask_h, mask_w);
  BAGS_REQUIRE(img_h >= 1 && img_w >= 1 && static_cast<long long>(img_h) * img_w <= 0x7fffffffLL,
               "bags_segm_rle: canvas %d x %d must be positive and hold at most 2^31 - 1 pixels", img_h, img_w);
  if (n == 0) return BAGS_OK;
  BAGS_REQUIRE(probs && boxes_host && boxes && lengths, "bags_segm_rle: NULL argument");
  for (int d = 0; d < n; ++d) {
    const int32_t* b = boxes_host + 4 * static_cast<size_t>(d);
    BAGS_REQUIRE(b[2] >= 1 && b[3] >= 1, "bags_segm_rle: detection %d has an empty box (w = %d, h = %d)", d, b[2], b[3]);
    BAGS_REQUIRE(b[0] >= 0 && b[1] >= 0 && b[2] <= img_w - b[0] && b[3] <= img_h - b[1],
                 "bags_segm_rle: detection %d's box (left %d, top %d, w %d, h %d) leaves the %d x %d canvas", d, b[0],
                 b[1], b[2], b[3], img_h, img_w);
  }
  BAGS_REQUIRE((reinterpret_cast<uintptr_t>(boxes) & 15) == 0, "bags_segm_rle: boxes must be 16-byte aligned");
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  // pageable source: staged by the driver before the call returns, no wait on the device
  BAGS_CUDA(cudaMemcpyAsync(boxes, boxes_host, 16 * static_cast<size_t>(n), cudaMemcpyHostToDevice, stream));
  bags_segm_rle_kernel<<<n, kSegmThreads, 0, stream>>>(probs, mask_h, mask_w, reinterpret_cast<const int4*>(boxes),
                                                       img_h, img_w, thr, reinterpret_cast<long long*>(lengths), out);
  BAGS_CUDA(cudaGetLastError());
  return BAGS_OK;
}

// ----------------------------------------------------------------------------
// training mask targets (see bags_mask_target.cuh)
// ----------------------------------------------------------------------------
extern "C" int bags_mask_target(const float* const* boxes_host, const int64_t* const* gt_inds_host,
                                const uint8_t* const* masks_host, const int32_t* sizes_host, int n_images, int mask_h,
                                int mask_w, float* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  BAGS_REQUIRE(n_images >= 0, "bags_mask_target: n_images = %d < 0", n_images);
  BAGS_REQUIRE(mask_h >= 1 && mask_w >= 1 && mask_h <= kMaskTargetMaxSize && mask_w <= kMaskTargetMaxSize,
               "bags_mask_target: mask size %d x %d outside [1, %d]", mask_h, mask_w, kMaskTargetMaxSize);
  if (n_images == 0) return BAGS_OK;
  BAGS_REQUIRE(boxes_host && gt_inds_host && masks_host && sizes_host, "bags_mask_target: NULL argument");
  long long rows = 0;
  for (int i = 0; i < n_images; ++i) {
    const int32_t* s = sizes_host + 4 * static_cast<size_t>(i);
    BAGS_REQUIRE(s[0] >= 0 && s[1] >= 0 && s[2] >= 0 && s[3] >= 0,
                 "bags_mask_target: image %d has a negative size (num_pos %d, num_gt %d, H %d, W %d)", i, s[0], s[1],
                 s[2], s[3]);
    BAGS_REQUIRE(s[0] == 0 || (boxes_host[i] && gt_inds_host[i]), "bags_mask_target: image %d: NULL boxes or gt_inds",
                 i);
    BAGS_REQUIRE(static_cast<long long>(s[1]) * s[2] * s[3] == 0 || masks_host[i],
                 "bags_mask_target: image %d: NULL masks", i);
    BAGS_REQUIRE(s[0] == 0 || (aligned(boxes_host[i], 4) && aligned(gt_inds_host[i], 8)),
                 "bags_mask_target: image %d: boxes must be 4-byte and gt_inds 8-byte aligned", i);
    rows += s[0];
  }
  BAGS_REQUIRE(rows <= 0x7fffffffLL, "bags_mask_target: %lld positive RoIs: at most 2^31 - 1", rows);
  if (rows == 0) return BAGS_OK;
  BAGS_REQUIRE(out, "bags_mask_target: NULL argument");
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  // the per-image table travels as a kernel argument: kMaskTargetMaxImages images per launch
  long long done = 0;
  for (int i0 = 0; i0 < n_images; i0 += kMaskTargetMaxImages) {
    MaskTargetParams p{};
    p.n_images = n_images - i0 < kMaskTargetMaxImages ? n_images - i0 : kMaskTargetMaxImages;
    p.mask_h = mask_h;
    p.mask_w = mask_w;
    p.out = out + done * mask_h * mask_w;
    int begin = 0;
    for (int k = 0; k < p.n_images; ++k) {
      const int32_t* s = sizes_host + 4 * static_cast<size_t>(i0 + k);
      p.img[k] = MaskTargetImage{boxes_host[i0 + k], reinterpret_cast<const long long*>(gt_inds_host[i0 + k]),
                                 masks_host[i0 + k], begin, s[1], s[2], s[3]};
      begin += s[0];
    }
    if (begin > 0) bags_mask_target_kernel<<<begin, kMaskTargetThreads, 0, stream>>>(p);
    BAGS_CUDA(cudaGetLastError());
    done += begin;
  }
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
  BAGS_REQUIRE((reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 7) == 0,
               "bags_cast_bf16: src must be 16-byte and dst 8-byte aligned");
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
  const bool bf = dtype == BAGS_DTYPE_BF16;
  BAGS_REQUIRE(bf || dtype == BAGS_DTYPE_F32, "bags_gemm_probe: bad dtype");
  // the kernels the product runs: kk the forward GEMM, kmn the merged backward's dX units alone (a = dz [M, K],
  // b = W [K, N]), mnmn its split-K dW units alone (a = dz [K, M], b = x [K, N])
  const bool kk = !a_mn && !b_mn && epi == 0, kmn = !a_mn && b_mn && epi == (bf ? 1 : 0);
  const bool mnmn = a_mn && b_mn && epi == 2;
  BAGS_REQUIRE(block_n == 256 && (kk || kmn || mnmn),
               "bags_gemm_probe: configuration a_mn=%d b_mn=%d block_n=%d epi=%d dtype=%d not instantiated", a_mn, b_mn,
               block_n, epi, dtype);
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  if (kk) {
    GemmArgs ga{};
    ga.a = a; ga.lda = lda;
    ga.b = b; ga.ldb = ldb;
    ga.M = M; ga.N = N; ga.K = K; ga.dtype = dtype; ga.splits = 1;
    ga.p.out = out; ga.p.ldo = ldo;
    return bf ? launch_gemm<256, EPI_STORE_F32, false, 4>(ga, di, stream)
              : launch_gemm<256, EPI_STORE_F32, true, 4>(ga, di, stream);
  }
  // in bags_bwd's terms: kmn has M RoIs, N features and K logits; mnmn has K RoIs, N features and M logits
  BwdMergedParams bp{};
  if (kmn) {
    bp.dx.out = out; bp.dx.ldo = ldo;
    return bf ? launch_bwd_merged<false>(a, lda, nullptr, 0, b, b, ldb, M, N, K, 0, bp, di, stream)
              : launch_bwd_merged<true>(a, lda, nullptr, 0, b, b, ldb, M, N, K, 0, bp, di, stream);
  }
  bp.dw.out = out; bp.dw.ldo = ldo;
  if (splits < 1) splits = 1;
  return bf ? launch_bwd_merged<false>(a, lda, b, ldb, nullptr, nullptr, 0, K, N, M, splits, bp, di, stream)
            : launch_bwd_merged<true>(a, lda, b, ldb, nullptr, nullptr, 0, K, N, M, splits, bp, di, stream);
}
