/*
 * bags_b200.h -- C ABI of the H100-native Balanced Group Softmax (BAGS) RoI
 * classification head hot path.
 *
 * This is the drop-in boundary for the reference's fc_cls -> grouped softmax /
 * cross-entropy path (FishYuLi/BalancedGroupSoftmax, mmdetection v1.0rc0 fork):
 *
 *   reference interface                                   replaced by
 *   ---------------------------------------------------   -------------------------
 *   ConvFCBBoxHead.forward: self.fc_cls(x_cls)            bags_linear_act_fwd
 *     mmdet/models/bbox_heads/convfc_bbox_head.py:166
 *   GSBBoxHeadWith0._sample_others                        bags_sample_others
 *     mmdet/models/bbox_heads/gs_bbox_head_with0.py:63-89
 *   GSBBoxHeadWith0._remap_labels (avg_factor)            bags_mask_avg
 *     gs_bbox_head_with0.py:91-112 (:109)
 *   _remap_labels + _slice_preds + 5x CrossEntropyLoss    bags_group_ce
 *     gs_bbox_head_with0.py:134-171 ;
 *     mmdet/models/losses/cross_entropy_loss.py:9-19,86-103 ;
 *     mmdet/models/losses/utils.py:26-53
 *   fc_cls + loss in one call                             bags_fwd
 *   ReweightBBoxHead.loss: fc_cls + weighted softmax CE   bags_ce_fwd
 *     + accuracy (reweight_bbox_head.py:36-55)
 *   autograd backward of the above (dW, db, dX)           bags_bwd
 *     triggered at mmdet/core/utils/dist_utils.py:53
 *   GSBBoxHeadWith0._merge_score                          bags_merge_scores
 *     gs_bbox_head_with0.py:239-273
 *   allreduce_grads / _allreduce_coalesced                bags_grad_allreduce
 *     mmdet/core/utils/dist_utils.py:9-41
 *
 * The reference's own native plugins export pybind11 `forward`/`backward`
 * functions over at::Tensor (e.g. mmdet/ops/sigmoid_focal_loss/src/
 * sigmoid_focal_loss.cpp:40-45) and launch on the current stream.  This ABI is
 * the torch-free equivalent: plain device pointers + sizes + an explicit
 * cudaStream_t, loadable with ctypes / dlopen.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in `_host`
 *   - the caller owns all buffers, including workspaces; the library allocates nothing
 *   - no call synchronises the device or reads device data on the host
 *   - return value 0 = success; otherwise a negative error code and a message
 *     retrievable with bags_last_error() (thread-local)
 *   - dtype: BAGS_DTYPE_F32 = fp32 operands (TF32 tensor-core products, fp32 accumulate)
 *            BAGS_DTYPE_BF16 = bf16 operands (fp32 accumulate, fp32 softmax / loss)
 *   - `stream` is a cudaStream_t passed as void*
 *   - slices_host is int32 [G,2] = (start, len) per bin, ascending and non-overlapping
 *     (tools/lvis_analyse.py:45-50), G <= BAGS_MAX_BINS
 *   - requires an sm_90 (H100) device; there is no CPU or other-arch fallback
 */
#ifndef BAGS_B200_H_
#define BAGS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BAGS_ABI_VERSION 2
#define BAGS_MAX_BINS 8
#define BAGS_DTYPE_F32 0
#define BAGS_DTYPE_BF16 1
#define BAGS_WEIGHTS_U8 0    /* per-RoI sample weights: 0/1 bytes */
#define BAGS_WEIGHTS_F32 1   /* per-RoI sample weights: fp32 (reweight head variant) */

#define BAGS_OK 0
#define BAGS_ERR_INVALID (-1)   /* bad argument / unsupported shape */
#define BAGS_ERR_CUDA (-2)      /* CUDA runtime / driver error */
#define BAGS_ERR_ARCH (-3)      /* device is not sm_90 */

int bags_abi_version(void);
const char* bags_last_error(void);

/* bytes the caller must provide (zero-initialised ONCE) as `workspace` to bags_group_ce / bags_fwd: one workspace per
 * stream, kept across calls (it holds the fused forward's exchange counters, which are never reset) */
size_t bags_workspace_bytes(void);

/* wmask[G,N] (uint8 0/1) and avg[G] = max(sum w, 1): bin 0 all ones; bins >= 1 keep every in-bin row
 * and a uniform random subset of k = int(F * ratio) "others" rows (F = #in-bin rows), exactly as
 * _sample_others does, but on the device with a counter-based RNG keyed by the effective seed
 * seed + (*seed_step) * 0x9E3779B97F4A7C15, read on the DEVICE (seed_step may be NULL: the seed as given).
 * seed_step serves CUDA-graph replays, where by-value arguments are frozen at capture time: the caller advances the
 * counter between replays (not with the kernel that immediately precedes this one in the stream). */
int bags_sample_others(const int64_t* labels, const int32_t* label2bin, int N, int G, int classes,
                       double ratio, uint64_t seed, const uint64_t* seed_step, uint8_t* wmask,
                       float* avg, void* stream);

/* avg[g] = max(sum_n wmask[g,n], 1) for caller-provided masks */
int bags_mask_avg(const uint8_t* wmask, int N, int G, float* avg, void* stream);

/* Per-bin softmax cross-entropy over logit slices.
 *   loss[g] = sum_n w[g,n] * (logsumexp(z[n, slice_g]) - z[n, start_g + label2bin[g, labels[n]]]) / avg[g]
 * Optional outputs (NULL to skip): lse[N,G]; dz[N,ldd] (dtype elements) = w/avg * (softmax - onehot),
 * i.e. d(sum_g loss_g)/dz before the per-bin upstream gradients are applied; colsum[C] = sum_n dz.
 * weights: [G,N] sample weights w of type weights_dtype -- BAGS_WEIGHTS_U8 (0/1 bytes, the sampler's masks) or
 * BAGS_WEIGHTS_F32 (the reweight head variant's bags_reweight output); NULL => all ones.  avg NULL => N.
 * C % 4 == 0, ldz % 4 == 0, C <= 4096. */
int bags_group_ce(const float* logits, long long ldz, const int64_t* labels,
                  const int32_t* label2bin, const int32_t* slices_host, const void* weights,
                  int weights_dtype, const float* avg, int N, int C, int G, int classes, float* loss,
                  float* lse, void* dz, long long ldd, int dz_dtype, float* colsum, void* workspace,
                  size_t workspace_bytes, void* stream);

/* 1 if bags_fwd can run its fused kernel (logits == NULL) for this bin table: C <= 1280, G <= 6, C % 4 == 0,
 * bins tile [0, C) contiguously. */
int bags_fused_eligible(const int32_t* slices_host, int G, int C);

/* fc_cls + grouped softmax-CE (+ dz, colsum) in one call; weights / weights_dtype as in bags_group_ce.
 *   logits == NULL : fused kernel -- the logits stay in registers and never reach HBM
 *                    (requires bags_fused_eligible); ldz is ignored.
 *   logits != NULL : bags_linear_act_fwd (fp32 output, no activation) into `logits` followed by bags_group_ce
 *                    (same arguments).
 * colsum (optional) is [colsum_tiles, C] with colsum_tiles = ceil(N/128): per-128-row-tile partial column sums
 * of dz (written with plain stores, no pre-zeroing needed); their sum over tiles is sum_n dz[n, :].
 * clear (optional, NULL / 0 = none): `clear_bytes` bytes at `clear` (16-byte aligned, a multiple of 16; typically the
 * caller's dW) are set to zero -- by the fused kernel while its CTAs wait for each other's softmax partials, or by a memset on the
 * materialised route.  Together with `colsum` this lets bags_bwd run without any preparation work (flag
 * BAGS_BWD_DW_PREZEROED, no column-sum job).
 * The fused kernel is launched with programmatic dependent launch: when the preceding kernel in the stream is
 * bags_sample_others / bags_mask_avg, its GEMM mainloop overlaps them and only the epilogue waits.  It is also a
 * cooperative launch of at most one 4-CTA group per 4 SMs that loops over the row tiles (no limit on N); where that
 * grid cannot be resident at once, bags_fwd returns BAGS_ERR_CUDA. */
int bags_fwd(const void* x, long long ldx, const void* w, long long ldw, const float* bias,
             const int64_t* labels, const int32_t* label2bin, const int32_t* slices_host,
             const void* weights, int weights_dtype, const float* avg, int N, int K, int C, int G, int classes,
             int dtype, float* logits, long long ldz, float* loss, float* lse, void* dz,
             long long ldd, float* colsum, int colsum_tiles, void* workspace, size_t workspace_bytes,
             void* clear, size_t clear_bytes, void* stream);

/* fc_cls + softmax cross-entropy over all C logits (ReweightBBoxHead, mmdet/models/bbox_heads/reweight_bbox_head.py;
 * BBoxHead.loss, bbox_head.py:97-129), logits kept on chip -- the fused kernel of bags_fwd with the single bin (0, C):
 *   loss[0] = sum_n w[n] * (logsumexp(z[n,:]) - z[n, labels[n]]) / avg[0]      (weights NULL => w = 1, avg NULL => N)
 *   acc[0]  = 100 * #{n : z[n, labels[n]] == max_c z[n, c]} / N                (optional, NULL to skip; mmdet accuracy,
 *             topk = 1.  A tie with the row maximum counts as correct.  N <= 2^24 when requested: the count is exact)
 * weights: fp32 [N] per-RoI weights (cls_weight[labels] for ReweightBBoxHead).
 * dz, colsum, clear, workspace: as bags_fwd (ldd % 8 == 0, colsum [ceil(N/128), C]); dW, db and dX then come from
 * bags_bwd with the single slice (0, C) and gout = dL/dloss[0].
 * 1 <= C <= 1280, any C (not only multiples of 4); labels in [0, C) (a label outside it is scored against column 0).
 * N == 0: loss = 0, acc = 0. */
int bags_ce_fwd(const void* x, long long ldx, const void* w, long long ldw, const float* bias, const int64_t* labels,
                const float* weights, const float* avg, int N, int K, int C, int dtype, float* loss, float* acc,
                void* dz, long long ldd, float* colsum, int colsum_tiles, void* workspace, size_t workspace_bytes,
                void* clear, size_t clear_bytes, void* stream);

/* ---- reweight head variant (GSBBoxHeadWith0Reweight, mmdet/models/bbox_heads/gs_bbox_head_with0_reweight.py:57-109):
 * per-(bin, RoI) fp32 weights instead of 0/1 masks, consumed by bags_fwd / bags_group_ce as BAGS_WEIGHTS_F32. ----
 * bags_reweight: wfloat[g,n] = wmask[g,n] * cls_weight[g, label2bin[g, labels[n]]] for g >= 1 (bin 0: wmask as is),
 *                avg[g] = max(sum_n wfloat[g,n], 1).  cls_weight is [G, wstride] fp32 (row 0 unused, index 0 = "others"). */
int bags_reweight(const int64_t* labels, const int32_t* label2bin, const uint8_t* wmask, const float* cls_weight,
                  int wstride, int N, int G, int classes, float* wfloat, float* avg, void* stream);

/* bytes of `wscratch` bags_bwd needs (row-scaled copy of w + bias-gradient partials) */
size_t bags_bwd_scratch_bytes(int C, long long ldw, int dtype);

/* Backward of bags_fwd given dz saved by the forward and gout[G] = dL/dloss_g (NULL => 1):
 *   dW[C,K]  = (gout ⊙ dz)^T x      fp32, overwritten         (NULL to skip)
 *   db[C]    = gout ⊙ sum_n dz[n,:]  fp32                      (NULL to skip)
 *   dX[N,K]  = (gout ⊙ dz) w         dtype elements            (NULL to skip)
 * colsum: optional [colsum_tiles, C] partial column sums of dz from the forward; NULL => recomputed from dz.
 * wscratch: 256-byte aligned, bags_bwd_scratch_bytes() bytes; required when (dX and gout) or (db without colsum).
 * flags: BAGS_BWD_DW_PREZEROED = dW is already zero on entry (stream-ordered), e.g. by bags_fwd's clear hook.
 * Launch structure: one small preparation kernel (zero dW, scaled W, column-sum partials) whose execution is
 * overlapped by the dW GEMM's mainloop (programmatic dependent launch), then the dX GEMM. */
#define BAGS_BWD_DW_PREZEROED 1
int bags_bwd(const void* dz, long long ldd, const void* x, long long ldx, const void* w,
             long long ldw, const float* gout, const int32_t* slices_host, const float* colsum,
             int colsum_tiles, float* dW, long long lddw, float* db, void* dX, long long lddx,
             void* wscratch, size_t wscratch_bytes, int N, int K, int C, int G, int dtype, int flags, void* stream);

/* scores[N,classes]: scores[:,0] = softmax(z[:,slice_0])[:,0];
 * scores[:,c] = softmax(z[:,slice_0])[:,1] * softmax(z[:,slice_g])[:,j] where cls2col[c] = start_g + j.
 * cls2col: int32 [classes] (device), -1 => score 0. */
int bags_merge_scores(const float* logits, long long ldz, const int32_t* slices_host,
                      const int32_t* cls2col, int N, int C, int G, int classes, float* scores,
                      long long lds, void* stream);

/* Data-parallel exchange of the head's gradient bucket over NVLink peer memory -- replaces the reference's
 * flatten + dist.all_reduce + div_(world_size) + copy-back (mmdet/core/utils/dist_utils.py:9-41) by ONE kernel:
 * cross-rank barrier, two-shot all-reduce (rank r reduces slice r and broadcasts it), cross-rank barrier.
 *   peer_bufs_host : HOST array [world] of this process's device mappings of every rank's bucket (symmetric /
 *                    peer-mapped memory, same layout on every rank; entry `rank` is the local bucket)
 *   mc_buf         : multicast (NVLS) mapping of the same bucket, or NULL -> plain peer loads / stores
 *   count          : fp32 elements at the start of the bucket to reduce in place (multiple of 4)
 *   flag_off_bytes : offset, inside the same allocation, of bags_grad_allreduce_flag_bytes(world) bytes of flag
 *                    words that the caller zeroes ONCE (before the first exchange, on every rank); every call
 *                    leaves them zero
 *   scale          : applied to the sum (1/world = the reference's mean)
 *   max_blocks     : grid size limit (0 = the library's default for the transport; every rank the same value);
 *                    a NEGATIVE value selects the soft-failure mode of a construction-time self test (see below)
 * Every rank must issue the call with the same (count, world, max_blocks).  Stream-ordered after the local
 * gradients' producer.  A rank that never arrives at the exchange (BAGS_AR_TIMEOUT_MS, default 30 s -- generous
 * against checkpoint / evaluation hooks and data-loader stalls) makes the waiting kernels set the uint32 status word at
 * flag_off_bytes + bags_grad_allreduce_status_offset(world) to 1 and TRAP: the process fails with a sticky CUDA
 * error instead of continuing on un-averaged gradients (the reference's NCCL all-reduce would wait for ever).  In the
 * soft mode (max_blocks < 0, 3 s) the kernel only sets the status word and returns without exchanging, so that a
 * self test at construction can fall back to NCCL. */
size_t bags_grad_allreduce_flag_bytes(int world);
long long bags_grad_allreduce_status_offset(int world);
int bags_grad_allreduce(void* const* peer_bufs_host, void* mc_buf, long long flag_off_bytes, long long count,
                        int rank, int world, float scale, int max_blocks, void* stream);

/* Per-class greedy NMS, the test-time consumer of bags_merge_scores -- one launch instead of the reference's Python loop
 * over 1230 classes (mmdet/core/post_processing/bbox_nms.py:34-54, IoU convention of
 * mmdet/ops/nms/src/nms_kernel.cu:13-21: "+1" widths, a box is suppressed when IoU with a kept higher-score box >
 * iou_thr), without any host-side candidate compaction (no device->host sync):
 *   order  [S, n] int32 : RoI index of the i-th best score of foreground class s+1 (one batched descending sort)
 *   counts [S]   int32 : how many of them exceed score_thr (bbox_nms.py:36), clamped to n by the kernel
 *   boxes  [n, box_cols] fp32 decoded boxes, box_cols == 4 (class-agnostic) or 4 * (S + 1) (per class; bbox_nms.py:39-42)
 *   keep   [S, n] uint8 out (0 beyond counts[s]); *overflow (device int32, zeroed by the caller) is set to 1 when a
 *   class has more than 1024 candidates (its tail is dropped). */
int bags_class_nms_dense(const float* boxes, int box_cols, const int32_t* order, const int32_t* counts,
                         int num_classes_fg, int n, float iou_thr, uint8_t* keep, int32_t* overflow, void* stream);

/* test hook: launch `blocks` x `threads` threads that wait `micros` microseconds and exit */
int bags_debug_spin(int blocks, int threads, int micros, void* stream);

/* The head's trunk, the step before the path (SURVEY.md 8f-3; convfc_bbox_head.py:138-143 shared FCs + ReLU, :167 fc_reg):
 * out[N,C] = act(x[N,K] W[C,K]^T + bias), act = ReLU when relu != 0, on the wgmma GEMM.  With relu = 0 and fp32 output
 * it is also fc_cls (the materialised logits of bags_fwd).
 * dtype = operand dtype of x and W; out_dtype: BAGS_DTYPE_F32 (out and bias 16-byte aligned), or BAGS_DTYPE_BF16
 * (bf16 operands only: feeds the next layer). */
int bags_linear_act_fwd(const void* x, long long ldx, const void* w, long long ldw, const float* bias,
                        void* out, long long ldo, int N, int K, int C, int dtype, int out_dtype, int relu,
                        void* stream);

/* The same layer in two passes for shapes with few output tiles and a long contraction (shared_fcs.0: 8 x 4 tiles,
 * K = 12544): split-K GEMM with red.add into the zeroed fp32 workspace ws [N, ldws] (ldws % 4 == 0, >= C), then
 * out = act(ws + bias).  bags_linear_act_splits() returns the split count worth using (1: call bags_linear_act_fwd). */
int bags_linear_act_splits(int N, int K, int C, int dtype);
int bags_linear_act_fwd_splitk(const void* x, long long ldx, const void* w, long long ldw, const float* bias,
                               void* out, long long ldo, int N, int K, int C, int dtype, int out_dtype, int relu,
                               float* ws, long long ldws, int splits, void* stream);

/* Its backward up to the contractions: g[rows, cols] = (y > 0 ? dy : 0) in dtype g_dtype (y == NULL: a plain cast of dy);
 * dW / db / dX then come from bags_bwd(g, ...) with a single slice (0, cols) and gout == NULL.  cols % 4 == 0. */
int bags_act_bwd(const void* dy, long long lddy, int dy_dtype, const void* y, long long ldy, int y_dtype,
                 void* g, long long ldg, int g_dtype, int rows, int cols, void* stream);

/* dst[rows, cols] (bf16, leading dim ldd) = bf16(src[rows, cols] fp32, leading dim lds); cols % 4 == 0 */
int bags_cast_bf16(const float* src, long long lds, void* dst, long long ldd, int rows, int cols,
                   void* stream);

/* Test hook: one wgmma GEMM, out[M,N] = A * B^T with either operand K-major ([rows,K]) or
 * MN-major ([K,rows]).  epi: 0 = fp32 store, 1 = bf16 store, 2 = fp32 reduce-add (split-K).  block_n = 256. */
int bags_gemm_probe(const void* a, long long lda, int a_mn, const void* b, long long ldb, int b_mn,
                    void* out, long long ldo, int M, int N, int K, int dtype, int block_n,
                    int splits, int epi, void* stream);

/* Test hook: point the fused forward (bags_fwd / bags_ce_fwd without logits) and the gradient-exchange kernel
 * (bags_grad_allreduce) at a device buffer of int64 %globaltimer stamps, [blocks][8] slots per kernel.  The fused
 * forward writes rows [0, blocks) (at most 256 CTAs; tools/fused_fwd_phases.py reads its phases), the gradient
 * exchange rows from 4096 on.  The GEMM and backward kernels do not stamp it.  NULL (the default) disables it.
 * Not thread-safe; for profiling only. */
int bags_debug_set_timing(void* dev_ptr);

/* The library reads its tuning / experiment switches (BAGS_* environment variables) once per name and caches them;
 * this drops the cache so that the next call re-reads the environment (tests flip switches inside one process). */
int bags_reload_env(void);

#ifdef __cplusplus
}
#endif
#endif /* BAGS_B200_H_ */
