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
 *   fc_cls + FocalLoss (sigmoid) + accuracy              bags_focal_fwd
 *     focal_loss.py:29-88, sigmoid_focal_loss_cuda.cu:23-96
 *   fc_reg + gather + SmoothL1Loss (class-specific)       bags_box_fwd / bags_box_bwd
 *     bbox_head.py:118-128, smooth_l1_loss.py
 *   conv_logits + mask_cross_entropy (class-specific)  bags_mask_fwd / bags_mask_bwd
 *     fcn_mask_head.py:82,102,114-123, cross_entropy_loss.py:54-61
 *   conv_logits + the label channel of each detection     bags_mask_logits
 *     (test time) fcn_mask_head.py:125-181, htc.py:403-421
 *   autograd backward of the above (dW, db, dX)           bags_bwd
 *     triggered at mmdet/core/utils/dist_utils.py:53
 *   GSBBoxHeadWith0._merge_score                          bags_merge_scores
 *     gs_bbox_head_with0.py:239-273
 *   FCNMaskHead.get_seg_masks: resize, paste, RLE     bags_segm_rle
 *     fcn_mask_head.py:125-239
 *   FCNMaskHead.get_target: crop + resize gt masks    bags_mask_target
 *     mmdet/core/mask/mask_target.py
 *   SingleRoIExtractor.forward + RoIAlign                 bags_roi_align_fwd / bags_roi_align_bwd
 *     single_level.py, roi_align_kernel.cu
 *   RPNHead.get_bboxes: RPN proposals                     bags_rpn_proposals (+ bags_rpn_scratch_bytes)
 *     rpn_head.py:55-104, anchor_head.py:250-276, nms_kernel.cu
 *   RPNHead.loss: RPN training targets                    bags_anchor_target (+ bags_anchor_target_scratch_bytes)
 *     anchor_target.py, max_iou_assigner.py, base_sampler.py / random_sampler.py
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
 * counter between replays (not with the kernel that immediately precedes this one in the stream).
 * An empty batch (N == 0; labels and wmask may then be NULL) sets every avg[g] to 1. */
int bags_sample_others(const int64_t* labels, const int32_t* label2bin, int N, int G, int classes,
                       double ratio, uint64_t seed, const uint64_t* seed_step, uint8_t* wmask,
                       float* avg, void* stream);

/* avg[g] = max(sum_n wmask[g,n], 1) for caller-provided masks (wmask may be NULL when N == 0) */
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
 * grid cannot be resident at once, bags_fwd returns BAGS_ERR_CUDA.
 * Operands of the fused kernel (bags_fwd with logits == NULL, bags_ce_fwd, bags_focal_fwd), when N > 0: x [N, K] and
 * W [C, K] 16-byte aligned, ldx >= K and ldw >= K, and both row strides multiples of 16 bytes (ldx, ldw % 8 == 0 for
 * bf16, % 4 == 0 for fp32); checked before anything touches the device. */
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
 *             topk = 1.  A tie with the row maximum counts as correct; a label outside [0, C) never counts as correct.
 *             N <= 2^24 when requested: the count is exact)
 * weights: fp32 [N] per-RoI weights (cls_weight[labels] for ReweightBBoxHead).
 * dz, colsum, clear, workspace: as bags_fwd (ldd % 8 == 0, colsum [ceil(N/128), C]); dW, db and dX then come from
 * bags_bwd with the single slice (0, C) and gout = dL/dloss[0].
 * 1 <= C <= 1280, any C (not only multiples of 4); labels in [0, C) (a label outside it is scored against column 0).
 * N == 0: loss = 0, acc = 0. */
int bags_ce_fwd(const void* x, long long ldx, const void* w, long long ldw, const float* bias, const int64_t* labels,
                const float* weights, const float* avg, int N, int K, int C, int dtype, float* loss, float* acc,
                void* dz, long long ldd, float* colsum, int colsum_tiles, void* workspace, size_t workspace_bytes,
                void* clear, size_t clear_bytes, void* stream);

/* fc_cls + the sigmoid focal loss over all C logits, logits kept on chip -- replaces FocalLoss.forward
 * (mmdet/models/losses/focal_loss.py:63-88), sigmoid_focal_loss + weight_reduce_loss (:29-43, losses/utils.py:26-53) and
 * the op's forward and backward kernels (mmdet/ops/sigmoid_focal_loss/src/sigmoid_focal_loss_cuda.cu:23-96), with the
 * fused kernel of bags_ce_fwd in its focal variant:
 *   loss[0] = sum_n sum_c w[n] * l(z[n,c], t[n]) / norm                          (weights NULL => w = 1)
 *   dz      = w[n] / norm * g(z[n,c], t[n])                                      (the op's analytic gradient)
 *   acc[0]  = 100 * #{n : z[n, labels[n]] == max_c z[n, c]} / N                  (optional; as bags_ce_fwd)
 * targets: int64 [N] in the op's convention, read as int: column t - 1 is positive, every other column negative, and a
 *          row with t < 0 contributes nothing.  FocalLoss.forward passes F.one_hot(labels, 1231) as the targets and the
 *          op reads its first N entries: t[n] = (labels[n / 1231] == n % 1231).
 * With p = sigmoid(z) and log1m = -z [z >= 0] - log(1 + exp(-|z|)):
 *   positive: l = -alpha (1-p)^gamma log(max(p, FLT_MIN))   g = -alpha (1-p)^gamma (1 - p - gamma p log(max(p, FLT_MIN)))
 *   negative: l = -(1-alpha) p^gamma log1m                  g = -(1-alpha) p^gamma (gamma (1-p) log1m - p)
 * norm: the host-known divisor, N * 1231 for FocalLoss (which ignores the caller's avg_factor); no device read.
 * labels: int64 [N], needed only for acc (a label outside [0, C) never counts as correct).  Without acc the CTAs of the
 * kernel do not wait for each other.
 * weights, dz, colsum, clear, workspace: as bags_ce_fwd; dW, db and dX then come from bags_bwd with the single slice
 * (0, C) and gout = dL/dloss[0].  1 <= C <= 1280.  N == 0: loss = 0, acc = 0. */
int bags_focal_fwd(const void* x, long long ldx, const void* w, long long ldw, const float* bias, const int64_t* targets,
                   const int64_t* labels, const float* weights, float norm, float gamma, float alpha, int N, int K, int C,
                   int dtype, float* loss, float* acc, void* dz, long long ldd, float* colsum, int colsum_tiles,
                   void* workspace, size_t workspace_bytes, void* clear, size_t clear_bytes, void* stream);

/* Class-specific box regression fused with its SmoothL1 loss -- replaces, for the training loss, fc_reg's
 * [N, 4 * classes] GEMM (convfc_bbox_head.py:167), the gather bbox_pred.view(N, -1, 4)[pos_inds, labels[pos_inds]] of
 * BBoxHead.loss (bbox_head.py:118-128, with its nonzero() host sync) and SmoothL1Loss 'mean'
 * (mmdet/models/losses/smooth_l1_loss.py, losses/utils.py:26-53).  A RoI n is positive when 0 < l = labels[n] < classes;
 * only its four columns are computed, with fp32 products and accumulation, from the fp32 master W:
 *   pred[n,j] = sum_k x[n,k] W[4l+j, k] + bias[4l+j]          d = pred[n,j] - targets[n,j]
 *   sl1(d)    = |d| < beta ? 0.5 d^2 / beta : |d| - 0.5 beta
 *   loss[0]   = sum_{n positive, j} weights[n,j] sl1(d) / avg  (summed in a fixed order: bit-identical across runs)
 *   g[n,j]    = weights[n,j] sl1'(d) / avg, sl1' = d / beta for |d| < beta, sign(d) otherwise; 0 for other rows
 * x: [N, K] (ldx) bf16 or fp32 (dtype), rows 8- (bf16) or 16-byte (fp32) aligned, ldx % 4 == 0, K % 4 == 0.
 * W: [4 * classes, K] fp32 (ldw % 4 == 0, 16-byte aligned); bias: [4 * classes] fp32 or NULL.  labels: int64 [N]; a
 * label >= classes (or <= 0) contributes nothing.  targets, weights, g, pred: contiguous fp32 [N, 4], 16-byte aligned.
 * pred (optional, NULL to skip) holds the four predictions of each positive row and 0 elsewhere.
 * avg: the host-known normaliser (bbox_targets.size(0)), never read from the device; beta > 0.  1 <= classes <= 8192.
 * index: int32 [classes + 1 + N], written for bags_box_bwd -- offsets [classes + 1] of each class's positives, then the
 * positive RoIs sorted by class, ascending RoI id inside a class (a stable counting sort built on the device).
 * workspace: as bags_fwd (its counter is left at zero).  One launch, no host sync.  N == 0: loss = 0. */
int bags_box_fwd(const void* x, long long ldx, int dtype, const float* w, long long ldw, const float* bias,
                 const int64_t* labels, const float* targets, const float* weights, float beta, float avg, int N, int K,
                 int classes, float* loss, float* g, float* pred, int32_t* index, void* workspace,
                 size_t workspace_bytes, void* stream);

/* Backward of bags_box_fwd (the autograd backward of the gather + SmoothL1, scatter and fc_reg's dW / db / dX GEMMs),
 * given its g, index and gout = dL/dloss[0] (device fp32 [1]; NULL => 1):
 *   dW[4c+j, :] = sum_{n of class c, ascending} gout g[n,j] x[n,:]   fp32 [4 * classes, K] (lddw), FULLY overwritten:
 *                                                                   rows of classes without a positive are zero
 *   db[4c+j]    = sum_{n of class c, ascending} gout g[n,j]          fp32 [4 * classes]
 *   dX[n, :]    = sum_j gout g[n,j] W[4l+j, :]                       x's dtype [N, K] (lddx); 0 for non-positive rows
 * Each output is optional (NULL to skip).  One launch; no atomics, so every output is bit-identical across runs and
 * CUDA-graph replays.  Operand rules as bags_box_fwd; dW 16-byte aligned rows, dX aligned like x. */
int bags_box_bwd(const float* g, const float* gout, const void* x, long long ldx, int dtype, const float* w, long long ldw,
                 const int64_t* labels, const int32_t* index, int N, int K, int classes, float* dW, long long lddw,
                 float* db, void* dX, long long lddx, void* stream);

/* Class-specific mask logits fused with their BCE loss -- replaces, for the training loss, conv_logits' 1x1 conv into
 * [P, classes, H, W] (fcn_mask_head.py:82,102), the channel gather pred[arange(P), labels] of mask_cross_entropy and
 * its BCE-with-logits 'mean' (FCNMaskHead.loss, fcn_mask_head.py:114-123; cross_entropy_loss.py:54-61).  A row p is
 * valid when 0 <= l = labels[p] < classes (class-agnostic heads pass label 0 to one channel); only channel l of it is
 * computed, with fp32 products and accumulation from the fp32 W, over the HW = H * W pixels q:
 *   z[p,q]  = bias[l] + sum_c W[l,c] y[p,c,q]
 *   loss[0] = sum_{p valid, q} (max(z,0) - z t[p,q] + log1p(exp(-|z|))) / (P HW)   (fixed order: bit-identical runs)
 *   g[p,q]  = (sigmoid(z) - t[p,q]) / (P HW); 0 on an invalid row, which still counts in P HW
 * y: contiguous [P, Cin, HW] bf16 or fp32 (dtype); W: [classes, Cin] fp32 (ldw >= Cin); bias: [classes] fp32 or NULL;
 * labels: int64 [P]; targets, g: contiguous fp32 [P, HW].  1 <= classes <= 8192.  P == 0: loss = 0.
 * rsum: fp32 scratch of at least P * ceil(HW / BAGS_MASK_TILE) * (Cin + 2) floats, written for bags_mask_bwd: each
 * (RoI, pixel tile)'s sum_q g y per channel and sum_q g, then the tile losses.  index: int32 [classes + 1 + P], the
 * valid RoIs sorted by class (as bags_box_fwd's).  workspace: as bags_fwd (its counter is left at zero).
 * Two launches, no host sync; y is read from memory once. */
#define BAGS_MASK_TILE 64
int bags_mask_fwd(const void* y, int dtype, const float* w, long long ldw, const float* bias, const int64_t* labels,
                  const float* targets, int P, int Cin, int HW, int classes, float* loss, float* g, float* rsum,
                  size_t rsum_floats, int32_t* index, void* workspace, size_t workspace_bytes, void* stream);

/* Backward of bags_mask_fwd (the gather's scatter and conv_logits' dW / db / dX), given its g, rsum, index and
 * gout = dL/dloss[0] (device fp32 [1]; NULL => 1):
 *   dW[l, c]   = gout sum_{p of class l} sum_q g[p,q] y[p,c,q]              fp32 [classes, Cin] (lddw), FULLY
 *                                                                          overwritten: absent classes are zero
 *   db[l]      = gout sum_{p of class l} sum_q g[p,q]                       fp32 [classes]
 *   dY[p,c,q]  = gout g[p,q] W[l,c]                                         dtype [P, Cin, HW]; 0 on invalid rows
 * The class sums run in an order fixed by the labels alone (the class's RoIs ascending, per-tile partials dealt to 8
 * warps, the warps added in order).  Each output is optional (NULL to skip).  One launch; no atomics, so every output
 * is bit-identical across runs and CUDA-graph replays. */
int bags_mask_bwd(const float* g, const float* rsum, const float* gout, int dtype, const float* w, long long ldw,
                  const int64_t* labels, const int32_t* index, int P, int Cin, int HW, int classes, float* dW,
                  long long lddw, float* db, void* dY, void* stream);

/* Test-time mask logits of one channel per detection -- replaces, where the caller reads only channel c_d of each
 * detection d, conv_logits' 1x1 conv into [n, classes, H, W] (fcn_mask_head.py:82,102) followed by the channel
 * selection of get_seg_masks (mask_pred[i, label], fcn_mask_head.py:125-181) or HTC's mask_pred.gather(1, labels)
 * (htc.py:403-421):
 *   out[d, q] = bias[c_d] + sum_k W[c_d, k] y[d, k, q]        c_d = channels[d], q < HW = H * W
 * with fp32 products and accumulation from the fp32 W, in the summation order of bags_mask_fwd's logits, rounded once
 * to y's dtype.  y: contiguous [n, Cin, HW] bf16 or fp32 (dtype); W: [classes, Cin] fp32 (ldw >= Cin); bias: [classes]
 * fp32 or NULL; channels: int64 [n] (device); out: contiguous [n, HW] in y's dtype.  A channel outside [0, classes)
 * gives a row of NaN and reads nothing of W, bias or y.  1 <= classes <= 8192.  One launch, no host sync, no atomics;
 * y is read from memory once.  n == 0: nothing is launched. */
int bags_mask_logits(const void* y, int dtype, const float* w, long long ldw, const float* bias, const int64_t* channels,
                     int n, int Cin, int HW, int classes, void* out, void* stream);

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
 * Bins need not tile [0, C): with gout given, a dz column outside every bin is scaled by 0 (it contributes to none of
 * dW, db, dX); with gout NULL every column is scaled by 1.
 * colsum: optional [colsum_tiles, C] partial column sums of dz from the forward; NULL => recomputed from dz.
 * wscratch: 256-byte aligned, bags_bwd_scratch_bytes() bytes; required when (dX and gout) or (db without colsum).
 * flags: BAGS_BWD_DW_PREZEROED = dW is already zero on entry (stream-ordered), e.g. by bags_fwd's clear hook.
 * Launch structure: one small preparation kernel (zero dW, scaled W, column-sum partials), then one merged launch whose
 * work list holds the requested contractions (split-K dW tiles, dX tiles, or both) and whose mainloop overlaps the
 * preparation kernel (programmatic dependent launch).  db without dW takes one more small kernel. */
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
 *                    words that the caller zeroes ONCE (before the first exchange, on every rank); the calls
 *                    keep them consistent from then on (epoch counters: no reset, also across CUDA-graph replays)
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

/* Test-time masks as COCO compressed RLE -- replaces the per-detection loop of FCNMaskHead.get_seg_masks /
 * get_seg_masks_without (fcn_mask_head.py:125-239: cv2 INTER_LINEAR resize to the box, "> thr", paste into an empty
 * img_h x img_w image, pycocotools.mask.encode) without materialising the image:
 *   probs     device fp32 [n, mask_h, mask_w], mask_h, mask_w >= 2: each detection's probability map (its channel)
 *   boxes_host int32 [n, 4] (left, top, w, h): w, h >= 1 and the box inside the canvas (checked here; the caller
 *             handles boxes that leave it); copied stream-ordered into boxes (int32 [n, 4], 16-byte aligned)
 *   thr       a pixel is set when (double) resized > thr (pass float32(thr) for a float32 comparison)
 *   lengths   device int64 [n]
 *   out       NULL: the sizing pass, which writes each detection's string length to lengths[d].  Otherwise the write
 *             pass, given the lengths of the sizing pass: it writes detection d's string (pycocotools' rleToString of
 *             the column-major run lengths, not NUL-terminated) at out + lengths[0] + ... + lengths[d-1].
 * The resize reproduces OpenCV's float32 INTER_LINEAR bitwise (dsize == ssize copies).  One launch per pass, no host
 * sync; the caller reads the lengths back between the passes. */
int bags_segm_rle(const float* probs, int n, int mask_h, int mask_w, const int32_t* boxes_host, int32_t* boxes,
                  int img_h, int img_w, double thr, int64_t* lengths, char* out, void* stream);

/* Training mask targets -- replaces the per-RoI loop of mask_target / mask_target_single
 * (mmdet/core/mask/mask_target.py: boxes and gt indices to the host, gt_masks[gt][y1:y1 + h, x1:x1 + w] per RoI,
 * mmcv.imresize to mask_size, a stacked float upload).  For image i and its positive RoI r:
 *   (x1, y1, x2, y2) = boxes[r] truncated as numpy's astype(np.int32), w = max(x2 - x1 + 1, 1), h likewise
 *   crop = masks[gt_inds[r]][y1:y1 + h, x1:x1 + w] by numpy's slice rules (a negative start counts from the end)
 *   out[row] = cv2.resize(crop, (mask_w, mask_h), INTER_LINEAR) as float, bitwise (8-bit fixed point; a crop of
 *              exactly the output size is copied, one of exactly twice it on both axes is averaged over 2 x 2 blocks)
 * with rows of image i after those of the images before it.  A gt index outside [0, num_gt), or a crop the slicing
 * leaves empty (where the reference raises), gives a row of NaN.  Any uint8 mask values, not only 0 / 1.
 *   boxes_host   HOST array [n_images] of device fp32 [num_pos, 4] (x1, y1, x2, y2), 4-byte aligned
 *   gt_inds_host HOST array [n_images] of device int64 [num_pos], 8-byte aligned
 *   masks_host   HOST array [n_images] of device uint8 [num_gt, H, W], contiguous
 *   sizes_host   int32 [n_images, 4]: (num_pos, num_gt, H, W), each >= 0
 *   out          device fp32 [sum num_pos, mask_h, mask_w]; 1 <= mask_h, mask_w <= 256
 * Pointers of an image without positives (boxes, gt_inds) or without mask pixels (masks) may be NULL.  One launch per
 * 64 images, no host sync, nothing read on the host from the device: capturable in a CUDA graph. */
int bags_mask_target(const float* const* boxes_host, const int64_t* const* gt_inds_host, const uint8_t* const* masks_host,
                     const int32_t* sizes_host, int n_images, int mask_h, int mask_w, float* out, void* stream);

/* FPN RoI feature extractor -- replaces SingleRoIExtractor.forward (mmdet/models/roi_extractors/single_level.py:
 * map_roi_levels :56-75, the per-level loop :93-108 with its host syncs on inds.any(), rois[inds] and
 * roi_feats[inds] = ...; the len(feats) == 1 path :94-95) and the RoIAlign op it calls per level
 * (mmdet/ops/roi_align/src/roi_align_kernel.cu: ROIAlignForward :61-119 with bilinear_interpolate :16-59).
 * Every RoI of every image in one launch:
 *   level  = clamp(floor(log2f(sqrt((x2 - x1 + 1) (y2 - y1 + 1)) * fp32(1 / finest_scale) + fp32(1e-6))), 0, L - 1),
 *            each step rounded to fp32 as torch evaluates the reference's expression on CUDA; 0 when L == 1
 *   out[r] = ROIAlignForward<float> of rois[r] on level `level`, bitwise (its -O2 sm_90a rounding sequence)
 * A RoI whose level is NaN, or whose batch index (int)rois[r][0] lies outside [0, B), gives a zero row.
 *   feats_host   HOST array [L] of device fp32 [B, C, H_l, W_l], contiguous, 4-byte aligned; L <= 8
 *   sizes_host   int32 [L, 2]: (H_l, W_l), each >= 1;  scales_host fp32 [L]: spatial_scale of each level
 *   rois_map     device fp32 [k, 5] (batch, x1, y1, x2, y2) the levels are mapped from
 *   rois         device fp32 [k, 5] the RoIs pooled (== rois_map unless roi_scale_factor rescales them)
 *   out_h, out_w 1 to 64;  sample_num <= 0: ceil(bin size) samples per bin, as the reference
 *   finest_scale > 0 (unused with one level)
 *   out          device fp32 [k, C, out_h, out_w];  levels (optional, NULL to skip): int32 [k], -1 for a NaN level
 * k == 0: nothing is launched.  No host sync: capturable in a CUDA graph. */
int bags_roi_align_fwd(const float* const* feats_host, const int32_t* sizes_host, const float* scales_host, int n_levels,
                       int B, int C, const float* rois_map, const float* rois, int k, int out_h, int out_w,
                       int sample_num, float finest_scale, float* out, int32_t* levels, void* stream);

/* Backward of bags_roi_align_fwd -- replaces ROIAlignBackward (roi_align_kernel.cu:164-282) launched once per level
 * and the scatter of roi_feats[inds] = ...: the terms gout w_i / count of each sample's four corners, for every RoI
 * and level in one launch, ADDED to grads_host[level] (the caller zeroes them on the stream).  A CTA sums each pixel
 * its RoI touches in registers, in a fixed order, and adds it with one reduction; the order across RoIs is open, so
 * the result is not bitwise reproducible.  grads_host: HOST array [L] of device fp32 [B, C, H_l, W_l] (contiguous,
 * 4-byte aligned), or NULL for a level that takes no gradient; gout: device fp32 [k, C, out_h, out_w].  Other
 * arguments as bags_roi_align_fwd.  Zero rows of the forward take no gradient.  k == 0, or every level NULL: nothing
 * is launched. */
int bags_roi_align_bwd(const float* gout, float* const* grads_host, const int32_t* sizes_host, const float* scales_host,
                       int n_levels, int B, int C, const float* rois_map, const float* rois, int k, int out_h,
                       int out_w, int sample_num, float finest_scale, void* stream);

/* RPN proposals -- replaces RPNHead.get_bboxes (mmdet/models/anchor_heads/anchor_head.py:250-276: grid_anchors per
 * level, then the per-image loop) and RPNHead.get_bboxes_single (rpn_head.py:55-104: per level sigmoid, topk(nms_pre),
 * delta2bbox, min_bbox_size, the NMS op of mmdet/ops/nms/src/nms_kernel.cu:69-130 with its device-to-host copy of the
 * suppression matrix and CPU scan, [:nms_post]; then topk(min(max_num, total)) over the levels), for a sigmoid RPN
 * with nms_across_levels=False.  Every image and level in four launches, no host read, no allocation:
 *   scores   sigmoid(logit) as torch.sigmoid (1 / (1 + expf(-x)) in fp32), flat index (h W + w) A + a;
 *   select   the top nms_pre by (score desc, flat asc) when the level has more than nms_pre > 0 anchors, else all;
 *   anchors  base[a] + (w stride, h stride) in fp32;  boxes: delta2bbox with one fp32 rounding per torch op, clamped
 *            to [0, img_w - 1] x [0, img_h - 1] of the image (NaN kept); boxes with x2 - x1 + 1 or y2 - y1 + 1 below
 *            min_bbox_size > 0 are dropped;
 *   suppress greedy in (score desc, flat asc) order, IoU with "+1" widths, suppressed when IoU > nms_thr; the first
 *            nms_post survivors in the level's input order (score order when selected, anchor order when not);
 *   merge    the first min(max_num, total) survivors of the image by (score desc, level asc, position asc).
 *   logits_host  HOST array [L] of device fp32 [B, A_l, H_l, W_l], contiguous, 4-byte aligned; L in [1, 8]
 *   deltas_host  HOST array [L] of device fp32 [B, 4 A_l, H_l, W_l]
 *   levels_host  int32 [L, 4]: H_l, W_l (>= 0), A_l (1 to 16), stride_l (>= 1); a level may hold 0 anchors
 *   base_host    fp32 [sum A_l, 4]: each level's base anchors (x1, y1, x2, y2), level after level
 *   img_shapes_host int32 [B, 2]: (h, w) of img_shape per image, each >= 1;  B in [1, 32]
 *   nms_pre (<= 0: no selection), nms_post >= 1, max_num >= 1; each level's candidate count (nms_pre when selected,
 *            else its anchor count) at most 4096
 *   means_host, stds_host fp32 [4];  scratch: device, bags_rpn_scratch_bytes() bytes, 256-byte aligned
 *   out      device fp32 [B, max_num, 5] (x1, y1, x2, y2, score), zero rows after counts[b]; counts: device int32 [B]
 * No host sync: capturable in a CUDA graph. */
int bags_rpn_proposals(const float* const* logits_host, const float* const* deltas_host, const int32_t* levels_host,
                       const float* base_host, int n_levels, int B, const int32_t* img_shapes_host, int nms_pre,
                       int nms_post, int max_num, float nms_thr, float min_bbox_size, const float* means_host,
                       const float* stds_host, void* scratch, size_t scratch_bytes, float* out, int32_t* counts,
                       void* stream);

/* Scratch bytes bags_rpn_proposals needs for these level shapes (levels_host as there), B, nms_pre and nms_post; the
 * same argument checks.  Writes *bytes. */
int bags_rpn_scratch_bytes(const int32_t* levels_host, int n_levels, int B, int nms_pre, int nms_post, size_t* bytes);

/* RPN training targets -- replaces anchor_target (mmdet/core/anchor/anchor_target.py: per image anchor_inside_flags,
 * MaxIoUAssigner.assign of core/bbox/assigners/max_iou_assigner.py, the sampler of core/bbox/samplers/
 * base_sampler.py, bbox2delta and unmap) for an RPN without gt labels or ignored gts.  Every image in one memset and
 * four launches, no host read, no allocation:
 *   anchors  per image, level after level, location-major ((h W + w) A + a): base[a] + (w stride, h stride) in fp32;
 *            inside when h < valid_h and w < valid_w of the level and, when allowed_border >= 0, x1 >= -border,
 *            y1 >= -border, x2 < img_w + border and y2 < img_h + border (fp32 comparisons);
 *   assign   IoU = bbox_overlaps(gt, anchor) with one fp32 rounding per torch op (NaN propagates); per anchor the max
 *            over gts (first gt on ties, NaN wins), per gt the max over the inside anchors; ignored (-1) by default,
 *            negative when neg_on and neg_lo <= max < neg_hi, positive (argmax) when max >= pos_iou_thr, then for
 *            each gt in order with max >= min_pos_iou, every inside anchor at that max (or the first only, when
 *            gt_max_assign_all = 0) is given to it: the last gt wins;
 *   sample   key(n) = (sample_key(seed', image, n) << 32) | n with seed' = seed + *seed_step * 0x9E3779B97F4A7C15
 *            when seed_step is given; the k_pos = min(#pos, int(num pos_fraction)) positives and then the
 *            k_neg = min(#neg, num - k_pos, int(neg_pos_ub max(k_pos, 1)) when neg_pos_ub >= 0) negatives with the
 *            smallest keys: an exact-k uniform subset, not np.random.shuffle's;
 *   targets  labels int64 [B, N] 1 at sampled positives; label_weights fp32 [B, N] pos_weight (1 when <= 0) at
 *            sampled positives and 1 at sampled negatives; bbox_targets fp32 [B, N, 4] bbox2delta(anchor, gt) in
 *            torch's op sequence, then (d - means) / stds, and bbox_weights 1 at sampled positives; 0 elsewhere;
 *            totals int64 [3]: sum_b max(k_pos, 1), sum_b max(k_neg, 1) and their sum.
 *   levels_host  int32 [L, 4]: H_l, W_l (>= 0), A_l (1 to 16), stride_l (>= 1); L in [1, 8]; N = sum H W A >= 1
 *   base_host    fp32 [sum A_l, 4]: each level's base anchors, level after level
 *   images_host  int32 [B, 4 + 2 L]: img_h, img_w (>= 1), gt_off, gt_cnt (>= 1; the images' gts consecutive rows of
 *                gts), then valid_h, valid_w of every level (in [0, H] x [0, W]);  B in [1, 32]
 *   gts          device fp32 [total_gts, 4], 16-byte aligned;  num >= 0, pos_fraction in [0, 1]
 *   means_host, stds_host fp32 [4];  seed_step: optional device int64;  scratch: device,
 *   bags_anchor_target_scratch_bytes() bytes, 256-byte aligned;  bbox_targets / bbox_weights 16-byte aligned
 * No host sync: capturable in a CUDA graph. */
int bags_anchor_target(const int32_t* levels_host, const float* base_host, int n_levels, int B,
                       const int32_t* images_host, const float* gts, int total_gts, float pos_iou_thr, int neg_on,
                       float neg_lo, float neg_hi, float min_pos_iou, int gt_max_assign_all, double allowed_border,
                       int num, double pos_fraction, double neg_pos_ub, float pos_weight, const float* means_host,
                       const float* stds_host, uint64_t seed, const int64_t* seed_step, void* scratch,
                       size_t scratch_bytes, int64_t* labels, float* label_weights, float* bbox_targets,
                       float* bbox_weights, int64_t* totals, void* stream);

/* Scratch bytes bags_anchor_target needs for these level shapes (levels_host as there), B and total_gts; the same
 * argument checks.  Writes *bytes. */
int bags_anchor_target_scratch_bytes(const int32_t* levels_host, int n_levels, int B, int total_gts, size_t* bytes);

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

/* dst[rows, cols] (bf16, leading dim ldd) = bf16(src[rows, cols] fp32, leading dim lds), rounded to nearest even;
 * cols, lds and ldd % 4 == 0, src 16-byte and dst 8-byte aligned */
int bags_cast_bf16(const float* src, long long lds, void* dst, long long ldd, int rows, int cols,
                   void* stream);

/* Test hook: out[M,N] = A * B^T on the wgmma kernel the product runs for that layout, each operand K-major ([rows,K])
 * or MN-major ([K,rows]); block_n = 256:
 *   both K-major, epi 0 (fp32 store):                        the forward GEMM
 *   A K-major, B MN-major, epi 1 (bf16 store; bf16 operands)
 *                       or epi 0 (fp32 store; fp32 operands): the merged backward with dX units only
 *   both MN-major, epi 2 (fp32 reduce-add, `splits` split-K): the merged backward with dW units only
 * Any other combination is BAGS_ERR_INVALID. */
int bags_gemm_probe(const void* a, long long lda, int a_mn, const void* b, long long ldb, int b_mn,
                    void* out, long long ldo, int M, int N, int K, int dtype, int block_n,
                    int splits, int epi, void* stream);

/* Test hook: point the fused forward (bags_fwd / bags_ce_fwd without logits) and the gradient-exchange kernel
 * (bags_grad_allreduce) at a device buffer of int64 %globaltimer stamps, [blocks][8] slots per kernel.  The fused
 * forward writes rows [0, blocks) (at most 256 CTAs; tools/fused_fwd_phases.py reads its phases), the merged
 * backward two rows per CTA from row 1024 on, the backward's preparation kernel rows [2048, 4096) (one per CTA;
 * tools/bwd_phases.py reads both), the gradient exchange rows from 4096 on.  The GEMM kernels do not stamp it.
 * NULL (the default) disables it.  Not thread-safe; for profiling only. */
int bags_debug_set_timing(void* dev_ptr);

/* The library reads its tuning / experiment switches (BAGS_* environment variables) once per name and caches them;
 * this drops the cache so that the next call re-reads the environment (tests flip switches inside one process). */
int bags_reload_env(void);

#ifdef __cplusplus
}
#endif
#endif /* BAGS_B200_H_ */
