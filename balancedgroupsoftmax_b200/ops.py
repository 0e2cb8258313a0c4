"""Tensor-level wrappers over the C ABI + the autograd Functions of the BAGS head.

Layering (mirrors the reference's own plugin pattern, e.g.
mmdet/ops/sigmoid_focal_loss/sigmoid_focal_loss.py:8-35: an autograd.Function
whose forward/backward call a compiled ``forward``/``backward``):

    GroupSoftmaxFunction.forward/backward      <- torch.autograd.Function
        -> bags_fwd / bags_bwd                 <- C ABI (include/bags_b200.h), ctypes
            -> sm_90a kernels                  <- csrc/*.cuh

Nothing in this file computes on the CPU or with torch math ops; torch is used
for device memory, streams and autograd bookkeeping only.  Every entry point
raises if the inputs are not CUDA tensors or the extension is missing.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import _native as nat
from .tables import GroupTables


# --------------------------------------------------------------------------- helpers
def _stream_ptr(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def _require_cuda(*tensors) -> None:
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise nat.BagsNativeError(
                'BAGS ops run on an H100 GPU only (got a %s tensor); there is no CPU fallback' % t.device)


def _dtype_code(dt: torch.dtype) -> int:
    if dt == torch.float32:
        return nat.DTYPE_F32
    if dt == torch.bfloat16:
        return nat.DTYPE_BF16
    raise nat.BagsNativeError('unsupported operand dtype %s (float32 or bfloat16)' % dt)


def _row_major(t: torch.Tensor) -> torch.Tensor:
    if t.dim() != 2 or t.stride(1) != 1:
        t = t.contiguous()
    return t


_workspaces: Dict[Tuple[int, int], torch.Tensor] = {}


def _weights_arg(wmask: Optional[torch.Tensor]) -> Tuple[Optional[torch.Tensor], int]:
    """[G,N] sample weights as the kernels read them, with their weights_dtype code: contiguous 0/1 bytes (bool is
    the same storage), or fp32 (reweight head variant); other dtypes are cast to fp32."""
    if wmask is None:
        return None, nat.WEIGHTS_U8
    if wmask.dtype == torch.bool:
        wmask = wmask.view(torch.uint8)
    elif wmask.dtype not in (torch.uint8, torch.float32):
        wmask = wmask.to(torch.float32)
    return wmask.contiguous(), (nat.WEIGHTS_F32 if wmask.dtype == torch.float32 else nat.WEIGHTS_U8)


def _workspace(device: torch.device) -> torch.Tensor:
    key = (device.index if device.index is not None else torch.cuda.current_device(), _stream_ptr(device))
    ws = _workspaces.get(key)
    if ws is None:
        if len(_workspaces) >= 64:      # streams come and go (side streams, graph captures): keep the table bounded
            _workspaces.pop(next(iter(_workspaces)))
        ws = torch.zeros(nat.lib().bags_workspace_bytes(), dtype=torch.uint8, device=device)
        _workspaces[key] = ws
    return ws


@dataclass
class DeviceTables:
    """Group tables resident on one GPU (int32), converted once from the reference's int64 tables
    (gs_bbox_head_with0.py:37-49)."""
    G: int
    num_classes: int
    num_logits: int
    label2bin: torch.Tensor     # [G, num_classes] int32, device
    cls2col: torch.Tensor       # [num_classes] int32, device
    slices_host: C.Array        # int32 [G*2] host
    pred_slice: np.ndarray      # [G, 2] int64 host copy

    @staticmethod
    def from_tables(t: GroupTables, device) -> 'DeviceTables':
        if t.num_bins > nat.MAX_BINS:
            raise nat.BagsNativeError('at most %d bins are supported (got %d)' % (nat.MAX_BINS, t.num_bins))
        l2b = torch.from_numpy(np.ascontiguousarray(t.label2binlabel.astype(np.int32))).to(device)
        c2c = torch.from_numpy(np.ascontiguousarray(t.cls2col())).to(device)
        flat = [int(v) for v in np.asarray(t.pred_slice).reshape(-1)]
        return DeviceTables(t.num_bins, t.num_classes, t.num_logits, l2b, c2c, nat.int32_array(flat),
                            np.asarray(t.pred_slice, dtype=np.int64).copy())


def pad_cols(c: int, mult: int = 64) -> int:
    return (c + mult - 1) // mult * mult


# --------------------------------------------------------------------------- raw ops
def cast_bf16(src: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _require_cuda(src)
    src = _row_major(src)
    assert src.dtype == torch.float32
    rows, cols = src.shape
    if out is None:
        out = torch.empty((rows, cols), dtype=torch.bfloat16, device=src.device)
    nat.check(nat.lib().bags_cast_bf16(src.data_ptr(), src.stride(0), out.data_ptr(), out.stride(0), rows, cols,
                                       _stream_ptr(src.device)), 'bags_cast_bf16')
    return out


def linear_fwd(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor],
               out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[N,C] fp32 = x @ w^T + bias   (a1: convfc_bbox_head.py:166)."""
    _require_cuda(x, w, bias)
    x, w = _row_major(x), _row_major(w)
    if x.dtype != w.dtype:
        raise nat.BagsNativeError('x (%s) and w (%s) must share a dtype' % (x.dtype, w.dtype))
    N, K = x.shape
    Cc = w.shape[0]
    if out is None:
        # (any C: the GEMM epilogue stores column pairs only where ldo is even, single floats otherwise -- 1231 classes)
        out = torch.empty((N, Cc), dtype=torch.float32, device=x.device)
    if bias is not None:
        bias = bias.contiguous()
        assert bias.dtype == torch.float32
    # the single-pass GEMM, never split-K (linear_act may choose it): the materialised logits keep one summation order
    nat.check(nat.lib().bags_linear_act_fwd(x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), nat.ptr(bias),
                                            out.data_ptr(), out.stride(0), N, K, Cc, _dtype_code(x.dtype),
                                            nat.DTYPE_F32, 0, _stream_ptr(x.device)), 'bags_linear_act_fwd')
    return out


def sample_others(labels: torch.Tensor, dt: DeviceTables, ratio: float, seed: int,
                  seed_step: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Device sampler: (wmask [G,N] uint8, avg [G] fp32)   (a3/a4).
    ``seed_step``: optional int64 device scalar added (times a odd constant) to the seed on the device, so that
    replays of a captured CUDA graph draw different subsets (advance it between replays)."""
    _require_cuda(labels, seed_step)
    labels = labels.contiguous()
    assert labels.dtype == torch.int64
    N = labels.numel()
    wmask = torch.empty((dt.G, N), dtype=torch.uint8, device=labels.device)
    avg = torch.empty((dt.G,), dtype=torch.float32, device=labels.device)
    if seed_step is not None:
        assert seed_step.dtype == torch.int64 and seed_step.numel() == 1
    nat.check(nat.lib().bags_sample_others(labels.data_ptr(), dt.label2bin.data_ptr(), N, dt.G, dt.num_classes,
                                           float(ratio), int(seed) & 0xFFFFFFFFFFFFFFFF, nat.ptr(seed_step),
                                           wmask.data_ptr(), avg.data_ptr(), _stream_ptr(labels.device)),
              'bags_sample_others')
    return wmask, avg


def reweight(labels: torch.Tensor, dt: DeviceTables, wmask: Optional[torch.Tensor], cls_weight: torch.Tensor
             ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Reweight head variant (gs_bbox_head_with0_reweight.py:57-109): (wfloat [G,N] fp32, avg [G]) with
    wfloat[g,n] = wmask[g,n] * cls_weight[g, in-bin label of n] for g >= 1 and avg[g] = max(sum_n wfloat[g,n], 1).
    ``cls_weight`` is [G, stride] fp32 on the device (row 0 unused; index 0 of a row is the "others" weight)."""
    _require_cuda(labels, wmask, cls_weight)
    labels = labels.contiguous()
    assert cls_weight.dtype == torch.float32 and cls_weight.dim() == 2 and cls_weight.shape[0] == dt.G
    cls_weight = cls_weight.contiguous()
    N = labels.numel()
    wfloat = torch.empty((dt.G, N), dtype=torch.float32, device=labels.device)
    avg = torch.empty((dt.G,), dtype=torch.float32, device=labels.device)
    nat.check(nat.lib().bags_reweight(labels.data_ptr(), dt.label2bin.data_ptr(), nat.ptr(wmask), cls_weight.data_ptr(),
                                      cls_weight.shape[1], N, dt.G, dt.num_classes, wfloat.data_ptr(), avg.data_ptr(),
                                      _stream_ptr(labels.device)), 'bags_reweight')
    return wfloat, avg


def mask_avg(wmask: torch.Tensor) -> torch.Tensor:
    _require_cuda(wmask)
    wmask = wmask.contiguous()
    assert wmask.dtype == torch.uint8 and wmask.dim() == 2
    G, N = wmask.shape
    avg = torch.empty((G,), dtype=torch.float32, device=wmask.device)
    nat.check(nat.lib().bags_mask_avg(wmask.data_ptr(), N, G, avg.data_ptr(), _stream_ptr(wmask.device)),
              'bags_mask_avg')
    return avg


def group_ce(logits: torch.Tensor, labels: torch.Tensor, dt: DeviceTables,
             wmask: Optional[torch.Tensor], avg: Optional[torch.Tensor], want_dz: bool = True,
             dz_dtype: torch.dtype = torch.bfloat16, want_lse: bool = False):
    """(loss[G], lse[N,G] | None, dz[N, ldd] | None, colsum[1,C] | None)   (a5-a7 + grad-in-forward)."""
    _require_cuda(logits, labels, wmask, avg)
    assert logits.dtype == torch.float32 and logits.dim() == 2 and logits.stride(1) == 1
    labels = labels.contiguous()
    N, Cc = logits.shape
    dev = logits.device
    loss = torch.empty((dt.G,), dtype=torch.float32, device=dev)
    lse = torch.empty((N, dt.G), dtype=torch.float32, device=dev) if want_lse else None
    dz = colsum = None
    ldd = 0
    if want_dz:
        ldd = pad_cols(Cc)
        dz = torch.empty((N, ldd), dtype=dz_dtype, device=dev)
        colsum = torch.empty((1, Cc), dtype=torch.float32, device=dev)
    ws = _workspace(dev)
    wmask, wcode = _weights_arg(wmask)
    nat.check(nat.lib().bags_group_ce(
        logits.data_ptr(), logits.stride(0), labels.data_ptr(), dt.label2bin.data_ptr(), dt.slices_host,
        nat.ptr(wmask), wcode, nat.ptr(avg), N, Cc, dt.G, dt.num_classes, loss.data_ptr(), nat.ptr(lse), nat.ptr(dz),
        ldd, _dtype_code(dz_dtype), nat.ptr(colsum), ws.data_ptr(), ws.numel(), _stream_ptr(dev)), 'bags_group_ce')
    return loss, lse, dz, colsum


def fused_eligible(dt: DeviceTables) -> bool:
    """True when bags_fwd can keep the logits on chip (fused GEMM + grouped CE kernel)."""
    return bool(nat.lib().bags_fused_eligible(dt.slices_host, dt.G, dt.num_logits))


def fused_fwd(x, w, bias, labels, dt: DeviceTables, wmask, avg, logits: Optional[torch.Tensor] = None,
              want_dz: bool = True, want_lse: bool = False, materialize: Optional[bool] = None,
              want_colsum: bool = False, clear: Optional[torch.Tensor] = None):
    """bags_fwd: fc_cls + grouped CE in one ABI call.  Returns (loss, logits | None, lse, dz, colsum).

    By default (``logits is None`` and the bin table is eligible) the fused kernel runs and no logits
    exist in HBM; pass a ``logits`` buffer or ``materialize=True`` for the GEMM -> fp32 logits -> CE route.
    ``want_colsum`` additionally returns the forward's bias-gradient partial column sums [ceil(N/128), C]
    (fused_bwd recomputes them from dz when they are not supplied).
    """
    _require_cuda(x, w, bias, labels, wmask, avg)
    x, w = _row_major(x), _row_major(w)
    if x.dtype != w.dtype:
        raise nat.BagsNativeError('x (%s) and w (%s) must share a dtype' % (x.dtype, w.dtype))
    labels = labels.contiguous()
    N, K = x.shape
    Cc = w.shape[0]
    dev = x.device
    if materialize is None:
        materialize = (logits is not None) or not fused_eligible(dt)
    if materialize and logits is None:
        logits = torch.empty((N, Cc), dtype=torch.float32, device=dev)
    if not materialize:
        logits = None
    loss = torch.empty((dt.G,), dtype=torch.float32, device=dev)
    lse = torch.empty((N, dt.G), dtype=torch.float32, device=dev) if want_lse else None
    dz = colsum = None
    ldd = 0
    if want_dz:
        ldd = pad_cols(Cc)
        dz = torch.empty((N, ldd), dtype=x.dtype, device=dev)
        if want_colsum:   # per-row-tile partials; by default the backward recomputes them from dz instead
            colsum = torch.empty((max((N + 127) // 128, 1), Cc), dtype=torch.float32, device=dev)
    ws = _workspace(dev)
    wmask, wcode = _weights_arg(wmask)
    if clear is not None:
        # ``clear``: a contiguous buffer (the caller's dW) that the forward zeroes, on the fused route while its CTAs
        # exchange their softmax partials
        assert clear.is_contiguous() and (clear.numel() * clear.element_size()) % 16 == 0
    nat.check(nat.lib().bags_fwd(
        x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), nat.ptr(bias), labels.data_ptr(),
        dt.label2bin.data_ptr(), dt.slices_host, nat.ptr(wmask), wcode, nat.ptr(avg), N, K, Cc, dt.G, dt.num_classes,
        _dtype_code(x.dtype), nat.ptr(logits), logits.stride(0) if logits is not None else 0, loss.data_ptr(),
        nat.ptr(lse), nat.ptr(dz), ldd, nat.ptr(colsum), colsum.shape[0] if colsum is not None else 0, ws.data_ptr(),
        ws.numel(), nat.ptr(clear), clear.numel() * clear.element_size() if clear is not None else 0,
        _stream_ptr(dev)), 'bags_fwd')
    return loss, logits, lse, dz, colsum


def ce_fwd(x, w, bias, labels, weights=None, avg=None, want_acc: bool = False, want_dz: bool = True,
           want_colsum: bool = False, clear: Optional[torch.Tensor] = None, acc_out: Optional[torch.Tensor] = None):
    """bags_ce_fwd: fc_cls + softmax CE over all C logits in the fused kernel (ReweightBBoxHead / BBoxHead.loss).
    Returns (loss [1], acc [1] | None, dz [N, pad_cols(C)] | None, colsum [ceil(N/128), C] | None).

    ``weights``: fp32 [N] per-RoI weights (None: 1); ``avg``: fp32 [1] normaliser on the device (None: N).
    ``want_acc``: also the top-1 accuracy in percent (ties with the row maximum count as correct), written into
    ``acc_out`` when given.  ``clear``: as in ``fused_fwd``."""
    _require_cuda(x, w, bias, labels, weights, avg, clear, acc_out)
    x, w = _row_major(x), _row_major(w)
    if x.dtype != w.dtype:
        raise nat.BagsNativeError('x (%s) and w (%s) must share a dtype' % (x.dtype, w.dtype))
    labels = labels.contiguous()
    N, K = x.shape
    Cc = w.shape[0]
    dev = x.device
    if bias is not None:
        assert bias.dtype == torch.float32
        bias = bias.contiguous()
    if weights is not None:
        weights = weights.to(torch.float32).contiguous()
        assert weights.numel() == N
    if avg is not None:
        assert avg.dtype == torch.float32 and avg.numel() >= 1
    loss = torch.empty((1,), dtype=torch.float32, device=dev)
    acc = None
    if want_acc:
        acc = acc_out if acc_out is not None else torch.empty((1,), dtype=torch.float32, device=dev)
        assert acc.dtype == torch.float32 and acc.numel() == 1
    dz = colsum = None
    ldd = 0
    if want_dz:
        ldd = pad_cols(Cc)
        dz = torch.empty((N, ldd), dtype=x.dtype, device=dev)
        if want_colsum:
            colsum = torch.empty((max((N + 127) // 128, 1), Cc), dtype=torch.float32, device=dev)
    if clear is not None:
        assert clear.is_contiguous() and (clear.numel() * clear.element_size()) % 16 == 0
    ws = _workspace(dev)
    nat.check(nat.lib().bags_ce_fwd(
        x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), nat.ptr(bias), labels.data_ptr(), nat.ptr(weights),
        nat.ptr(avg), N, K, Cc, _dtype_code(x.dtype), loss.data_ptr(), nat.ptr(acc), nat.ptr(dz), ldd, nat.ptr(colsum),
        colsum.shape[0] if colsum is not None else 0, ws.data_ptr(), ws.numel(), nat.ptr(clear),
        clear.numel() * clear.element_size() if clear is not None else 0, _stream_ptr(dev)), 'bags_ce_fwd')
    return loss, acc, dz, colsum


_scratch_cache: Dict[Tuple, torch.Tensor] = {}


def bwd_scratch(w: torch.Tensor, cached: bool = False) -> torch.Tensor:
    """Scratch buffer for fused_bwd (row-scaled copy of W + bias-gradient partials), reusable across calls.
    ``cached``: one buffer per (device, stream, shape) -- safe because consecutive launches on a stream are ordered."""
    key = None
    if cached:
        key = (w.device.index, _stream_ptr(w.device), w.shape[0], w.stride(0), w.dtype)
        hit = _scratch_cache.get(key)
        if hit is not None:
            return hit
    nbytes = nat.lib().bags_bwd_scratch_bytes(w.shape[0], w.stride(0), _dtype_code(w.dtype))
    buf = torch.empty(nbytes, dtype=torch.uint8, device=w.device)
    if cached:
        if len(_scratch_cache) > 32:
            _scratch_cache.clear()
        _scratch_cache[key] = buf
    return buf


def fused_bwd(dz, x, w, gout, dt: DeviceTables, colsum=None, need_dw=True, need_db=True, need_dx=True,
              dW: Optional[torch.Tensor] = None, dX: Optional[torch.Tensor] = None,
              wscratch: Optional[torch.Tensor] = None, db: Optional[torch.Tensor] = None, dw_prezeroed: bool = False):
    """bags_bwd: (dW fp32 [C,K] | None, db fp32 [C] | None, dX [N,K] operand dtype | None)   (a8).
    ``colsum`` (forward's column-sum partials) is optional; without it db is recomputed from dz.
    ``dw_prezeroed``: the given ``dW`` is already zero (``fused_fwd(clear=dW)``): no zeroing job in the backward."""
    _require_cuda(dz, x, w, gout, colsum)
    x, w = _row_major(x), _row_major(w)
    N, K = x.shape
    Cc = w.shape[0]
    dev = x.device
    if need_dw and dW is None:
        dW = torch.empty((Cc, K), dtype=torch.float32, device=dev)
    if need_db and db is None:
        db = torch.empty((Cc,), dtype=torch.float32, device=dev)
    if not need_db:
        db = None
    if need_dx and dX is None:
        dX = torch.empty((N, K), dtype=x.dtype, device=dev)
    if wscratch is None and ((need_dx and gout is not None) or (need_db and colsum is None)):
        # (not under stream capture: a captured graph must own its buffers)
        wscratch = bwd_scratch(w, cached=not torch.cuda.is_current_stream_capturing())
    if gout is not None:
        gout = gout.contiguous()
        assert gout.dtype == torch.float32 and gout.numel() == dt.G
    nat.check(nat.lib().bags_bwd(
        dz.data_ptr(), dz.stride(0), x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), nat.ptr(gout),
        dt.slices_host, nat.ptr(colsum), (colsum.shape[0] if colsum.dim() == 2 else 1) if colsum is not None else 0,
        nat.ptr(dW) if need_dw else None, dW.stride(0) if need_dw else 0,
        nat.ptr(db), nat.ptr(dX) if need_dx else None, dX.stride(0) if need_dx else 0,
        nat.ptr(wscratch), wscratch.numel() * wscratch.element_size() if wscratch is not None else 0,
        N, K, Cc, dt.G, _dtype_code(x.dtype), 1 if (dw_prezeroed and need_dw) else 0, _stream_ptr(dev)), 'bags_bwd')
    return (dW if need_dw else None), db, (dX if need_dx else None)


def merge_scores(logits: torch.Tensor, dt: DeviceTables) -> torch.Tensor:
    """scores [N, num_classes] fp32   (a10: gs_bbox_head_with0.py:239-273)."""
    _require_cuda(logits)
    if logits.dtype != torch.float32:
        raise nat.BagsNativeError('merge_scores expects fp32 logits')
    logits = _row_major(logits)
    N, Cc = logits.shape
    scores = torch.empty((N, dt.num_classes), dtype=torch.float32, device=logits.device)
    nat.check(nat.lib().bags_merge_scores(logits.data_ptr(), logits.stride(0), dt.slices_host,
                                          dt.cls2col.data_ptr(), N, Cc, dt.G, dt.num_classes, scores.data_ptr(),
                                          scores.stride(0), _stream_ptr(logits.device)), 'bags_merge_scores')
    return scores


def multiclass_nms(multi_bboxes: torch.Tensor, multi_scores: torch.Tensor, score_thr: float, iou_thr: float,
                   max_num: int = -1) -> Tuple[torch.Tensor, torch.Tensor]:
    """mmdet/core/post_processing/bbox_nms.py:6-66 (hard NMS) with the per-class Python loop -- 1230 NMS launches and as
    many host syncs per image -- replaced by device-side work and ONE sync for the size of the result:

        one batched descending sort of the class scores  ->  per-class candidate counts (score > score_thr) on the device
        ->  bags_class_nms_dense: one CTA per class gathers its candidates' boxes and suppresses (IoU with "+1" widths,
            mmdet/ops/nms/src/nms_kernel.cu:13-21,60)  ->  top-``max_num`` by score of the survivors (bbox_nms.py:55-61)

    Returns (dets [k,5], labels [k] 0-based): class-major / score-descending order when nothing is cut, score order
    when ``max_num`` cuts -- as the reference; ``max_num = -1`` drops the lowest-scored detection, as the reference does."""
    _require_cuda(multi_bboxes, multi_scores)
    n, num_classes = multi_scores.shape
    dev = multi_scores.device
    S = num_classes - 1
    if n == 0 or S <= 0:
        return multi_bboxes.new_zeros((0, 5)), multi_bboxes.new_zeros((0,), dtype=torch.long)
    boxes = multi_bboxes.float().contiguous()
    if boxes.shape[1] not in (4, 4 * num_classes):
        raise nat.BagsNativeError('multi_bboxes must be [n, 4] or [n, 4 * num_classes]')
    vals, order = multi_scores[:, 1:].float().t().contiguous().sort(dim=1, descending=True, stable=True)   # [S, n]
    counts = (vals > score_thr).sum(dim=1, dtype=torch.int32)
    order32 = order.to(torch.int32)
    keep = torch.empty((S, n), dtype=torch.uint8, device=dev)
    overflow = torch.zeros(1, dtype=torch.int32, device=dev)
    nat.check(nat.lib().bags_class_nms_dense(boxes.data_ptr(), boxes.shape[1], order32.data_ptr(), counts.data_ptr(), S, n,
                                             float(iou_thr), keep.data_ptr(), overflow.data_ptr(), _stream_ptr(dev)),
              'bags_class_nms_dense')
    kept = keep.bool()
    flat = torch.where(kept, vals, torch.full_like(vals, float('-inf'))).reshape(-1)
    cap = min(max_num, S * n) if max_num >= 0 else S * n
    topv, topi = flat.topk(cap)                                      # survivors by descending score, then -inf padding
    total, ovf = (int(v) for v in torch.stack([kept.sum(), overflow[0].to(torch.int64)]).tolist())   # the one sync
    if ovf:
        raise nat.BagsNativeError('multiclass_nms: a class has more than 1024 candidates above score_thr (n = %d)' % n)
    if total > max_num:                                              # bbox_nms.py:57-61 (true for max_num = -1 as well)
        k = max_num if max_num >= 0 else total + max_num             # inds[:max_num]: a negative bound drops the tail
        sel = topi[:max(min(k, total), 0)]
    else:
        sel = topi[:total].sort().values                             # class-major, score-descending inside a class
    cls = torch.div(sel, n, rounding_mode='floor')
    rows = order.reshape(-1)[sel]
    b4 = boxes[rows] if boxes.shape[1] == 4 else boxes.view(n, num_classes, 4)[rows, cls + 1]
    dets = torch.cat([b4, vals.reshape(-1)[sel][:, None]], 1)
    return dets, cls


def gemm_probe(a, a_mn: bool, b, b_mn: bool, M: int, N: int, K: int, block_n: int = 256, splits: int = 1,
               epi: int = 0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Test hook for one wgmma GEMM (see bags_gemm_probe)."""
    _require_cuda(a, b)
    dev = a.device
    if out is None:
        out_dtype = torch.bfloat16 if epi == 1 else torch.float32
        out = torch.zeros((M, (N + 7) // 8 * 8), dtype=out_dtype, device=dev)[:, :N]  # 16-byte aligned rows
    nat.check(nat.lib().bags_gemm_probe(a.data_ptr(), a.stride(0), int(a_mn), b.data_ptr(), b.stride(0), int(b_mn),
                                        out.data_ptr(), out.stride(0), M, N, K, _dtype_code(a.dtype), block_n,
                                        splits, epi, _stream_ptr(dev)), 'bags_gemm_probe')
    return out


# --------------------------------------------------------------------------- the trunk's linear layers
def linear_act(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], relu: bool,
               out_dtype: Optional[torch.dtype] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[N,C] = act(x @ w^T + bias), act = ReLU or identity, on the wgmma GEMM (convfc_bbox_head.py:138-143,167).
    x and w share the operand dtype (bf16, or fp32 = TF32 products); out is fp32 or (bf16 operands) bf16."""
    _require_cuda(x, w, bias)
    x, w = _row_major(x), _row_major(w)
    if x.dtype != w.dtype:
        raise nat.BagsNativeError('x (%s) and w (%s) must share a dtype' % (x.dtype, w.dtype))
    N, K = x.shape
    Cc = w.shape[0]
    if out_dtype is None:
        out_dtype = x.dtype
    if out is None:
        out = torch.empty((N, Cc), dtype=out_dtype, device=x.device)
    if bias is not None:
        bias = bias.contiguous()
        assert bias.dtype == torch.float32
    splits = nat.lib().bags_linear_act_splits(N, K, Cc, _dtype_code(x.dtype)) if N > 0 else 1
    if splits > 1:
        # few output tiles, long contraction (shared_fcs.0): split-K into an fp32 workspace, then bias + activation
        ws = torch.empty((N, (Cc + 3) // 4 * 4), dtype=torch.float32, device=x.device)
        nat.check(nat.lib().bags_linear_act_fwd_splitk(x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), nat.ptr(bias),
                                                       out.data_ptr(), out.stride(0), N, K, Cc, _dtype_code(x.dtype),
                                                       _dtype_code(out.dtype), 1 if relu else 0, ws.data_ptr(),
                                                       ws.stride(0), splits, _stream_ptr(x.device)),
                  'bags_linear_act_fwd_splitk')
        return out
    nat.check(nat.lib().bags_linear_act_fwd(x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), nat.ptr(bias),
                                            out.data_ptr(), out.stride(0), N, K, Cc, _dtype_code(x.dtype),
                                            _dtype_code(out.dtype), 1 if relu else 0, _stream_ptr(x.device)),
              'bags_linear_act_fwd')
    return out


def act_bwd(dy: torch.Tensor, y: Optional[torch.Tensor], g_dtype: torch.dtype) -> torch.Tensor:
    """g [rows, pad64(cols)] = (y > 0 ? dy : 0) in ``g_dtype`` (y None: a cast of dy): the A operand of the layer's
    backward contractions, with the padded leading dimension bags_bwd wants."""
    _require_cuda(dy, y)
    dy = _row_major(dy)
    rows, cols = dy.shape
    g = torch.empty((rows, pad_cols(cols)), dtype=g_dtype, device=dy.device)
    if y is not None:
        y = _row_major(y)
    nat.check(nat.lib().bags_act_bwd(dy.data_ptr(), dy.stride(0), _dtype_code(dy.dtype), nat.ptr(y),
                                     y.stride(0) if y is not None else 0,
                                     _dtype_code(y.dtype) if y is not None else nat.DTYPE_F32, g.data_ptr(), g.stride(0),
                                     _dtype_code(g_dtype), rows, cols, _stream_ptr(dy.device)), 'bags_act_bwd')
    return g


_operand_cache: Dict[int, tuple] = {}   # id(parameter) -> (weakref to it, version, bf16 copy)


def _bf16_operand(t: torch.Tensor) -> torch.Tensor:
    """bf16 copy of an fp32 master parameter, re-made only when the parameter changed (its version counter moves with
    every in-place optimizer update) -- shared_fcs.0.weight alone is 51 MB."""
    import weakref
    if t.dtype == torch.bfloat16:
        return _row_major(t)
    key = id(t)
    hit = _operand_cache.get(key)
    if hit is not None and hit[0]() is t and hit[1] == t._version and hit[2].device == t.device:
        return hit[2]
    c = cast_bf16(_row_major(t.detach().float()))
    if len(_operand_cache) > 64:      # parameters that went away
        for k in [k for k, v in _operand_cache.items() if v[0]() is None]:
            del _operand_cache[k]
    _operand_cache[key] = (weakref.ref(t), t._version, c)
    return c


def _single_slice_tables(cols: int, device) -> DeviceTables:
    """One bin (0, cols): the table of bags_bwd for a plain layer or the softmax-CE head."""
    return DeviceTables(1, 1, cols, torch.zeros(1, 1, dtype=torch.int32, device=device),
                        torch.zeros(1, dtype=torch.int32, device=device), nat.int32_array([0, cols]),
                        np.array([[0, cols]], dtype=np.int64))


class LinearActFunction(torch.autograd.Function):
    """y = act(x W^T + b) for the head's shared FCs (ReLU) and fc_reg (identity) -- nn.Linear (+ nn.ReLU) of the
    reference (convfc_bbox_head.py:138-143,167) on this library's wgmma GEMMs, forward and backward:

    forward : bags_linear_act_fwd (bias + activation in the GEMM epilogue; bf16 output feeds the next layer)
    backward: bags_act_bwd (ReLU mask + cast) -> bags_bwd (dW = g^T x, db, dX = g W: preparation + one merged launch)"""

    @staticmethod
    def forward(ctx, x, weight, bias, relu, compute_dtype, out_dtype):
        _require_cuda(x, weight, bias)
        xin = x.detach()
        if compute_dtype == torch.bfloat16:
            xc = _row_major(xin) if xin.dtype == torch.bfloat16 else cast_bf16(_row_major(xin.float()))
            wc = _bf16_operand(weight)
        elif compute_dtype == torch.float32:
            xc, wc = _row_major(xin.float()), _row_major(weight.detach().float())
        else:
            raise nat.BagsNativeError('compute_dtype must be torch.bfloat16 or torch.float32')
        b32 = None if bias is None else bias.detach().float().contiguous()
        y = linear_act(xc, wc, b32, bool(relu), out_dtype=out_dtype)
        ctx.relu = bool(relu)
        ctx.meta = (x.dtype, weight.dtype, None if bias is None else bias.dtype)
        if any(ctx.needs_input_grad[:3]):
            ctx.save_for_backward(xc, wc, y if relu else None)
        return y

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        xc, wc, y = ctx.saved_tensors
        xd, wd, bd = ctx.meta
        g = act_bwd(grad_out.detach(), y, xc.dtype)
        dt1 = _single_slice_tables(wc.shape[0], xc.device)
        dW, db, dX = fused_bwd(g, xc, wc, None, dt1, None, need_dw=ctx.needs_input_grad[1],
                               need_db=ctx.needs_input_grad[2] and bd is not None, need_dx=ctx.needs_input_grad[0])
        return (None if dX is None else dX.to(xd), None if dW is None else dW.to(wd),
                None if db is None else db.to(bd), None, None, None)


# --------------------------------------------------------------------------- autograd
# where the backward's preparation work runs: 1 = dW is zeroed by the fused forward kernel (idle producer warps)
PREP_IN_FORWARD = os.environ.get('BAGS_PREP_IN_FORWARD', '1') != '0'
# 1 = the bias-gradient column sums come from the forward's epilogue as well (otherwise a job of the backward's
# preparation kernel).  Off by default on one GPU; with a grad_bucket (data-parallel schedule)
# it is always on: the dW + db launch -- on the critical path before the exchange -- then has nothing to prepare.
FWD_COLSUM = os.environ.get('BAGS_FWD_COLSUM', '0') == '1'


def _fc_cls_operands(x, weight, bias, compute_dtype):
    """(xc, wc, b32): the fc_cls operands the fused forward reads.  bf16: fp32 masters are cast (the weight only when
    it changed); float32: fp32 operands, TF32 products.  The bias is always fp32."""
    if compute_dtype == torch.bfloat16:
        xc = _row_major(x) if x.dtype == torch.bfloat16 else cast_bf16(_row_major(x.float()))
        wc = _bf16_operand(weight)      # fp32 master: re-cast only when the parameter changed (version counter)
    elif compute_dtype == torch.float32:
        if x.dtype != torch.float32 or weight.dtype != torch.float32:
            raise nat.BagsNativeError('float32 compute needs float32 x and weight')
        xc, wc = _row_major(x), _row_major(weight)
    else:
        raise nat.BagsNativeError('compute_dtype must be torch.bfloat16 or torch.float32')
    if bias is None or (bias.dtype == torch.float32 and bias.is_contiguous()):
        b32 = bias
    else:
        b32 = bias.float().contiguous()
    return xc, wc, b32


def _save_param_dtypes(ctx, x, weight, bias) -> None:
    ctx.x_dtype = x.dtype
    ctx.w_dtype = weight.dtype
    ctx.has_bias = bias is not None
    ctx.bias_dtype = None if bias is None else bias.dtype


def _gout(grad_loss: torch.Tensor) -> torch.Tensor:
    return grad_loss if (grad_loss.dtype == torch.float32 and grad_loss.is_contiguous()) \
        else grad_loss.to(torch.float32).contiguous()


def _grads_in_param_dtypes(ctx, dX, dW, db):
    """dX, dW, db in the dtypes of x, the weight and the bias (the kernels produce dX in the operand dtype, dW / db
    in fp32)."""
    if dX is not None and dX.dtype != ctx.x_dtype:
        dX = dX.to(ctx.x_dtype)
    if dW is not None and dW.dtype != ctx.w_dtype:
        dW = dW.to(ctx.w_dtype)
    if db is not None and db.dtype != ctx.bias_dtype:
        db = db.to(ctx.bias_dtype)
    return dX, dW, db


class GroupSoftmaxFunction(torch.autograd.Function):
    """losses[G] = BAGS(fc_cls(x)) with a fused backward.

    forward : bags_fwd  (fused kernel: wgmma fc_cls GEMM with the grouped softmax-CE in its epilogue;
              logits stay on chip unless a ``logits_out`` buffer is given; saves dz~ and its column sums)
    backward: bags_bwd  (dW = dz^T x, db, dX = dz W on wgmma; per-bin upstream gradients applied
              in the GEMM epilogue / on a scaled copy of W)

    compute_dtype torch.bfloat16: x and W are used as bf16 operands (fp32 masters are cast by
    bags_cast_bf16); torch.float32: fp32 operands, TF32 products.  Accumulation, softmax, loss
    and dW/db are always fp32.
    """

    @staticmethod
    def forward(ctx, x, weight, bias, labels, dt: DeviceTables, wmask, avg, compute_dtype, logits_out, grad_bucket=None):
        """``grad_bucket`` (optional, data-parallel training): an object with ``views = (dW [C,K] fp32, db [C] fp32)`` living
        in the ranks' exchange bucket and ``exchange_overlapped()`` -- e.g. ``dist.PeerGradBucket``.  The backward then
        writes dW / db straight into the bucket, starts the exchange as soon as they are complete and computes dX while
        the gradients travel (the reference exchanges after the whole backward, dist_utils.py:51-58);
        the returned weight / bias gradients ARE the bucket views, holding the mean over ranks."""
        _require_cuda(x, weight, bias, labels)
        # (autograd does not record inside Function.forward: the inputs are used as they are, no detach() round trips)
        xc, wc, b32 = _fc_cls_operands(x, weight, bias, compute_dtype)
        need_grad = any(ctx.needs_input_grad[:3])
        # dW is allocated here and zeroed by the forward kernel (its split-K red.add in the
        # backward then needs no zeroing job); BAGS_FWD_COLSUM=1 also takes the bias-gradient partials from the forward
        dW = None
        ctx.grad_bucket = grad_bucket if (grad_bucket is not None and need_grad and ctx.needs_input_grad[1]) else None
        if ctx.grad_bucket is not None:
            dW = grad_bucket.views[0]
            assert dW.dtype == torch.float32 and tuple(dW.shape) == (wc.shape[0], wc.shape[1]) and dW.is_contiguous()
            if logits_out is not None or not PREP_IN_FORWARD:
                dW.zero_()
        elif need_grad and ctx.needs_input_grad[1] and logits_out is None and PREP_IN_FORWARD:
            dW = torch.empty((wc.shape[0], wc.shape[1]), dtype=torch.float32, device=xc.device)
        loss, _, _, dz, colsum = fused_fwd(xc, wc, b32, labels, dt, wmask, avg, logits=logits_out,
                                           want_dz=need_grad, clear=dW,
                                           want_colsum=(dW is not None and bias is not None and
                                                        (FWD_COLSUM or ctx.grad_bucket is not None)))
        ctx.dW = dW
        ctx.colsum = colsum if dW is not None else None
        ctx.dt = dt
        _save_param_dtypes(ctx, x, weight, bias)
        if need_grad:
            ctx.save_for_backward(xc, wc, dz)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_loss):
        xc, wc, dz = ctx.saved_tensors
        need_dx, need_dw, need_db = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        gout = _gout(grad_loss)
        dW0, ctx.dW = ctx.dW, None                      # (a second backward through a retained graph zeroes again)
        bucket = ctx.grad_bucket
        if bucket is not None and need_dw:
            # dW + db first, straight into the exchange bucket; the exchange starts when they are complete and runs
            # while the dX contraction does
            if dW0 is None:
                bucket.views[0].zero_()
            db_view = bucket.views[1] if (need_db and ctx.has_bias and len(bucket.views) > 1) else None
            dW, db, _ = fused_bwd(dz, xc, wc, gout, ctx.dt, ctx.colsum, need_dw=True,
                                  need_db=(need_db and ctx.has_bias), need_dx=False, dW=bucket.views[0], db=db_view,
                                  dw_prezeroed=True)
            join = bucket.exchange_overlapped()
            dX = None
            if need_dx:
                _, _, dX = fused_bwd(dz, xc, wc, gout, ctx.dt, None, need_dw=False, need_db=False, need_dx=True)
            join()
        else:
            dW, db, dX = fused_bwd(dz, xc, wc, gout, ctx.dt, ctx.colsum, need_dw=need_dw,
                                   need_db=(need_db and ctx.has_bias), need_dx=need_dx,
                                   dW=dW0 if need_dw else None, dw_prezeroed=dW0 is not None)
        dX, dW, db = _grads_in_param_dtypes(ctx, dX, dW, db)
        return dX, dW, db, None, None, None, None, None, None, None


class SoftmaxCEFunction(torch.autograd.Function):
    """loss[1] = softmax CE of fc_cls(x) over all C logits, per-RoI weighted (ReweightBBoxHead.loss) -- the
    single-bin counterpart of ``GroupSoftmaxFunction``, with the same operand casting:

    forward : bags_ce_fwd (fused fc_cls GEMM + softmax-CE; logits stay on chip; saves dz~; optional top-1 accuracy
              into ``acc_out``, a [1] fp32 tensor, which is not differentiable)
    backward: bags_bwd over the single slice (0, C); dX only when x needs a gradient (head-only training freezes
              the trunk), dW zeroed by the forward kernel."""

    @staticmethod
    def forward(ctx, x, weight, bias, labels, weights, avg, compute_dtype, acc_out=None):
        _require_cuda(x, weight, bias, labels)
        xc, wc, b32 = _fc_cls_operands(x, weight, bias, compute_dtype)
        need_grad = any(ctx.needs_input_grad[:3])
        dW = None
        if need_grad and ctx.needs_input_grad[1] and PREP_IN_FORWARD:
            dW = torch.empty((wc.shape[0], wc.shape[1]), dtype=torch.float32, device=xc.device)
        loss, _, dz, _ = ce_fwd(xc, wc, b32, labels, weights, avg, want_acc=acc_out is not None, want_dz=need_grad,
                                clear=dW, acc_out=acc_out)
        ctx.dW = dW
        ctx.num_cols = wc.shape[0]
        _save_param_dtypes(ctx, x, weight, bias)
        if need_grad:
            ctx.save_for_backward(xc, wc, dz)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_loss):
        xc, wc, dz = ctx.saved_tensors
        need_dx, need_dw, need_db = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        dW0, ctx.dW = ctx.dW, None                      # (a second backward through a retained graph zeroes again)
        dW, db, dX = fused_bwd(dz, xc, wc, _gout(grad_loss), _single_slice_tables(ctx.num_cols, xc.device), None,
                               need_dw=need_dw, need_db=(need_db and ctx.has_bias), need_dx=need_dx,
                               dW=dW0 if need_dw else None, dw_prezeroed=dW0 is not None)
        dX, dW, db = _grads_in_param_dtypes(ctx, dX, dW, db)
        return dX, dW, db, None, None, None, None, None


class GroupCEFunction(torch.autograd.Function):
    """losses[G] from materialised logits (used when loss() is handed a plain cls_score tensor).
    backward returns d/dlogits = gout ⊙ dz~ (computed by torch on the saved dz~; this path exists for API
    completeness -- the hot path is GroupSoftmaxFunction)."""

    @staticmethod
    def forward(ctx, logits, labels, dt: DeviceTables, wmask, avg):
        _require_cuda(logits, labels)
        z = _row_major(logits.detach().float())
        need = ctx.needs_input_grad[0]
        loss, _, dz, _ = group_ce(z, labels, dt, wmask, avg, want_dz=need, dz_dtype=torch.float32)
        ctx.dt = dt
        ctx.in_dtype = logits.dtype
        if need:
            ctx.save_for_backward(dz)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_loss):
        (dz,) = ctx.saved_tensors
        dt = ctx.dt
        Cc = dt.num_logits
        out = torch.zeros((dz.shape[0], Cc), dtype=torch.float32, device=dz.device)
        for g in range(dt.G):
            s, l = int(dt.pred_slice[g, 0]), int(dt.pred_slice[g, 1])
            out[:, s:s + l] = dz[:, s:s + l] * grad_loss[g]
        return out.to(ctx.in_dtype), None, None, None, None
