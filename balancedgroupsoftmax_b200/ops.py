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


def mask_fwd(y, w, bias, labels, targets):
    """bags_mask_fwd: the class-specific channel of conv_logits (a 1x1 conv) fused with mask_cross_entropy -- BCE with
    logits, 'mean' over P * H * W (FCNMaskHead.loss).  Returns (loss [1], g [P, H, W], rsum, index int32
    [classes + 1 + P]); ``g``, ``rsum`` and ``index`` feed ``mask_bwd``.  ``y``: bf16 or fp32 [P, Cin, H, W] (made
    contiguous); ``w``: the fp32 [classes, Cin] weight (never cast to bf16); ``labels``: int64 [P], a row with a label
    outside [0, classes) contributes 0 but counts in the mean; ``targets``: [P, H, W]."""
    _require_cuda(y, w, bias, labels, targets)
    y = y.contiguous()
    w = _row_major(w.reshape(w.shape[0], -1))
    if w.dtype != torch.float32:
        raise nat.BagsNativeError('mask_fwd: the conv_logits weight must be float32 (got %s)' % w.dtype)
    P, Cin, H, W_ = y.shape
    classes = w.shape[0]
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.numel() == classes, 'mask_fwd: bias must be fp32 [classes]'
        bias = bias.contiguous()
    labels = labels.contiguous()
    assert w.shape[1] == Cin and labels.dtype == torch.int64 and labels.numel() == P
    targets = targets.to(torch.float32).contiguous()
    assert targets.shape == (P, H, W_)
    dev = y.device
    tiles = (H * W_ + nat.MASK_TILE - 1) // nat.MASK_TILE
    loss = torch.empty((1,), dtype=torch.float32, device=dev)
    g = torch.empty((P, H, W_), dtype=torch.float32, device=dev)
    rsum = torch.empty((P * tiles * (Cin + 2),), dtype=torch.float32, device=dev)
    index = torch.empty((classes + 1 + P,), dtype=torch.int32, device=dev)
    ws = _workspace(dev)
    nat.check(nat.lib().bags_mask_fwd(
        y.data_ptr(), _dtype_code(y.dtype), w.data_ptr(), w.stride(0), nat.ptr(bias), labels.data_ptr(),
        targets.data_ptr(), P, Cin, H * W_, classes, loss.data_ptr(), g.data_ptr(), rsum.data_ptr(), rsum.numel(),
        index.data_ptr(), ws.data_ptr(), ws.numel(), _stream_ptr(dev)), 'bags_mask_fwd')
    return loss, g, rsum, index


def mask_bwd(g, rsum, gout, w, labels, index, y_shape, y_dtype, need_dw: bool = True, need_db: bool = True,
             need_dy: bool = True):
    """bags_mask_bwd: (dW fp32 [classes, Cin] | None, db fp32 [classes] | None, dY [P, Cin, H, W] in ``y_dtype`` |
    None) from the ``g``, ``rsum`` and ``index`` of ``mask_fwd``; ``gout``: dL/dloss as a device fp32 [1] tensor, or
    None for 1."""
    _require_cuda(g, rsum, gout, w, labels, index)
    w = _row_major(w.reshape(w.shape[0], -1))
    P, Cin, H, W_ = y_shape
    classes = w.shape[0]
    dev = g.device
    if gout is not None:
        gout = _gout(gout)
        assert gout.numel() == 1
    dW = torch.empty((classes, Cin), dtype=torch.float32, device=dev) if need_dw else None
    db = torch.empty((classes,), dtype=torch.float32, device=dev) if need_db else None
    dY = torch.empty((P, Cin, H, W_), dtype=y_dtype, device=dev) if need_dy else None
    nat.check(nat.lib().bags_mask_bwd(
        g.data_ptr(), rsum.data_ptr(), nat.ptr(gout), _dtype_code(y_dtype), w.data_ptr(), w.stride(0),
        labels.contiguous().data_ptr(), index.data_ptr(), P, Cin, H * W_, classes, nat.ptr(dW), Cin, nat.ptr(db),
        nat.ptr(dY), _stream_ptr(dev)), 'bags_mask_bwd')
    return dW, db, dY


def mask_channel_logits(y, weight, bias, channels):
    """bags_mask_logits: [n, 1, H, W] logits in y's dtype of one conv_logits channel per row, channel ``channels[d]``
    of row d -- what conv_logits(y).gather(1, channels[:, None, None, None].expand(-1, 1, H, W)) selects, without the
    [n, classes, H, W] tensor.  fp32 products from the fp32 weight, summed in bags_mask_fwd's order.  ``y``: bf16 or
    fp32 [n, Cin, H, W] (made contiguous); ``weight``: conv_logits.weight ([classes, Cin, 1, 1] or [classes, Cin]);
    ``bias``: [classes] or None; ``channels``: int64 [n] on y's device.  A channel outside [0, classes) gives a map of
    NaN.  Not differentiable: for callers that record no gradient."""
    _require_cuda(y, weight, bias, channels)
    y = y.contiguous()
    n, Cin, H, W_ = y.shape
    _, w, bias = _fp32_master_operands(y, weight, bias)
    w = _row_major(w.reshape(w.shape[0], -1))
    classes = w.shape[0]
    if bias is not None:
        assert bias.numel() == classes, 'mask_channel_logits: bias must be [classes]'
        bias = bias.contiguous()
    assert w.shape[1] == Cin, 'mask_channel_logits: weight is [%d, %d], y has %d channels' % (classes, w.shape[1], Cin)
    assert channels.dtype == torch.int64 and channels.numel() == n, 'mask_channel_logits: channels must be int64 [n]'
    channels = channels.contiguous()
    out = torch.empty((n, 1, H, W_), dtype=y.dtype, device=y.device)
    nat.check(nat.lib().bags_mask_logits(
        y.data_ptr(), _dtype_code(y.dtype), w.data_ptr(), w.stride(0), nat.ptr(bias), channels.data_ptr(), n, Cin,
        H * W_, classes, out.data_ptr(), _stream_ptr(y.device)), 'bags_mask_logits')
    return out


def _fused_outputs(x, w, bias, G: int, want_acc: bool, want_dz: bool, want_colsum: bool,
                   clear: Optional[torch.Tensor], acc_out: Optional[torch.Tensor] = None):
    """Operands and outputs shared by bags_fwd, bags_ce_fwd and bags_focal_fwd: row-major x and w of one dtype, the
    fp32 bias, loss [G], acc [1] (``acc_out`` when given), dz [N, pad_cols(C)] in the operand dtype, the per-row-tile
    colsum [ceil(N/128), C] and the buffer to ``clear``.  Returns (x, w, bias, loss, acc, dz, colsum, tail), ``tail``
    being the calls' common last arguments (dz, ldd, colsum, colsum_tiles, workspace, workspace_bytes, clear,
    clear_bytes, stream)."""
    x, w = _row_major(x), _row_major(w)
    if x.dtype != w.dtype:
        raise nat.BagsNativeError('x (%s) and w (%s) must share a dtype' % (x.dtype, w.dtype))
    N = x.shape[0]
    Cc = w.shape[0]
    dev = x.device
    if bias is not None:
        assert bias.dtype == torch.float32
        bias = bias.contiguous()
    loss = torch.empty((G,), dtype=torch.float32, device=dev)
    acc = None
    if want_acc:
        acc = acc_out if acc_out is not None else torch.empty((1,), dtype=torch.float32, device=dev)
        assert acc.dtype == torch.float32 and acc.numel() == 1
    dz = colsum = None
    ldd = 0
    if want_dz:
        ldd = pad_cols(Cc)
        dz = torch.empty((N, ldd), dtype=x.dtype, device=dev)
        if want_colsum:   # per-row-tile partials; by default the backward recomputes them from dz instead
            colsum = torch.empty((max((N + 127) // 128, 1), Cc), dtype=torch.float32, device=dev)
    if clear is not None:
        # ``clear``: a contiguous buffer (the caller's dW) that the forward zeroes, on the fused route while its CTAs
        # exchange their softmax partials
        assert clear.is_contiguous() and (clear.numel() * clear.element_size()) % 16 == 0
    ws = _workspace(dev)
    tail = (nat.ptr(dz), ldd, nat.ptr(colsum), colsum.shape[0] if colsum is not None else 0, ws.data_ptr(), ws.numel(),
            nat.ptr(clear), clear.numel() * clear.element_size() if clear is not None else 0, _stream_ptr(dev))
    return x, w, bias, loss, acc, dz, colsum, tail


def _roi_weights(weights: Optional[torch.Tensor], N: int) -> Optional[torch.Tensor]:
    """fp32 [N] per-RoI weights of the single-bin losses (None: 1)."""
    if weights is None:
        return None
    weights = weights.to(torch.float32).contiguous()
    assert weights.numel() == N
    return weights


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
    x, w, bias, loss, _, dz, colsum, tail = _fused_outputs(x, w, bias, dt.G, False, want_dz, want_colsum, clear)
    labels = labels.contiguous()
    N, K = x.shape
    Cc = w.shape[0]
    if materialize is None:
        materialize = (logits is not None) or not fused_eligible(dt)
    if materialize and logits is None:
        logits = torch.empty((N, Cc), dtype=torch.float32, device=x.device)
    if not materialize:
        logits = None
    lse = torch.empty((N, dt.G), dtype=torch.float32, device=x.device) if want_lse else None
    wmask, wcode = _weights_arg(wmask)
    nat.check(nat.lib().bags_fwd(
        x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), nat.ptr(bias), labels.data_ptr(),
        dt.label2bin.data_ptr(), dt.slices_host, nat.ptr(wmask), wcode, nat.ptr(avg), N, K, Cc, dt.G, dt.num_classes,
        _dtype_code(x.dtype), nat.ptr(logits), logits.stride(0) if logits is not None else 0, loss.data_ptr(),
        nat.ptr(lse), *tail), 'bags_fwd')
    return loss, logits, lse, dz, colsum


def ce_fwd(x, w, bias, labels, weights=None, avg=None, want_acc: bool = False, want_dz: bool = True,
           want_colsum: bool = False, clear: Optional[torch.Tensor] = None, acc_out: Optional[torch.Tensor] = None):
    """bags_ce_fwd: fc_cls + softmax CE over all C logits in the fused kernel (ReweightBBoxHead / BBoxHead.loss).
    Returns (loss [1], acc [1] | None, dz [N, pad_cols(C)] | None, colsum [ceil(N/128), C] | None).

    ``weights``: fp32 [N] per-RoI weights (None: 1); ``avg``: fp32 [1] normaliser on the device (None: N).
    ``want_acc``: also the top-1 accuracy in percent (ties with the row maximum count as correct), written into
    ``acc_out`` when given.  ``clear``: as in ``fused_fwd``."""
    _require_cuda(x, w, bias, labels, weights, avg, clear, acc_out)
    x, w, bias, loss, acc, dz, colsum, tail = _fused_outputs(x, w, bias, 1, want_acc, want_dz, want_colsum, clear,
                                                             acc_out)
    labels = labels.contiguous()
    N, K = x.shape
    weights = _roi_weights(weights, N)
    if avg is not None:
        assert avg.dtype == torch.float32 and avg.numel() >= 1
    nat.check(nat.lib().bags_ce_fwd(
        x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), nat.ptr(bias), labels.data_ptr(), nat.ptr(weights),
        nat.ptr(avg), N, K, w.shape[0], _dtype_code(x.dtype), loss.data_ptr(), nat.ptr(acc), *tail), 'bags_ce_fwd')
    return loss, acc, dz, colsum


def focal_fwd(x, w, bias, targets, norm: float, gamma: float = 2.0, alpha: float = 0.25, labels=None, weights=None,
              want_acc: bool = False, want_dz: bool = True, want_colsum: bool = False,
              clear: Optional[torch.Tensor] = None, acc_out: Optional[torch.Tensor] = None):
    """bags_focal_fwd: fc_cls + the sigmoid focal loss over all C logits in the fused kernel (FocalLoss with
    ReweightBBoxHead).  Returns (loss [1], acc [1] | None, dz [N, pad_cols(C)] | None, colsum [ceil(N/128), C] | None).

    ``targets``: int64 [N] in the focal-loss op's convention (column t - 1 positive, t < 0 ignores the row; see
    ``losses.focal_targets``); ``norm``: the host-known divisor (N * 1231 for FocalLoss); ``labels``: int64 [N], for the
    accuracy only.  ``weights``, ``want_acc``, ``clear``, ``acc_out``: as in ``ce_fwd``."""
    _require_cuda(x, w, bias, targets, labels, weights, clear, acc_out)
    x, w, bias, loss, acc, dz, colsum, tail = _fused_outputs(x, w, bias, 1, want_acc, want_dz, want_colsum, clear,
                                                             acc_out)
    N, K = x.shape
    weights = _roi_weights(weights, N)
    targets = targets.contiguous()
    assert targets.dtype == torch.int64 and targets.numel() == N
    if want_acc:
        if labels is None:
            raise nat.BagsNativeError('focal_fwd: the accuracy needs the labels')
        labels = labels.contiguous()
        assert labels.dtype == torch.int64 and labels.numel() == N
    nat.check(nat.lib().bags_focal_fwd(
        x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), nat.ptr(bias), targets.data_ptr(),
        nat.ptr(labels) if want_acc else None, nat.ptr(weights), float(norm), float(gamma), float(alpha), N, K,
        w.shape[0], _dtype_code(x.dtype), loss.data_ptr(), nat.ptr(acc), *tail), 'bags_focal_fwd')
    return loss, acc, dz, colsum


def box_fwd(x, w, bias, labels, targets, weights, beta: float, avg: float, want_pred: bool = False):
    """bags_box_fwd: the class-specific fc_reg columns of the positive RoIs fused with SmoothL1 'mean' (BBoxHead's box
    loss).  Returns (loss [1], g [N, 4], index int32 [classes + 1 + N], pred [N, 4] | None); ``g`` and ``index`` feed
    ``box_bwd``.  ``w``: the fp32 [4 * classes, K] weight (never cast to bf16); ``x``: bf16 or fp32 [N, K];
    ``avg``: the host normaliser (bbox_targets.size(0))."""
    _require_cuda(x, w, bias, labels, targets, weights)
    x, w = _row_major(x), _row_major(w)
    if w.dtype != torch.float32:
        raise nat.BagsNativeError('box_fwd: the fc_reg weight must be float32 (got %s)' % w.dtype)
    if bias is not None:
        assert bias.dtype == torch.float32
        bias = bias.contiguous()
    labels = labels.contiguous()
    targets = targets.to(torch.float32).contiguous()
    weights = weights.to(torch.float32).contiguous()
    N, K = x.shape
    classes = w.shape[0] // 4
    assert w.shape[0] == 4 * classes and w.shape[1] == K
    assert labels.dtype == torch.int64 and labels.numel() == N and targets.shape == (N, 4) and weights.shape == (N, 4)
    dev = x.device
    loss = torch.empty((1,), dtype=torch.float32, device=dev)
    g = torch.empty((N, 4), dtype=torch.float32, device=dev)
    index = torch.empty((classes + 1 + N,), dtype=torch.int32, device=dev)
    pred = torch.empty((N, 4), dtype=torch.float32, device=dev) if want_pred else None
    ws = _workspace(dev)
    nat.check(nat.lib().bags_box_fwd(
        x.data_ptr(), x.stride(0), _dtype_code(x.dtype), w.data_ptr(), w.stride(0), nat.ptr(bias), labels.data_ptr(),
        targets.data_ptr(), weights.data_ptr(), float(beta), float(avg), N, K, classes, loss.data_ptr(), g.data_ptr(),
        nat.ptr(pred), index.data_ptr(), ws.data_ptr(), ws.numel(), _stream_ptr(dev)), 'bags_box_fwd')
    return loss, g, index, pred


def box_bwd(g, gout, x, w, labels, index, need_dw: bool = True, need_db: bool = True, need_dx: bool = True):
    """bags_box_bwd: (dW fp32 [4 * classes, K] | None, db fp32 [4 * classes] | None, dX [N, K] x's dtype | None) from
    the ``g`` and ``index`` of ``box_fwd``; ``gout``: dL/dloss as a device fp32 [1] tensor, or None for 1."""
    _require_cuda(g, gout, x, w, labels, index)
    x, w = _row_major(x), _row_major(w)
    N, K = x.shape
    classes = w.shape[0] // 4
    dev = x.device
    if gout is not None:
        gout = _gout(gout)
        assert gout.numel() == 1
    dW = torch.empty((4 * classes, K), dtype=torch.float32, device=dev) if need_dw else None
    db = torch.empty((4 * classes,), dtype=torch.float32, device=dev) if need_db else None
    dX = torch.empty((N, K), dtype=x.dtype, device=dev) if need_dx else None
    nat.check(nat.lib().bags_box_bwd(
        g.data_ptr(), nat.ptr(gout), x.data_ptr(), x.stride(0), _dtype_code(x.dtype), w.data_ptr(), w.stride(0),
        labels.contiguous().data_ptr(), index.data_ptr(), N, K, classes, nat.ptr(dW), K, nat.ptr(db), nat.ptr(dX), K,
        _stream_ptr(dev)), 'bags_box_bwd')
    return dW, db, dX


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

    Returns (dets [k,5], labels [k] 0-based) in the reference's order: when nothing is cut, class-major and ascending
    RoI index inside a class (the NMS op returns its kept indices sorted, nms_kernel.cu:127-130); score order when
    ``max_num`` cuts.  ``max_num = -1`` drops the lowest-scored detection, as the reference does.  A candidate is a
    score ``> score_thr`` compared in the scores' own dtype (bbox_nms.py:36), so a NaN score is never one.  Equal scores
    of a class are visited lower RoI index first (the reference's unstable sort leaves that order open)."""
    _require_cuda(multi_bboxes, multi_scores)
    n, num_classes = multi_scores.shape
    dev = multi_scores.device
    S = num_classes - 1
    if n == 0 or S <= 0:
        return multi_bboxes.new_zeros((0, 5)), multi_bboxes.new_zeros((0,), dtype=torch.long)
    boxes = multi_bboxes.float().contiguous()
    if boxes.data_ptr() % 16:                                        # a view at an odd offset: the kernel reads float4
        boxes = boxes.clone()
    if boxes.shape[1] not in (4, 4 * num_classes):
        raise nat.BagsNativeError('multi_bboxes must be [n, 4] or [n, 4 * num_classes]')
    cand = (multi_scores[:, 1:] > score_thr).t()                     # in the scores' dtype; NaN is never a candidate
    counts = cand.sum(dim=1, dtype=torch.int32)
    # non-candidates sort last, so each class's candidates are the first counts[s] of its row
    key = torch.where(cand, multi_scores[:, 1:].t().float(), float('-inf'))
    vals, order = key.contiguous().sort(dim=1, descending=True, stable=True)   # [S, n]
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
    else:                                                            # class-major, ascending RoI index inside a class
        sel = topi[:total]
        sel = sel[(torch.div(sel, n, rounding_mode='floor') * n + order.reshape(-1)[sel]).argsort()]
    cls = torch.div(sel, n, rounding_mode='floor')
    rows = order.reshape(-1)[sel]
    b4 = boxes[rows] if boxes.shape[1] == 4 else boxes.view(n, num_classes, 4)[rows, cls + 1]
    dets = torch.cat([b4, vals.reshape(-1)[sel][:, None]], 1)
    return dets, cls


def seg_masks_rle(probs: torch.Tensor, boxes: np.ndarray, img_h: int, img_w: int, thr: float) -> list:
    """COCO compressed RLE strings (the ``counts`` of pycocotools.mask.encode) of n test-time masks, each the map
    ``probs[d]`` (fp32 [n, h, w] on the GPU) resized to its box as cv2.INTER_LINEAR does, thresholded with ``> thr``
    and pasted at (left, top) into an empty ``img_h x img_w`` image (fcn_mask_head.py:160-179).  ``boxes``: int32
    [n, 4] (left, top, w, h), each inside the image.  The comparison is in float64 against ``thr`` as given, so pass
    ``float(np.float32(thr))`` for numpy's float32 comparison.  Two launches of bags_segm_rle and two host syncs:
    the string lengths, then the strings."""
    _require_cuda(probs)
    n = int(boxes.shape[0])
    if n == 0:
        return []
    dev = probs.device
    probs = probs.float().contiguous()
    if probs.dim() != 3 or probs.shape[0] != n:
        raise nat.BagsNativeError('seg_masks_rle: probs must be [n, h, w] with n = %d boxes' % n)
    boxes = np.ascontiguousarray(boxes, dtype=np.int32)
    boxes_dev = torch.empty((n, 4), dtype=torch.int32, device=dev)
    lengths = torch.empty((n,), dtype=torch.int64, device=dev)
    args = (probs.data_ptr(), n, probs.shape[1], probs.shape[2], boxes.ctypes.data, boxes_dev.data_ptr(), int(img_h),
            int(img_w), float(thr), lengths.data_ptr())
    nat.check(nat.lib().bags_segm_rle(*args, None, _stream_ptr(dev)), 'bags_segm_rle')
    lens = lengths.cpu().numpy()                                     # host sync: the sizes
    ends = np.cumsum(lens)
    out = torch.empty((max(int(ends[-1]), 1),), dtype=torch.uint8, device=dev)
    nat.check(nat.lib().bags_segm_rle(*args, out.data_ptr(), _stream_ptr(dev)), 'bags_segm_rle')
    data = out[:int(ends[-1])].cpu().numpy().tobytes()               # host sync: the strings
    return [data[e - l:e] for e, l in zip(ends.tolist(), lens.tolist())]


def upload_masks(gt_masks_list, device) -> list:
    """uint8 [num_gt, H, W] gt masks of each image on ``device``: CUDA tensors there as they are (made contiguous),
    everything else (mmdet's numpy masks) packed into one pinned host tensor and uploaded with one non-blocking copy.
    The caching host allocator keeps the pinned tensor until the copy has run, so nothing waits for it."""
    out = [None] * len(gt_masks_list)
    host = []
    for i, m in enumerate(gt_masks_list):
        if isinstance(m, torch.Tensor) and m.is_cuda:
            if m.device != torch.device(device) or m.dtype != torch.uint8 or m.dim() != 3:
                raise nat.BagsNativeError('mask_targets: CUDA gt masks must be uint8 [num_gt, H, W] on %s (got %s %s on '
                                          '%s)' % (device, m.dtype, tuple(m.shape), m.device))
            out[i] = m.contiguous()
        else:
            a = np.asarray(m.cpu() if isinstance(m, torch.Tensor) else m)
            if a.dtype != np.uint8 or a.ndim != 3:
                raise nat.BagsNativeError('mask_targets: gt masks must be uint8 [num_gt, H, W] (got %s %s)'
                                          % (a.dtype, a.shape))
            host.append((i, a))
    if host:
        staging = torch.empty((sum(a.size for _, a in host),), dtype=torch.uint8, pin_memory=True)
        flat, at = staging.numpy(), 0
        for _, a in host:
            flat[at:at + a.size].reshape(a.shape)[...] = a
            at += a.size
        dev_buf, at = staging.to(device, non_blocking=True), 0
        for i, a in host:
            out[i] = dev_buf[at:at + a.size].view(a.shape)
            at += a.size
    return out


def mask_targets(pos_proposals_list, pos_assigned_gt_inds_list, gt_masks_list, mask_size) -> torch.Tensor:
    """bags_mask_target: the mask heads' training targets (mmdet/core/mask/mask_target.py) of every image in one
    launch -- each positive RoI's gt mask cut to its proposal box (truncated to int32, at least one pixel wide and
    high, numpy slice rules) and resized to ``mask_size`` as cv2.resize(uint8, INTER_LINEAR) does, bitwise.  float32
    [sum P, h, w] on the proposals' device, images in order.  ``pos_proposals_list``: [P, >= 4] CUDA boxes per image;
    ``pos_assigned_gt_inds_list``: [P] integer gt indices; ``gt_masks_list``: uint8 [num_gt, H, W] per image, CUDA
    tensors (read in place) or numpy arrays (``upload_masks``).  A gt index outside [0, num_gt) or a crop the slicing
    leaves empty gives a row of NaN.  No host sync: with CUDA masks it can be captured in a CUDA graph."""
    mh, mw = (mask_size, mask_size) if isinstance(mask_size, int) else tuple(mask_size)
    n = len(pos_proposals_list)
    if not (len(pos_assigned_gt_inds_list) == len(gt_masks_list) == n) or n == 0:
        raise nat.BagsNativeError('mask_targets: one proposal tensor, gt index tensor and mask array per image '
                                  '(got %d, %d, %d)' % (n, len(pos_assigned_gt_inds_list), len(gt_masks_list)))
    _require_cuda(*pos_proposals_list, *pos_assigned_gt_inds_list)
    dev = pos_proposals_list[0].device
    boxes = [p[:, :4].float().contiguous() for p in pos_proposals_list]
    gt_inds = [g.to(torch.int64).contiguous() for g in pos_assigned_gt_inds_list]
    masks = upload_masks(gt_masks_list, dev)
    sizes = np.array([(b.shape[0], m.shape[0], m.shape[1], m.shape[2]) for b, m in zip(boxes, masks)], dtype=np.int32)
    if any(g.numel() != b.shape[0] for b, g in zip(boxes, gt_inds)):
        raise nat.BagsNativeError('mask_targets: one gt index per positive proposal')
    out = torch.empty((int(sizes[:, 0].sum()), mh, mw), dtype=torch.float32, device=dev)
    ptrs = lambda ts: (C.c_void_p * n)(*[t.data_ptr() if t.numel() else None for t in ts])   # noqa: E731
    nat.check(nat.lib().bags_mask_target(ptrs(boxes), ptrs(gt_inds), ptrs(masks), sizes.ctypes.data, n, mh, mw,
                                         out.data_ptr(), _stream_ptr(dev)), 'bags_mask_target')
    return out


# --------------------------------------------------------------------------- RPN proposals
def _rpn_levels(cls_scores, bbox_preds, base_anchors, strides):
    L = len(cls_scores)
    if not (L == len(bbox_preds) == len(base_anchors) == len(strides)) or not 1 <= L <= 8:
        raise nat.BagsNativeError('rpn_proposals: %d score levels, %d delta levels, %d base-anchor tables and %d '
                                  'strides (1 to 8 levels, the same count of each)'
                                  % (L, len(bbox_preds), len(base_anchors), len(strides)))
    B = cls_scores[0].shape[0] if cls_scores[0].dim() == 4 else -1
    levels = np.zeros((L, 4), dtype=np.int32)
    for l, (s, d, base) in enumerate(zip(cls_scores, bbox_preds, base_anchors)):
        A = s.shape[1] if s.dim() == 4 else -1
        if s.dim() != 4 or d.dim() != 4 or s.shape[0] != B or tuple(d.shape) != (B, 4 * A) + tuple(s.shape[2:]):
            raise nat.BagsNativeError('rpn_proposals: level %d: scores must be [B, A, H, W] and deltas [B, 4A, H, W] '
                                      'with one B (got %s and %s)' % (l, tuple(s.shape), tuple(d.shape)))
        if tuple(np.shape(base)) != (A, 4):
            raise nat.BagsNativeError('rpn_proposals: level %d: %d anchors per location but base anchors of shape %s'
                                      % (l, A, tuple(np.shape(base))))
        levels[l] = (s.shape[2], s.shape[3], A, int(strides[l]))
    return B, levels


def rpn_scratch_bytes(levels: np.ndarray, B: int, nms_pre: int, nms_post: int) -> int:
    """bags_rpn_scratch_bytes: device scratch bags_rpn_proposals needs; ``levels`` int32 [L, 4] (H, W, A, stride)."""
    levels = np.ascontiguousarray(levels, dtype=np.int32)
    out = C.c_size_t(0)
    nat.check(nat.lib().bags_rpn_scratch_bytes(levels.ctypes.data, levels.shape[0], int(B), int(nms_pre),
                                               int(nms_post), C.byref(out)), 'bags_rpn_scratch_bytes')
    return out.value


def rpn_proposals(cls_scores, bbox_preds, base_anchors, strides, img_shapes, nms_pre: int, nms_post: int,
                  max_num: int, nms_thr: float, min_bbox_size: float = 0.0, means=(0., 0., 0., 0.),
                  stds=(1., 1., 1., 1.)):
    """bags_rpn_proposals: the proposals of a sigmoid RPN for every image and level in one call (four launches), with
    no host sync -- capturable in a CUDA graph.

    ``cls_scores`` / ``bbox_preds``: per level, CUDA fp32 [B, A, H, W] logits and [B, 4A, H, W] deltas (made
    contiguous); ``base_anchors``: per level [A, 4] (AnchorGenerator.base_anchors); ``strides``: per level;
    ``img_shapes``: per image (h, w, ...).  Returns ``(proposals, counts)``: fp32 [B, max_num, 5] rows (x1, y1, x2, y2,
    score), the first counts[b] of image b valid and the rest zero, and int32 [B] counts.  Equal to RPNHead.get_bboxes
    (nms_across_levels=False) per image where no tie decides the result; ties are broken by (score desc, flat index
    asc) within a level and (score desc, level asc, position asc) across levels."""
    cls_scores, bbox_preds = list(cls_scores), list(bbox_preds)
    for t in cls_scores + bbox_preds:
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32:
            raise nat.BagsNativeError('rpn_proposals: scores and deltas must be CUDA fp32 tensors (got %s)'
                                      % (t.dtype if isinstance(t, torch.Tensor) else type(t).__name__,))
    B, levels = _rpn_levels(cls_scores, bbox_preds, base_anchors, strides)
    if len(img_shapes) != B:
        raise nat.BagsNativeError('rpn_proposals: %d img_shapes for %d images' % (len(img_shapes), B))
    dev = cls_scores[0].device
    cls_scores = [t.detach().contiguous() for t in cls_scores]
    bbox_preds = [t.detach().contiguous() for t in bbox_preds]
    base = np.ascontiguousarray(np.concatenate([np.asarray(torch.as_tensor(b, dtype=torch.float32).cpu(),
                                                           dtype=np.float32).reshape(-1, 4) for b in base_anchors]))
    shapes = np.array([(int(s[0]), int(s[1])) for s in img_shapes], dtype=np.int32).reshape(B, 2)
    mean = np.asarray(means, dtype=np.float32).reshape(4)
    std = np.asarray(stds, dtype=np.float32).reshape(4)
    nbytes = rpn_scratch_bytes(levels, B, nms_pre, nms_post)
    scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    max_num = int(max_num)
    out = torch.empty((B, max(max_num, 0), 5), dtype=torch.float32, device=dev)
    counts = torch.empty((B,), dtype=torch.int32, device=dev)
    L = len(cls_scores)
    lp = (C.c_void_p * L)(*[t.data_ptr() for t in cls_scores])
    dp = (C.c_void_p * L)(*[t.data_ptr() for t in bbox_preds])
    nat.check(nat.lib().bags_rpn_proposals(lp, dp, levels.ctypes.data, base.ctypes.data, L, B, shapes.ctypes.data,
                                           int(nms_pre), int(nms_post), max_num, float(nms_thr), float(min_bbox_size),
                                           mean.ctypes.data, std.ctypes.data, scratch.data_ptr(), nbytes,
                                           out.data_ptr(), counts.data_ptr(), _stream_ptr(dev)), 'bags_rpn_proposals')
    return out, counts


# --------------------------------------------------------------------------- RPN training targets
def valid_size(pad_shape, stride: int, featmap_size) -> Tuple[int, int]:
    """AnchorHead.get_anchors' valid_flags size of one level: (min(ceil(pad_h / stride), feat_h), same for w)."""
    return (min(int(np.ceil(pad_shape[0] / stride)), int(featmap_size[0])),
            min(int(np.ceil(pad_shape[1] / stride)), int(featmap_size[1])))


def _anchor_target_levels(featmap_sizes, base_anchors, strides):
    L = len(featmap_sizes)
    if not (L == len(base_anchors) == len(strides)) or not 1 <= L <= 8:
        raise nat.BagsNativeError('anchor_targets: %d feature maps, %d base-anchor tables and %d strides (1 to 8 '
                                  'levels, the same count of each)' % (L, len(base_anchors), len(strides)))
    levels = np.zeros((L, 4), dtype=np.int32)
    for l, ((h, w), base) in enumerate(zip(featmap_sizes, base_anchors)):
        levels[l] = (int(h), int(w), int(np.shape(base)[0]), int(strides[l]))
    base = np.ascontiguousarray(np.concatenate([np.asarray(torch.as_tensor(b, dtype=torch.float32).cpu(),
                                                           dtype=np.float32).reshape(-1, 4) for b in base_anchors]))
    return levels, base


def anchor_target_scratch_bytes(levels: np.ndarray, B: int, total_gts: int) -> int:
    """bags_anchor_target_scratch_bytes: device scratch bags_anchor_target needs; ``levels`` int32 [L, 4]
    (H, W, A, stride)."""
    levels = np.ascontiguousarray(levels, dtype=np.int32)
    out = C.c_size_t(0)
    nat.check(nat.lib().bags_anchor_target_scratch_bytes(levels.ctypes.data, levels.shape[0], int(B), int(total_gts),
                                                         C.byref(out)), 'bags_anchor_target_scratch_bytes')
    return out.value


def anchor_targets(featmap_sizes, base_anchors, strides, img_shapes, pad_shapes, gt_bboxes, pos_iou_thr=0.7,
                   neg_iou_thr=0.3, min_pos_iou=0.3, gt_max_assign_all=True, allowed_border=0, num=256,
                   pos_fraction=0.5, neg_pos_ub=-1, pos_weight=-1, means=(0., 0., 0., 0.), stds=(1., 1., 1., 1.),
                   seed: int = 0, seed_step: Optional[torch.Tensor] = None):
    """bags_anchor_target: anchor_target of an RPN (MaxIoUAssigner + the base sampler, no gt labels, no ignored gts)
    for every image in one call (a memset and four launches), with no host sync -- capturable in a CUDA graph.

    ``featmap_sizes``: per level (H, W); ``base_anchors``: per level [A, 4] (AnchorGenerator.base_anchors);
    ``strides``: per level; ``img_shapes`` / ``pad_shapes``: per image (h, w, ...); ``gt_bboxes``: per image a CUDA
    [G_i, 4] tensor, G_i >= 1.  The assigner's and sampler's parameters as in their configs: ``neg_iou_thr`` a float
    (negatives 0 <= max < thr) or a tuple (lo <= max < hi); any other type gives no negatives, as in the reference.
    ``seed`` / ``seed_step`` pick the sample as in sample_others: the k positives and then the k negatives with the
    smallest (sample_key(seed, image, n) << 32 | n), an exact-k uniform subset (statistically, not bitwise, the
    reference's np.random.shuffle draw).

    Returns ``(labels, label_weights, bbox_targets, bbox_weights, totals)``: int64 [B, N], fp32 [B, N], fp32
    [B, N, 4], fp32 [B, N, 4] over the N anchors of an image (level after level, location-major), zero outside the
    inside anchors, and int64 [3] device totals (num_total_pos, num_total_neg, num_total_samples)."""
    gt_bboxes = list(gt_bboxes)
    for t in gt_bboxes:
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dim() != 2 or t.shape[1] != 4 or t.shape[0] < 1:
            raise nat.BagsNativeError('anchor_targets: gt_bboxes must be CUDA [G, 4] tensors with G >= 1 (got %s)'
                                      % (tuple(t.shape) if isinstance(t, torch.Tensor) else type(t).__name__,))
    _require_cuda(seed_step)
    levels, base = _anchor_target_levels(featmap_sizes, base_anchors, strides)
    B, L = len(gt_bboxes), levels.shape[0]
    if len(img_shapes) != B or len(pad_shapes) != B:
        raise nat.BagsNativeError('anchor_targets: %d img_shapes and %d pad_shapes for %d images'
                                  % (len(img_shapes), len(pad_shapes), B))
    images = np.zeros((B, 4 + 2 * L), dtype=np.int32)
    off = 0
    for b in range(B):
        g = int(gt_bboxes[b].shape[0])
        images[b, :4] = (int(img_shapes[b][0]), int(img_shapes[b][1]), off, g)
        off += g
        for l in range(L):
            images[b, 4 + 2 * l: 6 + 2 * l] = valid_size(pad_shapes[b], int(strides[l]), featmap_sizes[l])
    if isinstance(neg_iou_thr, float):
        neg = (1, 0.0, neg_iou_thr)
    elif isinstance(neg_iou_thr, tuple):
        assert len(neg_iou_thr) == 2
        neg = (1, float(neg_iou_thr[0]), float(neg_iou_thr[1]))
    else:   # the reference's assigner tests neither branch: no negatives
        neg = (0, 0.0, 0.0)
    if seed_step is not None:
        assert seed_step.dtype == torch.int64 and seed_step.numel() == 1
    dev = gt_bboxes[0].device
    gts = torch.cat([t.detach().float() for t in gt_bboxes]).contiguous()
    mean = np.asarray(means, dtype=np.float32).reshape(4)
    std = np.asarray(stds, dtype=np.float32).reshape(4)
    N = int(sum(int(h) * int(w) * int(a) for h, w, a, _ in levels))
    nbytes = anchor_target_scratch_bytes(levels, B, off)
    scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    labels = torch.empty((B, N), dtype=torch.int64, device=dev)
    label_weights = torch.empty((B, N), dtype=torch.float32, device=dev)
    bbox_targets = torch.empty((B, N, 4), dtype=torch.float32, device=dev)
    bbox_weights = torch.empty((B, N, 4), dtype=torch.float32, device=dev)
    totals = torch.empty((3,), dtype=torch.int64, device=dev)
    images = np.ascontiguousarray(images)
    nat.check(nat.lib().bags_anchor_target(
        levels.ctypes.data, base.ctypes.data, L, B, images.ctypes.data, gts.data_ptr(), off, float(pos_iou_thr),
        neg[0], neg[1], neg[2], float(min_pos_iou), int(bool(gt_max_assign_all)), float(allowed_border), int(num),
        float(pos_fraction), float(neg_pos_ub), float(pos_weight), mean.ctypes.data, std.ctypes.data,
        int(seed) & 0xFFFFFFFFFFFFFFFF, nat.ptr(seed_step), scratch.data_ptr(), nbytes, labels.data_ptr(),
        label_weights.data_ptr(), bbox_targets.data_ptr(), bbox_weights.data_ptr(), totals.data_ptr(),
        _stream_ptr(dev)), 'bags_anchor_target')
    return labels, label_weights, bbox_targets, bbox_weights, totals


# --------------------------------------------------------------------------- FPN RoI feature extractor
@dataclass(frozen=True)
class RoIAlignSpec:
    """What bags_roi_align_fwd / _bwd take besides the tensors: the output size, each level's spatial_scale (as the
    reference's op receives it, a C++ float), the samples per bin (<= 0: adaptive) and map_roi_levels' finest_scale
    (unused with one level)."""
    out_size: Tuple[int, int]
    scales: Tuple[float, ...]
    sample_num: int = 0
    finest_scale: float = 56.0


def _roi_align_args(spec: RoIAlignSpec, shapes, rois: torch.Tensor, rois_map: torch.Tensor):
    L = len(shapes)
    if L != len(spec.scales) or not 1 <= L <= 8:
        raise nat.BagsNativeError('roi_align: %d feature levels and %d scales (1 to 8 levels)' % (L, len(spec.scales)))
    B, Cc = shapes[0][0], shapes[0][1]
    if any(len(s) != 4 or s[0] != B or s[1] != Cc for s in shapes):
        raise nat.BagsNativeError('roi_align: every level must be [B, C, H, W] with the same B and C (got %s)'
                                  % [tuple(s) for s in shapes])
    for r in (rois, rois_map):
        if r.dtype != torch.float32 or r.dim() != 2 or r.shape[1] != 5 or not r.is_contiguous():
            raise nat.BagsNativeError('roi_align: rois must be contiguous fp32 [k, 5] (got %s %s)'
                                      % (r.dtype, tuple(r.shape)))
    if rois_map.shape[0] != rois.shape[0]:
        raise nat.BagsNativeError('roi_align: %d RoIs to map, %d to pool' % (rois_map.shape[0], rois.shape[0]))
    sizes = np.array([(s[2], s[3]) for s in shapes], dtype=np.int32)
    scales = np.array(spec.scales, dtype=np.float32)
    oh, ow = spec.out_size
    return (sizes, scales, L, B, Cc, rois_map.data_ptr(), rois.data_ptr(), rois.shape[0], oh, ow, spec.sample_num,
            float(spec.finest_scale))


def roi_align_fwd(feats, rois: torch.Tensor, spec: RoIAlignSpec, rois_map: Optional[torch.Tensor] = None,
                  want_levels: bool = False):
    """bags_roi_align_fwd: every RoI pooled from its level in one launch, bitwise the reference's op; fp32
    [k, C, out_h, out_w].  ``feats``: contiguous fp32 [B, C, H_l, W_l] per level; ``rois`` (and ``rois_map``, the RoIs
    the levels are mapped from, ``rois`` when None): contiguous fp32 [k, 5].  With ``want_levels`` also returns the
    int32 [k] level of each RoI (-1: a NaN scale, which gives a zero row, as a batch index outside [0, B) does)."""
    feats = list(feats)
    _require_cuda(rois, rois_map, *feats)
    rois_map = rois if rois_map is None else rois_map
    for f in feats:
        if f.dtype != torch.float32 or not f.is_contiguous():
            raise nat.BagsNativeError('roi_align: features must be contiguous fp32 (got %s)' % f.dtype)
    args = _roi_align_args(spec, [f.shape for f in feats], rois, rois_map)
    sizes, scales, L, B, Cc, pm, pr, k, oh, ow = args[:10]
    dev = rois.device
    out = torch.empty((k, Cc, oh, ow), dtype=torch.float32, device=dev)
    levels = torch.empty((k,), dtype=torch.int32, device=dev) if want_levels else None
    ptrs = (C.c_void_p * L)(*[f.data_ptr() for f in feats])
    nat.check(nat.lib().bags_roi_align_fwd(ptrs, sizes.ctypes.data, scales.ctypes.data, *args[2:], nat.ptr(out),
                                           nat.ptr(levels), _stream_ptr(dev)), 'bags_roi_align_fwd')
    return (out, levels) if want_levels else out


def roi_align_bwd(gout: torch.Tensor, shapes, rois: torch.Tensor, spec: RoIAlignSpec,
                  rois_map: Optional[torch.Tensor] = None, needs=None):
    """bags_roi_align_bwd: the gradient of roi_align_fwd for every level in one launch, into fp32 gradients zeroed on
    the stream.  ``shapes``: each level's [B, C, H, W]; ``needs``: which levels want a gradient (all when None).
    Returns one fp32 gradient per level, None where it is not wanted; nothing is launched when none is."""
    _require_cuda(gout, rois, rois_map)
    rois_map = rois if rois_map is None else rois_map
    needs = [True] * len(shapes) if needs is None else list(needs)
    args = _roi_align_args(spec, shapes, rois, rois_map)
    sizes, scales, L = args[:3]
    dev = gout.device
    gout = gout.float().contiguous()
    if tuple(gout.shape) != (args[7], args[4]) + tuple(spec.out_size):
        raise nat.BagsNativeError('roi_align: gout must be [k, C, out_h, out_w] (got %s)' % (tuple(gout.shape),))
    grads = [torch.zeros(tuple(s), dtype=torch.float32, device=dev) if n else None for s, n in zip(shapes, needs)]
    if any(needs):
        ptrs = (C.c_void_p * L)(*[nat.ptr(g) for g in grads])
        nat.check(nat.lib().bags_roi_align_bwd(gout.data_ptr(), ptrs, sizes.ctypes.data, scales.ctypes.data, *args[2:],
                                               _stream_ptr(dev)), 'bags_roi_align_bwd')
    return grads


class RoIAlignFunction(torch.autograd.Function):
    """out = roi_align_fwd(feats, rois, spec, rois_map) as an autograd Function over ``(rois, *feats)``; fp32
    contiguous features (the callers cast).  Its backward is one bags_roi_align_bwd launch for the levels that need a
    gradient, none when no level does; the RoIs get no gradient, as in the reference."""

    @staticmethod
    def forward(ctx, spec: RoIAlignSpec, rois_map, rois, *feats):
        ctx.spec = spec
        ctx.shapes = [tuple(f.shape) for f in feats]
        ctx.save_for_backward(rois, rois_map)
        return roi_align_fwd(feats, rois, spec, rois_map)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gout):
        rois, rois_map = ctx.saved_tensors
        needs = ctx.needs_input_grad[3:]
        grads = roi_align_bwd(gout, ctx.shapes, rois, ctx.spec, rois_map, needs) if any(needs) else [None] * len(needs)
        return (None, None, None) + tuple(grads)


def roi_align_apply(feats, rois: torch.Tensor, spec: RoIAlignSpec, rois_map: Optional[torch.Tensor] = None):
    """RoIAlignFunction on any floating features: non-fp32 ones are cast to fp32 first (force_fp32) and take their
    gradient back through the cast; features and RoIs are made contiguous."""
    _require_cuda(rois, rois_map, *feats)
    rois = rois.float().contiguous()
    rois_map = rois if rois_map is None else rois_map.float().contiguous()
    feats = [f.float().contiguous() for f in feats]
    return RoIAlignFunction.apply(spec, rois_map, rois, *feats)


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
        _save_param_dtypes(ctx, x, weight, bias)
        if any(ctx.needs_input_grad[:3]):
            ctx.save_for_backward(xc, wc, y if relu else None)
        return y

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        xc, wc, y = ctx.saved_tensors
        g = act_bwd(grad_out.detach(), y, xc.dtype)
        dt1 = _single_slice_tables(wc.shape[0], xc.device)
        dW, db, dX = fused_bwd(g, xc, wc, None, dt1, None, need_dw=ctx.needs_input_grad[1],
                               need_db=ctx.needs_input_grad[2] and ctx.has_bias, need_dx=ctx.needs_input_grad[0])
        return _grads_in_param_dtypes(ctx, dX, dW, db) + (None, None, None)


# --------------------------------------------------------------------------- autograd
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


def _fused_loss_prologue(ctx, x, weight, bias, compute_dtype, clear_dw: bool = True):
    """Forward prologue of the fused-loss Functions: (xc, wc, b32, dW).  xc, wc, b32: the fc_cls operands
    (``_fc_cls_operands``); dW: when the weight needs a gradient and ``clear_dw``, its fp32 [C, K] buffer for the fused
    forward to zero (its ``clear``), so that the backward's split-K red.add needs no zeroing job; None otherwise."""
    xc, wc, b32 = _fc_cls_operands(x, weight, bias, compute_dtype)
    _save_param_dtypes(ctx, x, weight, bias)
    dW = None
    if ctx.needs_input_grad[1] and clear_dw:
        dW = torch.empty((wc.shape[0], wc.shape[1]), dtype=torch.float32, device=xc.device)
    return xc, wc, b32, dW


def _fused_loss_saved(ctx, xc, wc, dz, dW) -> None:
    """What ``_fused_loss_bwd`` reads: the dW the forward zeroed, and dz~ with the operands when a gradient is needed."""
    ctx.dW = dW
    if any(ctx.needs_input_grad[:3]):
        ctx.save_for_backward(xc, wc, dz)


def _fused_loss_bwd(ctx, grad_loss, dt: Optional[DeviceTables] = None, colsum: Optional[torch.Tensor] = None,
                    bucket=None):
    """(dX, dW, db) in the parameters' dtypes from the dz~ a fused-loss forward saved: one bags_bwd over the bin table
    ``dt`` (None: the single slice (0, C)), with the forward's column-sum partials ``colsum`` when it took them; dX only
    when x needs a gradient, dW zeroed by the forward kernel when ``ctx.dW`` is set.

    With a gradient ``bucket`` (``views = (dW, db)``, ``exchange_overlapped()``) and a weight gradient wanted, dW + db
    go straight into the bucket views in a first bags_bwd, the exchange starts as soon as they are complete, and dX is
    a second bags_bwd that runs while the gradients travel; the exchange is joined before returning."""
    xc, wc, dz = ctx.saved_tensors
    need_dx, need_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
    need_db = ctx.needs_input_grad[2] and ctx.has_bias
    split = bucket is not None and need_dw
    dW0, ctx.dW = ctx.dW, None                      # (a second backward through a retained graph zeroes again)
    if dt is None:
        dt = _single_slice_tables(wc.shape[0], xc.device)
    gout = _gout(grad_loss)
    if split and dW0 is None:
        dW0 = bucket.views[0].zero_()
    dW, db, dX = fused_bwd(dz, xc, wc, gout, dt, colsum, need_dw=need_dw, need_db=need_db,
                           need_dx=need_dx and not split, dW=dW0 if need_dw else None, dw_prezeroed=dW0 is not None,
                           db=bucket.views[1] if (split and need_db and len(bucket.views) > 1) else None)
    if split:
        join = bucket.exchange_overlapped()
        if need_dx:
            _, _, dX = fused_bwd(dz, xc, wc, gout, dt, None, need_dw=False, need_db=False, need_dx=True)
        join()
    return _grads_in_param_dtypes(ctx, dX, dW, db)


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
        ctx.grad_bucket = grad_bucket if (grad_bucket is not None and ctx.needs_input_grad[1]) else None
        xc, wc, b32, dW = _fused_loss_prologue(ctx, x, weight, bias, compute_dtype,
                                               clear_dw=ctx.grad_bucket is None and logits_out is None)
        if ctx.grad_bucket is not None:
            # the forward zeroes the bucket's dW as well, and takes the bias-gradient partials: the dW + db launch -- on
            # the critical path before the exchange -- then has nothing to prepare
            dW = grad_bucket.views[0]
            assert dW.dtype == torch.float32 and tuple(dW.shape) == (wc.shape[0], wc.shape[1]) and dW.is_contiguous()
            if logits_out is not None:
                dW.zero_()
        loss, _, _, dz, colsum = fused_fwd(xc, wc, b32, labels, dt, wmask, avg, logits=logits_out,
                                           want_dz=any(ctx.needs_input_grad[:3]), clear=dW,
                                           want_colsum=ctx.grad_bucket is not None and bias is not None)
        ctx.dt = dt
        ctx.colsum = colsum
        _fused_loss_saved(ctx, xc, wc, dz, dW)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_loss):
        return _fused_loss_bwd(ctx, grad_loss, ctx.dt, ctx.colsum, ctx.grad_bucket) + (None,) * 7


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
        xc, wc, b32, dW = _fused_loss_prologue(ctx, x, weight, bias, compute_dtype)
        loss, _, dz, _ = ce_fwd(xc, wc, b32, labels, weights, avg, want_acc=acc_out is not None,
                                want_dz=any(ctx.needs_input_grad[:3]), clear=dW, acc_out=acc_out)
        _fused_loss_saved(ctx, xc, wc, dz, dW)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_loss):
        return _fused_loss_bwd(ctx, grad_loss) + (None,) * 5


class SigmoidFocalFunction(torch.autograd.Function):
    """loss[1] = sigmoid focal loss of fc_cls(x) over all C logits, per-RoI weighted, divided by ``norm``
    (FocalLoss(use_sigmoid=True) in ReweightBBoxHead.loss) -- the focal counterpart of ``SoftmaxCEFunction``:

    forward : bags_focal_fwd (fused fc_cls GEMM + the focal loss and the op's analytic gradient per element; logits stay
              on chip; saves dz~; optional top-1 accuracy of ``labels`` into ``acc_out``)
    backward: bags_bwd over the single slice (0, C), as SoftmaxCEFunction.  ``norm`` is a host number (from shapes): no
              host sync."""

    @staticmethod
    def forward(ctx, x, weight, bias, targets, weights, norm, gamma, alpha, compute_dtype, labels=None, acc_out=None):
        _require_cuda(x, weight, bias, targets)
        xc, wc, b32, dW = _fused_loss_prologue(ctx, x, weight, bias, compute_dtype)
        loss, _, dz, _ = focal_fwd(xc, wc, b32, targets, norm, gamma, alpha, labels=labels, weights=weights,
                                   want_acc=acc_out is not None, want_dz=any(ctx.needs_input_grad[:3]), clear=dW,
                                   acc_out=acc_out)
        _fused_loss_saved(ctx, xc, wc, dz, dW)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_loss):
        return _fused_loss_bwd(ctx, grad_loss) + (None,) * 8


def _fp32_master_operands(x, weight, bias):
    """(xc, wc, b32) of the kernels that multiply in fp32 from the fp32 master weight (box and mask losses): x stays
    bf16 or fp32, anything else becomes fp32; the weight and the bias are fp32."""
    xc = x if x.dtype in (torch.bfloat16, torch.float32) else x.float()
    wc = weight if weight.dtype == torch.float32 else weight.float()
    b32 = None if bias is None else (bias if bias.dtype == torch.float32 else bias.float())
    return xc, wc, b32


class SmoothL1BoxFunction(torch.autograd.Function):
    """loss[1] = SmoothL1 'mean' of the class-specific box deltas of the positive RoIs, fc_reg included
    (BBoxHead._bbox_loss on fc_reg(x) with loss_weight 1) -- only the four columns each positive RoI's loss reads:

    forward : bags_box_fwd (fp32 products from the fp32 master weight, the loss, its gradient g and the class index;
              no host sync: ``avg`` is a host number, bbox_targets.size(0))
    backward: bags_box_bwd (dW fully written -- zero rows for absent classes --, db, dX), only what autograd needs."""

    @staticmethod
    def forward(ctx, x, weight, bias, labels, targets, weights, beta, avg):
        _require_cuda(x, weight, bias, labels, targets, weights)
        xc, wc, b32 = _fp32_master_operands(x, weight, bias)
        labels = labels.contiguous()
        loss, g, index, _ = box_fwd(xc, wc, b32, labels, targets, weights, beta, avg)
        _save_param_dtypes(ctx, x, weight, bias)
        if any(ctx.needs_input_grad[:3]):
            ctx.save_for_backward(g, index, _row_major(xc), _row_major(wc), labels)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_loss):
        g, index, xc, wc, labels = ctx.saved_tensors
        dW, db, dX = box_bwd(g, grad_loss, xc, wc, labels, index, need_dw=ctx.needs_input_grad[1],
                             need_db=ctx.needs_input_grad[2] and ctx.has_bias, need_dx=ctx.needs_input_grad[0])
        dX, dW, db = _grads_in_param_dtypes(ctx, dX, dW, db)
        return dX, dW, db, None, None, None, None, None


class MaskBCEFunction(torch.autograd.Function):
    """loss[1] = mask_cross_entropy of the class-specific 1x1 conv_logits, the conv included (FCNMaskHead.loss on
    conv_logits(y) with loss_weight 1) -- only the channel of each RoI's label:

    forward : bags_mask_fwd (fp32 products from the fp32 weight, the loss, its gradient g, the per-tile sums of g y for
              dW and the class index; no host sync)
    backward: bags_mask_bwd (dW fully written -- zero rows for absent classes --, db, dY), only what autograd needs.

    ``weight`` may be the conv's [classes, Cin, 1, 1] parameter; its gradient comes back in that shape."""

    @staticmethod
    def forward(ctx, y, weight, bias, labels, targets):
        _require_cuda(y, weight, bias, labels, targets)
        yc, wc, b32 = _fp32_master_operands(y, weight, bias)
        labels = labels.contiguous()
        loss, g, rsum, index = mask_fwd(yc, wc, b32, labels, targets)
        _save_param_dtypes(ctx, y, weight, bias)
        ctx.y_shape, ctx.y_cdtype, ctx.w_shape = tuple(yc.shape), yc.dtype, weight.shape
        if any(ctx.needs_input_grad[:3]):
            ctx.save_for_backward(g, rsum, index, wc.reshape(wc.shape[0], -1), labels)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_loss):
        g, rsum, index, wc, labels = ctx.saved_tensors
        dW, db, dY = mask_bwd(g, rsum, grad_loss, wc, labels, index, ctx.y_shape, ctx.y_cdtype,
                              need_dw=ctx.needs_input_grad[1], need_db=ctx.needs_input_grad[2] and ctx.has_bias,
                              need_dy=ctx.needs_input_grad[0])
        dY, dW, db = _grads_in_param_dtypes(ctx, dY, dW, db)
        if dW is not None:
            dW = dW.reshape(ctx.w_shape)
        return dY, dW, db, None, None


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
