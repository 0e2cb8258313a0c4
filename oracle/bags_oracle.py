"""CPU oracle for the BAGS head hot path -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline /
``--impl reference`` legs may import this module.  The product package
(``balancedgroupsoftmax_b200``) never imports it and has no CPU path.

It restates, in plain PyTorch (CPU, fp32 or fp64) + numpy, the reference's
algorithm for the path, function by function:

  fc_cls                  mmdet/models/bbox_heads/convfc_bbox_head.py:166
  sample_others           mmdet/models/bbox_heads/gs_bbox_head_with0.py:63-89
  remap_labels            gs_bbox_head_with0.py:91-112
  slice_preds             gs_bbox_head_with0.py:134-145
  cross_entropy           mmdet/models/losses/cross_entropy_loss.py:9-19
  weight_reduce_loss      mmdet/models/losses/utils.py:26-53
  bags_loss               gs_bbox_head_with0.py:147-171
  merge_score             gs_bbox_head_with0.py:239-273
  closed_form_grads       what autograd produces for the above

Parity pinning: the reference ships no tests / golden vectors for this path
(, §8c), so the oracle is pinned against the reference's OWN source
executed in place on CPU through ``oracle/ref_shim.py`` (tests/test_oracle_vs_reference.py,
run wherever /root/reference is reachable) and against the committed fixtures in
``tests/golden/`` that the same shim generated (tests/golden/make_golden.py).
The only known-answer numbers the reference holds near the path -- the
``weighted_loss`` doctest in losses/utils.py:66-83 -- are checked in
tests/test_oracle.py.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------- fc_cls
def fc_cls(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor]) -> torch.Tensor:
    """cls_score = x_cls @ W^T + b   (convfc_bbox_head.py:166, nn.Linear)."""
    return F.linear(x, weight, bias)


# --------------------------------------------------------------------------- label remap
def sample_others(bin_label: torch.Tensor, ratio: float) -> torch.Tensor:
    """gs_bbox_head_with0.py:63-89.  Uses numpy's GLOBAL RNG exactly like the
    reference (np.random.choice(bg_idx, (k,), replace=False)), so seeding
    np.random identically reproduces the reference's masks."""
    fg = torch.where(bin_label > 0, torch.ones_like(bin_label), torch.zeros_like(bin_label))
    fg_idx = fg.nonzero(as_tuple=True)[0]
    fg_num = fg_idx.shape[0]
    if fg_num == 0:
        return torch.zeros_like(bin_label)
    bg = 1 - fg
    bg_idx = bg.nonzero(as_tuple=True)[0]
    bg_num = bg_idx.shape[0]
    bg_sample_num = int(fg_num * ratio)
    if bg_sample_num >= bg_num:
        return torch.ones_like(bin_label)
    sample_idx = np.random.choice(bg_idx.cpu().numpy(), (bg_sample_num,), replace=False)
    fg = fg.clone()
    fg[torch.from_numpy(sample_idx)] = 1
    return fg


def remap_labels(labels: torch.Tensor, label2binlabel: torch.Tensor, ratio: float
                 ) -> Tuple[List[torch.Tensor], List[torch.Tensor], List[float]]:
    """gs_bbox_head_with0.py:91-112."""
    new_labels, new_weights, new_avg = [], [], []
    for i in range(label2binlabel.shape[0]):
        new_bin_label = label2binlabel[i][labels]
        if i < 1:
            weight = torch.ones_like(new_bin_label)
        else:
            weight = sample_others(new_bin_label, ratio)
        new_labels.append(new_bin_label)
        new_weights.append(weight)
        new_avg.append(max(torch.sum(weight).float().item(), 1.))
    return new_labels, new_weights, new_avg


def remap_labels_reweight(labels: torch.Tensor, label2binlabel: torch.Tensor, ratio: float,
                          cls_weights: Sequence[torch.Tensor]
                          ) -> Tuple[List[torch.Tensor], List[torch.Tensor], List[float]]:
    """Reweight head variant, gs_bbox_head_with0_reweight.py:57-109: like ``remap_labels``, but the sampled 0/1 weight
    of a foreground bin is multiplied by ``cls_weights[bin-1][in-bin label]`` (all zeros when the bin has no
    foreground RoI, :66-67), and the normaliser is max(sum of the products, 1)."""
    new_labels, new_weights, new_avg = [], [], []
    for i in range(label2binlabel.shape[0]):
        new_bin_label = label2binlabel[i][labels]
        if i < 1:
            weight = torch.ones_like(new_bin_label)
        else:
            weight = sample_others(new_bin_label, ratio)
            if (new_bin_label > 0).any():          # (the reference returns integer zeros before the multiply otherwise)
                weight = weight * cls_weights[i - 1][new_bin_label]
        new_labels.append(new_bin_label)
        new_weights.append(weight)
        new_avg.append(max(torch.sum(weight).float().item(), 1.))
    return new_labels, new_weights, new_avg


def slice_preds(cls_score: torch.Tensor, pred_slice: torch.Tensor) -> List[torch.Tensor]:
    """gs_bbox_head_with0.py:134-145."""
    return [cls_score.narrow(1, int(pred_slice[i, 0]), int(pred_slice[i, 1]))
            for i in range(pred_slice.shape[0])]


# --------------------------------------------------------------------------- loss
def weight_reduce_loss(loss, weight=None, reduction='mean', avg_factor=None):
    """losses/utils.py:26-53."""
    if weight is not None:
        loss = loss * weight
    if avg_factor is None:
        if reduction == 'mean':
            return loss.mean()
        if reduction == 'sum':
            return loss.sum()
        return loss
    if reduction == 'mean':
        return loss.sum() / avg_factor
    if reduction != 'none':
        raise ValueError('avg_factor can not be used with reduction="sum"')
    return loss


def cross_entropy(pred, label, weight=None, reduction='mean', avg_factor=None):
    """losses/cross_entropy_loss.py:9-19."""
    loss = F.cross_entropy(pred, label, reduction='none')
    if weight is not None:
        weight = weight.to(loss.dtype)
    return weight_reduce_loss(loss, weight=weight, reduction=reduction, avg_factor=avg_factor)


def bags_loss(cls_score: torch.Tensor, labels: torch.Tensor, label2binlabel: torch.Tensor,
              pred_slice: torch.Tensor, ratio: float = 8.0, loss_weight: float = 1.0,
              remapped=None) -> Dict[str, torch.Tensor]:
    """Classification part of GSBBoxHeadWith0.loss (gs_bbox_head_with0.py:157-171).

    ``remapped`` = (new_labels, new_weights, new_avgfactors) to reuse masks
    recorded elsewhere (e.g. from the reference shim); otherwise they are drawn
    here with numpy's global RNG like the reference does.
    """
    if remapped is None:
        remapped = remap_labels(labels, label2binlabel, ratio)
    new_labels, new_weights, new_avg = remapped
    new_preds = slice_preds(cls_score, pred_slice)
    losses = {}
    for i in range(len(new_labels)):
        losses['loss_cls_bin{}'.format(i)] = loss_weight * cross_entropy(
            new_preds[i], new_labels[i], new_weights[i], reduction='mean', avg_factor=new_avg[i])
    return losses


def closed_form_grads(x, weight, bias, labels, label2binlabel, pred_slice, remapped,
                      gout: Optional[Sequence[float]] = None):
    """dz, dW, db, dX of sum_g gout[g] * loss_g by the closed form
        dz[n, s_g + j] = gout_g * w_g[n]/avg_g * (softmax(z[n, slice_g])[j] - [j == t_g[n]])
    Independent of autograd, so tests can cross-check both."""
    new_labels, new_weights, new_avg = remapped
    z = fc_cls(x, weight, bias)
    dz = torch.zeros_like(z)
    G = pred_slice.shape[0]
    for g in range(G):
        s, l = int(pred_slice[g, 0]), int(pred_slice[g, 1])
        p = torch.softmax(z[:, s:s + l], dim=1)
        onehot = F.one_hot(new_labels[g], l).to(z.dtype)
        coef = new_weights[g].to(z.dtype) / new_avg[g]
        if gout is not None:
            coef = coef * float(gout[g])
        dz[:, s:s + l] = coef[:, None] * (p - onehot)
    dW = dz.t() @ x
    db = dz.sum(0)
    dX = dz @ weight
    return dz, dW, db, dX


# --------------------------------------------------------------------------- inference
def merge_score(cls_score: torch.Tensor, pred_slice: torch.Tensor,
                fg_splits: Sequence[torch.Tensor], num_classes: int) -> torch.Tensor:
    """gs_bbox_head_with0.py:239-273 (the variant get_det_bboxes uses)."""
    num_proposals = cls_score.shape[0]
    new_preds = slice_preds(cls_score, pred_slice)
    new_scores = [F.softmax(pred, dim=1) for pred in new_preds]
    bg_score = new_scores[0]
    fg_score = new_scores[1:]
    fg_merge = torch.zeros((num_proposals, num_classes), dtype=cls_score.dtype)
    merge = torch.zeros((num_proposals, num_classes), dtype=cls_score.dtype)
    for i, split in enumerate(fg_splits):
        fg_merge[:, split] = fg_score[i][:, 1:]
    weight = bg_score.narrow(1, 1, 1)
    fg_merge = weight * fg_merge
    merge[:, 0] = bg_score[:, 0]
    merge[:, 1:] = fg_merge[:, 1:]
    return merge


# --------------------------------------------------------------------------- full step (CPU baseline)
def head_step(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, labels: torch.Tensor,
              label2binlabel: torch.Tensor, pred_slice: torch.Tensor, ratio: float = 8.0,
              need_dx: bool = True):
    """fc_cls -> BAGS loss -> sum -> backward (dW, db, dX): the unit bench.py's
    cpu_baseline times.  Returns (losses dict, dW, db, dX-or-None)."""
    x = x.detach().requires_grad_(need_dx)
    w = weight.detach().requires_grad_(True)
    b = bias.detach().requires_grad_(True)
    z = fc_cls(x, w, b)
    losses = bags_loss(z, labels, label2binlabel, pred_slice, ratio)
    total = sum(losses.values())
    total.backward()
    return losses, w.grad, b.grad, (x.grad if need_dx else None)


# ---------------------------------------------------------------------------------------------------
# test-time consumer of the merged scores: per-class NMS
# ---------------------------------------------------------------------------------------------------
def iou_plus1_fp32(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """devIoU of the reference op (mmdet/ops/nms/src/nms_kernel.cu:13-21) in its own fp32 arithmetic and operation
    order: "+1" widths, CUDA's float max/min (fmaxf/fminf: a NaN operand yields the other one).  a, b [..., 4]
    broadcast; every step rounds to fp32 once, so with integer coordinates below 2^11 the division is the only
    rounding."""
    a = np.asarray(a, dtype=np.float32)
    b = np.asarray(b, dtype=np.float32)
    one, zero = np.float32(1), np.float32(0)
    with np.errstate(invalid='ignore', divide='ignore', over='ignore'):
        left, right = np.fmax(a[..., 0], b[..., 0]), np.fmin(a[..., 2], b[..., 2])
        top, bottom = np.fmax(a[..., 1], b[..., 1]), np.fmin(a[..., 3], b[..., 3])
        width, height = np.fmax(right - left + one, zero), np.fmax(bottom - top + one, zero)
        inter = width * height
        sa = (a[..., 2] - a[..., 0] + one) * (a[..., 3] - a[..., 1] + one)
        sb = (b[..., 2] - b[..., 0] + one) * (b[..., 3] - b[..., 1] + one)
        return inter / (sa + sb - inter)


def greedy_keep(boxes: np.ndarray, iou_thr: float) -> np.ndarray:
    """The reference op's greedy scan over boxes already in visiting order: box j is removed when a box i < j that
    is still alive has IoU(i, j) > fp32(iou_thr) (nms_kernel.cu:60,117-126).  -> bool keep [n]."""
    boxes = np.asarray(boxes, dtype=np.float32).reshape(-1, 4)
    n = boxes.shape[0]
    thr = np.float32(iou_thr)
    removed = np.zeros(n, dtype=bool)
    for i in range(n):
        if not removed[i] and i + 1 < n:
            removed[i + 1:] |= iou_plus1_fp32(boxes[i], boxes[i + 1:]) > thr
    return ~removed


def nms_plus1(dets: torch.Tensor, iou_thr: float) -> Tuple[torch.Tensor, torch.Tensor]:
    """Greedy NMS with the reference op's conventions (mmdet/ops/nms/src/nms_kernel.cu:13-21,60,76-78,127-130):
    boxes visited in descending score order, fp32 IoU with "+1" widths (iou_plus1_fp32), a box is dropped when its
    IoU with a kept box is > fp32(iou_thr); the kept rows are returned in ASCENDING index order, as the op returns
    them.  Equal scores are visited lower index first (the op's unstable sort leaves their order open).
    dets [n,5] (x1,y1,x2,y2,score) -> (dets[inds], inds)."""
    if dets.shape[0] == 0:
        return dets, dets.new_zeros(0, dtype=torch.long)
    d = dets.detach().float().cpu().numpy()
    order = np.argsort(-d[:, 4], kind='stable')
    keep = greedy_keep(d[order, :4], iou_thr)
    inds = torch.as_tensor(np.sort(order[keep]).astype(np.int64))
    return dets[inds], inds


def multiclass_nms(multi_bboxes: torch.Tensor, multi_scores: torch.Tensor, score_thr: float, iou_thr: float,
                   max_num: int = -1, nms_op=None) -> Tuple[torch.Tensor, torch.Tensor]:
    """mmdet/core/post_processing/bbox_nms.py:6-66 restated (nms_cfg = dict(type='nms', iou_thr=...)): column 0 of the
    scores is background and ignored; per class keep score > score_thr, NMS, label = class - 1; concatenate in class
    order; ``if n > max_num`` sort by score and keep ``[:max_num]`` -- including the reference's behaviour for
    max_num = -1 (n > -1 always holds, so the lowest-scored detection is dropped).  ``score > score_thr`` compares in
    the scores' own dtype.  ``nms_op(dets, iou_thr) -> (dets, inds)`` is the per-class NMS (default nms_plus1; the
    reference's compiled op through oracle.ref_nms.nms_wrapper_op plugs in here)."""
    nms_op = nms_plus1 if nms_op is None else nms_op
    num_classes = multi_scores.shape[1]
    bboxes, labels = [], []
    for i in range(1, num_classes):
        cls_inds = multi_scores[:, i] > score_thr
        if not cls_inds.any():
            continue
        _b = multi_bboxes[cls_inds, :] if multi_bboxes.shape[1] == 4 else multi_bboxes[cls_inds, i * 4:(i + 1) * 4]
        cls_dets, _ = nms_op(torch.cat([_b, multi_scores[cls_inds, i][:, None]], 1), iou_thr)
        bboxes.append(cls_dets)
        labels.append(multi_bboxes.new_full((cls_dets.shape[0],), i - 1, dtype=torch.long))
    if not bboxes:
        return multi_bboxes.new_zeros((0, 5)), multi_bboxes.new_zeros((0,), dtype=torch.long)
    bboxes, labels = torch.cat(bboxes), torch.cat(labels)
    if bboxes.shape[0] > max_num:
        _, inds = bboxes[:, -1].sort(descending=True)
        inds = inds[:max_num]
        bboxes, labels = bboxes[inds], labels[inds]
    return bboxes, labels
