"""Loss modules the BAGS head's config blocks name.

``CrossEntropyLoss`` / ``SmoothL1Loss`` keep the constructor and call contract of
mmdet/models/losses/cross_entropy_loss.py:64-103 and smooth_l1_loss.py:20-45
(``loss_weight * reduce(elementwise * weight) / avg_factor``, reduction semantics
of losses/utils.py:26-53) so ``loss_bin`` / ``loss_cls`` / ``loss_bbox`` dicts
build unchanged.

They are NOT the hot path: inside ``GSBBoxHeadWith0.loss`` the five per-bin
``CrossEntropyLoss`` calls of the reference (gs_bbox_head_with0.py:164-171) are
replaced by one fused CUDA call (ops.GroupSoftmaxFunction); the per-bin modules
only contribute their ``loss_weight``.  ``SmoothL1Loss`` (<= 128x4 values per
image) stays plain PyTorch, as scopes it.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from .registry import LOSSES, register


def _reduce(loss, weight, reduction, avg_factor):
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


class CrossEntropyLoss(nn.Module):

    def __init__(self, use_sigmoid=False, use_mask=False, reduction='mean', loss_weight=1.0):
        super().__init__()
        assert (use_sigmoid is False) or (use_mask is False)
        self.use_sigmoid = use_sigmoid
        self.use_mask = use_mask
        self.reduction = reduction
        self.loss_weight = loss_weight

    def forward(self, cls_score, label, weight=None, avg_factor=None, reduction_override=None, **kwargs):
        assert reduction_override in (None, 'none', 'mean', 'sum')
        reduction = reduction_override if reduction_override else self.reduction
        if self.use_mask:
            raise NotImplementedError('mask cross-entropy is outside the BAGS head path')
        if weight is not None:
            weight = weight.float()
        if self.use_sigmoid:
            if cls_score.dim() != label.dim():
                onehot = label.new_zeros((label.size(0), cls_score.size(-1)))
                inds = torch.nonzero(label >= 1, as_tuple=False).squeeze(-1)
                if inds.numel() > 0:
                    onehot[inds, label[inds] - 1] = 1
                if weight is not None:
                    weight = weight.view(-1, 1).expand(weight.size(0), cls_score.size(-1))
                label = onehot
            loss = F.binary_cross_entropy_with_logits(cls_score, label.float(), weight, reduction='none')
            return self.loss_weight * _reduce(loss, None, reduction, avg_factor)
        loss = F.cross_entropy(cls_score, label, reduction='none')
        return self.loss_weight * _reduce(loss, weight, reduction, avg_factor)


def accuracy(pred, target, topk=1):
    """Top-k accuracy in percent, mmdet/models/losses/accuracy.py:4-21 (``losses['acc']`` of BBoxHead.loss)."""
    assert isinstance(topk, (int, tuple))
    return_single = isinstance(topk, int)
    if return_single:
        topk = (topk, )
    maxk = max(topk)
    _, pred_label = pred.topk(maxk, dim=1)
    pred_label = pred_label.t()
    correct = pred_label.eq(target.view(1, -1).expand_as(pred_label))
    res = [correct[:k].reshape(-1).float().sum(0, keepdim=True).mul_(100.0 / pred.size(0)) for k in topk]
    return res[0] if return_single else res


class SmoothL1Loss(nn.Module):

    def __init__(self, beta=1.0, reduction='mean', loss_weight=1.0):
        super().__init__()
        assert beta > 0
        self.beta = beta
        self.reduction = reduction
        self.loss_weight = loss_weight

    def forward(self, pred, target, weight=None, avg_factor=None, reduction_override=None, **kwargs):
        assert reduction_override in (None, 'none', 'mean', 'sum')
        reduction = reduction_override if reduction_override else self.reduction
        assert pred.size() == target.size() and target.numel() > 0
        diff = torch.abs(pred - target)
        loss = torch.where(diff < self.beta, 0.5 * diff * diff / self.beta, diff - 0.5 * self.beta)
        return self.loss_weight * _reduce(loss, weight, reduction, avg_factor)


register(LOSSES, CrossEntropyLoss)
register(LOSSES, SmoothL1Loss)
