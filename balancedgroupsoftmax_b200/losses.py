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

With ``use_mask=True`` ``CrossEntropyLoss`` is the reference's ``mask_cross_entropy`` on materialised mask logits;
the mask heads (mask_head.py) fuse it into conv_logits instead (ops.MaskBCEFunction).

``FocalLoss`` keeps the contract of mmdet/models/losses/focal_loss.py:46-88,
quirks included; on plain logits it restates the reference's op in torch, and
``ReweightBBoxHead`` fuses it into fc_cls (ops.SigmoidFocalFunction).
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


def mask_cross_entropy(pred, target, label, reduction='mean', avg_factor=None):
    """The mask loss of FCNMaskHead on materialised logits ``pred`` [P, classes, H, W]: each RoI p is scored on its
    own channel label[p] only, with a BCE-with-logits against ``target`` [P, H, W] averaged over all P * H * W pixels;
    returned as a [1] tensor.  Only reduction 'mean' without avg_factor exists, as in mmdet.  Heads with
    ``MaskPredHandle`` compute the same loss fused into conv_logits instead (ops.MaskBCEFunction)."""
    assert reduction == 'mean' and avg_factor is None, 'the mask loss supports reduction="mean" without avg_factor only'
    own_channel = pred[torch.arange(pred.shape[0], device=pred.device), label]
    return F.binary_cross_entropy_with_logits(own_channel, target, reduction='mean').reshape(1)


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
            return self.loss_weight * mask_cross_entropy(cls_score, label, weight, reduction=reduction,
                                                         avg_factor=avg_factor, **kwargs)
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


# FocalLoss.forward one-hot encodes its labels with this literal width, whatever the head's num_classes
FOCAL_ONE_HOT_CLASSES = 1231


def focal_targets(labels: torch.Tensor, num_rows: int) -> torch.Tensor:
    """The per-row targets the sigmoid focal-loss op sees under FocalLoss.forward (focal_loss.py:73-74): it is handed
    F.one_hot(labels, 1231) and reads the first ``num_rows`` entries of its flattened buffer, so
    t[n] = 1 if labels[n // 1231] == n % 1231 else 0 (int64, on the labels' device, no host sync).  Unlike F.one_hot
    it does not check the labels' range: a label outside [0, 1231) simply matches nothing."""
    n = torch.arange(num_rows, device=labels.device)
    return (labels.reshape(-1)[n // FOCAL_ONE_HOT_CLASSES] == n % FOCAL_ONE_HOT_CLASSES).to(torch.int64)


def sigmoid_focal_elementwise(z, t, gamma, alpha, with_grad=False):
    """The focal-loss op (sigmoid_focal_loss_cuda.cu:23-96) restated in torch, in z's dtype: the per-element loss
    [N, C] and, with ``with_grad``, the op's analytic gradient (:79-93).  Column d of row n is positive when
    t[n] == d + 1 and negative when t[n] >= 0 otherwise; rows with t < 0 are 0."""
    t = t.reshape(-1, 1).to(torch.int32)            # the op reads `int t = targets[n]`
    d = torch.arange(z.shape[1], device=z.device, dtype=torch.int32)[None, :]
    c1 = (t == d + 1).to(z.dtype)
    c2 = ((t >= 0) & (t != d + 1)).to(z.dtype)
    p = 1. / (1. + torch.exp(-z))
    logp = torch.log(p.clamp_min(torch.finfo(torch.float32).tiny))
    nonneg = (z >= 0).to(z.dtype)
    log1m = -z * nonneg - torch.log(1. + torch.exp(z - 2 * z * nonneg))
    pos_w, neg_w = torch.pow(1 - p, gamma), torch.pow(p, gamma)
    loss = -c1 * pos_w * logp * alpha - c2 * neg_w * log1m * (1 - alpha)
    if not with_grad:
        return loss
    grad = -c1 * pos_w * (1 - p - p * gamma * logp) * alpha - c2 * neg_w * (log1m * (1 - p) * gamma - p) * (1 - alpha)
    return loss, grad


class _SigmoidFocalOp(torch.autograd.Function):
    """The op's forward / backward pair on materialised logits: the backward is its analytic gradient, not autograd of
    the forward."""

    @staticmethod
    def forward(ctx, z, t, gamma, alpha):
        loss, grad = sigmoid_focal_elementwise(z, t, gamma, alpha, with_grad=True)
        ctx.save_for_backward(grad)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_loss):
        (grad,) = ctx.saved_tensors
        return grad * d_loss, None, None, None


class FocalLoss(nn.Module):
    """FocalLoss of mmdet/models/losses/focal_loss.py:46-88 (sigmoid only), quirks included: the targets are the first N
    entries of F.one_hot(labels, 1231) (``focal_targets``), ``weight`` [N] is broadcast over the columns, and the
    caller's avg_factor is replaced by N * 1231 -- so 'mean' is sum / (N * 1231) and 'sum' raises.  Here the normaliser
    comes from the shape, without the reference's host sync.

    This module is the materialised route (plain logits on CPU or GPU, e.g. SharedFCBBoxHead); ReweightBBoxHead
    runs fc_cls and this loss in one fused kernel instead (ops.SigmoidFocalFunction)."""

    def __init__(self, use_sigmoid=True, gamma=2.0, alpha=0.25, reduction='mean', loss_weight=1.0):
        super().__init__()
        assert use_sigmoid is True, 'Only sigmoid focal loss supported now.'
        self.use_sigmoid = use_sigmoid
        self.gamma = gamma
        self.alpha = alpha
        self.reduction = reduction
        self.loss_weight = loss_weight

    def forward(self, pred, target, weight=None, avg_factor=None, reduction_override=None):
        assert reduction_override in (None, 'none', 'mean', 'sum')
        reduction = reduction_override if reduction_override else self.reduction
        avg_factor = max(float(target.numel() * FOCAL_ONE_HOT_CLASSES), 1.)
        loss = _SigmoidFocalOp.apply(pred, focal_targets(target, pred.shape[0]), float(self.gamma), float(self.alpha))
        if weight is not None:
            weight = weight.view(-1, 1)
        return self.loss_weight * _reduce(loss, weight, reduction, avg_factor)


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
register(LOSSES, FocalLoss)
