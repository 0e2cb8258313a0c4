"""GSBBoxHeadWith0 -- the Balanced Group Softmax RoI head behind the reference's BBoxHead API.

Reference surface mirrored here (constructor kwargs, attributes, state-dict keys, method
signatures and returned dict keys are identical so configs/bags/*.py blocks build unchanged):

    BBoxHead            mmdet/models/bbox_heads/bbox_head.py:13-239
    ConvFCBBoxHead      mmdet/models/bbox_heads/convfc_bbox_head.py:8-168
    SharedFCBBoxHead    mmdet/models/bbox_heads/convfc_bbox_head.py:171-185
    GSBBoxHeadWith0     mmdet/models/bbox_heads/gs_bbox_head_with0.py:14-380

What differs is the execution of the hot path:

  * ``fc_cls`` (convfc_bbox_head.py:166) runs on wgmma tensor cores through the C ABI
    (``bags_linear_act_fwd``) instead of cuBLAS SGEMM;
  * ``_remap_labels`` + ``_sample_others`` + ``_slice_preds`` + 5x ``CrossEntropyLoss``
    (gs_bbox_head_with0.py:63-171) -- ~70 small kernels and >=15 host syncs per call in the
    reference -- become one sampler launch plus ONE fused forward call and ONE fused backward
    call (``ops.GroupSoftmaxFunction``); nothing synchronises with the host;
  * in training ``forward`` returns a lazy ``ClsScoreHandle`` instead of materialised logits:
    ``loss`` consumes it to launch the fused kernels; any other use materialises it;
  * ``_merge_score`` (gs_bbox_head_with0.py:239-273) is one kernel (``bags_merge_scores``).

The shared FCs, ``fc_reg`` and the SmoothL1 box loss are neighbours of the path and stay
plain ``nn.Linear`` / PyTorch, exactly as scopes them -- unless the execution key ``fuse_bbox_loss`` is set: then
``forward`` returns a lazy ``BoxPredHandle`` for the class-specific ``bbox_pred`` and the box loss computes only the
positive RoIs' four deltas (``ops.SmoothL1BoxFunction``), with no host sync.
"""
from __future__ import annotations

import os
import pickle
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn.modules.utils import _pair

from . import ops
from .fp16 import auto_fp16, force_fp32
from .losses import CrossEntropyLoss, FocalLoss, SmoothL1Loss, accuracy  # noqa: F401  (registers them)
from .losses import FOCAL_ONE_HOT_CLASSES, focal_targets
from .registry import HEADS, build_loss, register
from .tables import GroupTables, load_reference_files


# --------------------------------------------------------------------------- mmdet.core glue
def _mmdet_core(name):
    try:  # pragma: no cover - mmdet is not installable in the build image
        import mmdet.core as core
        return getattr(core, name)
    except Exception:
        return None


def bbox2delta(proposals, gt, means=(0, 0, 0, 0), stds=(1, 1, 1, 1)):
    """Box encoding of the regression targets; same maths as mmdet/core/bbox/transforms.py:6-31 (legacy "+1" widths)."""
    assert proposals.size() == gt.size()
    proposals, gt = proposals.float(), gt.float()
    px = (proposals[..., 0] + proposals[..., 2]) * 0.5
    py = (proposals[..., 1] + proposals[..., 3]) * 0.5
    pw = proposals[..., 2] - proposals[..., 0] + 1.0
    ph = proposals[..., 3] - proposals[..., 1] + 1.0
    gx = (gt[..., 0] + gt[..., 2]) * 0.5
    gy = (gt[..., 1] + gt[..., 3]) * 0.5
    gw = gt[..., 2] - gt[..., 0] + 1.0
    gh = gt[..., 3] - gt[..., 1] + 1.0
    deltas = torch.stack([(gx - px) / pw, (gy - py) / ph, torch.log(gw / pw), torch.log(gh / ph)], dim=-1)
    means = deltas.new_tensor(means).unsqueeze(0)
    stds = deltas.new_tensor(stds).unsqueeze(0)
    return deltas.sub_(means).div_(stds)


def bbox_target(pos_bboxes_list, neg_bboxes_list, pos_gt_bboxes_list, pos_gt_labels_list, cfg, reg_classes=1,
                target_means=(.0, .0, .0, .0), target_stds=(1.0, 1.0, 1.0, 1.0), concat=True):
    """Per-image RoI targets, restating mmdet/core/bbox/bbox_target.py:7-63: positives first (their gt label, weight
    ``cfg.pos_weight`` or 1, encoded box target, box weight 1), negatives after (label 0, weight 1).  This is the
    producer of the ``labels`` vector the BAGS path consumes (its layout -- positives first in every image's block --
    is what bench.py's synthetic labels imitate).  ``reg_classes`` is accepted and unused, as in the reference."""
    pw = cfg['pos_weight'] if isinstance(cfg, dict) else cfg.pos_weight
    outs = ([], [], [], [])
    for pos_bboxes, neg_bboxes, pos_gt_bboxes, pos_gt_labels in zip(pos_bboxes_list, neg_bboxes_list,
                                                                      pos_gt_bboxes_list, pos_gt_labels_list):
        num_pos, num_neg = pos_bboxes.size(0), neg_bboxes.size(0)
        n = num_pos + num_neg
        labels = pos_bboxes.new_zeros(n, dtype=torch.long)
        label_weights = pos_bboxes.new_zeros(n)
        bbox_targets = pos_bboxes.new_zeros(n, 4)
        bbox_weights = pos_bboxes.new_zeros(n, 4)
        if num_pos > 0:
            labels[:num_pos] = pos_gt_labels
            label_weights[:num_pos] = 1.0 if pw <= 0 else pw
            bbox_targets[:num_pos, :] = bbox2delta(pos_bboxes, pos_gt_bboxes, target_means, target_stds)
            bbox_weights[:num_pos, :] = 1
        if num_neg > 0:
            label_weights[-num_neg:] = 1.0
        for o, v in zip(outs, (labels, label_weights, bbox_targets, bbox_weights)):
            o.append(v)
    if concat:
        return tuple(torch.cat(o, 0) for o in outs)
    return outs


def delta2bbox(rois, deltas, means=(0, 0, 0, 0), stds=(1, 1, 1, 1), max_shape=None, wh_ratio_clip=16 / 1000):
    """Box decoding used by get_det_bboxes / regress_by_class; same maths as
    mmdet/core/bbox/transforms.py:34-111 (consumer of the path, plain PyTorch)."""
    ext = _mmdet_core('delta2bbox')
    if ext is not None:  # pragma: no cover
        return ext(rois, deltas, means, stds, max_shape, wh_ratio_clip)
    reps = deltas.size(1) // 4
    d = deltas * deltas.new_tensor(stds).repeat(1, reps) + deltas.new_tensor(means).repeat(1, reps)
    max_ratio = abs(float(np.log(wh_ratio_clip)))
    dx, dy = d[:, 0::4], d[:, 1::4]
    dw = d[:, 2::4].clamp(min=-max_ratio, max=max_ratio)
    dh = d[:, 3::4].clamp(min=-max_ratio, max=max_ratio)
    px = ((rois[:, 0] + rois[:, 2]) * 0.5).unsqueeze(1)
    py = ((rois[:, 1] + rois[:, 3]) * 0.5).unsqueeze(1)
    pw = (rois[:, 2] - rois[:, 0] + 1.0).unsqueeze(1)
    ph = (rois[:, 3] - rois[:, 1] + 1.0).unsqueeze(1)
    gw, gh = pw * dw.exp(), ph * dh.exp()
    gx, gy = px + pw * dx, py + ph * dy
    x1, y1 = gx - gw * 0.5 + 0.5, gy - gh * 0.5 + 0.5
    x2, y2 = gx + gw * 0.5 - 0.5, gy + gh * 0.5 - 0.5
    if max_shape is not None:
        x1 = x1.clamp(min=0, max=max_shape[1] - 1)
        y1 = y1.clamp(min=0, max=max_shape[0] - 1)
        x2 = x2.clamp(min=0, max=max_shape[1] - 1)
        y2 = y2.clamp(min=0, max=max_shape[0] - 1)
    return torch.stack([x1, y1, x2, y2], dim=-1).view_as(deltas)


# --------------------------------------------------------------------------- lazy projections
class _LazyHandle(object):
    """A projection a training ``forward`` records instead of launching, so that ``loss`` can fuse it with its loss.
    Subclasses give ``shape``, ``device`` and ``tensor()`` (the materialised, autograd-connected output); indexing, any
    other attribute and any torch function handed a handle see ``tensor()``, so every other consumer keeps working."""

    def size(self, dim=None):
        return self.shape if dim is None else self.shape[dim]

    def dim(self):
        return 2

    def __getattr__(self, name):  # argmax, float, detach, ... -> materialise
        if name.startswith('_'):
            raise AttributeError(name)
        return getattr(self.tensor(), name)

    def __getitem__(self, idx):
        return self.tensor()[idx]

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        """torch.cat([cls_score, ...]), torch.softmax(cls_score, 1), F.cross_entropy(cls_score, ...) ...: any torch
        function handed a handle sees the materialised tensor (callers written for the reference's plain tensor)."""
        def unwrap(a):
            if isinstance(a, _LazyHandle):
                return a.tensor()
            if isinstance(a, (list, tuple)):
                return type(a)(unwrap(v) for v in a)
            if isinstance(a, dict):
                return {k: unwrap(v) for k, v in a.items()}
            return a
        return func(*unwrap(tuple(args)), **unwrap(kwargs or {}))


class ClsScoreHandle(_LazyHandle):
    """What ``GSBBoxHeadWith0.forward`` returns for ``cls_score`` in training mode.

    It records the fc_cls input instead of launching the projection, so that ``loss`` can run
    the fused forward (GEMM + grouped softmax-CE) without a logits round trip through autograd.
    ``tensor()`` (or any tensor attribute access) materialises real logits with the same
    wgmma kernel, autograd-connected, so every other consumer keeps working.
    """

    def __init__(self, head: 'GSBBoxHeadWith0', x_cls: torch.Tensor):
        self._head = head
        self.x_cls = x_cls
        self._logits = None

    @property
    def shape(self):
        return torch.Size((self.x_cls.shape[0], self._head.fc_cls.out_features))

    @property
    def device(self):
        return self.x_cls.device

    def tensor(self) -> torch.Tensor:
        if self._logits is None:
            self._logits = self._head._fc_cls_logits(self.x_cls)
        return self._logits


class BoxPredHandle(_LazyHandle):
    """What a head with ``fuse_bbox_loss`` returns for the class-specific ``bbox_pred`` in training mode.

    It records the fc_reg input, so that ``loss`` can compute only the four box deltas of each positive RoI inside its
    SmoothL1 loss (``ops.SmoothL1BoxFunction``) instead of the [N, 4 * num_classes] projection.  ``tensor()`` (or any
    tensor attribute access) materialises that projection through ``_fc_reg``, autograd-connected.
    """

    def __init__(self, head: 'NativeFcClsHead', x_reg: torch.Tensor):
        self._head = head
        self.x_reg = x_reg
        self._pred = None

    @property
    def shape(self):
        return torch.Size((self.x_reg.shape[0], self._head.fc_reg.out_features))

    @property
    def device(self):
        return self.x_reg.device

    def tensor(self) -> torch.Tensor:
        if self._pred is None:
            self._pred = self._head._fc_reg(self.x_reg)
        return self._pred


def _as_tensor(cls_score):
    return cls_score.tensor() if isinstance(cls_score, ClsScoreHandle) else cls_score


class FcClsFunction(torch.autograd.Function):
    """Materialised logits = x W^T + b on the wgmma GEMM (bags_linear_act_fwd); backward reuses bags_bwd."""

    @staticmethod
    def forward(ctx, x, weight, bias, compute_dtype):
        xin, win = x.detach(), weight.detach()
        if compute_dtype == torch.bfloat16:
            xc = xin if xin.dtype == torch.bfloat16 else ops.cast_bf16(ops._row_major(xin.float()))
            wc = win if win.dtype == torch.bfloat16 else ops.cast_bf16(ops._row_major(win.float()))
        else:
            xc, wc = ops._row_major(xin.float()), ops._row_major(win.float())
        b32 = None if bias is None else bias.detach().float().contiguous()
        out = ops.linear_fwd(xc, wc, b32)
        ctx.save_for_backward(xc, wc)
        ctx.meta = (x.dtype, weight.dtype, None if bias is None else bias.dtype)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        xc, wc = ctx.saved_tensors
        xd, wd, bd = ctx.meta
        N, Cc = grad_out.shape
        ldd = ops.pad_cols(Cc)
        dz = torch.zeros((N, ldd), dtype=xc.dtype, device=xc.device)
        dz[:, :Cc] = grad_out
        colsum = grad_out.float().sum(0, keepdim=True)
        dW, db, dX = ops.fused_bwd(dz, xc, wc, None, ops._single_slice_tables(Cc, xc.device), colsum,
                                   need_dw=ctx.needs_input_grad[1], need_db=ctx.needs_input_grad[2] and bd is not None,
                                   need_dx=ctx.needs_input_grad[0])
        return (None if dX is None else dX.to(xd), None if dW is None else dW.to(wd),
                None if db is None else db.to(bd), None)


# --------------------------------------------------------------------------- base heads
class BBoxHead(nn.Module):
    """Simplest RoI head (API contract of mmdet/models/bbox_heads/bbox_head.py:13-239)."""

    def __init__(self, with_avg_pool=False, with_cls=True, with_reg=True, roi_feat_size=7, in_channels=256,
                 num_classes=81, target_means=[0., 0., 0., 0.], target_stds=[0.1, 0.1, 0.2, 0.2],
                 reg_class_agnostic=False,
                 loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0),
                 loss_bbox=dict(type='SmoothL1Loss', beta=1.0, loss_weight=1.0)):
        super().__init__()
        assert with_cls or with_reg
        self.with_avg_pool = with_avg_pool
        self.with_cls = with_cls
        self.with_reg = with_reg
        self.roi_feat_size = _pair(roi_feat_size)
        self.roi_feat_area = self.roi_feat_size[0] * self.roi_feat_size[1]
        self.in_channels = in_channels
        self.num_classes = num_classes
        self.target_means = target_means
        self.target_stds = target_stds
        self.reg_class_agnostic = reg_class_agnostic
        self.fp16_enabled = False

        self.loss_cls = build_loss(loss_cls)
        self.loss_bbox = build_loss(loss_bbox)

        in_channels = self.in_channels
        if self.with_avg_pool:
            self.avg_pool = nn.AvgPool2d(self.roi_feat_size)
        else:
            in_channels *= self.roi_feat_area
        if self.with_cls:
            self.fc_cls = nn.Linear(in_channels, num_classes)
        if self.with_reg:
            self.fc_reg = nn.Linear(in_channels, 4 if reg_class_agnostic else 4 * num_classes)
        self.debug_imgs = None

    def init_weights(self):
        if self.with_cls:
            nn.init.normal_(self.fc_cls.weight, 0, 0.01)
            nn.init.constant_(self.fc_cls.bias, 0)
        if self.with_reg:
            nn.init.normal_(self.fc_reg.weight, 0, 0.001)
            nn.init.constant_(self.fc_reg.bias, 0)

    def get_target(self, sampling_results, gt_bboxes, gt_labels, rcnn_train_cfg):
        """(labels, label_weights, bbox_targets, bbox_weights) of the sampled RoIs (bbox_head.py:80-96).  Uses
        mmdet's ``bbox_target`` inside an mmdetection checkout, the restatement above otherwise (identical results)."""
        fn = _mmdet_core('bbox_target') or bbox_target
        reg_classes = 1 if self.reg_class_agnostic else self.num_classes
        return fn([r.pos_bboxes for r in sampling_results], [r.neg_bboxes for r in sampling_results],
                  [r.pos_gt_bboxes for r in sampling_results], [r.pos_gt_labels for r in sampling_results],
                  rcnn_train_cfg, reg_classes, target_means=self.target_means, target_stds=self.target_stds)

    @force_fp32(apply_to=('cls_score', 'bbox_pred'))
    def loss(self, cls_score, bbox_pred, labels, label_weights, bbox_targets, bbox_weights, reduction_override=None):
        """bbox_head.py:97-129: softmax CE over all classes (sample weights ``label_weights``), its top-1 ``acc`` and
        the box loss.  The normaliser max(#(label_weights > 0), 1) stays on the device (no host sync)."""
        losses = dict()
        if cls_score is not None:
            losses['loss_cls'] = self._cls_loss(cls_score, labels, label_weights, label_weights, reduction_override)
            losses['acc'] = accuracy(_as_tensor(cls_score), labels)
        if bbox_pred is not None:
            losses['loss_bbox'] = self._bbox_loss(bbox_pred, labels, bbox_targets, bbox_weights, reduction_override)
        return losses

    def _cls_loss(self, cls_score, labels, weight, label_weights, reduction_override):
        """loss_cls over materialised logits with avg_factor = max(#(label_weights > 0), 1) (None for 'sum')."""
        avg = (label_weights > 0).sum(dtype=torch.float32).clamp_min(1.0)
        return self.loss_cls(_as_tensor(cls_score), labels, weight,
                             avg_factor=None if reduction_override == 'sum' else avg,
                             reduction_override=reduction_override)

    def _nms(self, bboxes, scores, cfg):
        """multiclass_nms (mmdet/core/post_processing/bbox_nms.py): the native class-aware hard NMS, mmdet's own
        function for the other NMS types."""
        nms_cfg = _cfg_get(cfg, 'nms')
        nms_type = _cfg_get(nms_cfg, 'type', 'nms')
        if nms_type == 'nms' and os.environ.get('BAGS_NMS_NATIVE', '1') != '0':
            # hard NMS (every configs/bags/* file): the device-side class-aware NMS -- one sort, one kernel, one sync
            # instead of the reference's Python loop over 1230 classes (bbox_nms.py:34-54)
            return ops.multiclass_nms(bboxes, scores, float(_cfg_get(cfg, 'score_thr')),
                                      float(_cfg_get(nms_cfg, 'iou_thr')), int(_cfg_get(cfg, 'max_per_img')))
        multiclass_nms = _mmdet_core('multiclass_nms')
        if multiclass_nms is None:
            raise NotImplementedError('nms type %r is not implemented natively (hard NMS is); install mmdetection v1.x '
                                      'for soft-NMS' % (nms_type,))
        return multiclass_nms(bboxes, scores, cfg.score_thr, cfg.nms, cfg.max_per_img)

    @force_fp32(apply_to=('cls_score', 'bbox_pred'))
    def get_det_bboxes(self, rois, cls_score, bbox_pred, img_shape, scale_factor, rescale=False, cfg=None):
        """bbox_head.py:131-168: softmax over all classes, box decoding, class-aware NMS."""
        if isinstance(cls_score, list):
            cls_score = sum(_as_tensor(c) for c in cls_score) / float(len(cls_score))
        scores = F.softmax(_as_tensor(cls_score), dim=1) if cls_score is not None else None
        bboxes = self._decode(rois, bbox_pred, img_shape, scale_factor, rescale)
        if cfg is None:
            return bboxes, scores
        return self._nms(bboxes, scores, cfg)

    def _bbox_loss(self, bbox_pred, labels, bbox_targets, bbox_weights, reduction_override):
        pos_inds = labels > 0
        if self.reg_class_agnostic:
            pos_bbox_pred = bbox_pred.view(bbox_pred.size(0), 4)[pos_inds]
        else:
            pos_bbox_pred = bbox_pred.view(bbox_pred.size(0), -1, 4)[pos_inds, labels[pos_inds]]
        return self.loss_bbox(pos_bbox_pred, bbox_targets[pos_inds], bbox_weights[pos_inds],
                              avg_factor=bbox_targets.size(0), reduction_override=reduction_override)

    def _decode(self, rois, bbox_pred, img_shape, scale_factor, rescale):
        if bbox_pred is not None:
            bboxes = delta2bbox(rois[:, 1:], bbox_pred, self.target_means, self.target_stds, img_shape)
        else:
            bboxes = rois[:, 1:].clone()
            if img_shape is not None:
                bboxes[:, [0, 2]] = bboxes[:, [0, 2]].clamp(min=0, max=img_shape[1] - 1)
                bboxes[:, [1, 3]] = bboxes[:, [1, 3]].clamp(min=0, max=img_shape[0] - 1)
        if rescale:
            if isinstance(scale_factor, float):
                bboxes = bboxes / scale_factor
            else:
                bboxes = bboxes / torch.from_numpy(np.asarray(scale_factor)).to(bboxes.device)
        return bboxes

    @force_fp32(apply_to=('bbox_preds', ))
    def refine_bboxes(self, rois, labels, bbox_preds, pos_is_gts, img_metas):
        """Cascade refinement (bbox_head.py:169-208)."""
        img_ids = rois[:, 0].long().unique(sorted=True)
        assert img_ids.numel() == len(img_metas)
        bboxes_list = []
        for i in range(len(img_metas)):
            inds = torch.nonzero(rois[:, 0] == i, as_tuple=False).squeeze(-1)
            num_rois = inds.numel()
            bboxes = self.regress_by_class(rois[inds, 1:], labels[inds], bbox_preds[inds], img_metas[i])
            pos_is_gts_ = pos_is_gts[i]
            keep_inds = pos_is_gts_.new_ones(num_rois)
            keep_inds[:len(pos_is_gts_)] = 1 - pos_is_gts_
            bboxes_list.append(bboxes[keep_inds.bool()])
        return bboxes_list

    @force_fp32(apply_to=('bbox_pred', ))
    def regress_by_class(self, rois, label, bbox_pred, img_meta):
        """bbox_head.py:210-239."""
        assert rois.size(1) == 4 or rois.size(1) == 5
        if not self.reg_class_agnostic:
            label = label * 4
            inds = torch.stack((label, label + 1, label + 2, label + 3), 1)
            bbox_pred = torch.gather(bbox_pred, 1, inds)
        assert bbox_pred.size(1) == 4
        if rois.size(1) == 4:
            return delta2bbox(rois, bbox_pred, self.target_means, self.target_stds, img_meta['img_shape'])
        bboxes = delta2bbox(rois[:, 1:], bbox_pred, self.target_means, self.target_stds, img_meta['img_shape'])
        return torch.cat((rois[:, [0]], bboxes), dim=1)


class ConvFCBBoxHead(BBoxHead):
    """Shared-FC trunk + fc_cls / fc_reg (convfc_bbox_head.py:8-168).  Only the FC branches the
    BAGS configs use are supported; conv branches need mmdet's ConvModule and are out of scope."""

    def __init__(self, num_shared_convs=0, num_shared_fcs=0, num_cls_convs=0, num_cls_fcs=0, num_reg_convs=0,
                 num_reg_fcs=0, conv_out_channels=256, fc_out_channels=1024, conv_cfg=None, norm_cfg=None,
                 *args, **kwargs):
        super().__init__(*args, **kwargs)
        assert (num_shared_convs + num_shared_fcs + num_cls_convs + num_cls_fcs + num_reg_convs + num_reg_fcs > 0)
        if num_shared_convs or num_cls_convs or num_reg_convs:
            raise NotImplementedError('conv branches (ConvModule) are outside the BAGS head path')
        self.num_shared_convs, self.num_shared_fcs = num_shared_convs, num_shared_fcs
        self.num_cls_convs, self.num_cls_fcs = num_cls_convs, num_cls_fcs
        self.num_reg_convs, self.num_reg_fcs = num_reg_convs, num_reg_fcs
        self.conv_out_channels = conv_out_channels
        self.fc_out_channels = fc_out_channels
        self.conv_cfg, self.norm_cfg = conv_cfg, norm_cfg

        self.shared_convs, self.shared_fcs, last = self._add_fc_branch(self.num_shared_fcs, self.in_channels, True)
        self.shared_out_channels = last
        self.cls_convs, self.cls_fcs, self.cls_last_dim = self._add_fc_branch(self.num_cls_fcs, last)
        self.reg_convs, self.reg_fcs, self.reg_last_dim = self._add_fc_branch(self.num_reg_fcs, last)
        if self.num_shared_fcs == 0 and not self.with_avg_pool:
            if self.num_cls_fcs == 0:
                self.cls_last_dim *= self.roi_feat_area
            if self.num_reg_fcs == 0:
                self.reg_last_dim *= self.roi_feat_area
        self.relu = nn.ReLU(inplace=True)
        if self.with_cls:
            self.fc_cls = nn.Linear(self.cls_last_dim, self.num_classes)
        if self.with_reg:
            self.fc_reg = nn.Linear(self.reg_last_dim, 4 if self.reg_class_agnostic else 4 * self.num_classes)

    def _add_fc_branch(self, num_fcs, in_channels, is_shared=False):
        last = in_channels
        fcs = nn.ModuleList()
        if num_fcs > 0:
            if (is_shared or self.num_shared_fcs == 0) and not self.with_avg_pool:
                last *= self.roi_feat_area
            for i in range(num_fcs):
                fcs.append(nn.Linear(last if i == 0 else self.fc_out_channels, self.fc_out_channels))
            last = self.fc_out_channels
        return nn.ModuleList(), fcs, last

    def init_weights(self):
        super().init_weights()
        for module_list in [self.shared_fcs, self.cls_fcs, self.reg_fcs]:
            for m in module_list.modules():
                if isinstance(m, nn.Linear):
                    nn.init.xavier_uniform_(m.weight)
                    nn.init.constant_(m.bias, 0)

    def _trunk(self, x):
        if self.num_shared_fcs > 0:
            if self.with_avg_pool:
                x = self.avg_pool(x)
            x = x.view(x.size(0), -1)
            for fc in self.shared_fcs:
                x = self.relu(fc(x))
        x_cls, x_reg = x, x
        if x_cls.dim() > 2:
            if self.with_avg_pool:
                x_cls, x_reg = self.avg_pool(x_cls), self.avg_pool(x_reg)
            x_cls, x_reg = x_cls.view(x_cls.size(0), -1), x_reg.view(x_reg.size(0), -1)
        for fc in self.cls_fcs:
            x_cls = self.relu(fc(x_cls))
        for fc in self.reg_fcs:
            x_reg = self.relu(fc(x_reg))
        return x_cls, x_reg

    def forward(self, x):
        x_cls, x_reg = self._trunk(x)
        cls_score = self.fc_cls(x_cls) if self.with_cls else None
        bbox_pred = self.fc_reg(x_reg) if self.with_reg else None
        return cls_score, bbox_pred


class SharedFCBBoxHead(ConvFCBBoxHead):

    def __init__(self, num_fcs=2, fc_out_channels=1024, *args, **kwargs):
        assert num_fcs >= 1
        super().__init__(num_shared_convs=0, num_shared_fcs=num_fcs, num_cls_convs=0, num_cls_fcs=0,
                         num_reg_convs=0, num_reg_fcs=0, fc_out_channels=fc_out_channels, *args, **kwargs)


# --------------------------------------------------------------------------- the BAGS head
def _cfg_get(cfg, key, default=None):
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    return getattr(cfg, key, default)


_DTYPES = {'bf16': torch.bfloat16, 'bfloat16': torch.bfloat16, 'fp32': torch.float32, 'float32': torch.float32,
           'tf32': torch.float32}


class NativeFcClsHead(SharedFCBBoxHead):
    """What the heads with a native classifier share: the shared FCs and fc_reg on this library's wgmma GEMMs, fc_cls
    through ``FcClsFunction``, train / eval operand dtypes, and a training ``forward`` that returns a
    ``ClsScoreHandle`` so that ``loss`` can run fc_cls and the loss in one fused kernel.

    Execution keys, read from the head's own config dict (``gs_config`` / ``reweight_cfg``):
        compute_dtype      'bf16' (default) or 'fp32' (TF32 products) for the fc_cls contraction in training
        eval_compute_dtype 'fp32' (default) / 'bf16' for the test-time logits
        native_trunk       True (default): shared FCs / fc_reg on this library's wgmma GEMMs
        fuse_loss          True (default): training forward returns a ClsScoreHandle
        fuse_bbox_loss     False (default).  True: with class-specific regression, the training forward returns a
                           ``BoxPredHandle`` for ``bbox_pred`` and a 'mean' SmoothL1 ``loss_bbox`` computes only each
                           positive RoI's four deltas, with fp32 products, and no host sync
                           (``ops.SmoothL1BoxFunction``).  ``loss_bbox`` then differs from the default route by rounding
    """

    def _init_execution(self, cfg):
        cd = _cfg_get(cfg, 'compute_dtype', os.environ.get('BAGS_COMPUTE_DTYPE', 'bf16'))
        self.compute_dtype = _DTYPES[str(cd).lower()]
        # test-time logits: fp32 operands (TF32 products) by default -- a reference fp32 checkpoint scored through bf16
        # operands moves logits by ~1e-2, which reaches the score_thr / NMS ranking of rare classes
        ed = _cfg_get(cfg, 'eval_compute_dtype', os.environ.get('BAGS_EVAL_COMPUTE_DTYPE', 'fp32'))
        self.eval_compute_dtype = _DTYPES[str(ed).lower()]
        # shared FCs + fc_reg on this library's wgmma GEMMs (bias + ReLU in the epilogue) instead of nn.Linear / cuBLAS
        self.native_trunk = bool(_cfg_get(cfg, 'native_trunk', os.environ.get('BAGS_NATIVE_TRUNK', '1') != '0'))
        self.fuse_loss = bool(_cfg_get(cfg, 'fuse_loss', True))
        self.fuse_bbox_loss = bool(_cfg_get(cfg, 'fuse_bbox_loss', False))

    @staticmethod
    def _cuda_index(device) -> int:
        device = torch.device(device)
        if device.type != 'cuda':
            raise ops.nat.BagsNativeError(
                'the BAGS head hot path runs on an H100 GPU only (tensor on %s); there is no CPU fallback' % device)
        return device.index if device.index is not None else torch.cuda.current_device()

    def _active_dtype(self):
        return self.compute_dtype if self.training else self.eval_compute_dtype

    def _fc_cls_logits(self, x_cls):
        return FcClsFunction.apply(x_cls, self.fc_cls.weight, self.fc_cls.bias, self._active_dtype())

    def _use_native_trunk(self, x) -> bool:
        return (self.native_trunk and x.is_cuda and not self.with_avg_pool and self.num_shared_fcs > 0
                and self.num_cls_fcs == 0 and self.num_reg_fcs == 0)

    def _trunk(self, x):
        """convfc_bbox_head.py:132-160 for the FC-only configuration the BAGS configs use: flatten -> (Linear + ReLU) x
        num_shared_fcs, each one LinearActFunction (wgmma GEMM, bias + ReLU in its epilogue; the activations travel
        in the operand dtype)."""
        if not self._use_native_trunk(x):
            return super()._trunk(x)
        cd = self._active_dtype()
        act_dtype = torch.bfloat16 if cd == torch.bfloat16 else torch.float32
        x = x.reshape(x.size(0), -1)
        for fc in self.shared_fcs:
            x = ops.LinearActFunction.apply(x, fc.weight, fc.bias, True, cd, act_dtype)
        return x, x

    def _fc_reg(self, x_reg):
        if self.native_trunk and x_reg.is_cuda:
            return ops.LinearActFunction.apply(x_reg, self.fc_reg.weight, self.fc_reg.bias, False, self._active_dtype(),
                                               torch.float32)
        return self.fc_reg(x_reg)

    def _fused_bbox_loss_ok(self, reduction_override) -> bool:
        """True for a SmoothL1Loss with reduction 'mean' and no other reduction asked (recognised by type name and
        attributes, so mmdet's own class qualifies too)."""
        lb = self.loss_bbox
        return (reduction_override in (None, 'mean') and type(lb).__name__ == 'SmoothL1Loss'
                and getattr(lb, 'reduction', None) == 'mean'
                and all(isinstance(getattr(lb, k, None), (int, float)) for k in ('beta', 'loss_weight')))

    def _bbox_loss(self, bbox_pred, labels, bbox_targets, bbox_weights, reduction_override):
        """An unmaterialised ``BoxPredHandle`` with a 'mean' SmoothL1 takes the fused route (avg_factor =
        bbox_targets.size(0) from the shape); anything else the reference's op sequence on the materialised deltas."""
        if isinstance(bbox_pred, BoxPredHandle):
            if bbox_pred._pred is None and self._fused_bbox_loss_ok(reduction_override):
                lb = self.loss_bbox
                loss = ops.SmoothL1BoxFunction.apply(bbox_pred.x_reg, self.fc_reg.weight, self.fc_reg.bias, labels,
                                                     bbox_targets, bbox_weights, float(lb.beta),
                                                     float(bbox_targets.size(0)))[0]
                return loss if lb.loss_weight == 1.0 else loss * lb.loss_weight
            bbox_pred = bbox_pred.tensor()
        return super()._bbox_loss(bbox_pred, labels, bbox_targets, bbox_weights, reduction_override)

    @auto_fp16()
    def forward(self, x):
        x_cls, x_reg = self._trunk(x)
        bbox_pred = None
        if self.with_reg:
            if (self.fuse_bbox_loss and self.training and torch.is_grad_enabled() and not self.reg_class_agnostic
                    and x_reg.is_cuda):
                bbox_pred = BoxPredHandle(self, x_reg)
            else:
                bbox_pred = self._fc_reg(x_reg)
        if not self.with_cls:
            return None, bbox_pred
        if self.training and self.fuse_loss and torch.is_grad_enabled():
            return ClsScoreHandle(self, x_cls), bbox_pred
        return self._fc_cls_logits(x_cls), bbox_pred


class GSBBoxHeadWith0(NativeFcClsHead):
    """Balanced Group Softmax head (gs_bbox_head_with0.py:14-380), fused H100 execution.

    Extra, optional ``gs_config`` keys (all default to reference behaviour where one exists):
        tables            a ``GroupTables`` object instead of the three file paths
        compute_dtype     'bf16' (default) or 'fp32' (TF32 products) for the fc_cls contraction
        sampler           'device' (default; counter-based RNG on the GPU, no host sync) or
                          'numpy' (the reference's np.random.choice on the host -- bit-identical
                          masks for a given numpy seed, at the cost of the reference's syncs)
        fuse_loss         True (default): training forward returns a ClsScoreHandle
        graph_cache       False (default).  True: ``loss`` replays two CUDA graphs per recurring RoI count
                          (``api.GraphCachedHeadLoss``) -- graph-replay host cost with a data-dependent N
        native_trunk      True (default): shared FCs / fc_reg on this library's wgmma GEMMs
        eval_compute_dtype 'fp32' (default) / 'bf16' for the test-time logits
        fuse_bbox_loss    False (default).  True: fc_reg + the SmoothL1 box loss in one fused op (see NativeFcClsHead)
    """

    def __init__(self, num_fcs=2, fc_out_channels=1024, gs_config=None, *args, **kwargs):
        super().__init__(num_fcs=num_fcs, fc_out_channels=fc_out_channels, *args, **kwargs)
        assert gs_config is not None, 'GSBBoxHeadWith0 needs gs_config'
        num_bins = int(_cfg_get(gs_config, 'num_bins'))
        # 1236 = 1231 classes + one "others" slot per bin (gs_bbox_head_with0.py:28-29)
        self.fc_cls = nn.Linear(self.cls_last_dim, self.num_classes + num_bins)

        self.loss_bins = [build_loss(_cfg_get(gs_config, 'loss_bin')) for _ in range(num_bins)]

        tables = _cfg_get(gs_config, 'tables')
        if tables is None:
            tables = load_reference_files(_cfg_get(gs_config, 'label2binlabel'), _cfg_get(gs_config, 'pred_slice'),
                                          _cfg_get(gs_config, 'fg_split'))
        assert isinstance(tables, GroupTables)
        assert tables.num_bins == num_bins, 'gs_config.num_bins does not match the tables'
        assert tables.num_logits == self.num_classes + num_bins, 'pred_slice does not cover fc_cls outputs'
        self.tables = tables
        # limits of the native kernels, reported here rather than at the first loss / merge call
        if num_bins > ops.nat.MAX_BINS:
            raise ValueError('GSBBoxHeadWith0: %d bins, the native kernels support at most %d' % (num_bins, ops.nat.MAX_BINS))
        if tables.num_logits % 4 != 0:
            raise ValueError('GSBBoxHeadWith0: %d logits (classes + bins) -- the native kernels need a multiple of 4 '
                             '(the 5-bin LVIS tables give 1236); pad the bin table or use 1, 5 or 9 ... bins'
                             % tables.num_logits)
        for lb in self.loss_bins:
            if getattr(lb, 'reduction', 'mean') != 'mean':
                raise ValueError("GSBBoxHeadWith0: loss_bin.reduction=%r -- the fused path implements the reference's "
                                 "'mean' (sum / avg_factor, losses/utils.py:26-53)" % (lb.reduction,))
        # plain attributes like the reference (not buffers -> not in the state dict)
        self.label2binlabel = torch.from_numpy(tables.label2binlabel)
        self.pred_slice = torch.from_numpy(tables.pred_slice)
        self.fg_splits = [torch.from_numpy(s) for s in tables.fg_splits]
        self.others_sample_ratio = float(_cfg_get(gs_config, 'others_sample_ratio'))

        self._init_execution(gs_config)
        # opt-in: CUDA-graph replay per recurring RoI count behind loss() (api.GraphCachedHeadLoss)
        self.graph_cache = bool(_cfg_get(gs_config, 'graph_cache', os.environ.get('BAGS_GRAPH_CACHE', '0') == '1'))
        self._graph_loss = None
        self.sampler = str(_cfg_get(gs_config, 'sampler', 'device'))
        assert self.sampler in ('device', 'numpy')
        self._device_tables: Dict[int, ops.DeviceTables] = {}
        self._sample_calls = 0
        self.last_sample = None  # (wmask [G,N] uint8, avg [G]) of the latest loss() call, for inspection

    # ---- reference checkpoints -----------------------------------------------------------
    def load_reference_checkpoint(self, checkpoint, prefix: str = 'bbox_head.', strict: bool = True):
        """Load this head's parameters from a reference detector checkpoint (mmcv format: a dict with a
        ``'state_dict'`` entry, keys such as ``bbox_head.fc_cls.weight`` [1236,1024]; cascade / HTC checkpoints use
        ``bbox_head.<stage>.`` -- pass that as ``prefix``).  ``checkpoint`` is a path or an already loaded dict.
        Returns the (missing, unexpected) key lists of ``load_state_dict``."""
        if isinstance(checkpoint, (str, os.PathLike)):
            checkpoint = torch.load(checkpoint, map_location='cpu')
        sd = checkpoint.get('state_dict', checkpoint)
        if any(k.startswith('module.') for k in sd):      # saved from (Distributed)DataParallel
            sd = {(k[7:] if k.startswith('module.') else k): v for k, v in sd.items()}
        own = {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)} if prefix else dict(sd)
        if not own:
            raise KeyError('no key with prefix %r in the checkpoint' % prefix)
        want = self.state_dict()
        for k, v in own.items():
            if k in want and tuple(v.shape) != tuple(want[k].shape):
                raise ValueError('%s%s has shape %s, this head expects %s' % (prefix, k, tuple(v.shape),
                                                                             tuple(want[k].shape)))
        res = self.load_state_dict(own, strict=strict)
        return list(res.missing_keys), list(res.unexpected_keys)

    # ---- device-side tables -------------------------------------------------------------
    def device_tables(self, device) -> ops.DeviceTables:
        idx = self._cuda_index(device)
        dt = self._device_tables.get(idx)
        if dt is None:
            dt = ops.DeviceTables.from_tables(self.tables, torch.device(device))
            self._device_tables[idx] = dt
        return dt

    # ---- label remap / sampling ---------------------------------------------------------
    def _next_seed(self) -> int:
        self._sample_calls += 1
        rank = int(os.environ.get('RANK', '0'))
        return (torch.initial_seed() * 0x9E3779B97F4A7C15 + rank * 0xD1B54A32D192ED03 + self._sample_calls) \
            & 0xFFFFFFFFFFFFFFFF

    def _sample_others_numpy(self, bin_label_cpu: torch.Tensor) -> torch.Tensor:
        """Host sampler, statement for statement the reference's (gs_bbox_head_with0.py:63-89)."""
        fg = (bin_label_cpu > 0).to(torch.int64)
        fg_num = int(fg.sum())
        if fg_num == 0:
            return torch.zeros_like(bin_label_cpu)
        bg_idx = (1 - fg).nonzero(as_tuple=True)[0]
        bg_sample_num = int(fg_num * self.others_sample_ratio)
        if bg_sample_num >= bg_idx.shape[0]:
            return torch.ones_like(bin_label_cpu)
        sample_idx = np.random.choice(bg_idx.numpy(), (bg_sample_num, ), replace=False)
        fg[torch.from_numpy(sample_idx)] = 1
        return fg

    def _remap_labels(self, labels):
        """(wmask [G,N] uint8, avg [G] fp32) on the labels' device (gs_bbox_head_with0.py:91-112).
        The in-bin label gather itself happens inside the fused kernel."""
        dt = self.device_tables(labels.device)
        if self.sampler == 'device':
            return ops.sample_others(labels, dt, self.others_sample_ratio, self._next_seed())
        lab = labels.detach().cpu()
        rows = []
        for g in range(dt.G):
            t = self.label2binlabel[g][lab]
            rows.append(torch.ones_like(t) if g < 1 else self._sample_others_numpy(t))
        wmask = torch.stack(rows).to(torch.uint8).to(labels.device)
        return wmask, ops.mask_avg(wmask)

    def _slice_preds(self, cls_score):
        """Column views per bin (gs_bbox_head_with0.py:134-145); host ints, no device sync."""
        return [cls_score.narrow(1, int(s), int(l)) for s, l in self.tables.pred_slice.tolist()]

    # ---- loss ---------------------------------------------------------------------------
    @force_fp32(apply_to=('cls_score', 'bbox_pred'))
    def loss(self, cls_score, bbox_pred, labels, label_weights, bbox_targets, bbox_weights,
             reduction_override=None):
        losses = dict()
        if cls_score is not None:
            assert reduction_override in (None, 'none', 'mean', 'sum')
            dt = self.device_tables(labels.device)
            if (self.graph_cache and type(self)._remap_labels is GSBBoxHeadWith0._remap_labels and self.sampler == 'device'
                    and reduction_override in (None, 'mean') and isinstance(cls_score, ClsScoreHandle)
                    and cls_score._logits is None and torch.is_grad_enabled()):
                # opt-in (gs_config['graph_cache']): recurring RoI counts replay two CUDA graphs (sampler + fused forward;
                # preparation + merged backward) instead of paying the host work of every call; new counts run eagerly first
                if self._graph_loss is None:
                    from .api import GraphCachedHeadLoss
                    self._graph_loss = GraphCachedHeadLoss(dt, self.others_sample_ratio, compute_dtype=self.compute_dtype,
                                                           seed=self._next_seed())
                loss_vec = self._graph_loss(cls_score.x_cls, self.fc_cls.weight, self.fc_cls.bias, labels)
                self.last_sample = None
                for i in range(dt.G):
                    lw = self.loss_bins[i].loss_weight
                    losses['loss_cls_bin{}'.format(i)] = loss_vec[i] if lw == 1.0 else loss_vec[i] * lw
                if bbox_pred is not None:
                    losses['loss_bbox'] = self._bbox_loss(bbox_pred, labels, bbox_targets, bbox_weights, reduction_override)
                return losses
            wmask, avg = self._remap_labels(labels)
            self.last_sample = (wmask, avg)
            if reduction_override in ('none', 'sum'):
                # per-element / summed losses (only OHEM asks for these): materialised fallback through the
                # per-bin loss modules, the reference's own op sequence
                z = cls_score.tensor() if isinstance(cls_score, ClsScoreHandle) else cls_score
                preds = self._slice_preds(z)
                for i in range(dt.G):
                    t = dt.label2bin[i].long()[labels]
                    losses['loss_cls_bin{}'.format(i)] = self.loss_bins[i](
                        preds[i], t, wmask[i].float(), avg_factor=None if reduction_override == 'sum' else avg[i],
                        reduction_override=reduction_override)
            else:
                if isinstance(cls_score, ClsScoreHandle) and cls_score._logits is None:
                    loss_vec = ops.GroupSoftmaxFunction.apply(
                        cls_score.x_cls, self.fc_cls.weight, self.fc_cls.bias, labels, dt, wmask, avg,
                        self.compute_dtype, None)
                else:
                    z = cls_score.tensor() if isinstance(cls_score, ClsScoreHandle) else cls_score
                    loss_vec = ops.GroupCEFunction.apply(z, labels, dt, wmask, avg)
                for i in range(dt.G):
                    li = loss_vec[i]
                    lw = self.loss_bins[i].loss_weight
                    losses['loss_cls_bin{}'.format(i)] = li if lw == 1.0 else li * lw
        if bbox_pred is not None:
            losses['loss_bbox'] = self._bbox_loss(bbox_pred, labels, bbox_targets, bbox_weights,
                                                  reduction_override)
        return losses

    # ---- inference ------------------------------------------------------------------------
    @force_fp32(apply_to=('cls_score'))
    def _merge_score(self, cls_score):
        """[N,1236] logits -> [N,1231] scores (gs_bbox_head_with0.py:239-273), one kernel."""
        if isinstance(cls_score, ClsScoreHandle):
            cls_score = cls_score.tensor()
        z = cls_score.detach()
        if z.dtype != torch.float32:
            z = z.float()
        return ops.merge_scores(z, self.device_tables(z.device))

    @force_fp32(apply_to=('cls_score', 'bbox_pred'))
    def get_det_bboxes(self, rois, cls_score, bbox_pred, img_shape, scale_factor, rescale=False, cfg=None):
        if isinstance(cls_score, list):
            cls_score = [c.tensor() if isinstance(c, ClsScoreHandle) else c for c in cls_score]
            cls_score = sum(cls_score) / float(len(cls_score))
        scores = self._merge_score(cls_score)
        bboxes = self._decode(rois, bbox_pred, img_shape, scale_factor, rescale)
        if cfg is None:
            return bboxes, scores
        return self._nms(bboxes, scores, cfg)


class GSBBoxHead(GSBBoxHeadWith0):
    """Alias: two ablation configs name the class the reference deleted
    (configs/ablations/gs_faster_rcnn_r50_fpn_1x_lvis.py:35)."""


class GSBBoxHeadWith0Reweight(GSBBoxHeadWith0):
    """BAGS head with per-class loss weights inside the bins (gs_bbox_head_with0_reweight.py:14-109; used by
    configs/ablations/gs_faster_rcnn_r50_fpn_1x_lvis_with0_reweight.py).
    Differences from ``GSBBoxHeadWith0``: ``gs_config.bin_cls_weight`` names a pickle holding one weight
    vector per foreground bin (length = the bin's logit count, index 0 = "others"); the sampled 0/1 weight of every
    RoI is multiplied by the weight of its in-bin label and the per-bin normaliser is the sum of the products
    (``_sample_others`` :57-85, ``_remap_labels`` :87-109).  ``gs_config['cls_weights']`` may pass the vectors directly."""

    def __init__(self, *args, gs_config=None, **kwargs):
        super().__init__(*args, gs_config=gs_config, **kwargs)
        weights = _cfg_get(gs_config, 'cls_weights')
        if weights is None:
            import pickle
            with open(_cfg_get(gs_config, 'bin_cls_weight'), 'rb') as fin:
                weights = pickle.load(fin)
        weights = [torch.as_tensor(np.asarray(w), dtype=torch.float32) for w in weights]
        G = self.tables.num_bins
        assert len(weights) == G - 1, 'one weight vector per foreground bin'
        for g, w in enumerate(weights, start=1):
            assert w.numel() == int(self.tables.pred_slice[g, 1]), 'bin %d: %d weights for %d logits' % (
                g, w.numel(), int(self.tables.pred_slice[g, 1]))
        self.cls_weights = weights
        stride = max(int(w.numel()) for w in weights)
        table = torch.ones(G, stride, dtype=torch.float32)
        for g, w in enumerate(weights, start=1):
            table[g, :w.numel()] = w
        self._cls_weight_table = table
        self._cls_weight_dev: Dict[int, torch.Tensor] = {}

    def _remap_labels(self, labels):
        """(wfloat [G,N] fp32, avg [G] fp32): the base class's sampled masks times the per-class weights."""
        wmask, _ = super()._remap_labels(labels)
        dev = labels.device
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        if idx not in self._cls_weight_dev:
            self._cls_weight_dev[idx] = self._cls_weight_table.to(dev)
        return ops.reweight(labels, self.device_tables(dev), wmask, self._cls_weight_dev[idx])


class ReweightBBoxHead(NativeFcClsHead):
    """Class-reweighted softmax head (mmdet/models/bbox_heads/reweight_bbox_head.py), the re-weighting baselines of
    configs/transferred/faster_rcnn_r50_fpn_1x_lvis_reweight{all,head,head_bf,head_bfocal,head_bours}.py:
    softmax CE over all ``num_classes`` logits, each RoI weighted by ``cls_weight[label]``, normalised by
    max(#(label_weights > 0), 1); ``loss`` also returns the top-1 accuracy ``acc``.  The test path is BBoxHead's
    (softmax, decode, NMS).

    ``reweight_cfg.cls_weight`` names a ``torch.load``-able 1-D tensor of ``num_classes`` weights (the files
    ``python -m balancedgroupsoftmax_b200.tables --cls-weight ...`` writes); ``reweight_cfg.cls_weights`` may pass the
    vector directly.  It is kept as fp32 (the reference casts the gathered weights to fp32, cross_entropy_loss.py:15)
    and copied to a GPU when a loss first runs there.  ``reweight_cfg`` also takes the execution keys of
    ``NativeFcClsHead``.

    In training with a softmax ``CrossEntropyLoss`` (reduction 'mean') as ``loss_cls``, fc_cls, the weighted CE and the
    accuracy run in one fused kernel (``ops.SoftmaxCEFunction``: the [N, C] logits never reach memory) and the
    backward in one bags_bwd call; dX is computed only when the RoI features need a gradient.  A sigmoid ``FocalLoss``
    with reduction 'mean' (reweighthead_bfocal) takes the same fused route (``ops.SigmoidFocalFunction``).  Any other
    ``loss_cls`` or ``reduction_override`` runs the reference's op sequence on materialised logits."""

    def __init__(self, num_fcs=2, fc_out_channels=1024, reweight_cfg=None, *args, **kwargs):
        super().__init__(num_fcs=num_fcs, fc_out_channels=fc_out_channels, *args, **kwargs)
        assert reweight_cfg is not None, 'ReweightBBoxHead needs reweight_cfg'
        w = _cfg_get(reweight_cfg, 'cls_weights')
        if w is None:
            w = torch.load(_cfg_get(reweight_cfg, 'cls_weight'), map_location='cpu')
        w = torch.as_tensor(np.asarray(w.detach().cpu() if torch.is_tensor(w) else w)).to(torch.float32).reshape(-1)
        if w.numel() != self.num_classes:
            raise ValueError('ReweightBBoxHead: %d class weights for %d classes' % (w.numel(), self.num_classes))
        self.cls_weight = w          # a plain attribute as in the reference (not in the state dict)
        self._cls_weight_dev: Dict[int, torch.Tensor] = {}
        self._init_execution(reweight_cfg)

    def _reweight(self, labels):
        """cls_weight[labels] (reweight_bbox_head.py:29-33), gathered on the labels' device."""
        idx = self._cuda_index(labels.device) if labels.is_cuda else None
        if idx is None:
            return self.cls_weight[labels]
        w = self._cls_weight_dev.get(idx)
        if w is None:
            w = self._cls_weight_dev[idx] = self.cls_weight.to(labels.device)
        return w[labels]

    def _fused_loss_ok(self) -> Optional[str]:
        """'ce' for a softmax CrossEntropyLoss, 'focal' for a sigmoid FocalLoss, both with reduction 'mean' (recognised
        by type name and attributes, so mmdet's own classes qualify too); None: the materialised route."""
        lc = self.loss_cls
        if getattr(lc, 'reduction', None) != 'mean':
            return None
        name = type(lc).__name__
        if name == 'CrossEntropyLoss' and not getattr(lc, 'use_sigmoid', False) and not getattr(lc, 'use_mask', False):
            return 'ce'
        if (name == 'FocalLoss' and getattr(lc, 'use_sigmoid', False) is True
                and all(isinstance(getattr(lc, k, None), (int, float)) for k in ('gamma', 'alpha', 'loss_weight'))):
            return 'focal'
        return None

    @force_fp32(apply_to=('cls_score', 'bbox_pred'))
    def loss(self, cls_score, bbox_pred, labels, label_weights, bbox_targets, bbox_weights, reduction_override=None):
        losses = dict()
        if cls_score is not None:
            assert reduction_override in (None, 'none', 'mean', 'sum')
            weight = self._reweight(labels)
            kind = self._fused_loss_ok()
            if (reduction_override in (None, 'mean') and kind is not None and isinstance(cls_score, ClsScoreHandle)
                    and cls_score._logits is None):
                acc = torch.empty((1,), dtype=torch.float32, device=labels.device)
                if kind == 'focal':
                    # FocalLoss.forward: the one-hot targets' quirk, and avg_factor = N * 1231 whatever the caller passes
                    lc, N = self.loss_cls, labels.numel()
                    loss = ops.SigmoidFocalFunction.apply(
                        cls_score.x_cls, self.fc_cls.weight, self.fc_cls.bias, focal_targets(labels, N), weight,
                        max(float(N * FOCAL_ONE_HOT_CLASSES), 1.), float(lc.gamma), float(lc.alpha), self.compute_dtype,
                        labels, acc)[0]
                else:
                    avg = (label_weights > 0).sum(dtype=torch.float32).clamp_min(1.0).reshape(1)
                    loss = ops.SoftmaxCEFunction.apply(cls_score.x_cls, self.fc_cls.weight, self.fc_cls.bias, labels,
                                                       weight, avg, self.compute_dtype, acc)[0]
                lw = self.loss_cls.loss_weight
                losses['loss_cls'] = loss if lw == 1.0 else loss * lw
                losses['acc'] = acc
            else:
                losses['loss_cls'] = self._cls_loss(cls_score, labels, weight, label_weights, reduction_override)
                losses['acc'] = accuracy(_as_tensor(cls_score), labels)
        if bbox_pred is not None:
            losses['loss_bbox'] = self._bbox_loss(bbox_pred, labels, bbox_targets, bbox_weights, reduction_override)
        return losses


for _cls in (BBoxHead, ConvFCBBoxHead, SharedFCBBoxHead, GSBBoxHeadWith0, GSBBoxHead, GSBBoxHeadWith0Reweight,
             ReweightBBoxHead):
    register(HEADS, _cls)
