"""The RPN head: AnchorGenerator and RPNHead, with proposal generation on native kernels.

Drop-in for mmdet/core/anchor/anchor_generator.py and mmdet/models/anchor_heads/rpn_head.py (with the AnchorHead
parts it uses): the same constructors, attributes, layers and state-dict keys, so every LVIS config's ``rpn_head``
block builds unchanged.  ``RPNHead.get_bboxes`` is one ops.rpn_proposals call for the whole batch (four launches, no
host sync) followed by the batch's single host read of the per-image counts; the reference runs a Python loop per
image and level with a blocking device-to-host copy and a CPU scan in every NMS call.

The proposals equal the reference's bit for bit wherever no tie decides the result.  Ties, which the reference leaves
to torch's CUDA topk / sort, are broken by (score desc, flat index asc) within a level and by (score desc, level asc,
position asc) across levels.  Where the reference breaks, the native route returns: with min_bbox_size > 0 and exactly
one surviving box per level, that box (the reference's ``nonzero().squeeze()`` gives a 0-d index and its ``cat``
fails); a level with no candidate contributes nothing; an image with none gets a [0, 5] tensor.

A softmax RPN (``use_sigmoid=False``), ``nms_across_levels=True``, a level with more candidates than the kernel
holds (4096), more than 32 images or 16 anchors per location, or CPU tensors run mmdet's own ``get_bboxes_single``
per image when mmdet is importable (also under the drop-in, where this RPNHead is the one registered in mmdet's
HEADS), and raise NotImplementedError naming the setting otherwise.

``loss`` restates AnchorHead.loss with this package's losses.  Its targets are one ops.anchor_targets call for the
batch (a memset and four launches, no host sync): MaxIoUAssigner's assignment bit for bit the reference's, the box
targets bbox2delta's op sequence, and a sample drawn as the head's device sampler draws (an exact-k uniform subset by
counter-based keys; statistically, not bitwise, np.random.shuffle's).  With the device totals as avg_factor and the
sigmoid labels passed as [N, 1] columns (the one-hot CrossEntropyLoss would build, without its nonzero), the RPN
loss makes no host sync.  An image with no gt raises ValueError('No gt or bboxes') and one with no inside anchor
makes the loss None, both decided on the host from shapes and metadata.  A non-sampling RPN (Focal / GHM), another
assigner or sampler, add_gt_as_proposals=True, ignore_iof_thr > 0 with ignored gts, more than 8 levels, 32 images or
16 anchors per location, and CPU tensors take mmdet's ``anchor_target`` when mmdet is importable and raise
NotImplementedError naming the setting otherwise.
"""
from __future__ import annotations

import os

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from .fp16 import force_fp32
from .head import _mmdet_core
from .losses import CrossEntropyLoss, SmoothL1Loss  # noqa: F401  (registers them)
from .registry import HEADS, build_loss, register

MAX_CANDIDATES = 4096   # per (image, level): kRpnMaxCand in csrc/bags_rpn.cuh
MAX_IMAGES = 32
MAX_LEVELS = 8
MAX_ANCHORS = 16


class AnchorGenerator(object):
    """mmdet/core/anchor/anchor_generator.py: the base anchors of one level (``base_anchors``, [A, 4], on the CPU),
    the anchors of a feature map (``grid_anchors``, location-major: the A anchors of (0, 0), then (0, 1), ...) and the
    valid flags of a padded image."""

    def __init__(self, base_size, scales, ratios, scale_major=True, ctr=None):
        self.base_size = base_size
        self.scales = torch.Tensor(scales)
        self.ratios = torch.Tensor(ratios)
        self.scale_major = scale_major
        self.ctr = ctr
        self.base_anchors = self.gen_base_anchors()

    @property
    def num_base_anchors(self):
        return self.base_anchors.size(0)

    def gen_base_anchors(self):
        w = h = self.base_size
        x_ctr, y_ctr = (0.5 * (w - 1), 0.5 * (h - 1)) if self.ctr is None else self.ctr
        h_ratios = torch.sqrt(self.ratios)
        w_ratios = 1 / h_ratios
        if self.scale_major:
            ws = (w * w_ratios[:, None] * self.scales[None, :]).view(-1)
            hs = (h * h_ratios[:, None] * self.scales[None, :]).view(-1)
        else:
            ws = (w * self.scales[:, None] * w_ratios[None, :]).view(-1)
            hs = (h * self.scales[:, None] * h_ratios[None, :]).view(-1)
        return torch.stack([x_ctr - 0.5 * (ws - 1), y_ctr - 0.5 * (hs - 1),
                            x_ctr + 0.5 * (ws - 1), y_ctr + 0.5 * (hs - 1)], dim=-1).round()

    def _meshgrid(self, x, y, row_major=True):
        xx = x.repeat(len(y))
        yy = y.view(-1, 1).repeat(1, len(x)).view(-1)
        return (xx, yy) if row_major else (yy, xx)

    def grid_anchors(self, featmap_size, stride=16, device='cuda'):
        base_anchors = self.base_anchors.to(device)
        feat_h, feat_w = featmap_size
        shift_x = torch.arange(0, feat_w, device=device) * stride
        shift_y = torch.arange(0, feat_h, device=device) * stride
        shift_xx, shift_yy = self._meshgrid(shift_x, shift_y)
        shifts = torch.stack([shift_xx, shift_yy, shift_xx, shift_yy], dim=-1).type_as(base_anchors)
        return (base_anchors[None, :, :] + shifts[:, None, :]).view(-1, 4)

    def valid_flags(self, featmap_size, valid_size, device='cuda'):
        feat_h, feat_w = featmap_size
        valid_h, valid_w = valid_size
        assert valid_h <= feat_h and valid_w <= feat_w
        valid_x = torch.zeros(feat_w, dtype=torch.uint8, device=device)
        valid_y = torch.zeros(feat_h, dtype=torch.uint8, device=device)
        valid_x[:valid_w] = 1
        valid_y[:valid_h] = 1
        valid_xx, valid_yy = self._meshgrid(valid_x, valid_y)
        valid = valid_xx & valid_yy
        return valid[:, None].expand(valid.size(0), self.num_base_anchors).contiguous().view(-1)


def _multi_apply(func, *args, **kwargs):
    """mmdet/core/utils/misc.py:multi_apply."""
    import functools
    pfunc = functools.partial(func, **kwargs) if kwargs else func
    return tuple(map(list, zip(*map(pfunc, *args))))


def _images_to_levels(target, num_level_anchors):
    """anchor_target.py:images_to_levels on a batch tensor [B, N, ...]: per level [B, n_l, ...], squeezed at B = 1."""
    out, start = [], 0
    for n in num_level_anchors:
        out.append(target[:, start:start + n].squeeze(0))
        start += n
    return out


def _cfg(cfg, key, default=None):
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    return getattr(cfg, key, default)


def _mmdet_rpn_get_bboxes_single():
    """mmdet's own RPNHead.get_bboxes_single, or None when mmdet is not importable.

    Under the drop-in (INTEGRATION.md), mmdet/models/anchor_heads/__init__.py imports this package's RPNHead instead
    of mmdet's rpn_head module, and this RPNHead is registered in mmdet's HEADS.  Importing mmdet's module afterwards
    would register its RPNHead under the same name, which mmdet's Registry refuses with a KeyError.  So the entry is
    set aside while the module is imported and put back after it: the registered RPNHead stays this package's."""
    import importlib
    import sys
    name = 'mmdet.models.anchor_heads.rpn_head'
    mod = sys.modules.get(name)
    if mod is None:
        try:
            from mmdet.models.registry import HEADS as mmdet_heads
        except ImportError:
            return None
        table = getattr(mmdet_heads, '_module_dict', None)
        saved = table.pop('RPNHead', None) if table is not None else None
        try:
            mod = importlib.import_module(name)
        finally:
            if saved is not None:
                table['RPNHead'] = saved
    return mod.RPNHead.get_bboxes_single


class RPNHead(nn.Module):
    """mmdet's RPNHead (an AnchorHead with two classes): ``rpn_conv`` (3x3) + ReLU, then ``rpn_cls`` and ``rpn_reg``
    (1x1).  Constructor, attributes and state-dict keys as the reference's."""

    def __init__(self, in_channels, feat_channels=256, anchor_scales=[8, 16, 32], anchor_ratios=[0.5, 1.0, 2.0],
                 anchor_strides=[4, 8, 16, 32, 64], anchor_base_sizes=None, target_means=(.0, .0, .0, .0),
                 target_stds=(1.0, 1.0, 1.0, 1.0),
                 loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True, loss_weight=1.0),
                 loss_bbox=dict(type='SmoothL1Loss', beta=1.0 / 9.0, loss_weight=1.0)):
        super(RPNHead, self).__init__()
        num_classes = 2
        self.in_channels = in_channels
        self.num_classes = num_classes
        self.feat_channels = feat_channels
        self.anchor_scales = anchor_scales
        self.anchor_ratios = anchor_ratios
        self.anchor_strides = anchor_strides
        self.anchor_base_sizes = list(anchor_strides) if anchor_base_sizes is None else anchor_base_sizes
        self.target_means = target_means
        self.target_stds = target_stds
        self.use_sigmoid_cls = loss_cls.get('use_sigmoid', False)
        self.sampling = loss_cls['type'] not in ['FocalLoss', 'GHMC']
        self.cls_out_channels = num_classes - 1 if self.use_sigmoid_cls else num_classes
        if self.cls_out_channels <= 0:
            raise ValueError('num_classes={} is too small'.format(num_classes))
        self.loss_cls = build_loss(loss_cls)
        self.loss_bbox = build_loss(loss_bbox)
        self.fp16_enabled = False
        self.anchor_generators = [AnchorGenerator(base, anchor_scales, anchor_ratios)
                                  for base in self.anchor_base_sizes]
        self.num_anchors = len(self.anchor_ratios) * len(self.anchor_scales)
        self._init_layers()

    def _init_layers(self):
        self.rpn_conv = nn.Conv2d(self.in_channels, self.feat_channels, 3, padding=1)
        self.rpn_cls = nn.Conv2d(self.feat_channels, self.num_anchors * self.cls_out_channels, 1)
        self.rpn_reg = nn.Conv2d(self.feat_channels, self.num_anchors * 4, 1)

    def init_weights(self):
        for m in (self.rpn_conv, self.rpn_cls, self.rpn_reg):   # mmcv normal_init(std=0.01), bias 0
            nn.init.normal_(m.weight, 0, 0.01)
            nn.init.constant_(m.bias, 0)

    def forward_single(self, x):
        x = F.relu(self.rpn_conv(x), inplace=True)
        return self.rpn_cls(x), self.rpn_reg(x)

    def forward(self, feats):
        return _multi_apply(self.forward_single, feats)

    def get_anchors(self, featmap_sizes, img_metas, device='cuda'):
        """anchor_head.py:get_anchors: the anchors of every level (the same for every image) and each image's valid
        flags from its pad_shape."""
        num_levels = len(featmap_sizes)
        multi_level_anchors = [self.anchor_generators[i].grid_anchors(featmap_sizes[i], self.anchor_strides[i],
                                                                      device=device) for i in range(num_levels)]
        anchor_list = [multi_level_anchors for _ in img_metas]
        valid_flag_list = []
        for img_meta in img_metas:
            flags = []
            for i in range(num_levels):
                stride = self.anchor_strides[i]
                feat_h, feat_w = featmap_sizes[i]
                h, w, _ = img_meta['pad_shape']
                valid_h = min(int(np.ceil(h / stride)), feat_h)
                valid_w = min(int(np.ceil(w / stride)), feat_w)
                flags.append(self.anchor_generators[i].valid_flags((feat_h, feat_w), (valid_h, valid_w),
                                                                   device=device))
            valid_flag_list.append(flags)
        return anchor_list, valid_flag_list

    # ------------------------------------------------------------------ training loss
    def loss_single(self, cls_score, bbox_pred, labels, label_weights, bbox_targets, bbox_weights, num_total_samples,
                    cfg):
        if self.use_sigmoid_cls and self.cls_out_channels == 1 and isinstance(self.loss_cls, CrossEntropyLoss):
            # [N, 1] columns: the one-hot CrossEntropyLoss would build (labels are 0 / 1), without its nonzero sync
            labels = labels.reshape(-1, 1)
            label_weights = label_weights.reshape(-1, 1)
        else:
            labels = labels.reshape(-1)
            label_weights = label_weights.reshape(-1)
        cls_score = cls_score.permute(0, 2, 3, 1).reshape(-1, self.cls_out_channels)
        loss_cls = self.loss_cls(cls_score, labels, label_weights, avg_factor=num_total_samples)
        bbox_targets = bbox_targets.reshape(-1, 4)
        bbox_weights = bbox_weights.reshape(-1, 4)
        bbox_pred = bbox_pred.permute(0, 2, 3, 1).reshape(-1, 4)
        loss_bbox = self.loss_bbox(bbox_pred, bbox_targets, bbox_weights, avg_factor=num_total_samples)
        return loss_cls, loss_bbox

    def _next_seed(self) -> int:
        """The sampler's seed of this call: torch's initial seed, the process's rank and a per-call counter (as
        GSBBoxHeadWith0._next_seed)."""
        self._sample_calls = getattr(self, '_sample_calls', 0) + 1
        rank = int(os.environ.get('RANK', '0'))
        return (torch.initial_seed() * 0x9E3779B97F4A7C15 + rank * 0xD1B54A32D192ED03 + self._sample_calls) \
            & 0xFFFFFFFFFFFFFFFF

    def _targets_unsupported(self, cfg, cls_scores, gt_bboxes, gt_bboxes_ignore, n_images):
        """Why ops.anchor_targets cannot compute these targets, or None."""
        if not self.sampling:
            return 'sampling=False (a %s RPN)' % self.loss_cls.__class__.__name__
        assigner, sampler = _cfg(cfg, 'assigner'), _cfg(cfg, 'sampler')
        if _cfg(assigner, 'type') != 'MaxIoUAssigner':
            return 'the assigner %r (MaxIoUAssigner only)' % (_cfg(assigner, 'type'),)
        if _cfg(sampler, 'type') != 'RandomSampler':
            return 'the sampler %r (RandomSampler only)' % (_cfg(sampler, 'type'),)
        if _cfg(sampler, 'add_gt_as_proposals', True):
            return 'add_gt_as_proposals=True'
        if not 0 <= float(_cfg(sampler, 'pos_fraction')) <= 1:
            return 'pos_fraction=%r (0 to 1)' % (_cfg(sampler, 'pos_fraction'),)
        if _cfg(assigner, 'ignore_iof_thr', -1) > 0 and gt_bboxes_ignore is not None and \
                any(g is not None and g.numel() > 0 for g in gt_bboxes_ignore):
            return 'ignore_iof_thr > 0 with ignored gts'
        if not 1 <= len(cls_scores) <= MAX_LEVELS:
            return '%d levels (1 to %d)' % (len(cls_scores), MAX_LEVELS)
        if n_images > MAX_IMAGES:
            return '%d images per batch (at most %d)' % (n_images, MAX_IMAGES)
        if self.num_anchors > MAX_ANCHORS:
            return '%d anchors per location (at most %d)' % (self.num_anchors, MAX_ANCHORS)
        if not all(t.is_cuda for t in list(cls_scores) + list(gt_bboxes)):
            return 'CPU tensors (the native route runs on the GPU)'
        return None

    def _reference_anchor_target(self, why, featmap_sizes, gt_bboxes, img_metas, cfg, gt_bboxes_ignore, device):
        anchor_target = _mmdet_core('anchor_target')
        if anchor_target is None:
            raise NotImplementedError('RPNHead.loss: %s has no native route; install mmdetection v1.x for the '
                                      'reference anchor_target' % why)
        assert len(featmap_sizes) == len(self.anchor_generators)
        anchor_list, valid_flag_list = self.get_anchors(featmap_sizes, img_metas, device=device)
        label_channels = self.cls_out_channels if self.use_sigmoid_cls else 1
        return anchor_target(anchor_list, valid_flag_list, gt_bboxes, img_metas, self.target_means, self.target_stds,
                             cfg, gt_bboxes_ignore_list=gt_bboxes_ignore, gt_labels_list=None,
                             label_channels=label_channels, sampling=self.sampling)

    def _has_inside_anchor(self, featmap_sizes, img_meta, allowed_border):
        """Whether anchor_inside_flags keeps any anchor of this image: host arithmetic on its metadata, the same fp32
        adds and comparisons (anchors depend on shapes only)."""
        h, w = img_meta['img_shape'][:2]
        for l, size in enumerate(featmap_sizes):
            vh, vw = ops.valid_size(img_meta['pad_shape'], self.anchor_strides[l], size)
            if vh == 0 or vw == 0:
                continue
            if allowed_border < 0:
                return True
            base = self.anchor_generators[l].base_anchors.numpy().astype(np.float32)
            sx = (np.arange(vw) * self.anchor_strides[l]).astype(np.float32)
            sy = (np.arange(vh) * self.anchor_strides[l]).astype(np.float32)
            lo = np.float32(-allowed_border)
            for a in range(base.shape[0]):
                ok_x = ((base[a, 0] + sx >= lo) & (base[a, 2] + sx < np.float32(w + allowed_border))).any()
                ok_y = ((base[a, 1] + sy >= lo) & (base[a, 3] + sy < np.float32(h + allowed_border))).any()
                if ok_x and ok_y:
                    return True
        return False

    def anchor_targets(self, featmap_sizes, gt_bboxes, img_metas, cfg, seed=None, seed_step=None):
        """anchor_target on this head's anchors through ops.anchor_targets: (labels, label_weights, bbox_targets,
        bbox_weights, totals) as dense [B, N] / [B, N, 4] device tensors and int64 [3] device totals, with no host
        sync; None when an image has no inside anchor, and ValueError('No gt or bboxes') when one that has some has
        no gt (both decided from shapes and metadata, as the reference decides them)."""
        assigner, sampler = _cfg(cfg, 'assigner'), _cfg(cfg, 'sampler')
        allowed_border = _cfg(cfg, 'allowed_border', 0)
        inside = [self._has_inside_anchor(featmap_sizes, m, allowed_border) for m in img_metas]
        if any(ok and g.shape[0] == 0 for ok, g in zip(inside, gt_bboxes)):
            raise ValueError('No gt or bboxes')
        if not all(inside):
            return None
        L = len(featmap_sizes)
        return ops.anchor_targets(
            [tuple(int(v) for v in s) for s in featmap_sizes],
            [self.anchor_generators[i].base_anchors for i in range(L)], self.anchor_strides[:L],
            [m['img_shape'] for m in img_metas], [m['pad_shape'] for m in img_metas], gt_bboxes,
            pos_iou_thr=_cfg(assigner, 'pos_iou_thr'), neg_iou_thr=_cfg(assigner, 'neg_iou_thr'),
            min_pos_iou=_cfg(assigner, 'min_pos_iou', .0), gt_max_assign_all=_cfg(assigner, 'gt_max_assign_all', True),
            allowed_border=allowed_border, num=_cfg(sampler, 'num'), pos_fraction=_cfg(sampler, 'pos_fraction'),
            neg_pos_ub=_cfg(sampler, 'neg_pos_ub', -1), pos_weight=_cfg(cfg, 'pos_weight', -1),
            means=self.target_means, stds=self.target_stds,
            seed=self._next_seed() if seed is None else seed, seed_step=seed_step)

    @force_fp32(apply_to=('cls_scores', 'bbox_preds'))
    def loss(self, cls_scores, bbox_preds, gt_bboxes, img_metas, cfg, gt_bboxes_ignore=None):
        """RPNHead.loss / AnchorHead.loss (anchor_head.py:159-205).  The targets are one ops.anchor_targets call for
        the batch, split per level as images_to_levels splits them; with its device totals as avg_factor the loss
        makes no host sync.  Settings without a native route take mmdet's ``anchor_target``."""
        featmap_sizes = [featmap.size()[-2:] for featmap in cls_scores]
        why = self._targets_unsupported(cfg, cls_scores, gt_bboxes, gt_bboxes_ignore, len(img_metas))
        if why is not None:
            targets = self._reference_anchor_target(why, featmap_sizes, gt_bboxes, img_metas, cfg, gt_bboxes_ignore,
                                                    cls_scores[0].device)
            if targets is None:
                return None
            labels, label_weights, bbox_targets, bbox_weights, num_pos, num_neg = targets
            num_total_samples = num_pos + num_neg if self.sampling else num_pos
        else:
            assert len(featmap_sizes) == len(self.anchor_generators)
            targets = self.anchor_targets(featmap_sizes, gt_bboxes, img_metas, cfg)
            if targets is None:
                return None
            counts = [int(h) * int(w) * self.num_anchors for h, w in featmap_sizes]
            labels, label_weights, bbox_targets, bbox_weights = [_images_to_levels(t, counts) for t in targets[:4]]
            num_total_samples = targets[4][2]
        losses_cls, losses_bbox = _multi_apply(self.loss_single, cls_scores, bbox_preds, labels, label_weights,
                                               bbox_targets, bbox_weights, num_total_samples=num_total_samples,
                                               cfg=cfg)
        return dict(loss_rpn_cls=losses_cls, loss_rpn_bbox=losses_bbox)

    # ------------------------------------------------------------------ proposals
    def _unsupported(self, cfg, cls_scores, bbox_preds, n_images):
        """Why the native route cannot run these inputs, or None."""
        featmap_sizes = [c.shape[-2:] for c in cls_scores]
        if not self.use_sigmoid_cls:
            return 'a softmax RPN (use_sigmoid=False)'
        if _cfg(cfg, 'nms_across_levels', False):
            return 'nms_across_levels=True'
        if not 1 <= len(featmap_sizes) <= MAX_LEVELS:
            return '%d levels (1 to %d)' % (len(featmap_sizes), MAX_LEVELS)
        if n_images > MAX_IMAGES:
            return '%d images per batch (at most %d)' % (n_images, MAX_IMAGES)
        if self.num_anchors > MAX_ANCHORS:
            return '%d anchors per location (at most %d)' % (self.num_anchors, MAX_ANCHORS)
        nms_pre = int(_cfg(cfg, 'nms_pre', -1))
        for i, (h, w) in enumerate(featmap_sizes):
            n = int(h) * int(w) * self.num_anchors
            k = nms_pre if 0 < nms_pre < n else n
            if k > MAX_CANDIDATES:
                return 'level %d with %d candidates (nms_pre %d; at most %d)' % (i, k, nms_pre, MAX_CANDIDATES)
        if not all(t.is_cuda for t in list(cls_scores) + list(bbox_preds)):
            return 'CPU tensors (the native route runs on the GPU)'
        return None

    def _reference_get_bboxes(self, why, cls_scores, bbox_preds, img_metas, cfg, rescale):
        single = _mmdet_rpn_get_bboxes_single()
        if single is None:
            raise NotImplementedError('RPNHead.get_bboxes: %s has no native route; install mmdetection v1.x for the '
                                      'reference loop' % why)
        num_levels = len(cls_scores)
        device = cls_scores[0].device
        mlvl_anchors = [self.anchor_generators[i].grid_anchors(cls_scores[i].size()[-2:], self.anchor_strides[i],
                                                               device=device) for i in range(num_levels)]
        return [single(self, [cls_scores[i][b].detach() for i in range(num_levels)],
                       [bbox_preds[i][b].detach() for i in range(num_levels)], mlvl_anchors,
                       img_metas[b]['img_shape'], img_metas[b]['scale_factor'], cfg, rescale)
                for b in range(len(img_metas))]

    def proposals(self, cls_scores, bbox_preds, img_shapes, cfg):
        """ops.rpn_proposals on this head's anchors: (proposals [B, max_num, 5], counts [B] int32) on the device,
        with no host sync."""
        L = len(cls_scores)
        return ops.rpn_proposals(
            [c.float() for c in cls_scores], [b.float() for b in bbox_preds],
            [self.anchor_generators[i].base_anchors for i in range(L)], self.anchor_strides[:L], img_shapes,
            int(_cfg(cfg, 'nms_pre', -1)), int(_cfg(cfg, 'nms_post')), int(_cfg(cfg, 'max_num')),
            float(_cfg(cfg, 'nms_thr')), float(_cfg(cfg, 'min_bbox_size', 0)), self.target_means, self.target_stds)

    @force_fp32(apply_to=('cls_scores', 'bbox_preds'))
    def get_bboxes(self, cls_scores, bbox_preds, img_metas, cfg, rescale=False):
        """anchor_head.py:get_bboxes with rpn_head.py:get_bboxes_single: a list of [k_i, 5] proposals
        (x1, y1, x2, y2, score) per image.  One rpn_proposals call for the batch and one host read of its counts.
        ``rescale`` is ignored, as in the reference's RPN."""
        assert len(cls_scores) == len(bbox_preds)
        why = self._unsupported(cfg, cls_scores, bbox_preds, len(img_metas))
        if why is not None:
            return self._reference_get_bboxes(why, cls_scores, bbox_preds, img_metas, cfg, rescale)
        out, counts = self.proposals([c.detach() for c in cls_scores], [b.detach() for b in bbox_preds],
                                     [m['img_shape'] for m in img_metas], cfg)
        counts = counts.tolist()   # the batch's one host sync
        return [out[b, :counts[b]] for b in range(len(img_metas))]

    def get_bboxes_single(self, cls_scores, bbox_preds, mlvl_anchors, img_shape, scale_factor, cfg, rescale=False):
        """rpn_head.py:get_bboxes_single for one image ([A, H, W] scores and [4A, H, W] deltas per level), run as a
        batch of one.  The anchors are built on the device from this head's generators; ``mlvl_anchors`` must be
        theirs (``grid_anchors`` of each level)."""
        meta = dict(img_shape=img_shape, scale_factor=scale_factor)
        return self.get_bboxes([c[None] for c in cls_scores], [b[None] for b in bbox_preds], [meta], cfg,
                               rescale)[0]


register(HEADS, RPNHead)
