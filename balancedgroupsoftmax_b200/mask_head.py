"""FCNMaskHead and HTCMaskHead -- the mask branches of the LVIS mask configs behind the reference's API.

Reference surface mirrored here (constructor kwargs, attributes, ``init_weights``, state-dict keys and method
signatures are identical, so the ``mask_head=dict(type='FCNMaskHead' | 'HTCMaskHead', ...)`` blocks of
configs/bags/gs_mask_rcnn_r50_fpn_1x_lvis.py and configs/bags/gs_htc_*.py build unchanged):

    FCNMaskHead     mmdet/models/mask_heads/fcn_mask_head.py:14-123
    HTCMaskHead     mmdet/models/mask_heads/htc_mask_head.py:7-38
    ConvModule      mmdet/models/utils/conv_module.py (only conv_cfg=None, norm_cfg=None: biased conv, ReLU, kaiming)

The 3x3 convs and the deconv stay ``nn.Conv2d`` / ``nn.ConvTranspose2d``.  What differs is the training loss: a
training ``forward`` returns a lazy ``MaskPredHandle`` for ``mask_pred`` and ``loss`` computes only the channel of
each RoI's label inside its BCE (``ops.MaskBCEFunction``) instead of conv_logits' [P, num_classes, 28, 28] logits.
Everything else -- an eval-mode ``forward``, a materialised handle, another ``loss_mask`` -- runs the reference's ops.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn
from torch.nn.modules.utils import _pair

from . import ops
from .fp16 import auto_fp16, force_fp32
from .head import _LazyHandle, _mmdet_core
from .losses import CrossEntropyLoss  # noqa: F401  (registers it)
from .registry import HEADS, build_loss, register


# --------------------------------------------------------------------------- conv block
class ConvModule(nn.Module):
    """mmdet/models/utils/conv_module.py for ``conv_cfg=None, norm_cfg=None`` (every mask config): conv with bias, then
    ReLU; ``init_weights`` is mmcv's kaiming_init (normal, fan_out, relu; bias 0).  State-dict keys ``conv.*``."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 bias='auto', conv_cfg=None, norm_cfg=None, activation='relu', inplace=True,
                 order=('conv', 'norm', 'act')):
        super().__init__()
        if conv_cfg is not None or norm_cfg is not None:
            raise NotImplementedError('ConvModule: only conv_cfg=None and norm_cfg=None are supported (got conv_cfg=%r, '
                                      'norm_cfg=%r)' % (conv_cfg, norm_cfg))
        if activation not in ('relu', None):
            raise ValueError('{} is currently not supported.'.format(activation))
        assert isinstance(order, tuple) and set(order) == {'conv', 'norm', 'act'}
        self.conv_cfg, self.norm_cfg = conv_cfg, norm_cfg
        self.activation, self.inplace, self.order = activation, inplace, order
        self.with_norm = False
        self.with_activatation = activation is not None
        self.with_bias = True if bias == 'auto' else bias
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size, stride=stride, padding=padding,
                              dilation=dilation, groups=groups, bias=self.with_bias)
        self.in_channels, self.out_channels = self.conv.in_channels, self.conv.out_channels
        self.kernel_size, self.stride, self.padding = self.conv.kernel_size, self.conv.stride, self.conv.padding
        self.dilation, self.transposed = self.conv.dilation, self.conv.transposed
        self.output_padding, self.groups = self.conv.output_padding, self.conv.groups
        if self.with_activatation:
            self.activate = nn.ReLU(inplace=inplace)
        self.init_weights()

    def init_weights(self):
        nn.init.kaiming_normal_(self.conv.weight, mode='fan_out', nonlinearity='relu')
        if self.conv.bias is not None:
            nn.init.constant_(self.conv.bias, 0)

    def forward(self, x, activate=True, norm=True):
        for layer in self.order:
            if layer == 'conv':
                x = self.conv(x)
            elif layer == 'act' and activate and self.with_activatation:
                x = self.activate(x)
        return x


# --------------------------------------------------------------------------- lazy logits
class MaskPredHandle(_LazyHandle):
    """What a mask head's training ``forward`` returns for ``mask_pred``.

    It records the input ``y`` of ``conv_logits``, so that ``loss`` can compute only the channel of each RoI's label
    inside mask_cross_entropy (``ops.MaskBCEFunction``) instead of the [P, num_classes, H, W] logits.  ``tensor()`` (or
    any tensor attribute access, indexing or torch function) materialises them through ``conv_logits``,
    autograd-connected."""

    def __init__(self, head: 'FCNMaskHead', y: torch.Tensor):
        self._head = head
        self.y = y
        self._pred = None

    @property
    def shape(self):
        return torch.Size((self.y.shape[0], self._head.conv_logits.out_channels) + tuple(self.y.shape[2:]))

    @property
    def device(self):
        return self.y.device

    def dim(self):
        return len(self.shape)

    def tensor(self) -> torch.Tensor:
        if self._pred is None:
            self._pred = self._head.conv_logits(self.y)
        return self._pred


def _cfg_get(cfg, key):
    return cfg[key] if isinstance(cfg, dict) else getattr(cfg, key)


# --------------------------------------------------------------------------- mask targets and test-time masks
def _imresize_linear(img, size):
    """Resize ``img`` to ``size`` = (width, height) as mmcv.imresize does by default: cv2.resize, INTER_LINEAR."""
    try:
        import cv2
    except ImportError as e:  # pragma: no cover
        raise ImportError('the mask heads resize masks with OpenCV (cv2), as mmcv.imresize does; install '
                          'opencv-python') from e
    return cv2.resize(img, size, interpolation=cv2.INTER_LINEAR)


def _encode_rle(binary):
    """COCO run-length encoding of one uint8 [H, W] mask (pycocotools.mask.encode of its [H, W, 1] Fortran copy)."""
    try:
        import pycocotools.mask as coco_mask
    except ImportError as e:
        raise ImportError('get_seg_masks encodes masks as COCO RLE with pycocotools; install pycocotools') from e
    return coco_mask.encode(np.asfortranarray(binary[:, :, None]))[0]


def mask_target_single(pos_proposals, pos_assigned_gt_inds, gt_masks, cfg):
    """The targets of one image (mmdet/core/mask/mask_target.py): for each positive RoI, its gt mask cut to the
    proposal box truncated to int32 (at least one pixel wide and high) and resized as uint8 to ``cfg.mask_size``;
    float [num_pos, h, w] on the proposals' device."""
    out_h, out_w = _pair(_cfg_get(cfg, 'mask_size'))
    if pos_proposals.size(0) == 0:
        return pos_proposals.new_zeros((0, out_h, out_w))
    boxes = pos_proposals.cpu().numpy().astype(np.int32)
    gt_ids = pos_assigned_gt_inds.cpu().numpy()
    crops = []
    for (left, top, right, bottom), gt in zip(boxes, gt_ids):
        width, height = max(right - left + 1, 1), max(bottom - top + 1, 1)
        crops.append(_imresize_linear(gt_masks[gt][top:top + height, left:left + width], (out_w, out_h)))
    return torch.from_numpy(np.stack(crops)).float().to(pos_proposals.device)


def mask_target(pos_proposals_list, pos_assigned_gt_inds_list, gt_masks_list, cfg):
    """mmdet's own ``mask_target`` when mmdet is importable, otherwise ``mask_target_single`` per image,
    concatenated."""
    ext = _mmdet_core('mask_target')
    if ext is not None:  # pragma: no cover
        return ext(pos_proposals_list, pos_assigned_gt_inds_list, gt_masks_list, cfg)
    return torch.cat([mask_target_single(p, i, m, cfg) for p, i, m in
                      zip(pos_proposals_list, pos_assigned_gt_inds_list, gt_masks_list)])


def seg_masks(mask_pred, det_bboxes, det_labels, rcnn_test_cfg, ori_shape, scale_factor, rescale, num_classes,
              channel_of_label):
    """COCO-RLE masks per class from the test-time mask logits (fcn_mask_head.py:125-239).  ``mask_pred``: [n, C, h, w]
    logits (a tensor, squashed by a sigmoid) or probabilities (an ndarray, multi-scale testing); det_labels are
    0-based foreground labels, so class k's masks go to list k.  ``channel_of_label(label)`` picks the probability map
    of a 1-based label.  Each detection's map is resized to its box (the box divided by ``scale_factor`` and truncated
    to int32, at least one pixel), thresholded at ``rcnn_test_cfg.mask_thr_binary`` and pasted into an empty image of
    the original size (``rescale``) or of the scaled size."""
    if isinstance(mask_pred, torch.Tensor):
        mask_pred = mask_pred.sigmoid().cpu().numpy()
    assert isinstance(mask_pred, np.ndarray)
    probs = mask_pred.astype(np.float32)             # fp16 arrays under mixed precision
    per_class = [[] for _ in range(num_classes - 1)]
    boxes = det_bboxes.cpu().numpy()[:, :4]
    labels = det_labels.cpu().numpy() + 1
    if rescale:
        img_h, img_w = ori_shape[:2]
    else:
        img_h = np.round(ori_shape[0] * scale_factor).astype(np.int32)
        img_w = np.round(ori_shape[1] * scale_factor).astype(np.int32)
        scale_factor = 1.0
    thr = _cfg_get(rcnn_test_cfg, 'mask_thr_binary')
    for k in range(boxes.shape[0]):
        left, top, right, bottom = (boxes[k, :] / scale_factor).astype(np.int32)
        width, height = max(right - left + 1, 1), max(bottom - top + 1, 1)
        resized = _imresize_linear(probs[k, channel_of_label(labels[k]), :, :], (width, height))
        canvas = np.zeros((img_h, img_w), dtype=np.uint8)
        canvas[top:top + height, left:left + width] = (resized > thr).astype(np.uint8)
        per_class[labels[k] - 1].append(_encode_rle(canvas))
    return per_class


# --------------------------------------------------------------------------- heads
class FCNMaskHead(nn.Module):

    def __init__(self, num_convs=4, roi_feat_size=14, in_channels=256, conv_kernel_size=3, conv_out_channels=256,
                 upsample_method='deconv', upsample_ratio=2, num_classes=81, class_agnostic=False, conv_cfg=None,
                 norm_cfg=None, loss_mask=dict(type='CrossEntropyLoss', use_mask=True, loss_weight=1.0)):
        super().__init__()
        if upsample_method not in [None, 'deconv', 'nearest', 'bilinear']:
            raise ValueError('Invalid upsample method {}, accepted methods '
                             'are "deconv", "nearest", "bilinear"'.format(upsample_method))
        self.num_convs = num_convs
        self.roi_feat_size = _pair(roi_feat_size)   # reserved and not used, as in the reference
        self.in_channels = in_channels
        self.conv_kernel_size = conv_kernel_size
        self.conv_out_channels = conv_out_channels
        self.upsample_method = upsample_method
        self.upsample_ratio = upsample_ratio
        self.num_classes = num_classes
        self.class_agnostic = class_agnostic
        self.conv_cfg = conv_cfg
        self.norm_cfg = norm_cfg
        self.fp16_enabled = False
        self.loss_mask = build_loss(loss_mask)

        self.convs = nn.ModuleList()
        for i in range(self.num_convs):
            padding = (self.conv_kernel_size - 1) // 2
            self.convs.append(ConvModule(self.in_channels if i == 0 else self.conv_out_channels,
                                         self.conv_out_channels, self.conv_kernel_size, padding=padding,
                                         conv_cfg=conv_cfg, norm_cfg=norm_cfg))
        upsample_in_channels = self.conv_out_channels if self.num_convs > 0 else in_channels
        if self.upsample_method is None:
            self.upsample = None
        elif self.upsample_method == 'deconv':
            self.upsample = nn.ConvTranspose2d(upsample_in_channels, self.conv_out_channels, self.upsample_ratio,
                                               stride=self.upsample_ratio)
        else:
            self.upsample = nn.Upsample(scale_factor=self.upsample_ratio, mode=self.upsample_method)
        out_channels = 1 if self.class_agnostic else self.num_classes
        logits_in_channel = self.conv_out_channels if self.upsample_method == 'deconv' else upsample_in_channels
        self.conv_logits = nn.Conv2d(logits_in_channel, out_channels, 1)
        self.relu = nn.ReLU(inplace=True)
        self.debug_imgs = None

    def init_weights(self):
        for m in [self.upsample, self.conv_logits]:
            if m is None:
                continue
            nn.init.kaiming_normal_(m.weight, mode='fan_out', nonlinearity='relu')
            nn.init.constant_(m.bias, 0)

    def _logits(self, x):
        """conv_logits(x) -- or, in training with autograd on a GPU, the lazy handle the fused loss consumes."""
        if self.training and torch.is_grad_enabled() and x.is_cuda:
            return MaskPredHandle(self, x)
        return self.conv_logits(x)

    def _upsample(self, x):
        if self.upsample is not None:
            x = self.upsample(x)
            if self.upsample_method == 'deconv':
                x = self.relu(x)
        return x

    @auto_fp16()
    def forward(self, x):
        for conv in self.convs:
            x = conv(x)
        return self._logits(self._upsample(x))

    def get_target(self, sampling_results, gt_masks, rcnn_train_cfg):
        pos_proposals = [res.pos_bboxes for res in sampling_results]
        pos_assigned_gt_inds = [res.pos_assigned_gt_inds for res in sampling_results]
        return mask_target(pos_proposals, pos_assigned_gt_inds, gt_masks, rcnn_train_cfg)

    def _fused_loss_ok(self) -> bool:
        """True for a mask CrossEntropyLoss with reduction 'mean' (recognised by type name and attributes, so mmdet's
        own class qualifies too)."""
        lm = self.loss_mask
        return (type(lm).__name__ == 'CrossEntropyLoss' and getattr(lm, 'use_mask', False) is True
                and not getattr(lm, 'use_sigmoid', False) and getattr(lm, 'reduction', None) == 'mean'
                and isinstance(getattr(lm, 'loss_weight', None), (int, float)))

    @force_fp32(apply_to=('mask_pred', ))
    def loss(self, mask_pred, mask_targets, labels):
        """fcn_mask_head.py:114-123.  An unmaterialised ``MaskPredHandle`` with a 'mean' mask CrossEntropyLoss takes the
        fused route (only each RoI's label channel, ops.MaskBCEFunction); anything else the reference's op sequence on
        the materialised logits."""
        if self.class_agnostic:
            labels = torch.zeros_like(labels)
        if isinstance(mask_pred, MaskPredHandle):
            if mask_pred._pred is None and self._fused_loss_ok():
                lw = self.loss_mask.loss_weight
                loss_mask = ops.MaskBCEFunction.apply(mask_pred.y, self.conv_logits.weight, self.conv_logits.bias,
                                                      labels, mask_targets)
                return dict(loss_mask=loss_mask if lw == 1.0 else loss_mask * lw)
            mask_pred = mask_pred.tensor()
        return dict(loss_mask=self.loss_mask(mask_pred, mask_targets, labels))

    def get_seg_masks(self, mask_pred, det_bboxes, det_labels, rcnn_test_cfg, ori_shape, scale_factor, rescale):
        """fcn_mask_head.py:125-181: masks from the label's channel (channel 0 when class-agnostic)."""
        return seg_masks(mask_pred, det_bboxes, det_labels, rcnn_test_cfg, ori_shape, scale_factor, rescale,
                         self.num_classes, (lambda label: 0) if self.class_agnostic else (lambda label: label))

    def get_seg_masks_without(self, mask_pred, det_bboxes, det_labels, rcnn_test_cfg, ori_shape, scale_factor,
                              rescale):
        """fcn_mask_head.py:183-239: masks from channel 0 whatever the label (HTC's test path calls this variant,
        htc.py:419)."""
        return seg_masks(mask_pred, det_bboxes, det_labels, rcnn_test_cfg, ori_shape, scale_factor, rescale,
                         self.num_classes, lambda label: 0)


class HTCMaskHead(FCNMaskHead):

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.conv_res = ConvModule(self.conv_out_channels, self.conv_out_channels, 1, conv_cfg=self.conv_cfg,
                                   norm_cfg=self.norm_cfg)

    def init_weights(self):
        super().init_weights()
        self.conv_res.init_weights()

    def forward(self, x, res_feat=None, return_logits=True, return_feat=True):
        if res_feat is not None:
            x = x + self.conv_res(res_feat)
        for conv in self.convs:
            x = conv(x)
        res_feat = x
        outs = []
        if return_logits:
            outs.append(self._logits(self._upsample(x)))
        if return_feat:
            outs.append(res_feat)
        return outs if len(outs) > 1 else outs[0]


register(HEADS, FCNMaskHead)
register(HEADS, HTCMaskHead)
