"""FCNMaskHead and HTCMaskHead -- the mask branches of the LVIS mask configs behind the reference's API.

Reference surface mirrored here (constructor kwargs, attributes, ``init_weights``, state-dict keys and method
signatures are identical, so the ``mask_head=dict(type='FCNMaskHead' | 'HTCMaskHead', ...)`` blocks of
configs/bags/gs_mask_rcnn_r50_fpn_1x_lvis.py and configs/bags/gs_htc_*.py build unchanged):

    FCNMaskHead     mmdet/models/mask_heads/fcn_mask_head.py:14-123
    HTCMaskHead     mmdet/models/mask_heads/htc_mask_head.py:7-38
    ConvModule      mmdet/models/utils/conv_module.py (only conv_cfg=None, norm_cfg=None: biased conv, ReLU, kaiming)

The 3x3 convs and the deconv stay ``nn.Conv2d`` / ``nn.ConvTranspose2d``.  What differs is conv_logits: on a GPU, a
training ``forward`` (with autograd) and an eval ``forward`` return a lazy ``MaskPredHandle`` for ``mask_pred``
instead of its [n, num_classes, 28, 28] logits.  ``loss`` computes only the channel of each RoI's label inside its
BCE (``ops.MaskBCEFunction``); at test time ``get_seg_masks`` / ``get_seg_masks_without`` and HTC's
``mask_pred.gather(1, labels)`` compute only each detection's channel (``ops.mask_channel_logits``) when no gradient
is recorded.  Everything else -- a CPU input, a materialised handle, another ``loss_mask``, multi-scale testing's
``mask_pred.sigmoid()`` -- runs the reference's ops on the materialised logits.
"""
from __future__ import annotations

import os

import numpy as np
import torch
import torch.nn as nn
from torch.nn.modules.utils import _pair

from . import ops
from .fp16 import auto_fp16, force_fp32
from .head import _LazyHandle, _as_tensor, _mmdet_core, _pending_input, _weighted
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
    """What a mask head's ``forward`` returns for ``mask_pred`` on a GPU, in training with autograd and in eval.

    It records the input ``y`` of ``conv_logits``, so that its consumers can compute only the channel each RoI or
    detection reads instead of the [n, num_classes, H, W] logits: ``loss`` inside mask_cross_entropy
    (``ops.MaskBCEFunction``), ``seg_masks`` and ``gather`` at test time (``channel_logits``).  ``tensor()`` (or any
    other tensor attribute access, indexing or torch function) materialises them through ``conv_logits``,
    autograd-connected."""

    y = property(lambda self: self.input)          # earlier names, as in ClsScoreHandle
    _pred = property(lambda self: self._out)

    @property
    def shape(self):
        return torch.Size((self.input.shape[0], self._head.conv_logits.out_channels) + tuple(self.input.shape[2:]))

    def _project(self):
        return self._head.conv_logits(self.input)

    def label_only(self) -> bool:
        """True when ``channel_logits`` may stand in for the dense logits: the handle is pending, y is a bf16 or fp32
        CUDA tensor, and autograd would record nothing of conv_logits(y) (grad mode off, or none of y, the weight and
        the bias requires grad)."""
        conv = self._head.conv_logits
        y = self.input
        recorded = torch.is_grad_enabled() and any(t is not None and t.requires_grad
                                                   for t in (y, conv.weight, conv.bias))
        return self.pending and y.is_cuda and y.dtype in (torch.bfloat16, torch.float32) and not recorded

    def channel_logits(self, channels: torch.Tensor) -> torch.Tensor:
        """[n, 1, H, W] logits of channel ``channels[d]`` (int64 [n]) of each row d, without the dense tensor
        (``ops.mask_channel_logits``; NaN for a channel outside [0, num_classes)).  The handle stays pending."""
        conv = self._head.conv_logits
        return ops.mask_channel_logits(self.input, conv.weight, conv.bias, channels)

    def gather(self, dim, index, *, sparse_grad=False, out=None):
        """Tensor.gather on the logits.  HTC's test path (htc.py:403-421) gathers each detection's label channel with
        ``labels.expand(-1, -1, H, W)``: an int64 [n, 1, H, W] index on y's device that is constant along H and W
        (stride 0 or size 1) takes ``channel_logits(index[:, 0, 0, 0])`` when ``label_only()``.  Anything else
        gathers from the materialised logits."""
        y = self.input
        if (dim == 1 and not sparse_grad and out is None and isinstance(index, torch.Tensor)
                and index.dtype == torch.int64 and index.device == y.device and index.dim() == 4
                and index.shape[:2] == (y.shape[0], 1) and index.shape[2:] == y.shape[2:]
                and all(index.stride(i) == 0 or index.size(i) == 1 for i in (2, 3)) and self.label_only()):
            return self.channel_logits(index[:, 0, 0, 0])
        kw = {} if out is None else dict(out=out)
        return torch.gather(self.tensor(), dim, index, sparse_grad=sparse_grad, **kw)

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        """torch.gather(handle, ...) and Tensor.gather(handle, ...) go to ``gather``; every other function sees the
        materialised logits."""
        if func in (torch.gather, torch.Tensor.gather) and args and isinstance(args[0], MaskPredHandle):
            return args[0].gather(*args[1:], **(kwargs or {}))
        return super().__torch_function__(func, types, args, kwargs)


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


def _native_mask_target(pos_proposals_list, gt_masks_list) -> bool:
    """True when ``mask_target`` takes ``ops.mask_targets``: the positive proposals are on a GPU, every gt mask is a
    uint8 [num_gt, H, W] CUDA tensor, and BAGS_MASK_TARGET_NATIVE is not 0."""
    return (os.environ.get('BAGS_MASK_TARGET_NATIVE', '1') != '0' and len(pos_proposals_list) > 0
            and all(isinstance(p, torch.Tensor) and p.is_cuda for p in pos_proposals_list)
            and all(isinstance(m, torch.Tensor) and m.is_cuda and m.dtype == torch.uint8 and m.dim() == 3
                    for m in gt_masks_list))


def mask_target(pos_proposals_list, pos_assigned_gt_inds_list, gt_masks_list, cfg):
    """The mask heads' training targets.  With the proposals and the gt masks on a GPU, ``ops.mask_targets`` builds
    them in one launch, bitwise as the host loop, with no host sync (a gt index outside the image's masks, or a box the
    slicing leaves empty, gives a row of NaN where the host loop raises).  Otherwise mmdet's own ``mask_target`` when
    mmdet is importable, or ``mask_target_single`` per image, concatenated."""
    if _native_mask_target(pos_proposals_list, gt_masks_list):
        return ops.mask_targets(pos_proposals_list, pos_assigned_gt_inds_list, gt_masks_list,
                                _pair(_cfg_get(cfg, 'mask_size')))
    ext = _mmdet_core('mask_target')
    if ext is not None:  # pragma: no cover
        return ext(pos_proposals_list, pos_assigned_gt_inds_list, gt_masks_list, cfg)
    return torch.cat([mask_target_single(p, i, m, cfg) for p, i, m in
                      zip(pos_proposals_list, pos_assigned_gt_inds_list, gt_masks_list)])


def _paste_canvas(ori_shape, scale_factor, rescale):
    """(img_h, img_w, scale_factor) of the image the masks are pasted into (fcn_mask_head.py:164-170)."""
    if rescale:
        img_h, img_w = ori_shape[:2]
    else:
        img_h = np.round(ori_shape[0] * scale_factor).astype(np.int32)
        img_w = np.round(ori_shape[1] * scale_factor).astype(np.int32)
        scale_factor = 1.0
    return img_h, img_w, scale_factor


def _to_host(*tensors):
    """numpy copies of several device tensors through one device-to-host copy (one host sync)."""
    flat = [t.contiguous().reshape(-1).view(torch.uint8) for t in tensors]
    packed = torch.cat(flat).cpu().numpy()
    out, at = [], 0
    for t, f in zip(tensors, flat):
        dtype = torch.empty((), dtype=t.dtype).numpy().dtype
        out.append(packed[at:at + f.numel()].view(dtype).reshape(tuple(t.shape)))
        at += f.numel()
    return out


def seg_masks(mask_pred, det_bboxes, det_labels, rcnn_test_cfg, ori_shape, scale_factor, rescale, num_classes,
              label_channel):
    """COCO-RLE masks per class from the test-time mask logits (fcn_mask_head.py:125-239).  ``mask_pred``: [n, C, h, w]
    logits (a tensor, squashed by a sigmoid) or probabilities (an ndarray, multi-scale testing); det_labels are
    0-based foreground labels, so class k's masks go to list k.  Each detection's probability map is the channel of its
    1-based label (``label_channel``) or channel 0.  It is resized to its box (the box divided by ``scale_factor`` and
    truncated to int32, at least one pixel), thresholded at ``rcnn_test_cfg.mask_thr_binary`` and pasted into an empty
    image of the original size (``rescale``) or of the scaled size.

    With detections on the GPU this runs natively (``ops.seg_masks_rle``; BAGS_SEGM_NATIVE=0 turns it off): same
    masks, no pycocotools, three host syncs whatever n is.  A box that leaves the image takes the host loop, whose numpy
    slicing decides what such a paste gives.

    A ``MaskPredHandle`` (an eval ``forward`` on a GPU) gives only the channel each detection reads
    (``channel_logits``) when ``label_only()``; otherwise its materialised logits."""
    if isinstance(mask_pred, MaskPredHandle):
        if mask_pred.label_only():
            channel = det_labels + 1 if label_channel else torch.zeros_like(det_labels)
            mask_pred = mask_pred.channel_logits(channel.to(mask_pred.device, torch.int64))
            label_channel = False
        else:
            mask_pred = mask_pred.tensor()
    on_gpu = isinstance(mask_pred, np.ndarray) or (isinstance(mask_pred, torch.Tensor) and mask_pred.is_cuda)
    if (os.environ.get('BAGS_SEGM_NATIVE', '1') != '0' and on_gpu and isinstance(det_bboxes, torch.Tensor)
            and det_bboxes.is_cuda):
        boxes, labels = _to_host(det_bboxes[:, :4], det_labels)                # host sync 1
        per_class = _seg_masks_native(mask_pred, det_labels, boxes, labels + 1, rcnn_test_cfg, ori_shape,
                                      scale_factor, rescale, num_classes, label_channel)
        if per_class is not None:
            return per_class
    if isinstance(mask_pred, torch.Tensor):
        mask_pred = mask_pred.sigmoid().cpu().numpy()
    assert isinstance(mask_pred, np.ndarray)
    probs = mask_pred.astype(np.float32)             # fp16 arrays under mixed precision
    per_class = [[] for _ in range(num_classes - 1)]
    boxes = det_bboxes.cpu().numpy()[:, :4]
    labels = det_labels.cpu().numpy() + 1
    img_h, img_w, scale_factor = _paste_canvas(ori_shape, scale_factor, rescale)
    thr = _cfg_get(rcnn_test_cfg, 'mask_thr_binary')
    for k in range(boxes.shape[0]):
        left, top, right, bottom = (boxes[k, :] / scale_factor).astype(np.int32)
        width, height = max(right - left + 1, 1), max(bottom - top + 1, 1)
        resized = _imresize_linear(probs[k, labels[k] if label_channel else 0, :, :], (width, height))
        canvas = np.zeros((img_h, img_w), dtype=np.uint8)
        canvas[top:top + height, left:left + width] = (resized > thr).astype(np.uint8)
        per_class[labels[k] - 1].append(_encode_rle(canvas))
    return per_class


def _seg_masks_native(mask_pred, det_labels, boxes, labels, rcnn_test_cfg, ori_shape, scale_factor, rescale,
                      num_classes, label_channel):
    """seg_masks on the GPU, given the detections' boxes and 1-based labels on the host; None when a box leaves the
    image or the maps have a single row or column (cv2 resizes those by other arithmetic)."""
    if min(mask_pred.shape[-2:]) < 2:
        return None
    img_h, img_w, scale_factor = _paste_canvas(ori_shape, scale_factor, rescale)
    img_h, img_w = int(img_h), int(img_w)
    left, top, right, bottom = (boxes / scale_factor).astype(np.int32).T     # the host loop's expression, per row
    width, height = np.maximum(right - left + 1, 1), np.maximum(bottom - top + 1, 1)
    if ((left < 0) | (top < 0) | (left.astype(np.int64) + width > img_w) | (top.astype(np.int64) + height > img_h)).any():
        return None
    n = boxes.shape[0]
    dev = det_labels.device
    if isinstance(mask_pred, torch.Tensor):
        # the sigmoid is elementwise: these are bitwise the host loop's probabilities, in the logits' dtype first
        channel = det_labels + 1 if label_channel else torch.zeros_like(det_labels)
        probs = mask_pred[torch.arange(n, device=dev), channel].sigmoid().float()
    else:
        channel = labels if label_channel else np.zeros_like(labels)
        probs = torch.from_numpy(mask_pred[np.arange(n), channel].astype(np.float32)).to(dev, non_blocking=True)
    # ``resized > thr`` compares in numpy's promoted type: float32 for a Python float, float64 for np.float64
    thr = _cfg_get(rcnn_test_cfg, 'mask_thr_binary')
    thr = float(np.asarray(thr).astype(np.result_type(np.float32, thr)))
    counts = ops.seg_masks_rle(probs, np.stack([left, top, width, height], 1), img_h, img_w, thr)   # host syncs 2, 3
    per_class = [[] for _ in range(num_classes - 1)]
    for label, rle in zip(labels.tolist(), counts):
        per_class[label - 1].append({'size': [img_h, img_w], 'counts': rle})
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
        """conv_logits(x) -- or, on a GPU, the lazy handle: in training with autograd for the fused loss, in eval for the
        label-only test-time logits of seg_masks and MaskPredHandle.gather."""
        if x.is_cuda and (not self.training or torch.is_grad_enabled()):
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
        y = _pending_input(mask_pred)
        if y is not None and self._fused_loss_ok():
            loss_mask = ops.MaskBCEFunction.apply(y, self.conv_logits.weight, self.conv_logits.bias, labels, mask_targets)
            return dict(loss_mask=_weighted(loss_mask, self.loss_mask.loss_weight))
        return dict(loss_mask=self.loss_mask(_as_tensor(mask_pred), mask_targets, labels))

    def get_seg_masks(self, mask_pred, det_bboxes, det_labels, rcnn_test_cfg, ori_shape, scale_factor, rescale):
        """fcn_mask_head.py:125-181: masks from the label's channel (channel 0 when class-agnostic)."""
        return seg_masks(mask_pred, det_bboxes, det_labels, rcnn_test_cfg, ori_shape, scale_factor, rescale,
                         self.num_classes, not self.class_agnostic)

    def get_seg_masks_without(self, mask_pred, det_bboxes, det_labels, rcnn_test_cfg, ori_shape, scale_factor,
                              rescale):
        """fcn_mask_head.py:183-239: masks from channel 0 whatever the label (HTC's test path calls this variant,
        htc.py:419)."""
        return seg_masks(mask_pred, det_bboxes, det_labels, rcnn_test_cfg, ori_shape, scale_factor, rescale,
                         self.num_classes, False)


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
