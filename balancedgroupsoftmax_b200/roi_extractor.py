"""The FPN RoI feature extractor: SingleRoIExtractor and its RoIAlign layer on native kernels.

Drop-in for mmdet/models/roi_extractors/single_level.py and mmdet/ops/roi_align/roi_align.py: the same constructors,
attributes and methods, so every ``bbox_roi_extractor``, ``mask_roi_extractor`` and ``semantic_roi_extractor`` block
of the LVIS configs builds unchanged.  ``SingleRoIExtractor.forward`` is one bags_roi_align_fwd launch for every
level and image, with the levels mapped on the device (no host sync, capturable in a CUDA graph), and its backward
one bags_roi_align_bwd launch (see ops.RoIAlignFunction).  The forward equals the reference's loop over levels on its
own op bit for bit; where the reference is undefined it gives a zero row: a RoI whose level scale is NaN (a box with
exactly one negative side), or whose batch index lies outside [0, B).  CUDA tensors only.
"""
from __future__ import annotations

import torch
import torch.nn as nn
from torch.nn.modules.utils import _pair

from . import _native as nat
from . import ops
from .fp16 import force_fp32
from .registry import ROI_EXTRACTORS, register


def roi_align(features, rois, out_size, spatial_scale, sample_num=0):
    """mmdet.ops.roi_align.roi_align on one feature map: fp32 [k, C, out_h, out_w], every RoI pooled from
    ``features`` (no level mapping)."""
    out_h, out_w = _pair(out_size)
    assert isinstance(out_h, int) and isinstance(out_w, int)
    spec = ops.RoIAlignSpec((out_h, out_w), (float(spatial_scale),), int(sample_num))
    return ops.roi_align_apply([features], rois, spec)


class RoIAlign(nn.Module):
    """mmdet/ops/roi_align/roi_align.py:RoIAlign; ``use_torchvision=True`` calls torchvision's roi_align, as the
    reference does."""

    def __init__(self, out_size, spatial_scale, sample_num=0, use_torchvision=False):
        super(RoIAlign, self).__init__()
        self.out_size = _pair(out_size)   # as the reference: (h, w)
        self.spatial_scale = float(spatial_scale)
        self.sample_num = int(sample_num)
        self.use_torchvision = use_torchvision

    def forward(self, features, rois):
        if self.use_torchvision:
            from torchvision.ops import roi_align as tv_roi_align
            return tv_roi_align(features, rois, self.out_size, self.spatial_scale, self.sample_num)
        return roi_align(features, rois, self.out_size, self.spatial_scale, self.sample_num)

    def __repr__(self):
        return '%s(out_size=%s, spatial_scale=%s, sample_num=%s, use_torchvision=%s)' % (
            type(self).__name__, self.out_size, self.spatial_scale, self.sample_num, self.use_torchvision)


class SingleRoIExtractor(nn.Module):
    """RoI features from an FPN: each RoI is pooled by RoIAlign from the level its size maps it to (``map_roi_levels``;
    a single input level is used as it is).  Constructor, attributes and methods as mmdet's SingleRoIExtractor;
    ``roi_layer`` must be a RoIAlign dict (out_size, sample_num), ``featmap_strides`` gives one spatial_scale per level
    (1 / stride) and ``finest_scale`` the RoI size mapped to the boundary of level 0 and 1 (at 2 x finest_scale)."""

    def __init__(self, roi_layer, out_channels, featmap_strides, finest_scale=56):
        super(SingleRoIExtractor, self).__init__()
        self.roi_layers = self.build_roi_layers(roi_layer, featmap_strides)
        self.out_channels = out_channels
        self.featmap_strides = featmap_strides
        self.finest_scale = finest_scale
        self.fp16_enabled = False

    @property
    def num_inputs(self):
        return len(self.featmap_strides)

    def init_weights(self):
        pass

    def build_roi_layers(self, layer_cfg, featmap_strides):
        kwargs = dict(layer_cfg)
        kind = kwargs.pop('type')
        if kind != 'RoIAlign':
            raise NotImplementedError('SingleRoIExtractor: roi_layer type %r has no native kernel (RoIAlign only)'
                                      % (kind,))
        return nn.ModuleList(RoIAlign(spatial_scale=1 / stride, **kwargs) for stride in featmap_strides)

    def map_roi_levels(self, rois, num_levels):
        """[k] int64 level of each RoI [k, 5]: floor(log2(sqrt(w h) / finest_scale + 1e-6)) clamped to the levels, with
        w and h counted inclusively (x2 - x1 + 1).  These are the torch ops the reference runs; ``forward`` maps the
        RoIs on the device with the same fp32 rounding."""
        w = rois[:, 3] - rois[:, 1] + 1
        h = rois[:, 4] - rois[:, 2] + 1
        lvl = torch.floor(torch.log2(torch.sqrt(w * h) / self.finest_scale + 1e-6))
        return lvl.clamp(min=0, max=num_levels - 1).long()

    def roi_rescale(self, rois, scale_factor):
        """The RoIs [k, 5] scaled by ``scale_factor`` about their centres (inclusive widths), batch index kept."""
        x1, y1, x2, y2 = rois[:, 1], rois[:, 2], rois[:, 3], rois[:, 4]
        cx, cy = (x1 + x2) * 0.5, (y1 + y2) * 0.5
        half_w = (x2 - x1 + 1) * scale_factor * 0.5
        half_h = (y2 - y1 + 1) * scale_factor * 0.5
        return torch.stack((rois[:, 0], cx - half_w + 0.5, cy - half_h + 0.5, cx + half_w - 0.5, cy + half_h - 0.5),
                           dim=-1)

    @force_fp32(apply_to=('feats', ), out_fp16=True)
    def forward(self, feats, rois, roi_scale_factor=None):
        if len(feats) == 1:
            return self.roi_layers[0](feats[0], rois)
        if any(layer.use_torchvision for layer in self.roi_layers):
            raise NotImplementedError('SingleRoIExtractor: use_torchvision with several levels')
        for f in feats:
            if f.dim() != 4 or f.shape[1] != self.out_channels:
                raise nat.BagsNativeError('SingleRoIExtractor: features must be [B, %d, H, W] (got %s)'
                                          % (self.out_channels, tuple(f.shape)))
        layer = self.roi_layers[0]
        spec = ops.RoIAlignSpec(layer.out_size, tuple(lr.spatial_scale for lr in self.roi_layers[:len(feats)]),
                                layer.sample_num, float(self.finest_scale))
        pooled = rois if roi_scale_factor is None else self.roi_rescale(rois, roi_scale_factor)
        return ops.roi_align_apply(list(feats), pooled, spec, rois_map=rois)


register(ROI_EXTRACTORS, SingleRoIExtractor)
