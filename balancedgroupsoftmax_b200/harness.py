"""Synthetic-image detector harness around the BAGS head -- the CALLER of the hot path.

The reference's detectors (``TwoStageDetector.forward_train`` mmdet/models/detectors/two_stage.py:134-265,
``CascadeRCNN`` cascade_rcnn.py:152-298) feed the head like this, per image batch:

    backbone + FPN -> RPN proposals -> assign + sample 512 RoIs / image (25 % positives, gt boxes added)
    -> RoIAlign 7x7 -> head.forward -> head.get_target -> head.loss            (x 3 heads with refined boxes: cascade)

mmdetection / mmcv cannot be installed here, torchvision can: the trunk (ResNet-FPN, RPN, MultiScaleRoIAlign) is
torchvision's, FROZEN and untrained -- it only has to produce RoI features of the real shape ([N,256,7,7]) at the real
cost, so that the head's share of a detector step and full-detector images/s can be measured (tools/bench_detector.py).
Everything from the sampled RoIs onward is this repository's head: ``forward`` -> ``get_target`` -> ``loss`` ->
backward -> gradient exchange.  Not part of the hot path; no CUDA code here.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from .head import GSBBoxHeadWith0
from .tables import GroupTables


def box_iou_plus1(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """IoU with the reference's legacy "+1" box widths (mmdet/core/bbox/geometry.py:4-63), [len(a), len(b)]."""
    if a.numel() == 0 or b.numel() == 0:
        return a.new_zeros((a.size(0), b.size(0)))
    lt = torch.max(a[:, None, :2], b[None, :, :2])
    rb = torch.min(a[:, None, 2:], b[None, :, 2:])
    wh = (rb - lt + 1).clamp(min=0)
    inter = wh[..., 0] * wh[..., 1]
    area_a = (a[:, 2] - a[:, 0] + 1) * (a[:, 3] - a[:, 1] + 1)
    area_b = (b[:, 2] - b[:, 0] + 1) * (b[:, 3] - b[:, 1] + 1)
    return inter / (area_a[:, None] + area_b[None, :] - inter)


def sample_rois(proposals: torch.Tensor, gt_boxes: torch.Tensor, gt_labels: torch.Tensor, num: int = 512,
                pos_fraction: float = 0.25, pos_iou_thr: float = 0.5, neg_iou_thr: float = 0.5,
                add_gt_as_proposals: bool = True, generator: Optional[torch.Generator] = None) -> SimpleNamespace:
    """One image's RoI assignment + sampling, restating what the shipped configs ask of mmdet
    (``MaxIoUAssigner(pos_iou_thr=.5, neg_iou_thr=.5, min_pos_iou=.5)`` core/bbox/assigners/max_iou_assigner.py:7-152 and
    ``RandomSampler(num=512, pos_fraction=.25, neg_pos_ub=-1, add_gt_as_proposals=True)``
    core/bbox/samplers/base_sampler.py:30-78, random_sampler.py): gt boxes join the proposals, a proposal is positive
    when its best IoU >= pos_iou_thr (label = that gt's label), negative when < neg_iou_thr; up to num*pos_fraction
    positives and the rest negatives are drawn uniformly.  Returns the ``SamplingResult`` fields the head consumes
    (pos_bboxes, neg_bboxes, pos_gt_bboxes, pos_gt_labels, pos_is_gt)."""
    boxes = proposals[:, :4]
    is_gt = boxes.new_zeros(boxes.size(0), dtype=torch.bool)
    if add_gt_as_proposals and gt_boxes.numel() > 0:
        boxes = torch.cat([gt_boxes, boxes], 0)
        is_gt = torch.cat([is_gt.new_ones(gt_boxes.size(0)), is_gt], 0)
    if gt_boxes.numel() > 0:
        iou = box_iou_plus1(boxes, gt_boxes)
        best, arg = iou.max(1)
    else:
        best = boxes.new_zeros(boxes.size(0))
        arg = boxes.new_zeros(boxes.size(0), dtype=torch.long)
    pos_idx = torch.nonzero(best >= pos_iou_thr, as_tuple=False).squeeze(1)
    neg_idx = torch.nonzero(best < neg_iou_thr, as_tuple=False).squeeze(1)

    def choose(idx: torch.Tensor, k: int) -> torch.Tensor:
        if idx.numel() <= k:
            return idx
        perm = torch.randperm(idx.numel(), generator=generator, device='cpu')[:k].to(idx.device)
        return idx[perm]

    pos_idx = choose(pos_idx, int(num * pos_fraction))
    neg_idx = choose(neg_idx, num - pos_idx.numel())
    return SimpleNamespace(pos_bboxes=boxes[pos_idx], neg_bboxes=boxes[neg_idx], pos_gt_bboxes=gt_boxes[arg[pos_idx]],
                           pos_gt_labels=gt_labels[arg[pos_idx]], pos_is_gt=is_gt[pos_idx].to(torch.uint8))


class TorchvisionTrunk(nn.Module):
    """Frozen torchvision Faster R-CNN trunk: image normalisation / resize, ResNet-FPN, RPN proposals, RoIAlign 7x7."""

    def __init__(self, backbone: str = 'resnet50', min_size: int = 800, max_size: int = 1333,
                 proposals_per_image: int = 2000):
        super().__init__()
        from torchvision.models.detection import fasterrcnn_resnet50_fpn
        if backbone != 'resnet50':
            raise NotImplementedError('only the R50-FPN trunk is wired up (configs[2]); got %r' % backbone)
        m = fasterrcnn_resnet50_fpn(weights=None, weights_backbone=None, num_classes=2, min_size=min_size, max_size=max_size,
                                    rpn_post_nms_top_n_test=proposals_per_image,
                                    rpn_pre_nms_top_n_test=max(proposals_per_image, 2000))
        self.transform, self.backbone, self.rpn = m.transform, m.backbone, m.rpn
        self.box_roi_pool = m.roi_heads.box_roi_pool
        for p in self.parameters():
            p.requires_grad_(False)
        self.eval()

    def train(self, mode: bool = True):   # the trunk stays in eval mode (frozen BN, test-time RPN)
        return super().train(False)

    @torch.no_grad()
    def forward(self, images: Sequence[torch.Tensor]):
        """-> (FPN features, proposals per image [k,4] in resized-image coordinates, image sizes, scale factors)."""
        il, _ = self.transform(list(images), None)
        feats = self.backbone(il.tensors)
        proposals, _ = self.rpn(il, feats)
        scales = [il.image_sizes[i][0] / float(img.shape[-2]) for i, img in enumerate(images)]
        return feats, proposals, il.image_sizes, scales

    @torch.no_grad()
    def roi_features(self, feats: Dict[str, torch.Tensor], boxes: List[torch.Tensor], image_sizes) -> torch.Tensor:
        x = self.box_roi_pool(feats, boxes, image_sizes)
        # The trunk is untrained (no checkpoints in the image): fifty randomly initialised layers with identity batch-norm
        # statistics overflow, so its RoI features are not O(1) like a trained detector's.  Standardise every RoI's
        # feature block (and drop non-finite values) -- shape and cost are what the harness needs from the trunk.
        x = torch.nan_to_num(x.float(), nan=0.0, posinf=0.0, neginf=0.0)
        mu = x.mean(dim=(1, 2, 3), keepdim=True)
        sd = x.std(dim=(1, 2, 3), keepdim=True)
        return torch.relu((x - mu) / (sd + 1e-6))


class BagsDetectorHarness(nn.Module):
    """Frozen trunk + 1 (Faster R-CNN style) or 3 (cascade style) BAGS heads, trained on synthetic images.

    ``forward_train(images, gt_boxes, gt_labels)`` returns the loss dict of the reference's detectors
    (``loss_cls_bin0..4``, ``loss_bbox``; prefixed ``s{i}.`` and scaled by ``stage_loss_weights`` with several
    stages, cascade_rcnn.py:246-250)."""

    def __init__(self, tables: GroupTables, num_stages: int = 1, stage_loss_weights: Sequence[float] = (1.0,),
                 rois_per_image: int = 512, pos_fraction: float = 0.25, stage_iou_thrs: Sequence[float] = (0.5, 0.6, 0.7),
                 trunk: Optional[nn.Module] = None, fc_out_channels: int = 1024, compute_dtype: str = 'bf16',
                 reg_class_agnostic: bool = False, amp: bool = True, **trunk_kwargs):
        super().__init__()
        assert len(stage_loss_weights) == num_stages
        self.trunk = trunk if trunk is not None else TorchvisionTrunk(**trunk_kwargs)
        self.num_stages = num_stages
        self.stage_loss_weights = [float(w) for w in stage_loss_weights]
        self.stage_iou_thrs = [float(t) for t in stage_iou_thrs]
        self.rois_per_image, self.pos_fraction = rois_per_image, pos_fraction
        # shared FCs / fc_reg under bf16 autocast (cuBLAS; 11x the fc_cls FLOPs): the BAGS part takes the
        # bf16 activations as they come
        self.amp = bool(amp)
        # several stages regress class-agnostically, like the cascade configs (configs/bags/gs_cascade_*.py)
        agnostic = reg_class_agnostic or num_stages > 1
        stds = [[0.1, 0.1, 0.2, 0.2], [0.05, 0.05, 0.1, 0.1], [0.033, 0.033, 0.067, 0.067]]
        self.heads = nn.ModuleList([
            GSBBoxHeadWith0(num_fcs=2, in_channels=256, fc_out_channels=fc_out_channels, roi_feat_size=7,
                            num_classes=tables.num_classes, target_means=[0., 0., 0., 0.],
                            target_stds=stds[i if num_stages > 1 else 0], reg_class_agnostic=agnostic,
                            gs_config=dict(tables=tables, others_sample_ratio=8.0, num_bins=tables.num_bins,
                                           compute_dtype=compute_dtype,
                                           loss_bin=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0)))
            for i in range(num_stages)])
        for h in self.heads:
            h.init_weights()
        self.rcnn_cfg = dict(pos_weight=-1)
        self.generator = torch.Generator().manual_seed(0)

    def head_parameters(self):
        return [p for h in self.heads for p in h.parameters() if p.requires_grad]

    def head_inputs(self, feats, rois: List[torch.Tensor], gt_boxes, gt_labels, image_sizes, stage: int = 0):
        """The data either side of the path for one stage: sampled RoIs -> (x [N,256,7,7], sampling results)."""
        thr = self.stage_iou_thrs[stage] if self.num_stages > 1 else 0.5
        sampling = [sample_rois(r, gb, gl, self.rois_per_image, self.pos_fraction, thr, thr, generator=self.generator)
                    for r, gb, gl in zip(rois, gt_boxes, gt_labels)]
        boxes = [torch.cat([s.pos_bboxes, s.neg_bboxes], 0) for s in sampling]
        x = self.trunk.roi_features(feats, boxes, image_sizes)
        return x, sampling, boxes

    def run_head(self, head, x):
        if self.amp and x.is_cuda:
            with torch.autocast('cuda', dtype=torch.bfloat16):
                return head(x)
        return head(x)

    def forward_train(self, images: Sequence[torch.Tensor], gt_boxes: List[torch.Tensor], gt_labels: List[torch.Tensor]
                      ) -> Dict[str, torch.Tensor]:
        feats, proposals, image_sizes, scales = self.trunk(images)
        gt_boxes = [g * s for g, s in zip(gt_boxes, scales)]          # gt boxes follow the trunk's resize
        losses: Dict[str, torch.Tensor] = {}
        rois = proposals
        for i, head in enumerate(self.heads):
            x, sampling, boxes = self.head_inputs(feats, rois, gt_boxes, gt_labels, image_sizes, i)
            cls_score, bbox_pred = self.run_head(head, x)
            targets = head.get_target(sampling, gt_boxes, gt_labels, self.rcnn_cfg)
            stage_losses = head.loss(cls_score, bbox_pred, *targets)
            lw = self.stage_loss_weights[i]
            for k, v in stage_losses.items():
                losses[('s%d.%s' % (i, k)) if self.num_stages > 1 else k] = v * lw
            if i + 1 < self.num_stages:       # next stage trains on this stage's refined boxes (cascade_rcnn.py:253-262)
                with torch.no_grad():
                    batch_rois = torch.cat([torch.cat([b.new_full((b.size(0), 1), j), b], 1) for j, b in enumerate(boxes)], 0)
                    pos_is_gts = [s.pos_is_gt for s in sampling]
                    metas = [dict(img_shape=(int(sz[0]), int(sz[1]), 3)) for sz in image_sizes]
                    rois = head.refine_bboxes(batch_rois, targets[0], bbox_pred.detach().float(), pos_is_gts, metas)
        return losses


def synthetic_batch(imgs_per_gpu: int = 2, height: int = 800, width: int = 1333, gts_per_image: int = 12,
                    num_classes: int = 1231, device='cpu', generator: Optional[torch.Generator] = None
                    ) -> Tuple[List[torch.Tensor], List[torch.Tensor], List[torch.Tensor]]:
    """Random images with random ground-truth boxes / LVIS-range labels (there is no dataset in the image)."""
    g = generator if generator is not None else torch.Generator().manual_seed(0)
    images, boxes, labels = [], [], []
    for _ in range(imgs_per_gpu):
        images.append(torch.rand(3, height, width, generator=g).to(device))
        xy = torch.rand(gts_per_image, 2, generator=g) * torch.tensor([width * 0.7, height * 0.7])
        wh = torch.rand(gts_per_image, 2, generator=g) * torch.tensor([width * 0.25, height * 0.25]) + 16.0
        b = torch.cat([xy, xy + wh], 1)
        b[:, 2].clamp_(max=width - 1)
        b[:, 3].clamp_(max=height - 1)
        boxes.append(b.to(device))
        labels.append(torch.randint(1, num_classes, (gts_per_image,), generator=g).to(device))
    return images, boxes, labels
