"""Restatement of the reference's RPN proposal loop in torch (RPNHead.get_bboxes_single, rpn_head.py:55-104, with
delta2bbox of transforms.py:34-111 and grid_anchors of anchor_generator.py) -- TEST INFRASTRUCTURE.

The NMS is injected: ``nms(dets, thr) -> (dets[inds], inds)``, the kept rows in input order, as mmdet/ops/nms returns
them.  Ties follow the rule the native route pins: top-k and the final merge take (score desc, index asc), which a
stable descending sort gives, and greedy_nms visits (score desc, input position asc).  On tie-free inputs that is the
reference's own order.
"""
import numpy as np
import torch

from oracle.bags_oracle import iou_plus1_fp32


def grid_anchors(base, H, W, stride, device='cpu'):
    """anchor_generator.py:grid_anchors: base [A, 4] + (w stride, h stride), location-major."""
    base = torch.as_tensor(base, dtype=torch.float32).to(device)
    sx = torch.arange(0, W, device=device) * stride
    sy = torch.arange(0, H, device=device) * stride
    xx, yy = sx.repeat(len(sy)), sy.view(-1, 1).repeat(1, len(sx)).view(-1)
    shifts = torch.stack([xx, yy, xx, yy], dim=-1).type_as(base)
    return (base[None, :, :] + shifts[:, None, :]).view(-1, 4)


def delta2bbox(rois, deltas, means=(0, 0, 0, 0), stds=(1, 1, 1, 1), max_shape=None, wh_ratio_clip=16 / 1000):
    """The reference's delta2bbox, op for op (addcmul included)."""
    means = deltas.new_tensor(means).repeat(1, deltas.size(1) // 4)
    stds = deltas.new_tensor(stds).repeat(1, deltas.size(1) // 4)
    d = deltas * stds + means
    dx, dy, dw, dh = d[:, 0::4], d[:, 1::4], d[:, 2::4], d[:, 3::4]
    max_ratio = np.abs(np.log(wh_ratio_clip))
    dw = dw.clamp(min=-max_ratio, max=max_ratio)
    dh = dh.clamp(min=-max_ratio, max=max_ratio)
    px = ((rois[:, 0] + rois[:, 2]) * 0.5).unsqueeze(1).expand_as(dx)
    py = ((rois[:, 1] + rois[:, 3]) * 0.5).unsqueeze(1).expand_as(dy)
    pw = (rois[:, 2] - rois[:, 0] + 1.0).unsqueeze(1).expand_as(dw)
    ph = (rois[:, 3] - rois[:, 1] + 1.0).unsqueeze(1).expand_as(dh)
    gw = pw * dw.exp()
    gh = ph * dh.exp()
    gx = torch.addcmul(px, pw, dx, value=1)
    gy = torch.addcmul(py, ph, dy, value=1)
    x1 = gx - gw * 0.5 + 0.5
    y1 = gy - gh * 0.5 + 0.5
    x2 = gx + gw * 0.5 - 0.5
    y2 = gy + gh * 0.5 - 0.5
    if max_shape is not None:
        x1 = x1.clamp(min=0, max=max_shape[1] - 1)
        y1 = y1.clamp(min=0, max=max_shape[0] - 1)
        x2 = x2.clamp(min=0, max=max_shape[1] - 1)
        y2 = y2.clamp(min=0, max=max_shape[0] - 1)
    return torch.stack([x1, y1, x2, y2], dim=-1).view_as(deltas)


def _desc(scores):
    """Indices of ``scores`` by (score desc, index asc); NaN first, as torch's sort."""
    return torch.sort(scores, descending=True, stable=True)[1]


def greedy_nms(dets, thr):
    """CPU stand-in for mmdet/ops/nms: greedy over (score desc, input position asc) with the op's fp32 "+1" IoU,
    suppressing IoU > thr; returns (dets[inds], inds) with the kept indices ascending, as the op does."""
    if dets.shape[0] == 0:
        inds = torch.zeros(0, dtype=torch.long)
        return dets[inds], inds
    order = _desc(dets[:, 4].cpu()).numpy()
    boxes = dets[:, :4].detach().cpu().numpy().astype(np.float32)[order]
    removed = np.zeros(len(order), dtype=bool)
    keep = []
    for i in range(len(order)):
        if removed[i]:
            continue
        keep.append(order[i])
        removed[i + 1:] |= iou_plus1_fp32(boxes[i], boxes[i + 1:]) > np.float32(thr)
    inds = torch.as_tensor(sorted(keep), dtype=torch.long)
    return dets[inds.to(dets.device)], inds


def get_bboxes_single(cls_scores, bbox_preds, mlvl_anchors, img_shape, cfg, nms, means=(0, 0, 0, 0),
                      stds=(1, 1, 1, 1)):
    """rpn_head.py:get_bboxes_single for a sigmoid RPN with nms_across_levels=False, on [A, H, W] scores and
    [4A, H, W] deltas per level; ``cfg`` a dict.  Unlike the reference, exactly one box left by min_bbox_size stays
    a [1, 4] row."""
    mlvl = []
    for s, d, anchors in zip(cls_scores, bbox_preds, mlvl_anchors):
        scores = s.permute(1, 2, 0).reshape(-1).sigmoid()
        d = d.permute(1, 2, 0).reshape(-1, 4)
        if cfg['nms_pre'] > 0 and scores.shape[0] > cfg['nms_pre']:
            inds = _desc(scores)[:cfg['nms_pre']]
            d, anchors, scores = d[inds, :], anchors[inds, :], scores[inds]
        proposals = delta2bbox(anchors, d, means, stds, img_shape)
        if cfg['min_bbox_size'] > 0:
            w = proposals[:, 2] - proposals[:, 0] + 1
            h = proposals[:, 3] - proposals[:, 1] + 1
            valid = torch.nonzero((w >= cfg['min_bbox_size']) & (h >= cfg['min_bbox_size'])).view(-1)
            proposals, scores = proposals[valid, :], scores[valid]
        proposals = torch.cat([proposals, scores.unsqueeze(-1)], dim=-1)
        proposals, _ = nms(proposals, cfg['nms_thr'])
        mlvl.append(proposals[:cfg['nms_post'], :])
    proposals = torch.cat(mlvl, 0)
    num = min(cfg['max_num'], proposals.shape[0])
    return proposals[_desc(proposals[:, 4])[:num], :]


def get_bboxes(cls_scores, bbox_preds, base_anchors, strides, img_shapes, cfg, nms, means=(0, 0, 0, 0),
               stds=(1, 1, 1, 1)):
    """The per-image loop of anchor_head.py:get_bboxes over [B, A, H, W] / [B, 4A, H, W] levels."""
    dev = cls_scores[0].device
    anchors = [grid_anchors(b, s.shape[2], s.shape[3], st, dev) for b, s, st in zip(base_anchors, cls_scores, strides)]
    return [get_bboxes_single([s[i] for s in cls_scores], [d[i] for d in bbox_preds], anchors, img_shapes[i], cfg,
                              nms, means, stds) for i in range(cls_scores[0].shape[0])]
