"""Restatement of the RPN's training targets in torch -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

``anchor_target`` / ``anchor_target_single`` restate mmdet/core/anchor/anchor_target.py with MaxIoUAssigner.assign
(core/bbox/assigners/max_iou_assigner.py, its >50-gt CPU route included), the base sampler
(core/bbox/samplers/base_sampler.py) and bbox2delta (core/bbox/transforms.py), for an RPN (no gt labels, sampling,
add_gt_as_proposals=False).  The draw is injectable: ``numpy_shuffle`` is RandomSampler.random_choice (np.random.shuffle
of the whole gallery), ``native_rule(seed)`` is the rule of ops.anchor_targets, restated in numpy by ``native_select``:
key(n) = (sample_key(seed, image, n) << 32) | n over the image's flat anchor index n, and the k smallest keys.

Every op is a torch op on the tensors' device, so run on CUDA it is what the reference computes there.
"""
from __future__ import annotations

import numpy as np
import torch

import sampler_oracle as S


def grid_anchors(base, H, W, stride, device):
    """AnchorGenerator.grid_anchors: [H W A, 4], location-major."""
    base = base.to(device)
    sx = torch.arange(0, W, device=device) * stride
    sy = torch.arange(0, H, device=device) * stride
    xx, yy = sx.repeat(len(sy)), sy.view(-1, 1).repeat(1, len(sx)).view(-1)
    shifts = torch.stack([xx, yy, xx, yy], dim=-1).type_as(base)
    return (base[None, :, :] + shifts[:, None, :]).view(-1, 4)


def valid_flags(H, W, A, vh, vw, device):
    """AnchorGenerator.valid_flags of a (vh, vw) valid region of an H x W map."""
    vx = torch.zeros(W, dtype=torch.uint8, device=device)
    vy = torch.zeros(H, dtype=torch.uint8, device=device)
    vx[:vw] = 1
    vy[:vh] = 1
    v = vx.repeat(len(vy)) & vy.view(-1, 1).repeat(1, len(vx)).view(-1)
    return v[:, None].expand(v.size(0), A).contiguous().view(-1)


def multi_level(bases, sizes, strides, pad_shape, device):
    """(anchors, valid flags) of one image, concatenated over levels as anchor_target concatenates them."""
    anchors, flags = [], []
    for base, (H, W), s in zip(bases, sizes, strides):
        anchors.append(grid_anchors(base, H, W, s, device))
        vh = min(int(np.ceil(pad_shape[0] / s)), H)
        vw = min(int(np.ceil(pad_shape[1] / s)), W)
        flags.append(valid_flags(H, W, base.shape[0], vh, vw, device))
    return torch.cat(anchors), torch.cat(flags)


def inside_flags(anchors, valid, img_shape, allowed_border):
    h, w = img_shape[:2]
    if allowed_border < 0:
        return valid
    return valid & (anchors[:, 0] >= -allowed_border).type(torch.uint8) & \
        (anchors[:, 1] >= -allowed_border).type(torch.uint8) & \
        (anchors[:, 2] < w + allowed_border).type(torch.uint8) & (anchors[:, 3] < h + allowed_border).type(torch.uint8)


def bbox_overlaps(b1, b2):
    """geometry.py bbox_overlaps, mode 'iou', not aligned: [rows, cols]."""
    lt = torch.max(b1[:, None, :2], b2[:, :2])
    rb = torch.min(b1[:, None, 2:], b2[:, 2:])
    wh = (rb - lt + 1).clamp(min=0)
    overlap = wh[:, :, 0] * wh[:, :, 1]
    area1 = (b1[:, 2] - b1[:, 0] + 1) * (b1[:, 3] - b1[:, 1] + 1)
    area2 = (b2[:, 2] - b2[:, 0] + 1) * (b2[:, 3] - b2[:, 1] + 1)
    return overlap / (area1[:, None] + area2 - overlap)


def assign(anchors, gts, a):
    """MaxIoUAssigner.assign (no ignored gts, no labels): assigned_gt_inds on the anchors' device.  Above 50 gts the
    reference computes on the CPU; ``a['cpu_above'] = None`` keeps every size on the anchors' device."""
    if anchors.shape[0] == 0 or gts.shape[0] == 0:
        raise ValueError('No gt or bboxes')
    dev = anchors.device
    cut = a.get('cpu_above', 50)
    if cut is not None and gts.shape[0] > cut:
        anchors, gts = anchors.cpu(), gts.cpu()
    overlaps = bbox_overlaps(gts, anchors[:, :4])
    G, N = overlaps.shape
    out = overlaps.new_full((N,), -1, dtype=torch.long)
    max_o, arg_o = overlaps.max(dim=0)
    gt_max, gt_arg = overlaps.max(dim=1)
    neg = a['neg_iou_thr']
    if isinstance(neg, float):
        out[(max_o >= 0) & (max_o < neg)] = 0
    elif isinstance(neg, tuple):
        out[(max_o >= neg[0]) & (max_o < neg[1])] = 0
    pos = max_o >= a['pos_iou_thr']
    out[pos] = arg_o[pos] + 1
    for i in range(G):
        if gt_max[i] >= a.get('min_pos_iou', 0.0):
            if a.get('gt_max_assign_all', True):
                out[overlaps[i, :] == gt_max[i]] = i + 1
            else:
                out[gt_arg[i]] = i + 1
    return out.to(dev)


def bbox2delta(proposals, gt, means, stds):
    px = (proposals[..., 0] + proposals[..., 2]) * 0.5
    py = (proposals[..., 1] + proposals[..., 3]) * 0.5
    pw = proposals[..., 2] - proposals[..., 0] + 1.0
    ph = proposals[..., 3] - proposals[..., 1] + 1.0
    gx = (gt[..., 0] + gt[..., 2]) * 0.5
    gy = (gt[..., 1] + gt[..., 3]) * 0.5
    gw = gt[..., 2] - gt[..., 0] + 1.0
    gh = gt[..., 3] - gt[..., 1] + 1.0
    d = torch.stack([(gx - px) / pw, (gy - py) / ph, torch.log(gw / pw), torch.log(gh / ph)], dim=-1)
    return d.sub_(d.new_tensor(means).unsqueeze(0)).div_(d.new_tensor(stds).unsqueeze(0))


# ------------------------------------------------------------------------------------------------------- the draws
def numpy_shuffle(gallery, num, flat, img):
    """RandomSampler.random_choice."""
    cands = np.arange(len(gallery))
    np.random.shuffle(cands)
    return gallery[torch.from_numpy(cands[:num]).long().to(gallery.device)]


def native_select(seed, img, flat, k):
    """The native rule in numpy: the k of the flat anchor indices ``flat`` with the smallest
    (sample_key(seed, img, n) << 32) | n."""
    flat = np.asarray(flat, dtype=np.int64)
    if k <= 0:
        return flat[:0]
    key = (S.keys(seed, img, flat).astype(np.uint64) << np.uint64(32)) | flat.astype(np.uint64)
    return flat[np.argsort(key, kind='stable')[:k]]


def native_rule(seed):
    """A draw for ``anchor_target`` that picks as ops.anchor_targets does (``seed`` the effective seed)."""
    def draw(gallery, num, flat, img):
        chosen = set(native_select(seed, img, flat.cpu().numpy(), num).tolist())
        keep = torch.tensor([int(f) in chosen for f in flat.cpu().tolist()], dtype=torch.bool, device=gallery.device)
        return gallery[keep]
    return draw


def sample(assigned, s, draw, flat, img):
    """BaseSampler.sample with RandomSampler's _sample_pos / _sample_neg: (pos_inds, neg_inds) into the inside
    anchors."""
    def pick(mask, num):
        inds = torch.nonzero(mask).squeeze(1)
        if inds.numel() <= num:
            return inds
        return draw(inds, num, flat[inds], img)
    pos = pick(assigned > 0, int(s['num'] * s['pos_fraction'])).unique()
    num_neg = s['num'] - pos.numel()
    if s.get('neg_pos_ub', -1) >= 0:
        ub = int(s['neg_pos_ub'] * max(1, pos.numel()))
        num_neg = min(num_neg, ub)
    neg = pick(assigned == 0, num_neg).unique()
    return pos, neg


def anchor_target_single(anchors, valid, gts, img_meta, means, stds, cfg, draw, img=0):
    inside = inside_flags(anchors, valid, img_meta['img_shape'][:2], cfg['allowed_border'])
    if not inside.any():
        return (None,) * 6
    flat = torch.nonzero(inside).squeeze(1)
    ins = anchors[inside.bool(), :]
    assigned = assign(ins, gts, cfg['assigner'])
    pos, neg = sample(assigned, cfg['sampler'], draw, flat, img)
    n = ins.shape[0]
    bbox_targets = torch.zeros_like(ins)
    bbox_weights = torch.zeros_like(ins)
    labels = ins.new_zeros(n, dtype=torch.long)
    label_weights = ins.new_zeros(n, dtype=torch.float)
    if len(pos) > 0:
        bbox_targets[pos, :] = bbox2delta(ins[pos], gts[assigned[pos] - 1, :], means, stds)
        bbox_weights[pos, :] = 1.0
        labels[pos] = 1
        label_weights[pos] = 1.0 if cfg['pos_weight'] <= 0 else cfg['pos_weight']
    if len(neg) > 0:
        label_weights[neg] = 1.0

    def unmap(data):
        ret = data.new_full((anchors.size(0),) + data.size()[1:], 0)
        ret[inside.bool()] = data
        return ret
    return unmap(labels), unmap(label_weights), unmap(bbox_targets), unmap(bbox_weights), pos, neg


def anchor_target(bases, sizes, strides, gt_list, img_metas, means, stds, cfg, draw, device):
    """Dense per-image targets (labels, label_weights, bbox_targets, bbox_weights stacked to [B, N, ...]) and
    (num_total_pos, num_total_neg); None when an image has no inside anchor."""
    outs = []
    for b, (gts, meta) in enumerate(zip(gt_list, img_metas)):
        anchors, valid = multi_level(bases, sizes, strides, meta['pad_shape'], device)
        outs.append(anchor_target_single(anchors, valid, gts, meta, means, stds, cfg, draw, b))
    if any(o[0] is None for o in outs):
        return None
    stacked = [torch.stack([o[i] for o in outs]) for i in range(4)]
    return stacked, (sum(max(o[4].numel(), 1) for o in outs), sum(max(o[5].numel(), 1) for o in outs))
