"""The RPN target cases shared by tests/test_anchor_target_cpu.py (against the reference's own anchor_target) and
tests/test_gpu_anchor_target.py (the kernels against the restatement) -- TEST INFRASTRUCTURE."""
import numpy as np
import torch

import anchor_target_oracle as O

RPN_CFG = dict(assigner=dict(type='MaxIoUAssigner', pos_iou_thr=0.7, neg_iou_thr=0.3, min_pos_iou=0.3,
                             ignore_iof_thr=-1),
               sampler=dict(type='RandomSampler', num=256, pos_fraction=0.5, neg_pos_ub=-1, add_gt_as_proposals=False),
               allowed_border=0, pos_weight=-1, debug=False)

def _cfg(**kw):
    a = dict(RPN_CFG['assigner'])
    s = dict(RPN_CFG['sampler'])
    top = dict(allowed_border=RPN_CFG['allowed_border'], pos_weight=RPN_CFG['pos_weight'])
    for k, v in kw.items():
        (a if k in a or k in ('gt_max_assign_all',) else s if k in s else top)[k] = v
    return dict(assigner=a, sampler=s, **top)


def _boxes(gen, n, w, h, lo=4.0, hi=48.0):
    x1 = torch.rand(n, generator=gen) * (w - 8)
    y1 = torch.rand(n, generator=gen) * (h - 8)
    bw = lo + torch.rand(n, generator=gen) * (hi - lo)
    bh = lo + torch.rand(n, generator=gen) * (hi - lo)
    return torch.stack([x1, y1, (x1 + bw).clamp(max=w - 1), (y1 + bh).clamp(max=h - 1)], 1).round()


def _head_bases(strides=(4, 8, 16)):
    from balancedgroupsoftmax_b200.rpn_head import AnchorGenerator
    return [AnchorGenerator(s, [8], [0.5, 1.0, 2.0]).base_anchors for s in strides]


EDGE_BASE = torch.tensor([[0., 0., 13., 9.], [0., 0., 13., 6.], [0., 0., 5., 6.]])


def _ulp_gt(box, anchor, target, steps=2000):
    """A gt near ``box`` whose fp32 IoU with ``anchor`` is exactly ``target`` (fp32): the first hit among ``box`` with
    one coordinate moved by up to ``steps`` fp32 neighbours either way."""
    want = float(np.float32(target))
    for coord in (3, 2, 1, 0):
        v0 = np.float32(box[coord].item())
        vals, lo, hi = [v0], v0, v0
        for _ in range(steps):
            hi, lo = np.nextafter(hi, np.float32(np.inf)), np.nextafter(lo, np.float32(-np.inf))
            vals += [hi, lo]
        g = box.repeat(len(vals), 1)
        g[:, coord] = torch.from_numpy(np.array(vals, dtype=np.float32))
        hit = (O.bbox_overlaps(g, anchor[None])[:, 0] == want).nonzero()
        if len(hit):
            return g[hit[0, 0]]
    raise AssertionError('no gt at IoU %r' % target)


def edge_gts():
    """gts inside the first anchor of location (0, 0) (base [0, 0, 13, 9]) whose IoU with it is float32(0.7) /
    float32(0.3) and one ulp either side; each is best matched by another anchor of the location (its own box), so
    only steps 2 and 3 decide that anchor."""
    a0 = EDGE_BASE[0]
    out = []
    for t, box in ((0.7, EDGE_BASE[1]), (0.3, EDGE_BASE[2])):
        t32 = np.float32(t)
        for v in (np.nextafter(t32, np.float32(0)), t32, np.nextafter(t32, np.float32(1))):
            out.append(_ulp_gt(box, a0, float(v)))
    return out


def cases():
    """(name, bases, sizes, strides, metas, gts, cfg, means, stds): the CPU cases, shared with the GPU tests."""
    gen = torch.Generator().manual_seed(5)
    bases, sizes, strides = _head_bases(), [(16, 24), (8, 12), (4, 6)], [4, 8, 16]
    meta = dict(img_shape=(60, 90, 3), pad_shape=(64, 96, 3))
    meta2 = dict(img_shape=(50, 70, 3), pad_shape=(52, 72, 3))
    out = []

    def add(name, gts, cfg=None, metas=None, means=(0., 0., 0., 0.), stds=(1., 1., 1., 1.), b=None, z=None, t=None):
        out.append((name, b or bases, z or sizes, t or strides, metas or [meta] * len(gts), gts, cfg or _cfg(),
                    means, stds))
    r3 = _boxes(gen, 3, 90, 60)
    add('realistic', [r3])
    add('many_gts_cpu_route', [_boxes(gen, 60, 90, 60, 2, 40), _boxes(gen, 55, 70, 50, 2, 30)], metas=[meta, meta2])
    dup = torch.cat([r3, r3[:2], r3[1:2]])
    add('duplicates', [dup])
    add('duplicates_first_argmax', [dup], _cfg(gt_max_assign_all=False))
    far = torch.cat([r3, torch.tensor([[300., 300., 340., 330.]])])
    add('no_overlap', [far])
    add('no_overlap_min_pos_0', [far], _cfg(min_pos_iou=0.0))
    add('degenerate', [torch.cat([r3, torch.tensor([[20., 20., 19., 40.], [30., 10., 27., 8.], [5., 5., 4., 4.]])])])
    add('nan_gt', [torch.cat([r3, torch.tensor([[10., float('nan'), 30., 30.]])])])
    add('pad_differs', [r3, _boxes(gen, 4, 70, 50)], metas=[dict(img_shape=(40, 50, 3), pad_shape=(64, 96, 3)), meta2])
    for ab in (-1, 0, 16):
        add('border_%d' % ab, [r3], _cfg(allowed_border=ab))
    add('neg_tuple', [r3], _cfg(neg_iou_thr=(0.1, 0.4)))
    add('neg_pos_ub', [_boxes(gen, 6, 90, 60)], _cfg(neg_pos_ub=2))
    add('neg_pos_ub_0', [_boxes(gen, 6, 90, 60)], _cfg(neg_pos_ub=0))
    add('pos_weight', [r3], _cfg(pos_weight=2.5))
    add('means_stds', [r3], means=(0.1, -0.2, 0.05, 0.0), stds=(0.1, 0.1, 0.2, 0.3))
    add('b3', [r3, _boxes(gen, 5, 70, 50), _boxes(gen, 1, 90, 60)], metas=[meta, meta2, meta])
    add('small_sample', [_boxes(gen, 8, 90, 60)], _cfg(num=16, pos_fraction=0.25))
    edge = edge_gts()
    em = dict(img_shape=(64, 64, 3), pad_shape=(64, 64, 3))
    add('iou_at_thresholds', [torch.stack(edge)], b=[EDGE_BASE], z=[(4, 4)], t=[16], metas=[em])
    for i, g in enumerate(edge):   # one gt per image: the anchor's max is exactly that IoU
        add('iou_edge_%d' % i, [g[None]], b=[EDGE_BASE], z=[(4, 4)], t=[16], metas=[em])
    return out


