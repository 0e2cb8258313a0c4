"""Regenerate tests/golden/reference_outputs.npz: what the reference's own source (run in place through oracle/ref_shim.py,
CPU) returns for the inputs tests/test_oracle_vs_reference.py builds from fixed seeds.  Large outputs are stored as a
fixed row sample.  Needs a reference checkout (see oracle/ref_shim.py):

    python tests/golden/make_ref_golden.py
"""
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from balancedgroupsoftmax_b200.tables import synthetic_tables  # noqa: E402
from oracle import bags_oracle as O  # noqa: E402
from oracle import ref_shim  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'reference_outputs.npz')
LOSS_CASES = [(1, 1, 0), (1, 0, 1), (64, 16, 2), (300, 75, 3), (512, 128, 4), (40, 40, 5)]
DW_ROWS, DX_ROWS, MERGE_COLS = 16, 4, 37   # row / column sampling strides of the stored outputs
REWEIGHT_CASES = ((300, 75, 1), (64, 0, 2), (40, 40, 3), (512, 128, 4))


def loss_case_inputs(N, npos, seed, C, K=128):
    """Inputs of one loss/grad case, drawn in the order the reference head's parameters were re-drawn."""
    torch.manual_seed(seed)
    W = torch.empty(C, K).normal_(0, 0.2)
    b = torch.empty(C).normal_(0, 0.1)
    x = torch.relu(torch.randn(N, K))
    labels = torch.zeros(N, dtype=torch.long)
    labels[:npos] = torch.randint(1, 1231, (npos,))
    return W, b, x, labels


def bbox_inputs():
    g = torch.Generator().manual_seed(11)

    def boxes(n):
        xy = torch.rand(n, 2, generator=g) * 600
        wh = torch.rand(n, 2, generator=g) * 200 + 1
        return torch.cat([xy, xy + wh], 1)

    imgs = []
    for npos, nneg in ((5, 20), (0, 12), (7, 0), (1, 1)):
        imgs.append(SimpleNamespace(pos_bboxes=boxes(npos), neg_bboxes=boxes(nneg), pos_gt_bboxes=boxes(npos),
                                    pos_gt_labels=torch.randint(1, 1231, (npos,), generator=g)))
    return imgs


def nms_inputs():
    g = torch.Generator().manual_seed(5)
    n, classes = 60, 9
    xy = torch.rand(n, 2, generator=g) * 80
    wh = torch.rand(n, 2, generator=g) * 40 + 2
    boxes4 = torch.cat([xy, xy + wh], 1)
    boxes_pc = (boxes4[:, None, :] + torch.rand(n, classes, 4, generator=g)).reshape(n, classes * 4)
    scores = torch.rand(n, classes, generator=g) ** 3
    return boxes4, boxes_pc, scores


NMS_SETTINGS = ((0.05, 0.5, 20), (0.0, 0.3, 1000), (0.9999, 0.5, 10), (0.2, 0.5, -1))
MEANS, STDS = [0., 0., 0., 0.], [0.1, 0.1, 0.2, 0.2]


def reweight_weights(t):
    g = torch.Generator().manual_seed(21)
    return [torch.rand(int(t.pred_slice[b, 1]), generator=g) * 2 + 0.1 for b in range(1, t.num_bins)]


def main():
    assert ref_shim.available(), 'no reference checkout'
    out = {}
    t = synthetic_tables(1231, seed=0)
    head = ref_shim.build_reference_head(t, fc_out_channels=128)
    head.init_weights()
    for N, npos, seed in LOSS_CASES:
        W, b, x, labels = loss_case_inputs(N, npos, seed, head.fc_cls.out_features)
        with torch.no_grad():
            head.fc_cls.weight.copy_(W)
            head.fc_cls.bias.copy_(b)
        np.random.seed(seed)
        xr = x.clone().requires_grad_(True)
        head.zero_grad()
        losses = head.loss(head.fc_cls(xr), None, labels, None, None, None)
        sum(losses.values()).backward()
        key = 'loss_%d_%d_%d_' % (N, npos, seed)
        out[key + 'losses'] = np.array([losses['loss_cls_bin%d' % g].item() for g in range(5)], np.float64)
        out[key + 'dW'] = head.fc_cls.weight.grad[::DW_ROWS].numpy()
        out[key + 'db'] = head.fc_cls.bias.grad.numpy()
        out[key + 'dX'] = xr.grad[::DX_ROWS].numpy()
    torch.manual_seed(7)
    for i in range(3):
        z = torch.randn(200, t.num_logits) * 3
        a = head._merge_score(z)
        out['merge_%d_sample' % i] = a[:, ::MERGE_COLS].numpy()
        out['merge_%d_argmax' % i] = a.argmax(1).numpy()
    out['tables_label2binlabel'] = head.label2binlabel.numpy()
    out['tables_pred_slice'] = head.pred_slice.numpy()
    out['tables_fg_splits'] = np.concatenate([s.numpy() for s in head.fg_splits])
    out['tables_fg_split_lens'] = np.array([len(s) for s in head.fg_splits])
    out['tables_out_features'] = np.array(head.fc_cls.out_features)
    labels = torch.zeros(400, dtype=torch.long)
    labels[:90] = torch.randint(1, 1231, (90,), generator=torch.Generator().manual_seed(3))
    np.random.seed(11)
    _, ref_w, _ = head._remap_labels(labels)
    for g in range(1, 5):
        out['sampler_w%d' % g] = ref_w[g].numpy()

    ref_bbox_target, ref_bbox2delta = ref_shim.load_bbox_target()
    imgs = bbox_inputs()
    out['bbox2delta'] = ref_bbox2delta(imgs[0].pos_bboxes, imgs[0].pos_gt_bboxes, MEANS, STDS).numpy()
    for pos_weight in (-1, 2.5):
        cfg = ref_shim.AttrDict(pos_weight=pos_weight)
        args = ([r.pos_bboxes for r in imgs], [r.neg_bboxes for r in imgs], [r.pos_gt_bboxes for r in imgs],
                [r.pos_gt_labels for r in imgs], cfg)
        for i, a in enumerate(ref_bbox_target(*args, reg_classes=1231, target_means=MEANS, target_stds=STDS)):
            out['bbox_target_%s_%d' % (pos_weight, i)] = a.numpy()
        for i, la in enumerate(ref_bbox_target(*args, target_means=MEANS, target_stds=STDS, concat=False)):
            for j, a in enumerate(la):
                out['bbox_target_%s_split_%d_%d' % (pos_weight, i, j)] = a.numpy()

    ref_mc_nms = ref_shim.load_multiclass_nms(O.nms_plus1)
    boxes4, boxes_pc, scores = nms_inputs()
    for bi, mb in enumerate((boxes4, boxes_pc)):
        for si, (thr, iou, k) in enumerate(NMS_SETTINGS):
            dets, lab = ref_mc_nms(mb, scores.clone(), thr, dict(type='nms', iou_thr=iou), k)
            out['nms_%d_%d_dets' % (bi, si)] = dets.numpy()
            out['nms_%d_%d_labels' % (bi, si)] = lab.numpy()

    cls_weights = reweight_weights(t)
    rhead = ref_shim.build_reference_reweight_head(t, cls_weights, fc_out_channels=64)
    rhead.init_weights()
    for N, npos, seed in REWEIGHT_CASES:
        torch.manual_seed(seed)
        with torch.no_grad():
            rhead.fc_cls.weight.normal_(0, 0.2)
            rhead.fc_cls.bias.normal_(0, 0.1)
        x = torch.relu(torch.randn(N, 64))
        labels = torch.zeros(N, dtype=torch.long)
        labels[:npos] = torch.randint(1, 1231, (npos,))
        z = rhead.fc_cls(x).detach()
        np.random.seed(seed)
        want = rhead.loss(z, None, labels, None, None, None)
        np.random.seed(seed)
        _, rw, ra = rhead._remap_labels(labels)
        key = 'reweight_%d_' % seed
        out[key + 'losses'] = np.array([want['loss_cls_bin%d' % g].item() for g in range(5)], np.float64)
        out[key + 'avg'] = np.array([float(a) for a in ra], np.float64)
        for g, w in enumerate(rw):
            out[key + 'w%d' % g] = w.float().numpy()
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT))


if __name__ == '__main__':
    main()
