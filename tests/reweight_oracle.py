"""CPU oracle of the class-reweighted softmax head (ReweightBBoxHead) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restates, in plain PyTorch / numpy:

  reweight_ce_loss        mmdet/models/bbox_heads/reweight_bbox_head.py:36-55 (cls part) with
                          cross_entropy_loss.py:9-19 and losses/utils.py:26-53
  accuracy                mmdet/models/losses/accuracy.py:4-21
  ce_closed_form_grads    what autograd produces for the loss above
  class_weights_*         tools/lvis_analyse.py: get_cate_weight / get_cate_weight_bf / get_cate_weight_bours

and, where a reference checkout is reachable (``oracle.ref_shim.reference_dir()``), runs the reference's own
``ReweightBBoxHead`` and weight functions on CPU for tests/test_reweight_head_cpu.py and
tests/golden/make_reweight_golden.py.  The GPU tests read only the committed fixture.
"""
from __future__ import annotations

import os
import sys
import tempfile
import types
from typing import Mapping

import numpy as np
import torch
import torch.nn.functional as F

from oracle import ref_shim


# --------------------------------------------------------------------------- loss / accuracy
def reweight_ce_loss(cls_score, labels, cls_weight, label_weights, loss_weight=1.0):
    """loss_cls of ReweightBBoxHead: sum_n w[labels[n]] * CE_n / max(#(label_weights > 0), 1)."""
    avg_factor = max(torch.sum(label_weights > 0).float().item(), 1.)
    w = cls_weight[labels].float()
    loss = F.cross_entropy(cls_score, labels, reduction='none')
    return loss_weight * ((loss * w).sum() / avg_factor)


def accuracy(pred, target):
    """Top-1 accuracy in percent (accuracy.py, topk=1): argmax by ``topk``."""
    _, pred_label = pred.topk(1, dim=1)
    correct = pred_label.t().eq(target.view(1, -1))
    return correct.reshape(-1).float().sum(0, keepdim=True).mul_(100.0 / pred.size(0))


def correct_rows(z, labels):
    """Per row: z[target] == row max (a tie with the maximum counts as correct, as the fused kernel counts)."""
    return z.gather(1, labels[:, None])[:, 0] == z.max(1).values


def top2_gap(z):
    v = z.topk(2, dim=1).values
    return v[:, 0] - v[:, 1]


def ce_closed_form_grads(x, W, b, labels, weights, avg, gout=1.0):
    """dz, dW, db, dX of gout * sum_n w[n] * CE_n / avg by the closed form dz = gout * w/avg * (softmax - onehot)."""
    z = F.linear(x, W, b)
    p = torch.softmax(z, dim=1)
    onehot = F.one_hot(labels, z.shape[1]).to(z.dtype)
    coef = (weights.to(z.dtype) if weights is not None else torch.ones(z.shape[0], dtype=z.dtype)) / float(avg)
    dz = float(gout) * coef[:, None] * (p - onehot)
    return dz, dz.t() @ x, dz.sum(0), dz @ W


def ce_loss(x, W, b, labels, weights, avg):
    z = F.linear(x, W, b)
    ce = F.cross_entropy(z, labels, reduction='none')
    if weights is not None:
        ce = ce * weights.to(ce.dtype)
    return ce.sum() / float(avg)


# --------------------------------------------------------------------------- class weights
def _counts(instance_counts: Mapping[int, int], num_classes: int) -> np.ndarray:
    c = np.zeros((num_classes,), dtype=np.float64)
    for cid, n in instance_counts.items():
        c[cid] = n
    return c


def class_weights_inv(instance_counts, num_classes=1231):
    c = _counts(instance_counts, num_classes)
    c[0] = 1
    with np.errstate(divide='ignore'):
        w = 1.0 / c
    w = w / w[1:].mean()
    w[0] = 1
    return np.clip(w, 0.1, 5)


def class_weights_bf(instance_counts, num_classes=1231):
    c = _counts(instance_counts, num_classes)
    c[0] = c[1:].sum() * 3
    w = (1 - 0.999) / (1 - 0.999 ** c)
    return w / w.mean()


def class_weights_bours(instance_counts, num_classes=1231):
    c = _counts(instance_counts, num_classes)
    w = (1 - 0.999) / (1 - 0.999 ** c[1:])
    out = np.ones((num_classes,), dtype=np.float64)
    out[1:] = w / w.mean()
    return np.clip(out, 0.1, 5)


# --------------------------------------------------------------------------- the head fixture
FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reweight_head_ref_n256.npz')
FIX_N, FIX_IN, FIX_ROI, FIX_FC, FIX_C = 256, 16, 2, 64, 1231


def fixture_inputs():
    """Seeded parameters and inputs of the ReweightBBoxHead fixture (regenerated on every machine from the seed; the
    fixture stores only the outputs).  Parameters use the head's state-dict keys."""
    from balancedgroupsoftmax_b200.tables import class_weights, synthetic_instance_counts
    g = torch.Generator().manual_seed(1231)
    k0 = FIX_IN * FIX_ROI * FIX_ROI

    def rn(*shape, s=1.0):
        return torch.randn(*shape, generator=g) * s

    params = {
        'shared_fcs.0.weight': rn(FIX_FC, k0, s=0.15), 'shared_fcs.0.bias': rn(FIX_FC, s=0.1),
        'shared_fcs.1.weight': rn(FIX_FC, FIX_FC, s=0.15), 'shared_fcs.1.bias': rn(FIX_FC, s=0.1),
        'fc_cls.weight': rn(FIX_C, FIX_FC, s=0.3), 'fc_cls.bias': rn(FIX_C, s=0.2),
        'fc_reg.weight': rn(4 * FIX_C, FIX_FC, s=0.01), 'fc_reg.bias': rn(4 * FIX_C, s=0.01),
    }
    params['fc_cls.bias'][0] += 9.0                  # background wins on many RoIs: a non-trivial accuracy
    feats = rn(FIX_N, FIX_IN, FIX_ROI, FIX_ROI)
    npos = 96
    labels = torch.zeros(FIX_N, dtype=torch.long)
    labels[:npos] = torch.randint(1, FIX_C, (npos,), generator=g)
    label_weights = torch.ones(FIX_N)
    label_weights[-20:] = 0.                          # ignored RoIs: only the normaliser sees them
    bbox_targets = torch.zeros(FIX_N, 4)
    bbox_targets[:npos] = rn(npos, 4, s=0.2)
    bbox_weights = torch.zeros(FIX_N, 4)
    bbox_weights[:npos] = 1.
    cls_weight = torch.from_numpy(class_weights(synthetic_instance_counts(FIX_C - 1, seed=0), FIX_C, 'inv'))
    return dict(params=params, feats=feats, labels=labels, label_weights=label_weights, bbox_targets=bbox_targets,
                bbox_weights=bbox_weights, cls_weight=cls_weight)


# --------------------------------------------------------------------------- the reference, run in place
def build_reference_reweight_bbox_head(cls_weight_path: str, num_classes: int = 1231, in_channels: int = 256,
                                       fc_out_channels: int = 1024, roi_feat_size: int = 7):
    """The reference's ReweightBBoxHead on CPU (its ``.cuda()`` is the identity under ``ref_shim.load()``)."""
    ref_shim.load()
    md = os.path.join(ref_shim.reference_dir(), 'mmdet')
    # this repository's drop-in registers itself under the same name when an `mmdet` package is importable
    sys.modules['mmdet.models.registry'].HEADS._module_dict.pop('ReweightBBoxHead', None)
    mod = ref_shim._exec('mmdet.models.bbox_heads.reweight_bbox_head',
                         os.path.join(md, 'models', 'bbox_heads', 'reweight_bbox_head.py'))
    return mod.ReweightBBoxHead(
        num_fcs=2, in_channels=in_channels, fc_out_channels=fc_out_channels,
        reweight_cfg=ref_shim.AttrDict(cls_weight=cls_weight_path), roi_feat_size=roi_feat_size,
        num_classes=num_classes, target_means=[0., 0., 0., 0.], target_stds=[0.1, 0.1, 0.2, 0.2],
        reg_class_agnostic=False, loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0),
        loss_bbox=dict(type='SmoothL1Loss', beta=1.0, loss_weight=1.0))


def reference_accuracy():
    ref_shim.load()
    return sys.modules['mmdet.models.losses.accuracy'].accuracy


def reference_class_weights(instance_counts: Mapping[int, int], kind: str) -> np.ndarray:
    """Run tools/lvis_analyse.py's get_cate_weight{,_bf,_bours} in place: its LVIS reader is stubbed to yield the
    given counts, pdb.set_trace is a no-op, np.float is float (numpy >= 1.24 removed it), and it writes into a
    temporary ./data/lvis.  Returns the saved tensor as numpy."""
    root = ref_shim.reference_dir()
    import importlib.util
    import pdb

    class _LVIS(object):
        def __init__(self, ann_file):
            self.cats = {cid: {'instance_count': n} for cid, n in instance_counts.items()}

    stubs = {'lvis': types.ModuleType('lvis'), 'lvis.lvis': types.ModuleType('lvis.lvis'),
             'pycocotools': types.ModuleType('pycocotools'), 'pycocotools.coco': types.ModuleType('pycocotools.coco')}
    stubs['lvis.lvis'].LVIS = _LVIS
    stubs['pycocotools.coco'].COCO = object
    saved = {k: sys.modules.get(k) for k in stubs}
    had_float = hasattr(np, 'float')
    old_trace, old_cwd = pdb.set_trace, os.getcwd()
    sys.modules.update(stubs)
    np.float = float
    pdb.set_trace = lambda *a, **k: None
    try:
        spec = importlib.util.spec_from_file_location('_ref_lvis_analyse', os.path.join(root, 'tools', 'lvis_analyse.py'))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        fn = {'inv': mod.get_cate_weight, 'bf': mod.get_cate_weight_bf, 'bours': mod.get_cate_weight_bours}[kind]
        name = {'inv': 'cls_weight.pt', 'bf': 'cls_weight_bf.pt', 'bours': 'cls_weight_bours.pt'}[kind]
        with tempfile.TemporaryDirectory() as d:
            os.makedirs(os.path.join(d, 'data', 'lvis'))
            os.chdir(d)
            with np.errstate(divide='ignore'):
                fn()
            return torch.load(os.path.join(d, 'data', 'lvis', name)).numpy()
    finally:
        os.chdir(old_cwd)
        pdb.set_trace = old_trace
        if not had_float:
            del np.float
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
