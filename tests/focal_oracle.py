"""Float64 oracle of the sigmoid focal loss (FocalLoss with its op) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restates, in float64 torch, term by term:

  op_forward / op_backward   mmdet/ops/sigmoid_focal_loss/src/sigmoid_focal_loss_cuda.cu:23-96 (the per-element
                             loss and the op's analytic gradient; ``pin_reference_source`` checks those lines)
  focal_loss                 FocalLoss.forward, mmdet/models/losses/focal_loss.py:63-88, with sigmoid_focal_loss
                             (:29-43) and weight_reduce_loss (losses/utils.py:26-53)

The reference's op itself cannot be built against current torch (it uses the removed THC API), so where a reference
checkout is reachable (``oracle.ref_shim``) its FocalLoss and heads run in place with ``mmdet.ops.sigmoid_focal_loss``
replaced by ``Float64Op`` -- the float64 restatement -- for tests/test_focal_cpu.py and tests/golden/make_focal_golden.py.
The GPU tests read only the committed fixture.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

from oracle import ref_shim

FLT_MIN = float(np.finfo(np.float32).tiny)
ONE_HOT = 1231


# --------------------------------------------------------------------------- the op
def _cases(t, C, device):
    t = t.to(torch.int32).to(torch.int64).reshape(-1, 1)         # `int t = targets[n]`
    d = torch.arange(C, device=device).reshape(1, -1)
    c1 = (t == d + 1).to(torch.float64)
    c2 = ((t >= 0) & (t != d + 1)).to(torch.float64)
    return c1, c2


def op_forward(z, t, gamma, alpha):
    """Per-element loss [N, C] in float64 (sigmoid_focal_loss_cuda.cu:30-57)."""
    z = z.to(torch.float64)
    c1, c2 = _cases(t, z.shape[1], z.device)
    zn, zp = 1.0 - alpha, alpha
    p = 1. / (1. + torch.exp(-z))
    term1 = torch.pow(1. - p, gamma) * torch.log(torch.clamp(p, min=FLT_MIN))
    ge = (z >= 0).to(torch.float64)
    term2 = torch.pow(p, gamma) * (-1. * z * ge - torch.log(1. + torch.exp(z - 2. * z * ge)))
    return -c1 * term1 * zp - c2 * term2 * zn


def op_backward(z, t, gamma, alpha):
    """The op's analytic d loss / d z per element [N, C] in float64 (sigmoid_focal_loss_cuda.cu:66-94, d_losses = 1)."""
    z = z.to(torch.float64)
    c1, c2 = _cases(t, z.shape[1], z.device)
    zn, zp = 1.0 - alpha, alpha
    p = 1. / (1. + torch.exp(-z))
    term1 = torch.pow(1. - p, gamma) * (1. - p - (p * gamma * torch.log(torch.clamp(p, min=FLT_MIN))))
    ge = (z >= 0).to(torch.float64)
    term2 = torch.pow(p, gamma) * ((-1. * z * ge - torch.log(1. + torch.exp(z - 2. * z * ge))) * (1. - p) * gamma - p)
    return -c1 * term1 * zp - c2 * term2 * zn


def targets_of(labels, n=None):
    """What the op sees as targets under FocalLoss.forward: the first N entries of F.one_hot(labels, 1231)."""
    n = labels.numel() if n is None else n
    return torch.nn.functional.one_hot(labels, num_classes=ONE_HOT).reshape(-1)[:n]


def focal_loss(z, labels, weight=None, gamma=2.0, alpha=0.25, reduction='mean', loss_weight=1.0):
    """FocalLoss.forward in float64: (loss, dloss/dz by the op's gradient) for reduction 'mean' or 'none'."""
    el = op_forward(z, targets_of(labels, z.shape[0]), gamma, alpha)
    g = op_backward(z, targets_of(labels, z.shape[0]), gamma, alpha)
    w = torch.ones(z.shape[0], 1, dtype=torch.float64) if weight is None else weight.to(torch.float64).reshape(-1, 1)
    el, g = el * w, g * w
    if reduction == 'none':
        return loss_weight * el, loss_weight * g
    avg = max(float(labels.numel() * ONE_HOT), 1.)
    return loss_weight * el.sum() / avg, loss_weight * g / avg


def lipschitz_bound(gamma, alpha, lim=60.0, steps=240001):
    """max_z |d grad / dz| of both element kinds over [-lim, lim], by float64 differences on a fine grid."""
    z = torch.linspace(-lim, lim, steps, dtype=torch.float64).reshape(-1, 1)
    out = 0.
    for t in (1, 0):   # column 0 positive, then negative
        g = op_backward(z, torch.full((z.shape[0],), t), gamma, alpha)[:, 0]
        out = max(out, float(((g[1:] - g[:-1]).abs() / (z[1:, 0] - z[:-1, 0])).max()))
    return out


# --------------------------------------------------------------------------- the reference, run in place
SOURCE_PINS = {
    os.path.join('mmdet', 'ops', 'sigmoid_focal_loss', 'src', 'sigmoid_focal_loss_cuda.cu'): [
        'int t = targets[n];',
        'scalar_t c1 = (t == (d + 1));',
        'scalar_t c2 = (t >= 0 & t != (d + 1));',
        'scalar_t zn = (1.0 - alpha); scalar_t zp = (alpha);',
        'scalar_t p = 1. / (1. + expf(-logits[i]));',
        'scalar_t term1 = powf((1. - p), gamma) * logf(max(p, FLT_MIN));',
        'scalar_t term2 = powf(p, gamma) * (-1. * logits[i] * (logits[i] >= 0) - '
        'logf(1. + expf(logits[i] - 2. * logits[i] * (logits[i] >= 0))));',
        'losses[i] = 0.0; losses[i] += -c1 * term1 * zp; losses[i] += -c2 * term2 * zn;',
        'scalar_t term1 = powf((1. - p), gamma) * (1. - p - (p * gamma * logf(max(p, FLT_MIN))));',
        'scalar_t term2 = powf(p, gamma) * ((-1. * logits[i] * (logits[i] >= 0) - '
        'logf(1. + expf(logits[i] - 2. * logits[i] * (logits[i] >= 0)))) * (1. - p) * gamma - p);',
        'd_logits[i] = 0.0; d_logits[i] += -c1 * term1 * zp; d_logits[i] += -c2 * term2 * zn; '
        'd_logits[i] = d_logits[i] * d_losses[i];',
    ],
    os.path.join('mmdet', 'models', 'losses', 'focal_loss.py'): [
        "expand_target = F.one_hot(target, num_classes=1231) target = expand_target",
        "avg_factor = max(torch.sum(torch.ones_like(target) > 0).float().item(), 1.)",
        "if weight is not None: weight = weight.view(-1, 1) loss = weight_reduce_loss(loss, weight, reduction, avg_factor)",
        "assert use_sigmoid is True, 'Only sigmoid focal loss supported now.'",
    ],
    os.path.join('mmdet', 'ops', 'sigmoid_focal_loss', 'sigmoid_focal_loss.py'): [
        'loss = sigmoid_focal_loss_cuda.forward(input, target, num_classes, gamma, alpha)',
        'd_input = sigmoid_focal_loss_cuda.backward(input, target, d_loss, num_classes, gamma, alpha)',
    ],
}


def pin_reference_source():
    """{file: [pinned lines missing from it]} for the reference checkout (whitespace-normalised); empty when the
    restatement above reads what the reference says."""
    root = ref_shim.reference_dir()
    missing = {}
    for rel, lines in SOURCE_PINS.items():
        with open(os.path.join(root, rel)) as f:
            text = ' '.join(f.read().split())
        gone = [ln for ln in lines if ' '.join(ln.split()) not in text]
        if gone:
            missing[rel] = gone
    return missing


class Float64Op(torch.autograd.Function):
    """Stand-in for mmdet.ops.sigmoid_focal_loss (SigmoidFocalLossFunction): the float64 restatement, forward and the
    op's analytic backward, in float64."""

    @staticmethod
    def forward(ctx, z, t, gamma=2.0, alpha=0.25):
        t = t.reshape(-1)[:z.shape[0]]   # the op reads targets[n] for the N rows only, whatever the tensor's shape
        ctx.save_for_backward(z, t)
        ctx.gamma, ctx.alpha = gamma, alpha
        return op_forward(z, t, gamma, alpha)

    @staticmethod
    def backward(ctx, d_loss):
        z, t = ctx.saved_tensors
        g = op_backward(z, t, ctx.gamma, ctx.alpha) * d_loss
        return g.to(z.dtype), None, None, None


def load_reference_focal_loss():
    """The reference's focal_loss.py executed in place (registered in its LOSSES), its op replaced by Float64Op."""
    ref_shim.load()
    md = os.path.join(ref_shim.reference_dir(), 'mmdet')
    ops_mod = sys.modules.get('mmdet.ops')
    if ops_mod is None:
        ops_mod = ref_shim._shell('mmdet.ops', os.path.join(md, 'ops'))
    ops_mod.sigmoid_focal_loss = Float64Op.apply
    sys.modules['mmdet.models.registry'].LOSSES._module_dict.pop('FocalLoss', None)
    mod = ref_shim._exec('mmdet.models.losses.focal_loss', os.path.join(md, 'models', 'losses', 'focal_loss.py'))
    return mod.FocalLoss


# the bbox_head blocks of configs/transferred/faster_rcnn_r50_fpn_1x_lvis_{focalloss,focalloss_all}.py (the same block)
# and faster_rcnn_r50_fpn_1x_lvis_reweighthead_bfocal.py, lines 34-53
FOCAL_SHARED_LOSS = dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0)
FOCAL_BFOCAL_LOSS = dict(type='FocalLoss', use_sigmoid=True, gamma=0.5, alpha=1, loss_weight=1.0)


def head_blocks(cls_weight_path, in_channels=256, fc_out_channels=1024, roi_feat_size=7, num_classes=1231):
    common = dict(num_fcs=2, in_channels=in_channels, fc_out_channels=fc_out_channels, roi_feat_size=roi_feat_size,
                  num_classes=num_classes, target_means=[0., 0., 0., 0.], target_stds=[0.1, 0.1, 0.2, 0.2],
                  reg_class_agnostic=False, loss_bbox=dict(type='SmoothL1Loss', beta=1.0, loss_weight=1.0))
    return {
        'shared': dict(type='SharedFCBBoxHead', loss_cls=dict(FOCAL_SHARED_LOSS), **common),
        'bfocal': dict(type='ReweightBBoxHead', reweight_cfg=dict(cls_weight=cls_weight_path),
                       loss_cls=dict(FOCAL_BFOCAL_LOSS), **common),
    }


def build_reference_heads(cls_weight_path, **sizes):
    """The reference's SharedFCBBoxHead and ReweightBBoxHead (CPU) for the blocks of ``head_blocks``."""
    load_reference_focal_loss()
    md = os.path.join(ref_shim.reference_dir(), 'mmdet')
    sys.modules['mmdet.models.registry'].HEADS._module_dict.pop('ReweightBBoxHead', None)
    rw = ref_shim._exec('mmdet.models.bbox_heads.reweight_bbox_head',
                        os.path.join(md, 'models', 'bbox_heads', 'reweight_bbox_head.py'))
    shared = sys.modules['mmdet.models.bbox_heads.convfc_bbox_head'].SharedFCBBoxHead
    out = {}
    for key, cfg in head_blocks(cls_weight_path, **sizes).items():
        cfg = dict(cfg)
        cls = {'SharedFCBBoxHead': shared, 'ReweightBBoxHead': rw.ReweightBBoxHead}[cfg.pop('type')]
        if 'reweight_cfg' in cfg:
            cfg['reweight_cfg'] = ref_shim.AttrDict(cfg['reweight_cfg'])
        out[key] = cls(**cfg)
    return out


# --------------------------------------------------------------------------- the head fixture
FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'focal_head_ref_n256.npz')


def fixture_inputs():
    """The ReweightBBoxHead fixture's seeded parameters and inputs (tests/reweight_oracle.py), with the 'bf' class
    weights the bfocal config names (cls_weight_bf.pt)."""
    import reweight_oracle as R
    from balancedgroupsoftmax_b200.tables import class_weights, synthetic_instance_counts
    inp = R.fixture_inputs()
    # Under the one-hot quirk, row n has a positive column only if labels[n // 1231] == n % 1231: with 256 rows, only
    # row labels[0].  Label 37 puts it at row 37 (the seeded label would fall outside the 256 rows: an all-negative
    # batch, whose alpha = 1 loss is exactly 0).
    inp['labels'][0] = 37
    inp['cls_weight'] = torch.from_numpy(class_weights(synthetic_instance_counts(R.FIX_C - 1, seed=0), R.FIX_C, 'bf'))
    return inp


def fixture_sizes():
    import reweight_oracle as R
    return dict(in_channels=R.FIX_IN, fc_out_channels=R.FIX_FC, roi_feat_size=R.FIX_ROI, num_classes=R.FIX_C)


def run_head(head, inp, materialise=False, device='cpu', dtype=torch.float32):
    """Losses of ``head`` on the fixture inputs and the gradients of loss_cls + loss_bbox.  ``materialise``: this
    package's ReweightBBoxHead through nn.Linear logits (its materialised route) instead of its forward.  ``dtype``:
    of the parameters and the float inputs (float64 on CPU takes fp32 rounding out of a comparison with the fixture)."""
    head.load_state_dict(inp['params'], strict=True)
    head.to(device, dtype).train()
    head.zero_grad()
    inp = {k: (v.to(device, dtype) if torch.is_tensor(v) and v.is_floating_point() else
               v.to(device) if torch.is_tensor(v) else v) for k, v in inp.items()}
    feats = inp['feats'].clone().requires_grad_(True)
    if materialise:
        x_cls, x_reg = head._trunk(feats)
        cls_score, bbox_pred = head.fc_cls(x_cls), head.fc_reg(x_reg)
    else:
        cls_score, bbox_pred = head(feats)
    losses = head.loss(cls_score, bbox_pred, inp['labels'], inp['label_weights'], inp['bbox_targets'],
                       inp['bbox_weights'])
    (losses['loss_cls'] + losses['loss_bbox']).backward()
    return dict(loss_cls=losses['loss_cls'].detach(), acc=losses['acc'].detach(),
                loss_bbox=losses['loss_bbox'].detach(), dW4=head.fc_cls.weight.grad[::4].detach(),
                db=head.fc_cls.bias.grad.detach(), dX=feats.grad.detach())
