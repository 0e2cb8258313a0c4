"""Float64 oracle of the class-specific box term (fc_reg + gather + SmoothL1 'mean') -- TEST INFRASTRUCTURE.

Restates, in float64 torch and in closed form, what the reference's heads compute for ``loss_bbox``:

  pred      bbox_pred.view(N, -1, 4)[pos_inds, labels[pos_inds]] of fc_reg(x)      bbox_head.py:118-128
  loss      smooth_l1_loss + weight_reduce_loss, avg_factor = bbox_targets.size(0)  smooth_l1_loss.py, losses/utils.py
  g         d loss / d pred (autograd's derivative: d / beta inside, sign(d) from |d| == beta on, abs'(0) = 0)
  dW, db, dX  the chain through fc_reg

Positives are 0 < label < classes here (labels >= classes contribute nothing; the reference would raise an index
error).  Where a reference checkout is reachable (``oracle.ref_shim``) tests/test_box_loss_cpu.py runs the reference's
own BBoxHead.loss against this restatement and tests/golden/make_box_golden.py writes the reference heads' outputs to
``FIXTURE``; the GPU tests read only that file.
"""
from __future__ import annotations

import os
import sys

import torch

from oracle import ref_shim

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'box_loss_ref_n256.npz')
FIX_N, FIX_IN, FIX_ROI, FIX_FC = 256, 16, 2, 64
FIX_ROWS = slice(0, None, 7)          # the fixture keeps every 7th row of dW_reg


def box_terms(x, W, b, labels, targets, weights, beta, avg, gout=1.0):
    """{'loss', 'pred' [N,4] (0 on non-positive rows), 'g' [N,4], 'dW' [4C,K], 'db' [4C], 'dX' [N,K]} in float64."""
    x, W = x.double(), W.double()
    b = torch.zeros(W.shape[0], dtype=torch.float64) if b is None else b.double()
    t, w = targets.double(), weights.double()
    N, K = x.shape
    C = W.shape[0] // 4
    labels = labels.cpu()
    pos = ((labels > 0) & (labels < C)).nonzero().reshape(-1)
    rows = (4 * labels[pos]).reshape(-1, 1) + torch.arange(4).reshape(1, 4)          # [P, 4]
    p = torch.einsum('pk,pjk->pj', x[pos], W[rows]) + b[rows]
    d = p - t[pos]
    ad = d.abs()
    quad = ad < beta
    sl1 = torch.where(quad, 0.5 * ad * ad / beta, ad - 0.5 * beta)
    sp = torch.where(quad, d / beta, torch.sign(d))
    pred = torch.zeros(N, 4, dtype=torch.float64)
    pred[pos] = p
    g = torch.zeros(N, 4, dtype=torch.float64)
    g[pos] = w[pos] * sp / avg
    gg = g * float(gout)
    dW = torch.zeros(4 * C, K, dtype=torch.float64)
    dW.index_add_(0, rows.reshape(-1), (gg[pos].unsqueeze(2) * x[pos].unsqueeze(1)).reshape(-1, K))
    db = torch.zeros(4 * C, dtype=torch.float64)
    db.index_add_(0, rows.reshape(-1), gg[pos].reshape(-1))
    dX = torch.zeros(N, K, dtype=torch.float64)
    dX[pos] = torch.einsum('pj,pjk->pk', gg[pos], W[rows])
    loss = (w[pos] * sl1).sum() / avg if N > 0 else torch.zeros((), dtype=torch.float64)
    return dict(loss=loss, pred=pred, g=g, dW=dW, db=db, dX=dX)


def error_bounds(x, W, b, labels, weights, beta, avg, gout=1.0):
    """Per-element bounds on |fp32 kernel - float64| for pred, g, dW, db and dX, x and W taken as exact.  fp32
    accumulation of n products errs by at most (n + 1) u sum |terms| (u = 2^-24); |sl1'| <= 1 with slope 1 / beta, so
    g inherits pred's error times w / (beta avg), plus a few roundings; dW, db and dX sum |g| |x| or |g| |W| terms and
    carry g's error through them.  Each bound is doubled for margin."""
    u = 2.0 ** -24
    x, W = x.double().abs(), W.double().abs()
    N, K = x.shape
    C = W.shape[0] // 4
    labels = labels.cpu()
    pos = ((labels > 0) & (labels < C)).nonzero().reshape(-1)
    rows = (4 * labels[pos]).reshape(-1, 1) + torch.arange(4).reshape(1, 4)
    bb = torch.zeros(W.shape[0], dtype=torch.float64) if b is None else b.double().abs()
    e_pred = torch.zeros(N, 4, dtype=torch.float64)
    e_pred[pos] = (K + 2) * u * (torch.einsum('pk,pjk->pj', x[pos], W[rows]) + bb[rows])
    gmax = weights.double().abs() / avg * abs(float(gout))
    e_g = gmax * (e_pred / beta + 4 * u)
    ga = gmax + e_g
    counts = torch.bincount(labels[pos], minlength=C).double().repeat_interleave(4)
    dW = torch.zeros(4 * C, K, dtype=torch.float64)
    dW.index_add_(0, rows.reshape(-1), (ga[pos].unsqueeze(2) * x[pos].unsqueeze(1)).reshape(-1, K))
    db = torch.zeros(4 * C, dtype=torch.float64)
    db.index_add_(0, rows.reshape(-1), ga[pos].reshape(-1))
    dX = torch.zeros(N, K, dtype=torch.float64)
    dX[pos] = torch.einsum('pj,pjk->pk', ga[pos], W[rows])
    # e_g is already inside ga; the sums add (n + 2) u of their magnitude
    edW = torch.zeros_like(dW)
    edW.index_add_(0, rows.reshape(-1), (e_g[pos].unsqueeze(2) * x[pos].unsqueeze(1)).reshape(-1, K))
    edb = torch.zeros_like(db)
    edb.index_add_(0, rows.reshape(-1), e_g[pos].reshape(-1))
    edX = torch.zeros_like(dX)
    edX[pos] = torch.einsum('pj,pjk->pk', e_g[pos], W[rows])
    return dict(pred=2 * e_pred, g=2 * e_g,
                dW=2 * ((counts.reshape(-1, 1) + 2) * u * dW + edW), db=2 * ((counts + 2) * u * db + edb),
                dX=2 * (6 * u * dX + edX))


# --------------------------------------------------------------------------- the reference, run in place
def reference_bbox_loss():
    """The reference's BBoxHead.loss (bbox_head.py:97-129) on CPU, bound to a class-specific BBoxHead: call it as
    ``f(bbox_pred, labels, bbox_targets, bbox_weights, beta)`` -> loss_bbox."""
    ref_shim.load()
    BBoxHead = sys.modules['mmdet.models.bbox_heads.bbox_head'].BBoxHead

    def f(bbox_pred, labels, bbox_targets, bbox_weights, beta=1.0):
        C = bbox_pred.shape[1] // 4
        head = BBoxHead(in_channels=4, roi_feat_size=1, num_classes=C, reg_class_agnostic=False,
                        loss_bbox=dict(type='SmoothL1Loss', beta=beta, loss_weight=1.0))
        return head.loss(None, bbox_pred, labels, None, bbox_targets, bbox_weights)['loss_bbox']
    return f


def fixture_inputs(num_classes=1231):
    """Seeded trunk + fc_reg parameters and RoI inputs of the box fixture: 256 RoIs, 96 positives (labels 1 and
    num_classes - 1 among them, several in one class), fc_reg scaled so that |d| falls on both sides of beta = 1, and
    some zero box weights."""
    g = torch.Generator().manual_seed(4924)
    k0 = FIX_IN * FIX_ROI * FIX_ROI

    def rn(*shape, s=1.0):
        return torch.randn(*shape, generator=g) * s

    params = {
        'shared_fcs.0.weight': rn(FIX_FC, k0, s=0.15), 'shared_fcs.0.bias': rn(FIX_FC, s=0.1),
        'shared_fcs.1.weight': rn(FIX_FC, FIX_FC, s=0.15), 'shared_fcs.1.bias': rn(FIX_FC, s=0.1),
        'fc_reg.weight': rn(4 * num_classes, FIX_FC, s=0.2), 'fc_reg.bias': rn(4 * num_classes, s=0.1),
    }
    feats = rn(FIX_N, FIX_IN, FIX_ROI, FIX_ROI)
    npos = 96
    labels = torch.zeros(FIX_N, dtype=torch.long)
    labels[:npos] = torch.randint(1, num_classes, (npos,), generator=g)
    labels[0], labels[1] = 1, num_classes - 1
    labels[2:10] = 7                                   # one class with several positives
    bbox_targets = torch.zeros(FIX_N, 4)
    bbox_targets[:npos] = rn(npos, 4, s=1.0)
    bbox_weights = torch.zeros(FIX_N, 4)
    bbox_weights[:npos] = 1.
    bbox_weights[10:14, 1] = 0.
    label_weights = torch.ones(FIX_N)
    return dict(params=params, feats=feats, labels=labels, label_weights=label_weights, bbox_targets=bbox_targets,
                bbox_weights=bbox_weights)


def run_box_loss(head, inp, device='cpu', dtype=torch.float32):
    """loss_bbox of ``head`` on the fixture inputs and its gradients w.r.t. fc_reg.weight (FIX_ROWS), fc_reg.bias and
    the RoI features.  Only the trunk and fc_reg parameters are loaded; the classifier is not run."""
    missing, _ = head.load_state_dict(inp['params'], strict=False)
    assert all(not k.startswith(('shared_fcs', 'fc_reg')) for k in missing), missing
    head.to(device, dtype).train()
    head.zero_grad()
    feats = inp['feats'].to(device, dtype).clone().requires_grad_(True)
    _, bbox_pred = head(feats)
    loss = head.loss(None, bbox_pred, inp['labels'].to(device), inp['label_weights'].to(device, dtype),
                     inp['bbox_targets'].to(device, dtype), inp['bbox_weights'].to(device, dtype))['loss_bbox']
    loss.backward()
    return dict(loss_bbox=loss.detach().reshape(1), dW=head.fc_reg.weight.grad[FIX_ROWS].detach(),
                db=head.fc_reg.bias.grad.detach(), dX=feats.grad.detach())
