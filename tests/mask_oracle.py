"""Float64 oracle of the class-specific mask term (conv_logits + mask_cross_entropy) -- TEST INFRASTRUCTURE.

Restates, in float64 torch and in closed form, what the reference's mask heads compute for ``loss_mask``:

  z         conv_logits(y)[arange(P), labels]: b[l] + sum_c W[l,c] y[p,c,q]         fcn_mask_head.py:82,102,114-123
  loss      F.binary_cross_entropy_with_logits(z, t, reduction='mean')             cross_entropy_loss.py:54-61
  g         d loss / d z = (sigmoid(z) - t) / (P H W)
  dW, db, dY  the chain through the 1x1 conv

A row is valid when 0 <= label < classes; an invalid row contributes 0 but counts in P H W (the reference would raise an
index error).  Where a reference checkout is reachable (``oracle.ref_shim``) tests/test_mask_loss_cpu.py runs the
reference's own mask_cross_entropy and mask heads against this restatement, and tests/golden/make_mask_golden.py
writes the reference heads' outputs to ``FIXTURE``; the GPU tests read only that file.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import types

import torch
import torch.nn as nn

from oracle import ref_shim

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'mask_loss_ref_p12.npz')
FIX_P, FIX_IN, FIX_CONV, FIX_ROI = 12, 8, 8, 7        # RoIs, input / conv channels, RoI feature size (logits 14x14)
FIX_ROWS = slice(0, None, 5)                          # the fixture keeps every 5th row of dW
FIX_CLASSES = 1231


def mask_terms(y, W, b, labels, targets, gout=1.0):
    """{'loss', 'z' [P,HW] (0 on invalid rows), 'g' [P,HW], 'dW' [C,Cin], 'db' [C], 'dY' [P,Cin,H,W]} in float64."""
    y = y.double()
    P, Cin = y.shape[:2]
    yf = y.reshape(P, Cin, -1)
    HW = yf.shape[2]
    W = W.double().reshape(W.shape[0], -1)
    C = W.shape[0]
    b = torch.zeros(C, dtype=torch.float64) if b is None else b.double()
    t = targets.double().reshape(P, HW)
    labels = labels.cpu()
    valid = ((labels >= 0) & (labels < C)).nonzero().reshape(-1)
    lv = labels[valid]
    z = torch.zeros(P, HW, dtype=torch.float64)
    z[valid] = torch.einsum('pc,pcq->pq', W[lv], yf[valid]) + b[lv].unsqueeze(1)
    n = float(P * HW)
    ell = torch.clamp(z, min=0) - z * t + torch.log1p(torch.exp(-z.abs()))
    g = torch.zeros(P, HW, dtype=torch.float64)
    g[valid] = (torch.sigmoid(z[valid]) - t[valid]) / n
    gg = g * float(gout)
    dW = torch.zeros(C, Cin, dtype=torch.float64)
    dW.index_add_(0, lv, torch.einsum('pq,pcq->pc', gg[valid], yf[valid]))
    db = torch.zeros(C, dtype=torch.float64)
    db.index_add_(0, lv, gg[valid].sum(1))
    dY = torch.zeros(P, Cin, HW, dtype=torch.float64)
    dY[valid] = gg[valid].unsqueeze(1) * W[lv].unsqueeze(2)
    loss = ell[valid].sum() / n if P > 0 else torch.zeros((), dtype=torch.float64)
    return dict(loss=loss, z=z, g=g, dW=dW, db=db, dY=dY.reshape(y.shape))


# --------------------------------------------------------------------------- the reference, run in place
def _weight_init_stub():
    """mmcv.cnn's init helpers the reference's ConvModule calls (mmcv/cnn/weight_init.py)."""
    cnn = types.ModuleType('mmcv.cnn')

    def constant_init(module, val, bias=0):
        nn.init.constant_(module.weight, val)
        if getattr(module, 'bias', None) is not None:
            nn.init.constant_(module.bias, bias)

    def kaiming_init(module, mode='fan_out', nonlinearity='relu', bias=0, distribution='normal'):
        if distribution == 'uniform':
            nn.init.kaiming_uniform_(module.weight, mode=mode, nonlinearity=nonlinearity)
        else:
            nn.init.kaiming_normal_(module.weight, mode=mode, nonlinearity=nonlinearity)
        if getattr(module, 'bias', None) is not None:
            nn.init.constant_(module.bias, bias)
    cnn.constant_init, cnn.kaiming_init = constant_init, kaiming_init
    return cnn


def _imresize(img, size, return_scale=False, interpolation='bilinear'):
    import cv2
    assert interpolation == 'bilinear' and not return_scale
    return cv2.resize(img, size, interpolation=cv2.INTER_LINEAR)


def _exec(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


_ref = None


def reference():
    """The reference's mask_cross_entropy, FCNMaskHead, HTCMaskHead and mask_target_single, executed in place on CPU.
    Only mmcv.cnn's init helpers, pycocotools and (while the heads import) mmdet.core.mask_target are stubbed; the
    reference's own conv_module.py is loaded for ConvModule, and mmcv.imresize is cv2.resize INTER_LINEAR."""
    global _ref
    if _ref is not None:
        return _ref
    ns = ref_shim.load()
    md = os.path.join(ns.root, 'mmdet')
    mmcv = sys.modules['mmcv']
    if 'mmcv.cnn' not in sys.modules:
        sys.modules['mmcv.cnn'] = mmcv.cnn = _weight_init_stub()
    if not hasattr(mmcv, 'imresize'):
        mmcv.imresize = _imresize
    if 'pycocotools' not in sys.modules:
        pc = types.ModuleType('pycocotools')
        pc.mask = types.ModuleType('pycocotools.mask')
        sys.modules['pycocotools'], sys.modules['pycocotools.mask'] = pc, pc.mask
    mutils = sys.modules['mmdet.models.utils']
    _exec('mmdet.models.utils.conv_ws', os.path.join(md, 'models', 'utils', 'conv_ws.py'))
    _exec('mmdet.models.utils.norm', os.path.join(md, 'models', 'utils', 'norm.py'))
    cm = _exec('mmdet.models.utils.conv_module', os.path.join(md, 'models', 'utils', 'conv_module.py'))
    mutils.ConvModule = cm.ConvModule
    core = sys.modules['mmdet.core']
    heads = sys.modules['mmdet.models.registry'].HEADS
    for name in ('FCNMaskHead', 'HTCMaskHead'):      # this package registers its own under these names
        heads._module_dict.pop(name, None)
    core.mask_target = None
    try:
        ref_shim._shell('mmdet.models.mask_heads', os.path.join(md, 'models', 'mask_heads'))
        fcn = _exec('mmdet.models.mask_heads.fcn_mask_head', os.path.join(md, 'models', 'mask_heads',
                                                                          'fcn_mask_head.py'))
        htc = _exec('mmdet.models.mask_heads.htc_mask_head', os.path.join(md, 'models', 'mask_heads',
                                                                          'htc_mask_head.py'))
    finally:
        del core.mask_target
    mt = _exec('bags_reference_mask_target', os.path.join(md, 'core', 'mask', 'mask_target.py'))
    ce = sys.modules['mmdet.models.losses.cross_entropy_loss']
    _ref = types.SimpleNamespace(mask_cross_entropy=ce.mask_cross_entropy, CrossEntropyLoss=ce.CrossEntropyLoss,
                                 FCNMaskHead=fcn.FCNMaskHead, HTCMaskHead=htc.HTCMaskHead,
                                 mask_target_single=mt.mask_target_single, mask_target=mt.mask_target)
    return _ref


# --------------------------------------------------------------------------- the fixture
def head_kwargs(kind):
    """Constructor kwargs of the fixture's heads: FCNMaskHead (class-specific, 1231 classes) and class-agnostic
    HTCMaskHead, at small channel counts."""
    kw = dict(num_convs=2, in_channels=FIX_IN, conv_out_channels=FIX_CONV, num_classes=FIX_CLASSES,
              loss_mask=dict(type='CrossEntropyLoss', use_mask=True, loss_weight=1.0))
    if kind == 'htc':
        kw['class_agnostic'] = True
    return kw


def fixture_inputs():
    """Seeded head parameters (both heads) and RoI inputs: 12 RoIs, labels 0, 1, 1230 and one class with several RoIs
    among them, binary and fractional targets."""
    g = torch.Generator().manual_seed(2862)

    def rn(*shape, s=1.0):
        return torch.randn(*shape, generator=g) * s

    params = {}
    for i in range(2):
        params['convs.%d.conv.weight' % i] = rn(FIX_CONV, FIX_IN if i == 0 else FIX_CONV, 3, 3, s=0.25)
        params['convs.%d.conv.bias' % i] = rn(FIX_CONV, s=0.1)
    params['upsample.weight'] = rn(FIX_CONV, FIX_CONV, 2, 2, s=0.3)
    params['upsample.bias'] = rn(FIX_CONV, s=0.1)
    params['conv_res.conv.weight'] = rn(FIX_CONV, FIX_CONV, 1, 1, s=0.3)
    params['conv_res.conv.bias'] = rn(FIX_CONV, s=0.1)
    logits = {'fcn': (rn(FIX_CLASSES, FIX_CONV, 1, 1, s=0.5), rn(FIX_CLASSES, s=0.3)),
              'htc': (rn(1, FIX_CONV, 1, 1, s=0.5), rn(1, s=0.3))}
    feats = rn(FIX_P, FIX_IN, FIX_ROI, FIX_ROI)
    res_feat = rn(FIX_P, FIX_CONV, FIX_ROI, FIX_ROI)
    labels = torch.randint(0, FIX_CLASSES, (FIX_P,), generator=g)
    labels[0], labels[1], labels[2] = 0, 1, FIX_CLASSES - 1
    labels[3:7] = 42
    targets = (torch.rand(FIX_P, 2 * FIX_ROI, 2 * FIX_ROI, generator=g) > 0.5).float()
    targets[-1] = torch.rand(2 * FIX_ROI, 2 * FIX_ROI, generator=g)
    return dict(params=params, logits=logits, feats=feats, res_feat=res_feat, labels=labels, targets=targets)


def head_params(inp, kind):
    p = {k: v for k, v in inp['params'].items() if kind == 'htc' or not k.startswith('conv_res')}
    p['conv_logits.weight'], p['conv_logits.bias'] = inp['logits'][kind]
    return p


def run_mask_loss(head, inp, kind, device='cpu', dtype=torch.float32):
    """loss_mask of ``head`` on the fixture inputs and its gradients w.r.t. conv_logits.weight (FIX_ROWS of its
    [classes, Cin] view), conv_logits.bias and conv_logits' input y."""
    head.load_state_dict(head_params(inp, kind), strict=True)
    head.to(device, dtype).train()
    head.zero_grad()
    seen = {}

    def grab(module, args):
        args[0].retain_grad()
        seen['y'] = args[0]
    hook = head.conv_logits.register_forward_pre_hook(grab)
    try:
        feats = inp['feats'].to(device, dtype)
        if kind == 'htc':
            mask_pred = head(feats, inp['res_feat'].to(device, dtype), return_feat=False)
        else:
            mask_pred = head(feats)
        if 'y' not in seen and hasattr(mask_pred, 'y'):     # a lazy handle: conv_logits has not run
            seen['y'] = mask_pred.y
            mask_pred.y.retain_grad()
        loss = head.loss(mask_pred, inp['targets'].to(device, dtype), inp['labels'].to(device))['loss_mask']
        loss.sum().backward()
    finally:
        hook.remove()
    w = head.conv_logits.weight.grad.detach()
    return dict(loss_mask=loss.detach().reshape(1), dW=w.reshape(w.shape[0], -1)[FIX_ROWS],
                db=head.conv_logits.bias.grad.detach(), dY=seen['y'].grad.detach(), y=seen['y'].detach())
