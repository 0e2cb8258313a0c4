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
    """{'loss', 'z' [P,HW] (0 on invalid rows), 'g' [P,HW], 'dW' [C,Cin], 'db' [C], 'dY' [P,Cin,H,W]} in float64,
    on y's device."""
    y = y.double()
    dev = y.device
    P, Cin = y.shape[:2]
    yf = y.reshape(P, Cin, -1)
    HW = yf.shape[2]
    W = W.double().to(dev).reshape(W.shape[0], -1)
    C = W.shape[0]
    b = torch.zeros(C, dtype=torch.float64, device=dev) if b is None else b.double().to(dev)
    t = targets.double().to(dev).reshape(P, HW)
    labels = labels.to(dev)
    valid = ((labels >= 0) & (labels < C)).nonzero().reshape(-1)
    lv = labels[valid]
    z = torch.zeros(P, HW, dtype=torch.float64, device=dev)
    z[valid] = torch.einsum('pc,pcq->pq', W[lv], yf[valid]) + b[lv].unsqueeze(1)
    n = float(P * HW)
    ell = torch.clamp(z, min=0) - z * t + torch.log1p(torch.exp(-z.abs()))
    g = torch.zeros(P, HW, dtype=torch.float64, device=dev)
    g[valid] = (torch.sigmoid(z[valid]) - t[valid]) / n
    gg = g * float(gout)
    dW = torch.zeros(C, Cin, dtype=torch.float64, device=dev)
    dW.index_add_(0, lv, torch.einsum('pq,pcq->pc', gg[valid], yf[valid]))
    db = torch.zeros(C, dtype=torch.float64, device=dev)
    db.index_add_(0, lv, gg[valid].sum(1))
    dY = torch.zeros(P, Cin, HW, dtype=torch.float64, device=dev)
    dY[valid] = gg[valid].unsqueeze(1) * W[lv].unsqueeze(2)
    loss = ell[valid].sum() / n if P > 0 else torch.zeros((), dtype=torch.float64, device=dev)
    return dict(loss=loss, z=z, g=g, dW=dW, db=db, dY=dY.reshape(y.shape))


# --------------------------------------------------------------------------- per-element bounds of the fp32 kernels
U = 2.0 ** -24
TILE = 64                 # bags_mask_fwd's pixels per CTA (nat.MASK_TILE)
TINY = 2.0 ** -146        # a few subnormal ulps: what a rounding near the bottom of the fp32 range can add absolutely


def valid_rows(labels, classes):
    return (labels >= 0) & (labels < classes)


def reduction_bounds(g, y, labels, classes, gout=1.0):
    """Bounds on |fp32 kernel - float64| of dW [C, Cin] and db [C] summed from a given g [P, HW] (float64, e.g. the
    kernel's own g, or |g| plus its own bound): only the reduction's roundings.

    A product g y of pixel q in tile t goes through at most 2 fma of its lane, the 5 levels of the warp sum (rsum),
    ceil(pairs / 8) additions of its class-unit warp (pairs = the class's RoIs times its tiles), the 8 warp partials
    and the final fma(gout, total, 0): depth ceil(pairs / 8) + 16, each rounding at most u of a partial sum of
    magnitude below sum |g y|; a db term goes through one addition fewer.  So |err| <= depth u |gout| sum |g| |y|
    (and sum |g|), plus depth subnormal ulps per term for products near underflow."""
    dev = g.device
    g = g.double().abs()
    P = g.shape[0]
    yf = y.double().abs().reshape(P, y.shape[1], -1)
    HW = yf.shape[2]
    tiles = -(-HW // TILE)
    labels = labels.to(dev)
    valid = valid_rows(labels, classes).nonzero().reshape(-1)
    lv = labels[valid]
    counts = torch.bincount(lv, minlength=classes).double()
    depth = torch.ceil(counts * tiles / 8) + 16
    dW = torch.zeros(classes, yf.shape[1], dtype=torch.float64, device=dev)
    dW.index_add_(0, lv, torch.einsum('pq,pcq->pc', g[valid], yf[valid]))
    db = torch.zeros(classes, dtype=torch.float64, device=dev)
    db.index_add_(0, lv, g[valid].sum(1))
    go = abs(float(gout))
    tiny = depth * counts * HW * TINY
    return dict(dW=(depth * U * go).unsqueeze(1) * dW + tiny.unsqueeze(1), db=depth * U * go * db + tiny)


def error_bounds(y, W, b, labels, targets, gout=1.0, z_exact=False):
    """Per-element bounds on |fp32 kernel - float64 mask_terms| for g [P, HW], the loss, dW [C, Cin] and db [C].  y
    and W are taken as given (y already in its operand dtype); ``z_exact``: the logits are exact in fp32 (small
    integers, asserted by the caller), so only the kernel's own BCE arithmetic errs.  u = 2^-24 throughout.

    z = b[l] + sum_c W[l,c] y[p,c,q]: fma chains of ceil(Cin / NG) channels per channel group (NG = 16 for four
    pixels a thread, 4 for one), the min(Cin, NG) nonzero group sums added in order, then the bias: no term goes
    through more than Cin + 2 roundings, ez = (Cin + 2) u (sum_c |W y| + |b|).

    g = (s - t) / n, n = P H W (exact in fp32 below 2^24): e = expf(-|z|) errs by 2 ulp <= 4 u relative, 1 + e and
    the division by u each; s = 1 / (1 + e) or e / (1 + e) has |d ln s / d ln e| = 1 - s, so |ds| <= (4 u (1 - s)
    + 2 u) s <= 6 u s.  fl(s - t) adds u |s - t| and the division u |g|.  So |dg| <= (6 u s + 2 u |s - t|) / n +
    u |g| (the second u |s - t| covers the second order; a subnormal e or g adds a few ulps of 2^-149, TINY).  With an inexact z, g also moves by max |sigmoid'| ez <= (s (1 - s) + ez) ez / n, and s, |s - t| by ez.

    The loss: each pixel's fmaxf(z, 0) - z t + log1pf(e) rounds z t, the subtraction and the addition (u of |z t|,
    |max(z, 0) - z t| and the term), log1pf errs by 1 ulp (2 u) of log1p(E) and e's 4 u E <= 8 u log1p(E) more
    (E <= 2 log1p(E) for E <= 1), and an inexact z moves the term by at most ez (|d/dz| = |sigmoid(z) - t| <= 1).
    The terms are summed by a 5-level warp sum, the two warps of the tile, ceil(CTAs / 256) partials per thread of
    the last CTA, a 5-level warp sum and 8 warp totals: depth ceil(CTAs / 256) + 19 over sum |terms|; the division
    by n adds u |loss|.

    dW, db: reduction_bounds of |g| + its bound, plus sum |dg| |y| (and sum |dg|) of g's own error."""
    dev = y.device
    y = y.double()
    P, Cin = y.shape[:2]
    yf = y.reshape(P, Cin, -1)
    HW = yf.shape[2]
    n = float(P * HW)
    assert n < 2 ** 24, 'n must be exact in fp32'
    Wd = W.double().to(dev).reshape(W.shape[0], -1)
    C = Wd.shape[0]
    bb = torch.zeros(C, dtype=torch.float64, device=dev) if b is None else b.double().to(dev)
    labels = labels.to(dev)
    t = targets.double().to(dev).reshape(P, HW)
    o = mask_terms(y, Wd, bb, labels, t, gout=gout)
    vmask = valid_rows(labels, C)
    valid = vmask.nonzero().reshape(-1)
    lv = labels[valid]
    ez = torch.zeros(P, HW, dtype=torch.float64, device=dev)
    if not z_exact:
        ez[valid] = (Cin + 2) * U * (torch.einsum('pc,pcq->pq', Wd[lv].abs(), yf[valid].abs())
                                     + bb[lv].abs().unsqueeze(1))
    z = o['z']
    s = torch.sigmoid(z)
    d = (s - t).abs()
    e_g = ((6 * U * (s + ez) + 2 * U * (d + ez)) + (s * (1 - s) + ez) * ez) / n + U * (o['g'].abs() + ez / n) + TINY
    e_g[~vmask] = 0
    # the loss
    L1 = torch.log1p(torch.exp(-z.abs()))
    a = torch.clamp(z, min=0) - z * t
    term = a + L1
    e_term = U * ((z * t).abs() + a.abs() + term.abs() + 10 * L1) + ez + TINY
    tiles = -(-HW // TILE)
    depth = -(-(P * tiles) // 256) + 19
    vt = vmask.unsqueeze(1).expand(P, HW)
    e_loss = ((depth * U * term[vt].abs().sum() + e_term[vt].sum()) / n + U * o['loss'].abs()).item()
    # dW, db
    red = reduction_bounds(o['g'].abs() + e_g, yf, labels, C, gout)
    go = abs(float(gout))
    dW = torch.zeros(C, Cin, dtype=torch.float64, device=dev)
    dW.index_add_(0, lv, torch.einsum('pq,pcq->pc', e_g[valid], yf[valid].abs()))
    db = torch.zeros(C, dtype=torch.float64, device=dev)
    db.index_add_(0, lv, e_g[valid].sum(1))
    return dict(terms=o, g=e_g, loss=e_loss, dW=red['dW'] + go * dW, db=red['db'] + go * db)


# --------------------------------------------------------------------------- the three tiers of input
EXACT_LIMIT = 2.0 ** 20
SAT_W = 256.0
INVALID_LABELS = (-1, 'classes', 'classes+7', 2 ** 40)


def tier_inputs(tier, P, Cin, HW, classes, dtype=torch.float32, seed=0, soft=False, invalid=False, one_class=False):
    """(y [P, Cin, HW] in ``dtype``, W [classes, Cin], b [classes], labels [P], targets [P, HW]) on CPU.

    'exact'     y in [-2, 2] and W small integers (the range chosen so that z spreads over about +-30), b a multiple
                of 2^-3: z is exact in fp32 in any summation order (exact_partial_max < 2^20).
    'saturated' y[:, 0] = +-1 times W[:, 0] = +-256, the other channels y in {0, 1} times W in {0, +-1/8}, |b| <= 4:
                |z| >= 128 everywhere (saturated_min_abs_z), so expf(-|z|) is 0 and s is exactly 0 or 1; 0/1 targets.
    'numeric'   y = relu(normal), W normal / sqrt(Cin / 2), b normal / 10, as in real use.
    Targets are 0/1, or multiples of 1/8 with ``soft``.  ``invalid`` puts the labels -1, classes, classes + 7 and
    2^40 on rows 1, 3, 5, 7; ``one_class`` gives every RoI the same class."""
    g = torch.Generator().manual_seed(seed)
    if tier == 'exact':
        k = max(1, round((900.0 / Cin) ** 0.5))
        y = torch.randint(-2, 3, (P, Cin, HW), generator=g).float()
        W = torch.randint(-k, k + 1, (classes, Cin), generator=g).float()
        b = torch.randint(-16, 17, (classes,), generator=g).float() / 8
    elif tier == 'saturated':
        y = torch.randint(0, 2, (P, Cin, HW), generator=g).float()
        y[:, 0] = torch.randint(0, 2, (P, HW), generator=g).float() * 2 - 1
        W = torch.randint(-1, 2, (classes, Cin), generator=g).float() / 8
        W[:, 0] = SAT_W * (torch.randint(0, 2, (classes,), generator=g).float() * 2 - 1)
        b = torch.randint(-32, 33, (classes,), generator=g).float() / 8
        soft = False
    else:
        assert tier == 'numeric', tier
        y = torch.relu(torch.randn(P, Cin, HW, generator=g))
        W = torch.randn(classes, Cin, generator=g) * (2.0 / Cin) ** 0.5
        b = torch.randn(classes, generator=g) * 0.1
    y = y.to(dtype)
    if one_class:
        labels = torch.full((P,), classes // 2, dtype=torch.int64)
    else:
        labels = torch.randint(0, classes, (P,), generator=g)
    if invalid:
        for i, l in zip(range(1, P, 2), INVALID_LABELS):
            labels[i] = classes if l == 'classes' else classes + 7 if l == 'classes+7' else l
    if soft:
        t = torch.randint(0, 9, (P, HW), generator=g).float() / 8
        t[::2] = (t[::2] >= 0.5).float()
    else:
        t = torch.randint(0, 2, (P, HW), generator=g).float()
    return y, W, b, labels, t


def _row_sums(y, W, b, labels):
    P, Cin = y.shape[:2]
    yf = y.double().reshape(P, Cin, -1)
    C = W.shape[0]
    valid = valid_rows(labels, C).nonzero().reshape(-1)
    lv = labels[valid]
    b = torch.zeros(C) if b is None else b
    return yf, W.double()[lv], b.double()[lv], valid


def exact_partial_max(y, W, b, labels):
    """max over valid pixels of sum_c |W y| + |b|: every partial sum of z is below it in magnitude."""
    yf, Wl, bl, valid = _row_sums(y, W, b, labels)
    if valid.numel() == 0:
        return 0.0
    return (torch.einsum('pc,pcq->pq', Wl.abs(), yf[valid].abs()) + bl.abs().unsqueeze(1)).max().item()


def saturated_min_abs_z(y, W, b, labels):
    """min over valid pixels of |z|."""
    yf, Wl, bl, valid = _row_sums(y, W, b, labels)
    if valid.numel() == 0:
        return float('inf')
    return (torch.einsum('pc,pcq->pq', Wl, yf[valid]) + bl.unsqueeze(1)).abs().min().item()


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
    from balancedgroupsoftmax_b200.mask_head import MaskPredHandle
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
        if 'y' not in seen and isinstance(mask_pred, MaskPredHandle):     # a lazy handle: conv_logits has not run
            seen['y'] = mask_pred.input
            mask_pred.input.retain_grad()
        loss = head.loss(mask_pred, inp['targets'].to(device, dtype), inp['labels'].to(device))['loss_mask']
        loss.sum().backward()
    finally:
        hook.remove()
    w = head.conv_logits.weight.grad.detach()
    return dict(loss_mask=loss.detach().reshape(1), dW=w.reshape(w.shape[0], -1)[FIX_ROWS],
                db=head.conv_logits.bias.grad.detach(), dY=seen['y'].grad.detach(), y=seen['y'].detach())
