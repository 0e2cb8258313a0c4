"""GPU: the fused mask loss (bags_mask_fwd / bags_mask_bwd, ops.MaskBCEFunction, MaskPredHandle).

  * the kernels against the float64 oracle (tests/mask_oracle.py), bf16 and fp32 y, at the config shape and at the
    edges (P = 0, 1, 7, 1000, odd Cin and H x W, invalid labels, one channel), and against the materialised route;
  * the committed reference fixture (FCNMaskHead, class-agnostic HTCMaskHead) through the autograd function;
  * only the gradients autograd asks for; determinism of eager calls and CUDA-graph replays;
  * a head step through MaskPredHandle against the same step through a materialised handle, and the peak memory of
    the fused route against the size of one [P, classes, H, W] logits tensor.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import mask_oracle as MO
from balancedgroupsoftmax_b200 import mask_head as MH
from balancedgroupsoftmax_b200 import ops

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _inputs(P, Cin=256, H=28, W=28, C=1231, dtype=torch.bfloat16, seed=0, invalid=False, label_classes=None):
    g = torch.Generator().manual_seed(seed)
    y = torch.relu(torch.randn(P, Cin, H, W, generator=g)).to(dtype)
    Wt = torch.randn(C, Cin, generator=g) * (2.0 / Cin) ** 0.5
    b = torch.randn(C, generator=g) * 0.1
    labels = torch.randint(0, label_classes or C, (P,), generator=g)
    if P >= 4 and label_classes is None:
        labels[:4] = torch.tensor([0, C - 1, 17, 17]) % C
    if invalid and P >= 7:
        labels[4], labels[6] = C, -1
    t = (torch.rand(P, H, W, generator=g) > 0.5).float()
    return y, Wt, b, labels, t


def _fused(y, Wt, b, labels, t, gout=None, need=(True, True, True)):
    yd, Wd, bd, ld, td = (v.to(DEV) for v in (y, Wt, b, labels, t))
    loss, g, rsum, index = ops.mask_fwd(yd, Wd, bd, ld, td)
    go = None if gout is None else torch.tensor([gout], device=DEV)
    dW, db, dY = ops.mask_bwd(g, rsum, go, Wd, ld, index, tuple(yd.shape), yd.dtype, *need)
    return dict(loss=loss, g=g, index=index, dW=dW, db=db, dY=dY)


def _close(got, want, rtol, what):
    got, want = got.double().cpu(), want.double().cpu()
    err = (got - want).abs().max().item() if want.numel() else 0.0
    scale = want.abs().max().item() if want.numel() else 0.0
    assert err <= rtol * scale + 1e-12, '%s: max err %g vs scale %g' % (what, err, scale)


def _check(out, y, Wt, b, labels, t, gout=1.0):
    o = MO.mask_terms(y.float(), Wt, b, labels, t, gout=gout)
    P = y.shape[0]
    assert abs(out['loss'].item() - o['loss'].item()) <= 2e-5 * max(abs(o['loss'].item()), 1e-3), \
        (out['loss'].item(), o['loss'].item())
    _close(out['g'].reshape(P, -1), o['g'], 2e-5, 'g')
    rt = 2e-2 if y.dtype == torch.bfloat16 else 2e-5          # dY is stored in y's dtype
    for name, tol in (('dW', 2e-5), ('db', 2e-5), ('dY', rt)):
        if out[name] is not None:
            _close(out[name], o[name], tol, name)
    C = Wt.shape[0]
    absent = torch.ones(C, dtype=torch.bool)
    lv = labels[(labels >= 0) & (labels < C)]
    absent[lv] = False
    if out['dW'] is not None:
        assert (out['dW'].cpu()[absent] == 0).all()
    if out['db'] is not None:
        assert (out['db'].cpu()[absent] == 0).all()
    invalid = ~((labels >= 0) & (labels < C))
    if out['dY'] is not None and invalid.any():
        assert (out['dY'].cpu()[invalid] == 0).all()


CASES = {
    'p256': dict(P=256),
    'p1': dict(P=1),
    'p7_invalid': dict(P=7, invalid=True),
    'p1000': dict(P=1000, Cin=64),
    'odd': dict(P=37, Cin=13, H=13, W=17, invalid=True),
    'odd_hw_aligned': dict(P=9, Cin=7, H=6, W=10, C=5),
    'one_channel': dict(P=300, Cin=32, C=1),
    'skewed': dict(P=333, Cin=40, label_classes=3),     # many RoIs per class: the backward's split class sums
}


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32], ids=['bf16', 'fp32'])
@pytest.mark.parametrize('case', list(CASES))
def test_kernels_match_float64(case, dtype):
    kw = dict(CASES[case])
    y, Wt, b, labels, t = _inputs(dtype=dtype, **kw)
    if kw.get('C') == 1:
        labels.zero_()
    _check(_fused(y, Wt, b, labels, t, gout=-0.6), y, Wt, b, labels, t, gout=-0.6)


def test_no_rois():
    y, Wt, b, labels, t = _inputs(0)
    out = _fused(y, Wt, b, labels, t)
    assert out['loss'].item() == 0.0
    assert (out['dW'] == 0).all() and (out['db'] == 0).all() and out['dY'].shape == (0, 256, 28, 28)


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32], ids=['bf16', 'fp32'])
def test_matches_materialised_route(dtype):
    """The same loss and gradients as conv_logits + CrossEntropyLoss(use_mask=True) on the GPU (fp32 conv)."""
    from balancedgroupsoftmax_b200.losses import CrossEntropyLoss
    y, Wt, b, labels, t = (v.to(DEV) for v in _inputs(64, dtype=dtype, seed=2))
    W4 = Wt.reshape(*Wt.shape, 1, 1)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        yr, Wr, br = y.float().clone().requires_grad_(True), W4.clone().requires_grad_(True), b.clone().requires_grad_(True)
        ref = CrossEntropyLoss(use_mask=True)(F.conv2d(yr, Wr, br), t, labels)
        ref.sum().backward()
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    yf, Wf, bf = y.clone().requires_grad_(True), W4.clone().requires_grad_(True), b.clone().requires_grad_(True)
    got = ops.MaskBCEFunction.apply(yf, Wf, bf, labels, t)
    got.sum().backward()
    assert got.shape == ref.shape == (1,)
    torch.testing.assert_close(got, ref.detach(), rtol=2e-5, atol=0)
    assert yf.grad.dtype == dtype and Wf.grad.shape == Wr.shape and Wf.grad.dtype == torch.float32
    _close(Wf.grad, Wr.grad, 1e-4, 'dW')
    _close(bf.grad, br.grad, 1e-4, 'db')
    _close(yf.grad, yr.grad, 2e-2 if dtype == torch.bfloat16 else 1e-4, 'dY')


@pytest.mark.parametrize('kind', ['fcn', 'htc'])
def test_autograd_function_matches_reference_fixture(kind):
    """The fixture's reference loss and gradients from conv_logits' input y (computed in float64 by this package's
    convs, which the CPU test pins to the reference's)."""
    fix = np.load(MO.FIXTURE)
    inp = MO.fixture_inputs()
    cls = MH.HTCMaskHead if kind == 'htc' else MH.FCNMaskHead
    y = MO.run_mask_loss(cls(**MO.head_kwargs(kind)), inp, kind, dtype=torch.float64)['y']
    W, b = inp['logits'][kind]
    labels = torch.zeros_like(inp['labels']) if kind == 'htc' else inp['labels']
    yd = y.float().to(DEV).requires_grad_(True)
    Wd, bd = W.to(DEV).requires_grad_(True), b.to(DEV).requires_grad_(True)
    loss = ops.MaskBCEFunction.apply(yd, Wd, bd, labels.to(DEV), inp['targets'].to(DEV))
    loss.sum().backward()
    _close(loss, torch.from_numpy(fix['%s_loss_mask' % kind]), 1e-5, 'loss')
    _close(Wd.grad.reshape(Wd.shape[0], -1)[MO.FIX_ROWS], torch.from_numpy(fix['%s_dW' % kind]), 1e-5, 'dW')
    _close(bd.grad, torch.from_numpy(fix['%s_db' % kind]), 1e-5, 'db')
    _close(yd.grad, torch.from_numpy(fix['%s_dY' % kind]), 1e-5, 'dY')


@pytest.mark.parametrize('frozen', ['weight', 'input', 'bias'])
def test_only_requested_gradients(frozen):
    y, Wt, b, labels, t = (v.to(DEV) for v in _inputs(16, seed=5))
    yr = y.clone().requires_grad_(frozen != 'input')
    Wr = Wt.clone().requires_grad_(frozen != 'weight')
    br = b.clone().requires_grad_(frozen != 'bias')
    ops.MaskBCEFunction.apply(yr, Wr, br, labels, t).sum().backward()
    full = _fused(y.cpu(), Wt.cpu(), b.cpu(), labels.cpu(), t.cpu())
    for tensor, name, key in ((yr, 'input', 'dY'), (Wr, 'weight', 'dW'), (br, 'bias', 'db')):
        if name == frozen:
            assert tensor.grad is None
        else:
            assert torch.equal(tensor.grad, full[key]), key


def test_eager_and_graph_replays_are_bit_identical():
    y, Wt, b, labels, t = (v.to(DEV) for v in _inputs(256, invalid=True))
    gout = torch.tensor([0.75], device=DEV)

    def step():
        loss, g, rsum, index = ops.mask_fwd(y, Wt, b, labels, t)
        return (loss, g) + ops.mask_bwd(g, rsum, gout, Wt, labels, index, tuple(y.shape), y.dtype)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        e1 = [v.clone() for v in step()]
        e2 = [v.clone() for v in step()]
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            static = step()
    torch.cuda.current_stream().wait_stream(s)
    replays = []
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        replays.append([v.clone() for v in static])
    for a, b_ in zip(e1, e2):
        assert torch.equal(a, b_)
    for r in replays:
        for a, b_ in zip(e1, r):
            assert torch.equal(a, b_)


# --------------------------------------------------------------------------- heads
def _head(cls, seed=3, **kw):
    torch.manual_seed(seed)
    h = cls(num_convs=4, in_channels=256, conv_out_channels=256, num_classes=1231, **kw)
    h.init_weights()
    return h.to(DEV).train()


def _head_step(head, x, t, labels, materialise=False, htc=False):
    head.zero_grad()
    xr = x.clone().requires_grad_(True)
    pred = head(xr, return_feat=False) if htc else head(xr)
    assert isinstance(pred, MH.MaskPredHandle)
    if materialise:
        pred.float()
    loss = head.loss(pred, t, labels)['loss_mask']
    loss.sum().backward()
    return loss.detach(), {k: p.grad.clone() for k, p in head.named_parameters() if p.grad is not None}, xr.grad.clone()


@pytest.mark.parametrize('cls', ['FCNMaskHead', 'HTCMaskHead', 'HTCMaskHead_agnostic'])
def test_head_step_matches_materialised_handle(cls):
    kw = dict(class_agnostic=True) if cls.endswith('agnostic') else {}
    klass = getattr(MH, cls.replace('_agnostic', ''))
    g = torch.Generator().manual_seed(9)
    x = torch.randn(48, 256, 14, 14, generator=g).to(DEV)
    t = (torch.rand(48, 28, 28, generator=g) > 0.5).float().to(DEV)
    labels = torch.randint(0, 1231, (48,), generator=g).to(DEV)
    htc = klass is MH.HTCMaskHead
    fused = _head_step(_head(klass, **kw), x, t, labels, htc=htc)
    dense = _head_step(_head(klass, **kw), x, t, labels, materialise=True, htc=htc)
    torch.testing.assert_close(fused[0], dense[0], rtol=1e-3, atol=0)
    assert set(fused[1]) == set(dense[1]) and 'conv_logits.weight' in dense[1]
    for k in dense[1]:
        _close(fused[1][k], dense[1][k], 2e-2, k)      # the dense route's convs run TF32
    _close(fused[2], dense[2], 2e-2, 'dx')


def test_loss_weight_is_applied():
    x = torch.randn(8, 256, 14, 14, device=DEV)
    t = (torch.rand(8, 28, 28, device=DEV) > 0.5).float()
    labels = torch.randint(0, 1231, (8,), device=DEV)
    h1 = _head(MH.FCNMaskHead)
    h2 = _head(MH.FCNMaskHead, loss_mask=dict(type='CrossEntropyLoss', use_mask=True, loss_weight=0.25))
    l1 = h1.loss(h1(x), t, labels)['loss_mask']
    l2 = h2.loss(h2(x), t, labels)['loss_mask']
    torch.testing.assert_close(l2, l1 * 0.25)


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
def test_fused_route_never_allocates_the_logits(dtype):
    """The peak memory of the fused loss and backward, above what is live before it, stays below one [P, classes,
    H, W] logits tensor in y's dtype (the materialised route allocates at least that)."""
    P = 256
    y, Wt, b, labels, t = (v.to(DEV) for v in _inputs(P, dtype=dtype, seed=4))
    W4 = Wt.reshape(*Wt.shape, 1, 1).requires_grad_(True)
    br = b.clone().requires_grad_(True)
    yr = y.clone().requires_grad_(True)
    logits_bytes = P * 1231 * 28 * 28 * y.element_size()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ops.MaskBCEFunction.apply(yr, W4, br, labels, t).sum().backward()
    torch.cuda.synchronize()
    fused_peak = torch.cuda.max_memory_allocated() - base
    assert fused_peak < logits_bytes // 4, (fused_peak, logits_bytes)
    from balancedgroupsoftmax_b200.losses import CrossEntropyLoss
    yr.grad = W4.grad = br.grad = None
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    CrossEntropyLoss(use_mask=True)(F.conv2d(yr, W4.to(dtype), br.to(dtype)).float(), t, labels).backward()
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base >= logits_bytes
