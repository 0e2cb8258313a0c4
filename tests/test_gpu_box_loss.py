"""GPU: the fused class-specific box loss (bags_box_fwd / bags_box_bwd, ops.SmoothL1BoxFunction, fuse_bbox_loss).

  * the kernels against the float64 oracle (tests/box_oracle.py) with per-element bounds for fp32 accumulation over K,
    bf16 and fp32 x, at the bench shape and at the edges (odd N, K = 64, no positive, N = 0, one class, labels 0,
    classes - 1 and >= classes, zero box weights, |d| exactly at 0 and beta, beta 1 and 1/9, gout != 1), every output
    subset of the backward, and dW rows of absent classes exactly zero;
  * determinism: eager calls and CUDA-graph replays are bit-identical (the capture also proves there is no host sync);
  * the four heads with fuse_bbox_loss on and off, and against the committed reference fixture;
  * the fallbacks to today's route.
"""
import itertools

import numpy as np
import pytest
import torch

import box_oracle as BO
from balancedgroupsoftmax_b200 import ops

pytestmark = pytest.mark.gpu
DEV = 'cuda'
U = 2.0 ** -24


def _inputs(N, K, C=1231, frac=0.25, dtype=torch.bfloat16, seed=0, labels=None, beta=1.0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, K, generator=g).to(dtype)
    W = torch.randn(4 * C, K, generator=g) * (1.0 / K ** 0.5)
    b = torch.randn(4 * C, generator=g) * 0.1
    if labels is None:
        labels = torch.zeros(N, dtype=torch.int64)
        npos = int(N * frac)
        labels[:npos] = torch.randint(1, C, (npos,), generator=g)
        labels = labels[torch.randperm(N, generator=g)]
    targets = torch.randn(N, 4, generator=g) * 1.2 * beta
    weights = (torch.rand(N, 4, generator=g) > 0.1).float()
    return x, W, b, labels, targets, weights


def _edge_inputs(dtype, beta):
    """Labels 0, 1, C - 1, C and C + 7; class C - 1 has zero W rows and bias, so pred = 0 exactly and the targets put d
    at 0, +-beta and beta / 2; some zero box weights."""
    N, K, C = 67, 64, 1231
    x, W, b, labels, targets, weights = _inputs(N, K, C, frac=0.6, dtype=dtype, seed=3, beta=beta)
    W[4 * (C - 1):] = 0.
    b[4 * (C - 1):] = 0.
    labels[:6] = torch.tensor([C - 1, C - 1, 0, 1, C, C + 7])
    targets[:2] = torch.tensor([[0., beta, -beta, 0.5 * beta], [-0., -beta, beta, -0.5 * beta]])
    weights[3, 2] = 0.
    return x, W, b, labels, targets, weights


def _run(x, W, b, labels, targets, weights, beta, avg, gout=None, need=(True, True, True)):
    xd, Wd, bd = x.to(DEV), W.to(DEV), b.to(DEV)
    ld, td, wd = labels.to(DEV), targets.to(DEV), weights.to(DEV)
    loss, g, index, pred = ops.box_fwd(xd, Wd, bd, ld, td, wd, beta, avg, want_pred=True)
    go = None if gout is None else torch.tensor([gout], dtype=torch.float32, device=DEV)
    dW, db, dX = ops.box_bwd(g, go, xd, Wd, ld, index, *need)
    return dict(loss=loss, g=g, pred=pred, index=index, dW=dW, db=db, dX=dX)


def _check(out, x, W, b, labels, targets, weights, beta, avg, gout=None):
    go = 1.0 if gout is None else gout
    ref = BO.box_terms(x.float(), W, b, labels, targets, weights, beta, avg, gout=go)
    bnd = BO.error_bounds(x.float(), W, b, labels, weights, beta, avg, gout=go)
    bnd['g'] = BO.error_bounds(x.float(), W, b, labels, weights, beta, avg)['g']     # g itself does not carry gout
    for name in ('pred', 'g', 'dW', 'db', 'dX'):
        if out[name] is None:
            continue
        got = out[name].double().cpu()
        want = ref[name]
        tol = bnd[name]
        if name == 'dX' and x.dtype == torch.bfloat16:
            tol = tol + 2.0 ** -8 * want.abs()             # dX is stored in x's dtype
        bad = (got - want).abs() > tol
        assert not bad.any(), '%s: %d elements out of bound, first %s: got %r want %r tol %r' % (
            name, int(bad.sum()), bad.nonzero()[0].tolist(), got[bad][0].item(), want[bad][0].item(), tol[bad][0].item())
    # loss: pred's error moves sl1 by at most |sl1'| <= 1 times it; 4P + 2 roundings of the fixed-order sum
    C = W.shape[0] // 4
    pos = (labels > 0) & (labels < C)
    w = weights.double()
    e = (w * bnd['pred']).sum().item() / avg if len(labels) else 0.0
    mag = (w[pos] * (ref['pred'][pos] - targets.double()[pos]).abs()).sum().item() / avg if len(labels) else 0.0
    tol = 2 * e + (4 * int(pos.sum()) + 2) * U * mag + 1e-30
    assert abs(out['loss'].item() - ref['loss'].item()) <= tol, (out['loss'].item(), ref['loss'].item(), tol)
    if out['dW'] is not None:
        absent = torch.ones(C, dtype=torch.bool)
        absent[labels[pos]] = False
        rows = absent.repeat_interleave(4)
        assert torch.equal(out['dW'][rows.to(DEV)], torch.zeros_like(out['dW'][rows.to(DEV)])), 'absent-class dW rows'
    if out['db'] is not None:
        absent = torch.ones(C, dtype=torch.bool)
        absent[labels[pos]] = False
        assert (out['db'].cpu()[absent.repeat_interleave(4)] == 0).all()
    if out['dX'] is not None:
        assert (out['dX'].cpu()[~pos] == 0).all()


CASES = {
    'bench': dict(N=4096, K=1024),
    'odd_n': dict(N=257, K=1024),
    'k64': dict(N=300, K=64),
    'no_positive': dict(N=128, K=64, frac=0.0),
    'empty': dict(N=0, K=64),
    'bench_1024': dict(N=1024, K=1024),
}


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32], ids=['bf16', 'fp32'])
@pytest.mark.parametrize('case', list(CASES))
def test_kernels_match_float64(case, dtype):
    kw = dict(CASES[case])
    x, W, b, labels, targets, weights = _inputs(kw.pop('N'), kw.pop('K'), dtype=dtype, **kw)
    avg = float(max(len(labels), 1)) if len(labels) else 0.0
    out = _run(x, W, b, labels, targets, weights, 1.0, avg)
    _check(out, x, W, b, labels, targets, weights, 1.0, max(avg, 1.0))
    if not ((labels > 0) & (labels < 1231)).any():
        assert out['loss'].item() == 0.0
        assert (out['dW'] == 0).all() and (out['db'] == 0).all() and (out['dX'] == 0).all() and (out['g'] == 0).all()


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32], ids=['bf16', 'fp32'])
@pytest.mark.parametrize('beta', [1.0, 1.0 / 9], ids=['beta1', 'beta1_9'])
@pytest.mark.parametrize('gout', [None, -0.37], ids=['gout1', 'gout'])
def test_edges_match_float64(beta, dtype, gout):
    x, W, b, labels, targets, weights = _edge_inputs(dtype, beta)
    out = _run(x, W, b, labels, targets, weights, beta, float(len(labels)), gout=gout)
    _check(out, x, W, b, labels, targets, weights, beta, float(len(labels)), gout=gout)
    g = out['g'].cpu()
    # d = 0 -> 0; |d| = beta -> sign(d) (the linear branch); beta / 2 -> d / beta
    inv = np.float32(1.0) / np.float32(len(labels))
    want = torch.tensor([[0., -1., 1., -0.5], [0., 1., -1., 0.5]]) * weights[:2] * float(inv)
    assert torch.equal(g[:2], want)
    assert (g[2] == 0).all() and (g[4:6] == 0).all() and g[3, 2] == 0      # label 0, >= classes, zero weight


def test_every_positive_in_one_class():
    N, K = 1024, 256
    labels = torch.full((N,), 17, dtype=torch.int64)
    x, W, b, labels, targets, weights = _inputs(N, K, labels=labels, dtype=torch.bfloat16)
    out = _run(x, W, b, labels, targets, weights, 1.0, float(N))
    _check(out, x, W, b, labels, targets, weights, 1.0, float(N))
    idx = out['index'].cpu()
    assert idx[17].item() == 0 and idx[18].item() == N and torch.equal(idx[1232:], torch.arange(N, dtype=torch.int32))


def test_class_index_is_a_stable_sort():
    x, W, b, labels, targets, weights = _inputs(5000, 64, C=300, frac=0.5, seed=7)
    labels[:3] = torch.tensor([300, 0, 299])
    idx = _run(x, W, b, labels, targets, weights, 1.0, 5000.0)['index'].cpu().long()
    pos = ((labels > 0) & (labels < 300)).nonzero().reshape(-1)
    order = pos[torch.argsort(labels[pos], stable=True)]
    counts = torch.bincount(labels[pos], minlength=300)
    assert torch.equal(idx[:301], torch.cat([torch.zeros(1, dtype=torch.long), counts.cumsum(0)]))
    assert torch.equal(idx[301:301 + len(pos)], order)


@pytest.mark.parametrize('need', list(itertools.product([False, True], repeat=3)),
                         ids=lambda n: 'dW%d_db%d_dX%d' % n)
def test_backward_output_subsets(need):
    x, W, b, labels, targets, weights = _inputs(513, 512 + 64)          # two K slices, the second partial
    full = _run(x, W, b, labels, targets, weights, 1.0, 513.0, gout=2.5)
    part = _run(x, W, b, labels, targets, weights, 1.0, 513.0, gout=2.5, need=need)
    for flag, name in zip(need, ('dW', 'db', 'dX')):
        if flag:
            assert torch.equal(part[name], full[name]), name
        else:
            assert part[name] is None


def test_eager_and_graph_replays_are_bit_identical():
    x, W, b, labels, targets, weights = [t.to(DEV) for t in _inputs(4096, 1024)]
    gout = torch.tensor([0.75], device=DEV)

    def step():
        loss, g, index, _ = ops.box_fwd(x, W, b, labels, targets, weights, 1.0, 4096.0)
        return (loss, g) + ops.box_bwd(g, gout, x, W, labels, index)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        e1 = [t.clone() for t in step()]
        e2 = [t.clone() for t in step()]
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            static = step()
    torch.cuda.current_stream().wait_stream(s)
    replays = []
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        replays.append([t.clone() for t in static])
    for a, b_ in zip(e1, e2):
        assert torch.equal(a, b_)
    for r in replays:
        for a, b_ in zip(e1, r):
            assert torch.equal(a, b_)


def test_autograd_function_grads_in_parameter_dtypes():
    x, W, b, labels, targets, weights = [t.to(DEV) for t in _inputs(300, 64)]
    xr = x.clone().requires_grad_(True)
    Wr, br = W.clone().requires_grad_(True), b.clone().requires_grad_(True)
    loss = ops.SmoothL1BoxFunction.apply(xr, Wr, br, labels, targets, weights, 1.0, 300.0)
    (loss[0] * 3.0).backward()
    assert xr.grad.dtype == torch.bfloat16 and Wr.grad.dtype == torch.float32 and br.grad.dtype == torch.float32
    ref = _run(*[t.cpu() for t in (x, W, b, labels, targets, weights)], 1.0, 300.0, gout=3.0)
    assert torch.equal(Wr.grad, ref['dW']) and torch.equal(br.grad, ref['db']) and torch.equal(xr.grad, ref['dX'])
    # only what autograd asks for: a frozen weight gets no gradient
    xr.grad = None
    Wf = W.clone()
    ops.SmoothL1BoxFunction.apply(xr, Wf, br, labels, targets, weights, 1.0, 300.0)[0].backward()
    assert Wf.grad is None and xr.grad is not None


# --------------------------------------------------------------------------- heads
HEADS = ['GSBBoxHeadWith0', 'GSBBoxHead', 'GSBBoxHeadWith0Reweight', 'ReweightBBoxHead', 'GSBBoxHeadWith0_graph_cache']


def _head(name, fuse, params=None, **extra):
    from balancedgroupsoftmax_b200 import head as H
    from balancedgroupsoftmax_b200.tables import synthetic_tables
    tables = synthetic_tables()
    sizes = dict(num_fcs=2, in_channels=BO.FIX_IN, fc_out_channels=BO.FIX_FC, roi_feat_size=BO.FIX_ROI,
                 num_classes=1231, loss_bbox=dict(type='SmoothL1Loss', beta=1.0, loss_weight=1.0))
    sizes.update(extra)
    execution = dict(fuse_bbox_loss=fuse)
    torch.manual_seed(11)
    if name == 'ReweightBBoxHead':
        h = H.ReweightBBoxHead(reweight_cfg=dict(cls_weights=torch.rand(1231) + 0.5, **execution), **sizes)
    else:
        gs = dict(tables=tables, others_sample_ratio=8.0, num_bins=tables.num_bins,
                  loss_bin=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0), **execution)
        if name == 'GSBBoxHeadWith0Reweight':
            gs['cls_weights'] = [torch.rand(int(tables.pred_slice[g, 1])) + 0.5 for g in range(1, tables.num_bins)]
        if name.endswith('_graph_cache'):
            gs['graph_cache'] = True
        h = getattr(H, name.replace('_graph_cache', ''))(gs_config=gs, **sizes)
    h.init_weights()
    h.load_state_dict(BO.fixture_inputs()['params'] if params is None else params, strict=False)
    return h.to(DEV).train()


def _step(head, inp, loss_weight=None):
    from balancedgroupsoftmax_b200.head import BoxPredHandle
    feats = inp['feats'].to(DEV).clone().requires_grad_(True)
    head.zero_grad()
    cls_score, bbox_pred = head(feats)
    assert isinstance(bbox_pred, BoxPredHandle) == head.fuse_bbox_loss
    losses = head.loss(cls_score, bbox_pred, inp['labels'].to(DEV), inp['label_weights'].to(DEV),
                       inp['bbox_targets'].to(DEV), inp['bbox_weights'].to(DEV))
    sum(v for k, v in losses.items() if k != 'acc').backward()
    grads = {k: p.grad.detach().clone() for k, p in head.named_parameters() if p.grad is not None}
    grads['feats'] = feats.grad.detach().clone()
    return {k: v.detach().clone() for k, v in losses.items()}, grads


def _near(a, b, what, rel=2e-2):
    a, b = a.double().cpu(), b.double().cpu()
    assert (a - b).abs().max().item() <= rel * b.abs().max().item() + 1e-7, what


@pytest.mark.parametrize('name', HEADS)
def test_heads_fused_box_loss_matches_default_route(name):
    """The classifier entries and fc_cls gradients are those of the default route (the classifier's own backward
    reduces split-K with red.add, so they are compared at 1e-6 rather than bit for bit); loss_bbox and the fc_reg,
    shared-FC and feature gradients agree within the default route's bf16 tolerance."""
    inp = BO.fixture_inputs()
    on_l, on_g = _step(_head(name, True), inp)
    off_l, off_g = _step(_head(name, False), inp)
    assert set(on_l) == set(off_l) and set(on_g) == set(off_g)
    # the graph-cached classifier loss draws its "others" subset from a process-wide seed counter, so two heads in one
    # process sample differently: there only the box terms are compared
    box_only = name.endswith('_graph_cache')
    for k in on_l:
        if k == 'loss_bbox':
            _near(on_l[k], off_l[k], k, rel=1e-2)
        elif not box_only:
            torch.testing.assert_close(on_l[k], off_l[k], rtol=1e-6, atol=1e-7, msg=k)
    for k in on_g:
        if box_only and not k.startswith('fc_reg'):
            continue
        if k.startswith('fc_cls'):
            torch.testing.assert_close(on_g[k], off_g[k], rtol=1e-5, atol=1e-6 * off_g[k].abs().max().item(), msg=k)
        else:
            _near(on_g[k], off_g[k], k)


@pytest.mark.parametrize('name', ['GSBBoxHeadWith0', 'ReweightBBoxHead', 'GSBBoxHeadWith0Reweight'])
@pytest.mark.parametrize('fuse', [True, False], ids=['fused', 'default'])
def test_heads_match_reference_fixture(name, fuse):
    fix = np.load(BO.FIXTURE)
    key = 'reweight' if name == 'ReweightBBoxHead' else 'gs'
    got = BO.run_box_loss(_head(name, fuse), BO.fixture_inputs(), device=DEV)
    for k in ('loss_bbox', 'dW', 'db'):
        _near(got[k], torch.from_numpy(fix['%s_%s' % (key, k)]), k)
    # the feature gradient crosses the bf16 trunk twice, where a few ReLU masks differ from float64: both routes are
    # 16 % off in the largest element and 4.8 % in norm (a float32 restatement with bf16 rounding gives the same)
    a, b = got['dX'].double().cpu(), torch.from_numpy(fix['%s_dX' % key]).double()
    assert ((a - b).norm() / b.norm()).item() <= 0.08


# --------------------------------------------------------------------------- fallbacks
def _box_only(head, inp, materialise=None, reduction_override=None):
    feats = inp['feats'].to(DEV).clone().requires_grad_(True)
    head.zero_grad()
    _, bbox_pred = head(feats)
    if materialise is not None:
        materialise(bbox_pred)
    loss = head.loss(None, bbox_pred, inp['labels'].to(DEV), inp['label_weights'].to(DEV),
                     inp['bbox_targets'].to(DEV), inp['bbox_weights'].to(DEV),
                     reduction_override=reduction_override)['loss_bbox']
    loss.sum().backward()
    return loss.detach(), head.fc_reg.weight.grad.clone(), feats.grad.clone()


def _same_as_default(got, want):
    assert torch.equal(got[0], want[0])
    for a, b in zip(got[1:], want[1:]):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6 * b.abs().max().item())


@pytest.mark.parametrize('how', ['float', 'index', 'cat'])
def test_materialised_handle_takes_the_default_route(how):
    inp = BO.fixture_inputs()
    fn = {'float': lambda h: h.float(), 'index': lambda h: h[0], 'cat': lambda h: torch.cat([h, h])}[how]
    want = _box_only(_head('GSBBoxHeadWith0', False), inp)
    got = _box_only(_head('GSBBoxHeadWith0', True), inp, materialise=fn)
    _same_as_default(got, want)


def test_reduction_override_takes_the_default_route():
    inp = BO.fixture_inputs()
    want = _box_only(_head('GSBBoxHeadWith0', False), inp, reduction_override='none')
    got = _box_only(_head('GSBBoxHeadWith0', True), inp, reduction_override='none')
    assert got[0].shape == (96, 4)
    _same_as_default(got, want)
    # 'sum' with the avg_factor the head passes raises in the reference's weight_reduce_loss; both routes keep that
    for fuse in (False, True):
        with pytest.raises(ValueError):
            _box_only(_head('GSBBoxHeadWith0', fuse), inp, reduction_override='sum')


class _WeightedL1(torch.nn.Module):
    loss_weight = 1.0

    def forward(self, pred, target, weight=None, avg_factor=None, reduction_override=None):
        return (weight * (pred - target).abs()).sum() / avg_factor


def test_other_box_loss_takes_the_default_route():
    inp = BO.fixture_inputs()
    heads = [_head('ReweightBBoxHead', f) for f in (False, True)]
    for h in heads:
        h.loss_bbox = _WeightedL1()
    _same_as_default(_box_only(heads[1], inp), _box_only(heads[0], inp))


def test_class_agnostic_regression_returns_a_tensor():
    inp = BO.fixture_inputs()
    inp['params'] = {k: v for k, v in inp['params'].items() if not k.startswith('fc_reg')}
    heads = [_head('GSBBoxHeadWith0', f, params=inp['params'], reg_class_agnostic=True) for f in (False, True)]
    feats = inp['feats'].to(DEV)
    _, bbox_pred = heads[1](feats)
    assert type(bbox_pred) is torch.Tensor and bbox_pred.shape == (BO.FIX_N, 4)
    _same_as_default(_box_only(heads[1], inp), _box_only(heads[0], inp))
