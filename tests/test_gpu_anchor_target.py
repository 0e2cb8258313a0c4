"""GPU: ops.anchor_targets / RPNHead.loss against the restatement of anchor_target (tests/anchor_target_oracle.py)
run on CUDA, as the reference runs it (its >50-gt assignment on the CPU).

  * the assignment exhaustively and without randomness: with num >= the anchor count and pos_fraction = 1 the sampler
    takes every positive and every negative, so the labels, weights and box targets expose the whole assignment;
  * the sample byte for byte against the numpy restatement of the selection rule;
  * no host sync, CUDA-graph capture following the step counter, and RPNHead.loss end to end."""
import numpy as np
import pytest
import torch

import anchor_target_oracle as O
import sampler_oracle as S
from anchor_target_cases import RPN_CFG, _boxes, _cfg, _head_bases, cases
from balancedgroupsoftmax_b200 import ops
from balancedgroupsoftmax_b200.registry import HEADS, build_from_cfg

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
CASES = cases()
LVIS_SIZES = [(200, 336), (100, 168), (50, 84), (25, 42), (13, 21)]
LVIS_STRIDES = [4, 8, 16, 32, 64]
LVIS_METAS = [dict(img_shape=(800, 1333, 3), pad_shape=(800, 1344, 3)),
              dict(img_shape=(750, 1344, 3), pad_shape=(800, 1344, 3))]


def _native(bases, sizes, strides, metas, gts, cfg, means, stds, seed=0, seed_step=None):
    a, s = cfg['assigner'], cfg['sampler']
    return ops.anchor_targets(sizes, bases, strides, [m['img_shape'] for m in metas], [m['pad_shape'] for m in metas],
                              [g.to(DEV) for g in gts], pos_iou_thr=a['pos_iou_thr'], neg_iou_thr=a['neg_iou_thr'],
                              min_pos_iou=a.get('min_pos_iou', 0.), gt_max_assign_all=a.get('gt_max_assign_all', True),
                              allowed_border=cfg['allowed_border'], num=s['num'], pos_fraction=s['pos_fraction'],
                              neg_pos_ub=s.get('neg_pos_ub', -1), pos_weight=cfg['pos_weight'], means=means,
                              stds=stds, seed=seed, seed_step=seed_step)


def _bitwise(a, b):
    """Byte for byte, every NaN the same NaN."""
    a, b = a.contiguous(), b.contiguous()
    if a.is_floating_point():
        a = torch.where(torch.isnan(a), torch.full_like(a, float('nan')), a)
        b = torch.where(torch.isnan(b), torch.full_like(b, float('nan')), b)
        return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))
    return a.shape == b.shape and torch.equal(a, b)


def _check(got, want, what):
    (labels, lw, bt, bw), (npos, nneg) = want
    names = ('labels', 'label_weights', 'bbox_targets', 'bbox_weights')
    for name, g, w in zip(names, got[:4], (labels, lw, bt, bw)):
        assert _bitwise(g, w.to(DEV)), (what, name, int((g != w.to(DEV)).sum()))
    assert got[4].tolist() == [npos, nneg, npos + nneg], (what, got[4].tolist(), npos, nneg)


def _take_all(cfg, N):
    """The sampler settings under which every positive and every negative is drawn."""
    return dict(cfg, sampler=dict(cfg['sampler'], num=N, pos_fraction=1.0, neg_pos_ub=-1))


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_assignment_exhaustive_on_the_cpu_cases(case):
    name, bases, sizes, strides, metas, gts, cfg, means, stds = case
    N = sum(h * w * b.shape[0] for (h, w), b in zip(sizes, bases))
    cfg = _take_all(cfg, N)
    want = O.anchor_target(bases, sizes, strides, [g.to(DEV) for g in gts], metas, means, stds, cfg, None, DEV)
    got = _native(bases, sizes, strides, metas, gts, cfg, means, stds)
    _check(got, want, name)


def _lvis_gts(n, seed):
    gen = torch.Generator().manual_seed(seed)
    out = []
    for m in LVIS_METAS:
        h, w = m['img_shape'][:2]
        g = _boxes(gen, n, w, h, 4, 400)
        out.append(g)
    return out


@pytest.mark.parametrize('n', [3, 15, 50, 51, 100, 300])
def test_assignment_exhaustive_on_lvis_batches(n):
    bases = _head_bases(tuple(LVIS_STRIDES))
    N = sum(h * w * 3 for h, w in LVIS_SIZES)
    cfg = _take_all(_cfg(), N)
    gts = _lvis_gts(n, n)
    if n == 100:   # duplicates and a gt of another image's shape: ties in both maxes
        gts[0][50:60] = gts[0][:10]
    want = O.anchor_target(bases, LVIS_SIZES, LVIS_STRIDES, [g.to(DEV) for g in gts], LVIS_METAS, (0., 0., 0., 0.),
                           (1., 1., 1., 1.), cfg, None, DEV)
    got = _native(bases, LVIS_SIZES, LVIS_STRIDES, LVIS_METAS, gts, cfg, (0., 0., 0., 0.), (1., 1., 1., 1.))
    _check(got, want, n)
    assert (got[0] == 1).sum() > 0 and (got[1] > 0).sum() > (got[0] == 1).sum()


def test_torch_max_on_cuda_takes_the_first_index_and_nan_wins():
    """The per-anchor rule the kernels restate: torch.max(dim=0) on CUDA gives the first row among equal maxima and a
    NaN over any number."""
    gen = torch.Generator().manual_seed(0)
    x = torch.randint(0, 4, (70, 5000), generator=gen).float() / 4
    x[13, ::7] = float('nan')
    v, i = x.to(DEV).max(dim=0)
    ref_i = torch.tensor([int(np.argmax(np.where(np.isnan(c), np.inf, c))) for c in x.t().numpy()])
    assert torch.equal(i.cpu(), ref_i)
    assert torch.isnan(v.cpu()[::7]).all()
    gv, gi = x.to(DEV).max(dim=1)   # the per-gt argmax of gt_max_assign_all=False
    ref_gi = torch.tensor([int(np.argmax(np.where(np.isnan(r), np.inf, r))) for r in x.numpy()])
    assert torch.equal(gi.cpu(), ref_gi)


# -------------------------------------------------------------------------------------------------------- sampling
def _sampled(cfg, gts, seed, step=None, means=(0., 0., 0., 0.), stds=(1., 1., 1., 1.)):
    bases = _head_bases(tuple(LVIS_STRIDES))
    eff = S.effective_seed(seed, step)
    want = O.anchor_target(bases, LVIS_SIZES, LVIS_STRIDES, [g.to(DEV) for g in gts], LVIS_METAS, means, stds, cfg,
                           O.native_rule(eff), DEV)
    st = None if step is None else torch.tensor([step], dtype=torch.int64, device=DEV)
    got = _native(bases, LVIS_SIZES, LVIS_STRIDES, LVIS_METAS, gts, cfg, means, stds, seed=seed, seed_step=st)
    return got, want


@pytest.mark.parametrize('setting', ['configs', 'few_pos', 'k0_pos', 'k0_neg', 'neg_pos_ub', 'high_word', 'step',
                                     'step_minus_1', 'means_stds'])
def test_sample_bit_exact_against_the_rule(setting):
    cfg, seed, step, n = _cfg(), 0x1234_5678_9ABC_DEF0, None, 15
    means, stds = (0., 0., 0., 0.), (1., 1., 1., 1.)
    if setting == 'few_pos':
        n = 2   # an untruncated positive gallery
    elif setting == 'k0_pos':
        cfg = _cfg(pos_fraction=0.0)
    elif setting == 'k0_neg':
        cfg = _cfg(neg_pos_ub=0)
    elif setting == 'neg_pos_ub':
        cfg = _cfg(neg_pos_ub=1.5)
    elif setting == 'high_word':
        seed ^= 1 << 60
    elif setting == 'step':
        step = 2 ** 40
    elif setting == 'step_minus_1':
        step = -1
    elif setting == 'means_stds':
        means, stds = (0.1, -0.2, 0.05, 0.0), (0.1, 0.1, 0.2, 0.3)
    gts = _lvis_gts(n, 7)
    got, want = _sampled(cfg, gts, seed, step, means, stds)
    _check(got, want, setting)
    if setting == 'configs':
        assert got[4].tolist()[0] == 2 * 128 or (got[0] == 1).sum().item() < 256
        assert (got[1] > 0).sum().item() == 2 * 256


def test_seeds_differing_only_in_the_high_word_draw_differently():
    gts = _lvis_gts(15, 8)
    a, _ = _sampled(_cfg(), gts, 5, None)
    b = _native(_head_bases(tuple(LVIS_STRIDES)), LVIS_SIZES, LVIS_STRIDES, LVIS_METAS, gts, _cfg(), (0.,) * 4,
                (1.,) * 4, seed=5 + (1 << 32))
    assert not torch.equal(a[1], b[1])
    assert (a[1] > 0).sum() == (b[1] > 0).sum() and torch.equal(a[4], b[4])   # the same counts, other anchors


# --------------------------------------------------------------------------------------------- no sync and graphs
def test_no_host_sync_and_graph_replays_follow_the_step_counter():
    bases = _head_bases(tuple(LVIS_STRIDES))
    gts = [g.to(DEV) for g in _lvis_gts(15, 9)]
    cfg = _cfg()
    step = torch.zeros(1, dtype=torch.int64, device=DEV)
    _native(bases, LVIS_SIZES, LVIS_STRIDES, LVIS_METAS, gts, cfg, (0.,) * 4, (1.,) * 4, seed=3, seed_step=step)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        _native(bases, LVIS_SIZES, LVIS_STRIDES, LVIS_METAS, gts, cfg, (0.,) * 4, (1.,) * 4, seed=3, seed_step=step)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        _native(bases, LVIS_SIZES, LVIS_STRIDES, LVIS_METAS, gts, cfg, (0.,) * 4, (1.,) * 4, seed=3, seed_step=step)
        with torch.cuda.graph(g, stream=s):
            out = _native(bases, LVIS_SIZES, LVIS_STRIDES, LVIS_METAS, gts, cfg, (0.,) * 4, (1.,) * 4, seed=3,
                          seed_step=step)
    torch.cuda.current_stream().wait_stream(s)
    seen = []
    for k in (0, 1, 2, 1):
        step.fill_(k)
        g.replay()
        torch.cuda.synchronize()
        eager = _native(bases, LVIS_SIZES, LVIS_STRIDES, LVIS_METAS, gts, cfg, (0.,) * 4, (1.,) * 4, seed=3,
                        seed_step=torch.tensor([k], dtype=torch.int64, device=DEV))
        for a, b in zip(out, eager):
            assert torch.equal(a, b), k
        seen.append(out[1].clone())
    assert not torch.equal(seen[0], seen[1]) and not torch.equal(seen[1], seen[2]) and torch.equal(seen[1], seen[3])


# --------------------------------------------------------------------------------------------------- end to end
def _head():
    torch.manual_seed(0)
    head = build_from_cfg(dict(type='RPNHead', in_channels=16, feat_channels=16, anchor_scales=[8],
                               anchor_ratios=[0.5, 1.0, 2.0], anchor_strides=LVIS_STRIDES), HEADS)
    head.init_weights()
    return head.to(DEV)


def _reference_loss_single(head, cls_score, bbox_pred, labels, lw, bt, bw, avg):
    """AnchorHead.loss_single as the reference runs it: flat labels (CrossEntropyLoss's one-hot) and a python avg."""
    import torch.nn.functional as F
    labels, lw = labels.reshape(-1), lw.reshape(-1)
    cls = cls_score.permute(0, 2, 3, 1).reshape(-1, 1)
    onehot = labels.new_zeros((labels.size(0), 1))
    inds = torch.nonzero(labels >= 1).squeeze(-1)
    onehot[inds, labels[inds] - 1] = 1
    loss_cls = F.binary_cross_entropy_with_logits(cls, onehot.float(), lw.view(-1, 1).float(),
                                                  reduction='none').sum() / avg
    diff = torch.abs(bbox_pred.permute(0, 2, 3, 1).reshape(-1, 4) - bt.reshape(-1, 4))
    beta = 1.0 / 9.0
    sl1 = torch.where(diff < beta, 0.5 * diff * diff / beta, diff - 0.5 * beta)
    return loss_cls, (sl1 * bw.reshape(-1, 4)).sum() / avg


@pytest.mark.parametrize('B', [1, 2])
def test_rpn_head_loss_end_to_end_without_mmdet(B, monkeypatch):
    from balancedgroupsoftmax_b200 import rpn_head
    monkeypatch.setattr(rpn_head, '_mmdet_core', lambda name: None)
    head = _head()
    monkeypatch.setattr(head, '_next_seed', lambda: 99)
    metas = LVIS_METAS[:B]
    feats = [torch.randn(B, 16, h, w, device=DEV) for h, w in LVIS_SIZES]
    cls_scores, bbox_preds = head(feats)
    gts = [g.to(DEV) for g in _lvis_gts(15, 11)[:B]]
    cfg = dict(RPN_CFG)
    losses = head.loss(cls_scores, bbox_preds, gts, metas, cfg)
    bases = [g.base_anchors for g in head.anchor_generators]
    (labels, lw, bt, bw), (npos, nneg) = O.anchor_target(bases, LVIS_SIZES, LVIS_STRIDES, gts, metas, (0.,) * 4,
                                                         (1.,) * 4, cfg, O.native_rule(99), DEV)
    start = 0
    for l, (h, w) in enumerate(LVIS_SIZES):
        n = h * w * 3
        sl = slice(start, start + n)
        want_cls, want_box = _reference_loss_single(head, cls_scores[l], bbox_preds[l], labels[:, sl], lw[:, sl],
                                                    bt[:, sl], bw[:, sl], npos + nneg)
        # the device avg_factor divides once where the reference's python int multiplies by its reciprocal
        torch.testing.assert_close(losses['loss_rpn_cls'][l], want_cls, rtol=3e-7, atol=0)
        torch.testing.assert_close(losses['loss_rpn_bbox'][l], want_box, rtol=3e-7, atol=0)
        start += n
    total = sum(losses['loss_rpn_cls']) + sum(losses['loss_rpn_bbox'])
    total.backward()
    assert head.rpn_cls.weight.grad.abs().sum() > 0 and head.rpn_reg.weight.grad.abs().sum() > 0
    if B == 1:
        assert losses['loss_rpn_cls'][0].dim() == 0


def test_rpn_head_loss_makes_no_host_sync(monkeypatch):
    from balancedgroupsoftmax_b200 import rpn_head
    monkeypatch.setattr(rpn_head, '_mmdet_core', lambda name: None)
    head = _head()
    feats = [torch.randn(2, 16, h, w, device=DEV) for h, w in LVIS_SIZES]
    cls_scores, bbox_preds = head(feats)
    gts = [g.to(DEV) for g in _lvis_gts(15, 12)]
    head.loss(cls_scores, bbox_preds, gts, LVIS_METAS, dict(RPN_CFG))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        losses = head.loss(cls_scores, bbox_preds, gts, LVIS_METAS, dict(RPN_CFG))
        total = sum(losses['loss_rpn_cls']) + sum(losses['loss_rpn_bbox'])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(total)


def test_no_gt_raises_and_no_inside_anchor_gives_none(monkeypatch):
    from balancedgroupsoftmax_b200 import rpn_head
    monkeypatch.setattr(rpn_head, '_mmdet_core', lambda name: None)
    head = _head()
    sizes = [(16, 16), (8, 8), (4, 4), (2, 2), (1, 1)]
    cls = [torch.zeros(1, 3, h, w, device=DEV) for h, w in sizes]
    reg = [torch.zeros(1, 12, h, w, device=DEV) for h, w in sizes]
    meta = dict(img_shape=(64, 64, 3), pad_shape=(64, 64, 3))
    with pytest.raises(ValueError, match='No gt or bboxes'):
        head.loss(cls, reg, [torch.zeros(0, 4, device=DEV)], [meta], dict(RPN_CFG))
    tiny = dict(img_shape=(2, 2, 3), pad_shape=(64, 64, 3))   # every anchor crosses the border
    assert head.loss(cls, reg, [torch.tensor([[0., 0., 1., 1.]], device=DEV)], [tiny], dict(RPN_CFG)) is None
