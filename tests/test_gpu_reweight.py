"""GPU: the reweight head variant's device ops (bags_reweight, bags_fwd / bags_group_ce with fp32 weights) against the
oracle restatement of gs_bbox_head_with0_reweight.py (pinned to the reference class in tests/test_oracle_vs_reference.py)."""
import os

import numpy as np
import pytest
import torch

from balancedgroupsoftmax_b200.tables import synthetic_tables
from oracle import bags_oracle as O

pytestmark = [pytest.mark.gpu]


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _problem(N, npos):
    """Tables, device weights from bags_reweight, the oracle's losses and gradients, and the bf16 device operands."""
    from balancedgroupsoftmax_b200 import ops
    t = synthetic_tables(1231, seed=0)
    dt = ops.DeviceTables.from_tables(t, 'cuda')
    l2b, ps = torch.from_numpy(t.label2binlabel), torch.from_numpy(t.pred_slice)
    g = torch.Generator().manual_seed(N)
    cls_weights = [torch.rand(int(t.pred_slice[b, 1]), generator=g) * 2 + 0.1 for b in range(1, t.num_bins)]
    table = torch.ones(t.num_bins, max(w.numel() for w in cls_weights))
    for b, w in enumerate(cls_weights, start=1):
        table[b, :w.numel()] = w
    labels = torch.zeros(N, dtype=torch.long)
    labels[:npos] = torch.randint(1, 1231, (npos,), generator=g)
    x = torch.relu(torch.randn(N, 1024, generator=g))
    W = torch.randn(t.num_logits, 1024, generator=g) * 0.05
    b = torch.randn(t.num_logits, generator=g) * 0.1
    np.random.seed(N)
    remapped = O.remap_labels_reweight(labels, l2b, 8.0, cls_weights)
    masks = torch.stack([(w > 0).to(torch.uint8) for w in remapped[1]]).cuda()      # the sampled 0/1 masks
    wfloat, avg = ops.reweight(labels.cuda(), dt, masks, table.cuda())
    xr, Wr = x.bfloat16().float(), W.bfloat16().float()
    ref = O.bags_loss(O.fc_cls(xr, Wr, b), labels, l2b, ps, remapped=remapped)
    _, dW_ref, db_ref, dX_ref = O.closed_form_grads(xr, Wr, b, labels, l2b, ps, remapped)
    return (ops, t, dt, remapped, wfloat, avg, ref, (dW_ref, db_ref, dX_ref),
            (x.cuda().bfloat16(), W.cuda().bfloat16(), b.cuda(), labels.cuda()))


def _check(t, ref, refgrads, loss, dW, db, dX, what):
    dW_ref, db_ref, dX_ref = refgrads
    for gi in range(t.num_bins):
        r = ref['loss_cls_bin%d' % gi].item()
        assert abs(loss[gi].item() - r) <= 2e-3 * max(abs(r), 1e-3), (what, gi, loss[gi].item(), r)
    assert rel(dW, dW_ref) < 5e-3 and rel(db, db_ref) < 5e-3 and rel(dX.float(), dX_ref) < 5e-3, what


@pytest.mark.parametrize('N,npos', [(300, 75), (64, 0), (1024, 256)])
def test_reweight_ops_match_oracle(N, npos):
    ops, t, dt, remapped, wfloat, avg, ref, refgrads, (xc, wc, b, labels) = _problem(N, npos)
    want_w = torch.stack([w.float() for w in remapped[1]])
    assert torch.allclose(wfloat.cpu(), want_w, rtol=1e-6, atol=0)
    assert torch.allclose(avg.cpu(), torch.tensor(remapped[2]), rtol=1e-5)
    for materialize in (False, True):
        loss, _, _, dz, colsum = ops.fused_fwd(xc, wc, b, labels, dt, wfloat, avg, materialize=materialize)
        dW, db, dX = ops.fused_bwd(dz, xc, wc, None, dt, colsum)
        torch.cuda.synchronize()
        _check(t, ref, refgrads, loss, dW, db, dX, materialize)


@pytest.mark.parametrize('N,npos', [(300, 75), (1024, 256)])
def test_reweight_clear_hook_matches_oracle(N, npos):
    """fp32 weights with the forward's clear hook: the forward (fused kernel or materialised route) zeroes a dirty dW,
    then the backward skips its zeroing job (dw_prezeroed) and still gives the oracle's gradients."""
    ops, t, dt, remapped, wfloat, avg, ref, refgrads, (xc, wc, b, labels) = _problem(N, npos)
    for materialize in (False, True):
        dW = torch.full((t.num_logits, 1024), 123.0, device='cuda')
        loss, _, _, dz, colsum = ops.fused_fwd(xc, wc, b, labels, dt, wfloat, avg, materialize=materialize, clear=dW)
        torch.cuda.synchronize()
        assert dW.abs().max().item() == 0.0, materialize
        _, db, dX = ops.fused_bwd(dz, xc, wc, None, dt, colsum, dW=dW, dw_prezeroed=True)
        torch.cuda.synchronize()
        _check(t, ref, refgrads, loss, dW, db, dX, materialize)
