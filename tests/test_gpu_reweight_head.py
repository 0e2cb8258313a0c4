"""GPU: the softmax-CE head's fused forward (bags_ce_fwd), its backward through bags_bwd at any C, and
ReweightBBoxHead end to end, against the CPU oracle (tests/reweight_oracle.py) and the committed reference fixture."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import reweight_oracle as R
from oracle import bags_oracle as O

pytestmark = [pytest.mark.gpu]

LOSS_TOL = 2e-3        # as in test_gpu_reweight.py
GRAD_TOL = 5e-3


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _groups():
    """CTA groups of the fused forward's persistent grid (one per 4 SMs at one CTA per SM)."""
    return torch.cuda.get_device_properties(0).multi_processor_count // 4


def _problem(N, C, K, dtype, weighted, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.relu(torch.randn(N, K, generator=g))
    W = torch.randn(C, K, generator=g) * 0.08
    b = torch.randn(C, generator=g) * 0.5
    labels = torch.randint(0, C, (N,), generator=g)
    labels[: N // 2] = 0
    W[0] += 0.02                                       # class 0 wins on part of the rows: a non-trivial accuracy
    weights = (torch.rand(N, generator=g) * 2 + 0.1) if weighted else None
    avg = torch.tensor([max(N - 3, 1)], dtype=torch.float32)
    xr, Wr = x.to(dtype).float(), W.to(dtype).float()     # the operands the kernel reads
    dev = dict(x=x.cuda().to(dtype), W=W.cuda().to(dtype), b=b.cuda(), labels=labels.cuda(),
               weights=None if weights is None else weights.cuda(), avg=avg.cuda())
    return xr, Wr, b, labels, weights, avg, dev


N_CASES = [64, 300, 4096, 'groups']


@pytest.mark.parametrize('C', [1231, 1204, 1280, 7])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32], ids=['bf16', 'fp32'])
@pytest.mark.parametrize('weighted', [False, True], ids=['w1', 'wf32'])
@pytest.mark.parametrize('N', N_CASES)
def test_ce_fwd_matches_oracle(C, dtype, weighted, N):
    from balancedgroupsoftmax_b200 import ops
    if N == 'groups':
        N = 3 * 128 * _groups() + 5                  # every CTA group loops over 3-4 row tiles
    K = 256
    xr, Wr, b, labels, weights, avg, d = _problem(N, C, K, dtype, weighted, seed=N + C)
    loss, acc, dz, colsum = ops.ce_fwd(d['x'], d['W'], d['b'], d['labels'], d['weights'], d['avg'], want_acc=True,
                                       want_colsum=True)
    torch.cuda.synchronize()
    z = F.linear(xr.double(), Wr.double(), b.double())
    ref = R.ce_loss(xr.double(), Wr.double(), b.double(), labels, weights, avg.item())
    assert abs(loss.item() - ref.item()) <= LOSS_TOL * max(abs(ref.item()), 1e-3), (loss.item(), ref.item())
    # accuracy: exact on rows whose top-2 gap is clear; near-ties may go either way and are bounded
    # (bf16: the oracle has the kernel's operands, so only fp32 rounding separates them; fp32 operands enter the
    # tensor cores as TF32, which moves a logit by up to ~1e-2 here)
    correct = R.correct_rows(z, labels)
    clear = R.top2_gap(z) > (1e-3 if dtype == torch.bfloat16 else 5e-2)
    got = acc.item() * N / 100.0
    lo = correct[clear].sum().item()
    hi = lo + correct[~clear].numel()
    assert abs(got - round(got)) < 0.05, got
    assert lo <= round(got) <= hi, (got, lo, hi)
    assert (~clear).sum().item() <= N // 5 + 3
    # dz and its column sums
    dz_ref, _, _, _ = R.ce_closed_form_grads(xr.double(), Wr.double(), b.double(), labels, weights, avg.item())
    assert rel(dz[:, :C].float(), dz_ref) <= GRAD_TOL
    assert colsum.shape == ((N + 127) // 128, C)
    assert rel(colsum.sum(0), dz_ref.sum(0)) <= GRAD_TOL


@pytest.mark.parametrize('C', [1231, 7])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32], ids=['bf16', 'fp32'])
def test_ce_backward_matches_closed_form(C, dtype):
    """dW, db, dX through bags_bwd with the single slice (0, C): at C = 1231 the dz^T tensor map has an odd inner
    dimension and ldd = pad_cols(1231)."""
    from balancedgroupsoftmax_b200 import ops
    N, K = 300, 256
    xr, Wr, b, labels, weights, avg, d = _problem(N, C, K, dtype, True, seed=7 * C)
    gout = 0.75
    dW0 = torch.full((C, K), 5.0, device='cuda')
    _, _, dz, colsum = ops.ce_fwd(d['x'], d['W'], d['b'], d['labels'], d['weights'], d['avg'], want_colsum=True,
                                  clear=dW0)
    assert dz.stride(0) == ops.pad_cols(C)
    dt1 = ops._single_slice_tables(C, 'cuda')
    g = torch.tensor([gout], device='cuda')
    dW, db, dX = ops.fused_bwd(dz, d['x'], d['W'], g, dt1, colsum, dW=dW0, dw_prezeroed=True)
    dW2, db2, _ = ops.fused_bwd(dz, d['x'], d['W'], g, dt1, None, need_dx=False)
    torch.cuda.synchronize()
    _, dW_ref, db_ref, dX_ref = R.ce_closed_form_grads(xr.double(), Wr.double(), b.double(), labels, weights,
                                                       avg.item(), gout)
    errs = dict(dW=rel(dW, dW_ref), db=rel(db, db_ref), dX=rel(dX.float(), dX_ref), dW2=rel(dW2, dW_ref),
                db2=rel(db2, db_ref))
    assert max(errs.values()) <= GRAD_TOL, errs


def test_ce_fwd_eager_and_graph_replay_agree():
    """Three eager calls and two replays of a CUDA graph on one stream (one workspace) give bit-identical dz and acc.
    The loss agrees to fp32 rounding only: each CTA adds its rows' terms with shared-memory atomics, whose order
    varies from run to run (as in bags_fwd); the accuracy count adds whole numbers, so its order does not matter."""
    from balancedgroupsoftmax_b200 import ops
    _, _, _, _, _, _, d = _problem(4096 + 77, 1231, 1024, torch.bfloat16, True, seed=3)
    s = torch.cuda.Stream()
    outs = []
    with torch.cuda.stream(s):
        for _ in range(3):
            loss, acc, dz, _ = ops.ce_fwd(d['x'], d['W'], d['b'], d['labels'], d['weights'], d['avg'], want_acc=True)
            outs.append((loss.clone(), acc.clone(), dz.clone()))
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            gl, ga, gdz, _ = ops.ce_fwd(d['x'], d['W'], d['b'], d['labels'], d['weights'], d['avg'], want_acc=True)
        for _ in range(2):
            graph.replay()
            outs.append((gl.clone(), ga.clone(), gdz.clone()))
    torch.cuda.synchronize()
    for loss, acc, dz in outs[1:]:
        assert torch.equal(dz, outs[0][2]) and torch.equal(acc, outs[0][1])
        assert abs(loss.item() - outs[0][0].item()) <= 1e-6 * abs(outs[0][0].item())


# --------------------------------------------------------------------------- the head
def _head(inp, compute_dtype='fp32', **extra):
    from balancedgroupsoftmax_b200.head import ReweightBBoxHead
    head = ReweightBBoxHead(num_fcs=2, in_channels=R.FIX_IN, fc_out_channels=R.FIX_FC, roi_feat_size=R.FIX_ROI,
                            num_classes=R.FIX_C, reweight_cfg=dict(cls_weights=inp['cls_weight'],
                                                                   compute_dtype=compute_dtype, **extra),
                            target_means=[0., 0., 0., 0.], target_stds=[0.1, 0.1, 0.2, 0.2])
    head.load_state_dict(inp['params'])
    return head.cuda()


def _targets(inp):
    return tuple(inp[k].cuda() for k in ('labels', 'label_weights', 'bbox_targets', 'bbox_weights'))


@pytest.fixture(scope='module')
def fixture():
    return R.fixture_inputs(), np.load(R.FIXTURE)


@pytest.mark.parametrize('compute_dtype', ['fp32', 'bf16'])
def test_head_training_matches_reference_fixture(fixture, compute_dtype):
    from balancedgroupsoftmax_b200.head import ClsScoreHandle
    inp, fix = fixture
    head = _head(inp, compute_dtype).train()
    feats = inp['feats'].cuda().requires_grad_(True)
    cls_score, bbox_pred = head(feats)
    assert isinstance(cls_score, ClsScoreHandle) and cls_score._logits is None
    losses = head.loss(cls_score, bbox_pred, *_targets(inp))
    assert cls_score._logits is None                          # the fused kernel ran: no logits in memory
    assert sorted(losses) == ['acc', 'loss_bbox', 'loss_cls'] and losses['acc'].shape == (1,)
    (losses['loss_cls'] + losses['loss_bbox']).backward()
    torch.cuda.synchronize()
    tol = 1e-3 if compute_dtype == 'fp32' else 1e-2
    assert abs(losses['loss_cls'].item() - float(fix['loss_cls'])) <= tol * float(fix['loss_cls'])
    assert abs(losses['loss_bbox'].item() - float(fix['loss_bbox'])) <= tol * float(fix['loss_bbox'])
    assert abs(losses['acc'].item() - float(fix['acc'][0])) <= 100.0 / R.FIX_N + 1e-4   # one near-tie row at most
    # The fixture's background rows are confident (p0 close to 1), so dz = p - onehot is a small difference of O(1)
    # terms, and the operand rounding of logits around 10 (bf16 round-to-nearest; TF32 drops the low mantissa bits)
    # moves the gradients by about a percent.  test_ce_backward_matches_closed_form checks them tightly.
    gtol = 5e-2
    errs = dict(dW=rel(head.fc_cls.weight.grad[::4], torch.from_numpy(fix['dW4'])),
                db=rel(head.fc_cls.bias.grad, torch.from_numpy(fix['db'])),
                dX=rel(feats.grad, torch.from_numpy(fix['dX'])))
    assert max(errs.values()) <= gtol, errs


def test_head_only_training_computes_no_dx(fixture, monkeypatch):
    """The 'transferred' head-only configs train fc_cls alone: the trunk is frozen and the RoI features carry no
    gradient, so the backward runs no dX contraction; dW and db still match the reference fixture."""
    from balancedgroupsoftmax_b200 import ops
    inp, fix = fixture
    head = _head(inp).train()
    for n, prm in head.named_parameters():
        prm.requires_grad_(n.startswith('fc_cls.'))
    calls = []
    real = ops.fused_bwd

    def spy(*a, **k):
        calls.append(k.get('need_dx', True))
        return real(*a, **k)
    monkeypatch.setattr(ops, 'fused_bwd', spy)
    feats = inp['feats'].cuda()
    cls_score, bbox_pred = head(feats)
    losses = head.loss(cls_score, bbox_pred, *_targets(inp))
    (losses['loss_cls'] + losses['loss_bbox'] * 0).backward()
    torch.cuda.synchronize()
    assert calls == [False]
    assert head.shared_fcs[0].weight.grad is None
    errs = dict(dW=rel(head.fc_cls.weight.grad[::4], torch.from_numpy(fix['dW4'])),
                db=rel(head.fc_cls.bias.grad, torch.from_numpy(fix['db'])))
    assert max(errs.values()) <= 5e-2, errs   # (see test_head_training_matches_reference_fixture)


def test_head_loss_does_not_sync(fixture):
    """The classification loss, its normaliser and acc stay on the device (the reference's .item() is gone).  The box
    loss is left out: its positive-RoI selection is boolean indexing, which sizes its result on the host."""
    inp, _ = fixture
    head = _head(inp, 'bf16').train()
    feats = inp['feats'].cuda().requires_grad_(True)
    targets = _targets(inp)
    cls_score, _ = head(feats)
    head.loss(cls_score, None, *targets)                   # first call: weight table upload, operand casts
    torch.cuda.synchronize()
    cls_score, _ = head(feats)
    torch.cuda.set_sync_debug_mode('error')
    try:
        losses = head.loss(cls_score, None, *targets)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert sorted(losses) == ['acc', 'loss_cls']


def test_head_eval_detections_match_oracle(fixture):
    """Test path (BBoxHead.get_det_bboxes): softmax over the 1231 logits, decoding, native hard NMS -- against
    F.softmax of the oracle logits and the oracle NMS."""
    inp, _ = fixture
    head = _head(inp).eval()
    feats = inp['feats'].cuda()
    g = torch.Generator().manual_seed(2)
    xy = torch.rand(R.FIX_N, 2, generator=g) * 500
    rois = torch.cat([torch.zeros(R.FIX_N, 1), xy, xy + torch.rand(R.FIX_N, 2, generator=g) * 120 + 4], 1).cuda()
    with torch.no_grad():
        cls_score, bbox_pred = head(feats)
        assert cls_score.shape == (R.FIX_N, R.FIX_C)
        bboxes, scores = head.get_det_bboxes(rois, cls_score, bbox_pred, (600, 800, 3), 1.0)
        cfg = dict(score_thr=0.001, nms=dict(type='nms', iou_thr=0.5), max_per_img=100)
        dets, labels = head.get_det_bboxes(rois, cls_score, bbox_pred, (600, 800, 3), 1.0, cfg=cfg)
    # logits against the oracle trunk + fc_cls (TF32 operands)
    p = {k: v.double() for k, v in inp['params'].items()}
    x = inp['feats'].double().reshape(R.FIX_N, -1)
    for i in range(2):
        x = torch.relu(F.linear(x, p['shared_fcs.%d.weight' % i], p['shared_fcs.%d.bias' % i]))
    z = F.linear(x, p['fc_cls.weight'], p['fc_cls.bias'])
    assert rel(scores, torch.softmax(z, 1)) <= 5e-3
    ref_dets, ref_labels = O.multiclass_nms(bboxes.cpu(), scores.cpu(), 0.001, 0.5, 100)
    assert torch.equal(labels.cpu(), ref_labels)
    assert torch.allclose(dets.cpu(), ref_dets, rtol=0, atol=1e-5)
