"""GPU: the sigmoid focal loss fused into fc_cls (bags_focal_fwd, ops.SigmoidFocalFunction, ReweightBBoxHead with a
FocalLoss) against the float64 oracle of the op (tests/focal_oracle.py) on the operands the kernel reads.

Tolerances, per element:
  * the logits: the oracle's z is exact in float64 on the rounded operands.  The kernel's z differs by the fp32
    accumulation, at most (K + 2) * 2^-24 * (S + |b|) with S = |x| |W|^T; fp32 operands also enter the tensor cores as
    TF32, whose 10-bit mantissa adds up to 2^-9 * S (2^-10 per operand).  This is dzl.
  * dz = w/norm * g(z): |d g / dz| <= 1 (test_focal_cpu.py::test_gradient_lipschitz_bound), so the logits move dz by
    at most coef * dzl.  The fp32 math of one element (expf, a correctly rounded reciprocal, log1pf, logf-free logs and
    powf, each within a few ulp, and sums of same-signed terms) errs by at most 2^-18 relative.  A bf16 dz is rounded
    to 8 significant bits: 2^-8 relative.
  * loss: the same per-element terms with |dl/dz| <= 1 + |z| (the loss grows at most linearly), summed, plus 2^-14
    relative for the fp32 sums (at most a few hundred additions per value in any order).
  * acc: exact except at near-ties; a row counts as decided when its label logit is more than 2 * dzl away from the
    best other logit, and the kernel's count must lie between the decided-correct rows and those plus the undecided.
  * column sums: the kernel's own stored dz summed in float64, up to 2^-24 * (128 + tiles) * sum |dz| (fp32 sums).
  * dW, db, dX from bags_bwd: float64 contractions of the kernel's own dz with the same operands, up to
    (N + 2) * 2^-24 * |dz|^T |x| (fp32 sums, split-K in any order) plus TF32's 2^-9 relative for fp32 operands, plus
    2^-8 for a bf16 dX.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import focal_oracle as FO
from balancedgroupsoftmax_b200 import _native as nat
from balancedgroupsoftmax_b200 import losses as L
from balancedgroupsoftmax_b200 import ops

pytestmark = pytest.mark.gpu

SENTINEL = -1024.0   # exact in bf16
U = 2.0 ** -24
K = 96
CHUNK = 8192


def _case(N, C, mode, weighted, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, K, generator=g)
    W = torch.randn(C, K, generator=g) * 0.1
    b = (torch.rand(C, generator=g) * 2 - 1) * 38.0               # logits up to |z| ~ 40 through the bias
    b[:4] = torch.tensor([0., 1e-3, -17.5, 17.5])
    t = torch.randint(2, C + 1, (N,), generator=g)                # in range: column t - 1 positive
    kind = torch.randint(0, 5, (N,), generator=g)
    t = torch.where(kind == 0, torch.zeros_like(t), t)            # all negative
    t = torch.where(kind == 1, torch.ones_like(t), t)             # column 0 positive
    t = torch.where(kind == 2, C + 1 + torch.randint(0, 5, (N,), generator=g), t)   # out of range: all negative
    t = torch.where(kind == 3, -1 - torch.randint(0, 3, (N,), generator=g), t)      # ignored row
    w = (torch.rand(N, generator=g) * 2) if weighted else None
    dev = 'cuda'
    xc, Wc = x.to(dev).to(mode), W.to(dev).to(mode)
    z64 = _z64(xc, Wc, b.to(dev))
    labels = torch.randint(0, C, (N,), generator=g).to(dev)
    half = torch.arange(N, device=dev) % 2 == 0
    labels = torch.where(half, z64.argmax(1), labels)             # about half the rows correct
    return xc, Wc, b.to(dev), t.to(dev), labels, (w.to(dev) if weighted else None)


def _z64(xc, Wc, b):
    return xc.double() @ Wc.double().t() + b.double()


def _dzl(xc, Wc, b, rows):
    S = xc[rows].double().abs() @ Wc.double().abs().t()
    tf32 = 2.0 ** -9 * S if xc.dtype == torch.float32 else 0.
    return (K + 2) * U * (S + b.double().abs()) + tf32


def _raw_focal(xc, Wc, b, t, labels, w, norm, gamma, alpha, acc=True, colsum=True):
    N, C = xc.shape[0], Wc.shape[0]
    ldd = ops.pad_cols(C)
    dz = torch.full((N, ldd), SENTINEL, dtype=xc.dtype, device=xc.device)
    cs = torch.empty(((N + 127) // 128, C), dtype=torch.float32, device=xc.device) if colsum else None
    loss = torch.empty(1, dtype=torch.float32, device=xc.device)
    a = torch.empty(1, dtype=torch.float32, device=xc.device) if acc else None
    ws = ops._workspace(xc.device)
    nat.check(nat.lib().bags_focal_fwd(
        xc.data_ptr(), xc.stride(0), Wc.data_ptr(), Wc.stride(0), b.data_ptr(), t.data_ptr(),
        labels.data_ptr() if acc else None, nat.ptr(w), norm, gamma, alpha, N, K, C, ops._dtype_code(xc.dtype),
        loss.data_ptr(), nat.ptr(a), dz.data_ptr(), ldd, nat.ptr(cs), cs.shape[0] if colsum else 0, ws.data_ptr(),
        ws.numel(), None, 0, ops._stream_ptr(xc.device)), 'bags_focal_fwd')
    return loss, a, dz, cs


def _check_forward(xc, Wc, b, t, labels, w, gamma, alpha, loss, acc, dz, cs):
    N, C = xc.shape[0], Wc.shape[0]
    norm = float(N * FO.ONE_HOT)
    assert (dz[:, C:].float() == SENTINEL).all(), 'padding columns were written'
    bf16 = xc.dtype == torch.bfloat16
    loss_ref = loss_tol = 0.
    decided_ok = undecided = 0
    dzsum = torch.zeros(C, dtype=torch.float64, device='cuda')
    dzabs = torch.zeros(C, dtype=torch.float64, device='cuda')
    for r0 in range(0, N, CHUNK):
        rows = slice(r0, min(N, r0 + CHUNK))
        z = _z64(xc[rows], Wc, b)
        dzl = _dzl(xc, Wc, b, rows)
        coef = (w[rows].double() if w is not None else torch.ones(z.shape[0], dtype=torch.float64, device='cuda'))
        coef = (coef / norm)[:, None]
        el = FO.op_forward(z, t[rows], gamma, alpha)
        g = FO.op_backward(z, t[rows], gamma, alpha)
        ref = coef * g
        tol = coef * (dzl + 2.0 ** -18 * g.abs()) + (2.0 ** -8 * ref.abs() if bf16 else 0.) + 1e-30
        got = dz[rows, :C].double()
        bad = (got - ref).abs() > tol
        assert not bad.any(), ('dz', bad.nonzero()[:5].tolist(), got[bad][:5].tolist(), ref[bad][:5].tolist())
        loss_ref += float((coef * el).sum())
        loss_tol += float((coef * ((1 + z.abs()) * dzl + 2.0 ** -18 * el.abs())).sum())
        loss_tol += 2.0 ** -14 * float((coef * el.abs()).sum())
        dzsum += got.sum(0)
        dzabs += got.abs().sum(0)
        if acc is not None:
            lab = labels[rows]
            zl = z.gather(1, lab[:, None])[:, 0]
            other = z.scatter(1, lab[:, None], float('-inf')).max(1).values
            margin = 2 * dzl.max(1).values
            decided_ok += int((zl - other > margin).sum())
            undecided += int(((zl - other).abs() <= margin).sum())
    assert abs(loss.item() - loss_ref) <= loss_tol + 1e-30, (loss.item(), loss_ref, loss_tol)
    if acc is not None:
        count = round(acc.item() * N / 100.0)
        assert decided_ok <= count <= decided_ok + undecided, (count, decided_ok, undecided)
    if cs is not None:
        got = cs.double().sum(0)
        assert ((got - dzsum).abs() <= U * (128 + cs.shape[0]) * dzabs + 1e-30).all()


def _check_backward(xc, Wc, dz):
    N, C = xc.shape[0], Wc.shape[0]
    gout = torch.tensor([0.75], device='cuda')
    dW, db, dX = ops.fused_bwd(dz, xc, Wc, gout, ops._single_slice_tables(C, xc.device), None)
    d = dz[:, :C].double() * 0.75
    x64, W64 = xc.double(), Wc.double()
    tf32 = 2.0 ** -9 if xc.dtype == torch.float32 else 0.
    bound_w = (N + 2) * U * (d.abs().t() @ x64.abs())
    assert ((dW.double() - d.t() @ x64).abs() <= bound_w + tf32 * (d.abs().t() @ x64.abs()) + 1e-30).all()
    assert ((db.double() - d.sum(0)).abs() <= (N + 2) * U * d.abs().sum(0) + 1e-30).all()
    ref_x = d @ W64
    sx = d.abs() @ W64.abs()
    bound_x = (C + 2) * U * sx + tf32 * sx + (2.0 ** -8 * ref_x.abs() if xc.dtype == torch.bfloat16 else 0.)
    assert ((dX.double() - ref_x).abs() <= bound_x + 1e-30).all()


GA = [(0.0, 0.25), (0.5, 1.0), (2.0, 0.25), (0.0, 1.0), (0.5, 0.25), (2.0, 1.0)]
DT = {'bf16': torch.bfloat16, 'fp32': torch.float32}
CASES = []
for i, (C, dt, weighted) in enumerate([(C, dt, wt) for C in (1231, 1204, 1280, 7) for dt in DT for wt in (True, False)]):
    CASES.append((4173, C, dt, weighted) + GA[i % len(GA)])
CASES += [(N, 1231, 'bf16', True, 2.0, 0.25) for N in (1, 127, 131072 + 77)]
CASES += [(131072 + 77, 1204, 'fp32', False, 0.5, 1.0), (127, 7, 'fp32', True, 0.0, 0.25)]
CASES += [(4173, 1231, 'bf16', False) + ga for ga in GA]


@pytest.mark.parametrize('N,C,dt,weighted,gamma,alpha', CASES)
def test_focal_fwd_and_bwd_match_float64(N, C, dt, weighted, gamma, alpha):
    xc, Wc, b, t, labels, w = _case(N, C, DT[dt], weighted, seed=N * 7 + C)
    loss, acc, dz, cs = _raw_focal(xc, Wc, b, t, labels, w, float(N * FO.ONE_HOT), gamma, alpha)
    torch.cuda.synchronize()
    _check_forward(xc, Wc, b, t, labels, w, gamma, alpha, loss, acc, dz, cs)
    if N <= 4173:
        _check_backward(xc, Wc, dz)


def test_without_accuracy_the_loss_and_dz_are_the_same():
    """Without acc the CTAs skip the row max and the exchange: dz and the loss are bit-identical to the run with it."""
    xc, Wc, b, t, labels, w = _case(4173, 1231, torch.bfloat16, True, seed=5)
    a = _raw_focal(xc, Wc, b, t, labels, w, 4173. * 1231, 2.0, 0.25)
    n = _raw_focal(xc, Wc, b, t, labels, w, 4173. * 1231, 2.0, 0.25, acc=False, colsum=False)
    assert torch.equal(a[0], n[0]) and torch.equal(a[2], n[2])


def test_graph_replays_are_bit_identical_to_eager():
    xc, Wc, b, t, labels, w = _case(4173, 1231, torch.bfloat16, True, seed=9)
    eager = [ops.focal_fwd(xc, Wc, b, t, 4173. * 1231, 0.5, 1.0, labels=labels, weights=w, want_acc=True)
             for _ in range(2)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.focal_fwd(xc, Wc, b, t, 4173. * 1231, 0.5, 1.0, labels=labels, weights=w, want_acc=True)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ops.focal_fwd(xc, Wc, b, t, 4173. * 1231, 0.5, 1.0, labels=labels, weights=w, want_acc=True)
    for _ in range(3):
        graph.replay()
        torch.cuda.synchronize()
        for e in eager:   # (dz's padding columns are never written)
            assert torch.equal(out[2][:, :1231], e[2][:, :1231]) and torch.equal(out[1], e[1])
            assert torch.equal(out[0], e[0])


def _heads(compute_dtype, loss_cls=FO.FOCAL_BFOCAL_LOSS):
    from balancedgroupsoftmax_b200.head import ReweightBBoxHead
    inp = FO.fixture_inputs()
    sizes = FO.fixture_sizes()
    head = ReweightBBoxHead(num_fcs=2, reweight_cfg=dict(cls_weights=inp['cls_weight'], compute_dtype=compute_dtype),
                            loss_cls=dict(loss_cls), loss_bbox=dict(type='SmoothL1Loss', beta=1.0),
                            target_means=[0., 0., 0., 0.], target_stds=[0.1, 0.1, 0.2, 0.2], **sizes)
    return head, inp


def _count_fused_calls(monkeypatch):
    """Counts ops.SigmoidFocalFunction.apply calls: proof that a head took the fused route."""
    calls = []
    apply = ops.SigmoidFocalFunction.apply

    def counting(*args):
        calls.append(1)
        return apply(*args)
    monkeypatch.setattr(ops.SigmoidFocalFunction, 'apply', counting)
    return calls


def test_bfocal_head_fused_matches_materialised_and_fixture(monkeypatch):
    """fp32 compute: the fused route (one focal kernel for loss_cls and acc, TF32 products) against the materialised
    route (fp32 nn.Linear logits, the op's formula in fp32) and the reference fixture (float64 op).  With alpha = 1 only
    the one positive element counts (row 37, column 0, z = 11.54): its loss (1-p)^0.5 (-log p) and gradient change by
    about 1.5 relative per unit of z, and TF32 moves z by at most 2^-9 * |x_cls| |w_0| = 2^-9 * 8.78: 2.6 %.  The
    materialised route evaluates 1 - p (~1e-5) in fp32, which loses 2^-24 / (1 - p) = 0.6 % relative.  So loss_cls and
    the fc_cls gradients agree within 2^-5 (normwise); dX adds the same trunk backward to both routes.  acc may differ
    by the rows whose top two logits lie within TF32's error of each other: at most 2 of 256 here."""
    head, inp = _heads('fp32')
    calls = _count_fused_calls(monkeypatch)
    fused = FO.run_head(head, inp, device='cuda')
    assert len(calls) == 1
    mat = FO.run_head(head, inp, materialise=True, device='cuda')
    assert len(calls) == 1
    fix = np.load(FO.FIXTURE)
    assert mat['acc'].item() == float(fix['bfocal_acc'][0])
    assert abs(fused['acc'].item() - float(fix['bfocal_acc'][0])) <= 2 * 100.0 / 256
    for name in ('loss_cls', 'db', 'dW4', 'dX'):
        ref = mat[name].double().cpu().reshape(-1)
        got = fused[name].double().cpu().reshape(-1)
        assert float((got - ref).norm()) <= 2.0 ** -5 * float(ref.norm()) + 1e-30, name
    ref = float(fix['bfocal_loss_cls'])
    for route in (fused, mat):
        assert abs(route['loss_cls'].item() - ref) <= 2.0 ** -5 * abs(ref)


@pytest.mark.parametrize('gamma,alpha', [(2.0, 0.25), (0.5, 1.0)])
def test_focal_head_fused_matches_materialised_per_element(monkeypatch, gamma, alpha):
    """ReweightBBoxHead with a FocalLoss, fp32 compute, on one fc_cls input x: the fused route (bags_focal_fwd, TF32
    products) against the materialised route (fp32 nn.Linear logits, the op's formula in fp32), both bounded against
    the float64 op on exact logits z = x W^T + b.  alpha = 0.25 weighs the negatives of every row.  Per element, with
    S = |x| |W|^T and K = 64:
      fused logits        2^-9 S + (K + 2) 2^-24 (S + |b|)       (TF32 operands, fp32 sums)
      materialised logits (K + 2) 2^-24 (S + |b|)
      the fp32 formula    2^-18 |g| fused (module docstring), 2^-19 absolute materialised (a few ulp of terms <= 2)
    and |dl/dz| = |g| <= 2.  dW and db then follow through |x| and the sums: TF32 in the fused backward (2^-9), fp32
    sums in both (N + 2) 2^-24.  acc may differ only on rows whose top two exact logits lie within both logit errors."""
    from balancedgroupsoftmax_b200.head import ClsScoreHandle
    head, inp = _heads('fp32', dict(type='FocalLoss', use_sigmoid=True, gamma=gamma, alpha=alpha, loss_weight=1.0))
    head.load_state_dict(inp['params'])
    head.cuda().train()
    d = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in inp.items()}
    with torch.no_grad():
        x, _ = head._trunk(d['feats'])
    x = x.detach().float().contiguous()
    W, b = head.fc_cls.weight, head.fc_cls.bias
    labels, lw = d['labels'], d['label_weights']
    N = x.shape[0]
    calls = _count_fused_calls(monkeypatch)
    handle = ClsScoreHandle(head, x)
    out_f = head.loss(handle, None, labels, lw, None, None)
    assert len(calls) == 1 and handle.pending
    head.zero_grad(set_to_none=True)
    out_f['loss_cls'].backward()
    dW_f, db_f = W.grad.double(), b.grad.double()
    head.zero_grad(set_to_none=True)
    out_m = head.loss(F.linear(x, W, b), None, labels, lw, None, None)
    assert len(calls) == 1
    out_m['loss_cls'].backward()
    dW_m, db_m = W.grad.double(), b.grad.double()

    x64, W64, b64 = x.double(), W.detach().double(), b.detach().double()
    z = x64 @ W64.t() + b64
    S = x64.abs() @ W64.abs().t()
    K = x.shape[1]
    dz_m = (K + 2) * U * (S + b64.abs())
    dz_f = 2.0 ** -9 * S + dz_m
    t = L.focal_targets(labels, N)
    coef = (head.cls_weight.cuda()[labels].double() / (N * FO.ONE_HOT))[:, None]
    el, g = FO.op_forward(z, t, gamma, alpha), FO.op_backward(z, t, gamma, alpha)
    E = coef * (2 * (dz_f + dz_m) + 2.0 ** -18 * g.abs() + 2.0 ** -19)        # |dz_fused - dz_materialised|
    D = coef * g.abs() + E                                                     # |dz| of either route
    loss_tol = float((coef * (2 * (dz_f + dz_m) + 2.0 ** -18 * el.abs() + 2.0 ** -19 * (1 + el.abs()))).sum())
    loss_tol += 2.0 ** -13 * float((coef * el.abs()).sum())
    assert abs(out_f['loss_cls'].item() - out_m['loss_cls'].item()) <= loss_tol
    rounding = 2.0 ** -9 + 2 * (N + 2) * U
    assert ((dW_f - dW_m).abs() <= E.t() @ x64.abs() + rounding * (D.t() @ x64.abs()) + 1e-30).all()
    assert ((db_f - db_m).abs() <= E.sum(0) + 2 * (N + 2) * U * D.sum(0) + 1e-30).all()
    zl = z.gather(1, labels[:, None])[:, 0]
    other = z.scatter(1, labels[:, None], float('-inf')).max(1).values
    undecided = int(((zl - other).abs() <= 2 * (dz_f + dz_m).max(1).values).sum())
    assert abs(out_f['acc'].item() - out_m['acc'].item()) * N / 100.0 <= undecided + 1e-6


def test_bfocal_head_step_makes_no_host_sync(monkeypatch):
    head, inp = _heads('bf16')
    head.load_state_dict(inp['params'])
    head.cuda().train()
    d = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in inp.items()}
    FO.run_head(head, inp, device='cuda')   # warm-up: caches, weight copies
    head.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    from balancedgroupsoftmax_b200.head import ClsScoreHandle
    calls = _count_fused_calls(monkeypatch)
    try:   # the classification step (the box loss's boolean-mask gather syncs by itself)
        cls_score, _ = head(d['feats'])
        losses = head.loss(cls_score, None, d['labels'], d['label_weights'], d['bbox_targets'], d['bbox_weights'])
        losses['loss_cls'].backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert isinstance(cls_score, ClsScoreHandle) and cls_score.pending and len(calls) == 1
    assert head.fc_cls.weight.grad is not None


def test_focal_loss_module_on_gpu_matches_oracle():
    """The materialised route on GPU logits (SharedFCBBoxHead's) against the float64 oracle."""
    g = torch.Generator().manual_seed(3)
    z = (torch.randn(300, 1231, generator=g) * 8).cuda().requires_grad_(True)
    labels = torch.randint(0, 1231, (300,), generator=g).cuda()
    labels[0] = 17
    w = torch.rand(300, generator=g).cuda()
    out = L.FocalLoss()(z, labels, w)
    ref, gref = FO.focal_loss(z.detach(), labels, w)
    assert abs(out.item() - ref.item()) <= 1e-5 * abs(ref.item())
    out.backward()
    assert ((z.grad.double() - gref).abs() <= 1e-5 * gref.abs() + 1e-12).all()
