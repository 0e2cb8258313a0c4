"""GPU parity tests (run with ``-m gpu`` on an H100): the CUDA path, called through the C ABI
(balancedgroupsoftmax_b200.ops -> ctypes -> libbags_b200.so), against

  * the committed golden fixtures produced by the reference's own code (tests/golden/),
  * the CPU oracle on the same seeded inputs at sizes the oracle finishes in seconds,
  * size-independent properties at the full benchmark size (4096 RoIs).

Tolerances:
  integer outputs (in-bin labels, masks given as input, avg factors, argmax ids) .. bit-exact
  fp32 mode (fp32 operands, TF32 tensor-core products, fp32 accumulate) ........... loss rel <= 1e-3,
                                                              dW/db/dX Frobenius-rel <= 1e-3 vs the fp32 reference
  bf16 mode (bf16 operands + bf16 dz, fp32 accumulate/softmax) ..................... loss rel <= 2e-3,
                                                              grads Frobenius-rel <= 5e-3 vs the fp32 reference
"""
import glob
import os

import numpy as np
import pytest
import torch

from balancedgroupsoftmax_b200.tables import synthetic_tables
from oracle import bags_oracle as O

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
CASES = sorted(glob.glob(os.path.join(GOLDEN, 'ref_*.npz')))
TOL = {
    torch.float32: dict(loss=1e-3, grad=1e-3, logits=1e-3),
    torch.bfloat16: dict(loss=2e-3, grad=5e-3, logits=4e-3),
}


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


@pytest.fixture(scope='module')
def env():
    from balancedgroupsoftmax_b200 import ops
    assert torch.cuda.is_available()
    t = synthetic_tables(1231, seed=0)
    dt = ops.DeviceTables.from_tables(t, 'cuda')
    return ops, t, dt, torch.from_numpy(t.label2binlabel), torch.from_numpy(t.pred_slice)


def test_native_library_is_loaded():
    """The CUDA extension (not a fallback) is what runs: the .so is mapped into this process."""
    from balancedgroupsoftmax_b200 import _native
    _native.lib()
    maps = open('/proc/self/maps').read()
    assert 'libbags_b200.so' in maps


@pytest.mark.parametrize('mode', [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('path', CASES, ids=[os.path.basename(p)[:-4] for p in CASES])
def test_golden_fixture_through_c_abi(env, path, mode):
    """Reference-generated vectors: same inputs, the reference's own sampled masks -> losses and grads."""
    ops, t, dt, l2b, ps = env
    d = np.load(path)
    x = torch.from_numpy(d['x']).cuda().to(mode)
    W = torch.from_numpy(d['weight']).cuda().to(mode)
    b = torch.from_numpy(d['bias']).cuda()
    labels = torch.from_numpy(d['labels']).cuda()
    wmask = torch.from_numpy(d['wmask']).cuda()
    avg = ops.mask_avg(wmask)
    assert avg.cpu().double().tolist() == d['avg'].tolist()          # integer-valued, bit-exact
    gout = torch.from_numpy(d['gout']).cuda()
    tol = TOL[mode]
    ref_loss = d['losses']
    assert ops.fused_eligible(dt)
    # route 1: fused kernel (logits never leave the chip); route 2: GEMM -> fp32 logits -> grouped CE
    for materialize in (False, True):
        loss, logits, lse, dz, colsum = ops.fused_fwd(x, W, b, labels, dt, wmask, avg, want_lse=True,
                                                      materialize=materialize)
        dW, db, dX = ops.fused_bwd(dz, x, W, gout, dt, colsum)
        torch.cuda.synchronize()
        assert (logits is None) == (not materialize)
        for g in range(5):
            assert abs(loss[g].item() - ref_loss[g]) <= tol['loss'] * max(abs(ref_loss[g]), 1e-2), \
                (materialize, g, loss[g].item(), ref_loss[g])
        if materialize:
            assert np.abs(logits[:, ::29].cpu().numpy() - d['logits_sample']).max() <= \
                tol['logits'] * np.abs(d['logits_sample']).max()
        for name, got in (('dW', dW), ('db', db), ('dX', dX)):
            ref = torch.from_numpy(d[name])
            if ref.norm().item() == 0:
                assert got.float().abs().max().item() == 0
            else:
                assert rel(got.float(), ref) <= tol['grad'], (materialize, name, rel(got.float(), ref))
    # argmax class ids of the merged scores: bit-exact on fp32 logits computed by the oracle
    z = O.fc_cls(torch.from_numpy(d['x']), torch.from_numpy(d['weight']), torch.from_numpy(d['bias']))
    scores = ops.merge_scores(z.cuda(), dt).cpu()
    assert np.array_equal(scores.argmax(1).numpy(), d['merged_argmax'].astype(np.int64))
    assert np.array_equal((scores[:, 1:].argmax(1) + 1).numpy(), d['merged_fg_argmax'].astype(np.int64))
    assert np.allclose(scores[:, ::37].numpy(), d['merged_sample'], rtol=1e-5, atol=1e-7)


def _problem(N, K=1024, seed=0, wstd=0.05):
    t = synthetic_tables(1231, seed=0)
    g = torch.Generator().manual_seed(seed)
    x = torch.relu(torch.randn(N, K, generator=g))
    W = torch.randn(t.num_logits, K, generator=g) * wstd
    b = torch.randn(t.num_logits, generator=g) * 0.1
    labels = torch.zeros(N, dtype=torch.long)
    npos = N // 4
    labels[:npos] = torch.randint(1, t.num_classes, (npos,), generator=g)
    l2b, ps = torch.from_numpy(t.label2binlabel), torch.from_numpy(t.pred_slice)
    np.random.seed(seed)
    remapped = O.remap_labels(labels, l2b, 8.0)
    return x, W, b, labels, remapped


@pytest.mark.parametrize('materialize', [False, True], ids=['fused', 'materialized'])
@pytest.mark.parametrize('mode', [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('N', [1, 3, 130, 512, 1000])
def test_fused_fwd_bwd_vs_oracle(env, N, mode, materialize):
    ops, t, dt, l2b, ps = env
    x, W, b, labels, remapped = _problem(N, seed=N)
    gout = [1.0, 0.5, 0.25, 2.0, 1.5]
    z = O.fc_cls(x, W, b)
    ref = O.bags_loss(z, labels, l2b, ps, remapped=remapped)
    _, dW_ref, db_ref, dX_ref = O.closed_form_grads(x, W, b, labels, l2b, ps, remapped, gout=gout)
    wmask = torch.stack([w.to(torch.uint8) for w in remapped[1]]).cuda()
    avg = ops.mask_avg(wmask)
    assert avg.cpu().tolist() == [float(a) for a in remapped[2]]
    xc, wc = x.cuda().to(mode), W.cuda().to(mode)
    loss, logits, _, dz, colsum = ops.fused_fwd(xc, wc, b.cuda(), labels.cuda(), dt, wmask, avg,
                                                materialize=materialize)
    dW, db, dX = ops.fused_bwd(dz, xc, wc, torch.tensor(gout, device='cuda'), dt, colsum)
    torch.cuda.synchronize()
    tol = TOL[mode]
    if mode == torch.bfloat16 and N < 128:
        # a handful of rows: bf16 operand rounding is not averaged out -> check the loss against the oracle
        # fed the same rounded operands (tight) instead of the fp32 one
        ref = O.bags_loss(O.fc_cls(x.bfloat16().float(), W.bfloat16().float(), b), labels, l2b, ps, remapped=remapped)
    for g in range(5):
        r = ref['loss_cls_bin%d' % g].item()
        assert abs(loss[g].item() - r) <= tol['loss'] * max(abs(r), 1e-2), (g, loss[g].item(), r)
    if materialize:
        assert rel(logits, z) <= tol['logits']
    if dW_ref.norm() > 0:
        assert rel(dW, dW_ref) <= tol['grad']
        assert rel(db, db_ref) <= tol['grad']
        assert rel(dX.float(), dX_ref) <= tol['grad']


@pytest.mark.parametrize('mode', [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('gval', [1.0, 0.375])
def test_uniform_upstream_gradients_skip_the_scaled_weight_copy(env, mode, gval):
    """all gout[g] equal (every bin's loss has the same weight -- the reference's setting): the merged backward reads W
    itself and scales dX in its epilogue instead of making W' = diag(gout) W; db is recomputed from dz (no colsum)"""
    ops, t, dt, l2b, ps = env
    N = 700
    x, W, b, labels, remapped = _problem(N, seed=11)
    gout = [gval] * 5
    _, dW_ref, db_ref, dX_ref = O.closed_form_grads(x, W, b, labels, l2b, ps, remapped, gout=gout)
    wmask = torch.stack([w.to(torch.uint8) for w in remapped[1]]).cuda()
    avg = ops.mask_avg(wmask)
    xc, wc = x.cuda().to(mode), W.cuda().to(mode)
    loss, _, _, dz, _ = ops.fused_fwd(xc, wc, b.cuda(), labels.cuda(), dt, wmask, avg)
    for _ in range(2):   # twice: the second call must not depend on state the first one left
        dW, db, dX = ops.fused_bwd(dz, xc, wc, torch.tensor(gout, device='cuda'), dt, None)
    torch.cuda.synchronize()
    tol = TOL[mode]
    assert rel(dW, dW_ref) <= tol['grad']
    assert rel(db, db_ref) <= tol['grad']
    assert rel(dX.float(), dX_ref) <= tol['grad']


def test_bf16_matches_oracle_on_rounded_operands_tightly(env):
    """With the oracle fed the same bf16-rounded x/W the only differences left are accumulation
    order and the bf16 rounding of dz: loss <= 1e-5, dW <= 2e-3; db <= 2e-3 when it is recomputed from
    the bf16-rounded dz (default) and <= 1e-5 when the grouped-CE kernel's fp32 column sums are passed."""
    ops, t, dt, l2b, ps = env
    x, W, b, labels, remapped = _problem(768, seed=5)
    xo, Wo = x.bfloat16().float(), W.bfloat16().float()
    ref = O.bags_loss(O.fc_cls(xo, Wo, b), labels, l2b, ps, remapped=remapped)
    _, dW_ref, db_ref, dX_ref = O.closed_form_grads(xo, Wo, b, labels, l2b, ps, remapped)
    wmask = torch.stack([w.to(torch.uint8) for w in remapped[1]]).cuda()
    avg = ops.mask_avg(wmask)
    for materialize, db_tol in ((False, 2e-3), (True, 1e-5)):
        loss, _, _, dz, colsum = ops.fused_fwd(x.cuda().bfloat16(), W.cuda().bfloat16(), b.cuda(), labels.cuda(), dt,
                                               wmask, avg, materialize=materialize, want_colsum=materialize)
        dW, db, dX = ops.fused_bwd(dz, x.cuda().bfloat16(), W.cuda().bfloat16(), None, dt, colsum)
        for g in range(5):
            r = ref['loss_cls_bin%d' % g].item()
            assert abs(loss[g].item() - r) <= 1e-5 * max(abs(r), 1.0)
        assert rel(dW, dW_ref) <= 2e-3 and rel(db, db_ref) <= db_tol and rel(dX.float(), dX_ref) <= 4e-3


def test_group_assignment_is_bit_exact(env):
    """t_g[n] = label2binlabel[g, labels[n]]: checked through the kernel's onehot position --
    with zero logits, dz[n, s_g + j] = coef*(1/len_g - [j == t_g]) so the most negative entry of each
    slice marks t_g exactly."""
    ops, t, dt, l2b, ps = env
    N = 700
    g = torch.Generator().manual_seed(3)
    labels = torch.randint(0, t.num_classes, (N,), generator=g)
    z = torch.zeros(N, t.num_logits, device='cuda')
    loss, _, dz, _ = ops.group_ce(z, labels.cuda(), dt, None, None, want_dz=True, dz_dtype=torch.float32)
    dz = dz[:, :t.num_logits].cpu()
    for gi in range(5):
        s, l = int(ps[gi, 0]), int(ps[gi, 1])
        got = dz[:, s:s + l].argmin(1)
        assert torch.equal(got, l2b[gi][labels]), gi
        assert abs(loss[gi].item() - np.log(l)) < 1e-5     # all-ones weights, avg = N


def test_sampler_properties_full_size(env):
    """Device sampler at the benchmark size: exact-k subsets, in-bin rows always kept, avg = F + k,
    deterministic per seed, different across seeds, selection frequency ~ uniform."""
    ops, t, dt, l2b, ps = env
    N = 4096
    _, _, _, labels, _ = _problem(N, seed=9)
    lab = labels.cuda()
    w1, a1 = ops.sample_others(lab, dt, 8.0, 42)
    w1b, _ = ops.sample_others(lab, dt, 8.0, 42)
    assert torch.equal(w1, w1b)
    counts = torch.zeros(5, N)
    trials = 64
    for s in range(trials):
        w, a = ops.sample_others(lab, dt, 8.0, 1000 + s)
        counts += w.float().cpu()
        for g in range(5):
            tg = l2b[g][labels]
            F = int((tg > 0).sum())
            k = int(F * 8.0)
            exp = N if (g == 0 or (F > 0 and k >= N - F)) else (0 if F == 0 else F + k)
            assert int(w[g].sum()) == exp and a[g].item() == max(float(exp), 1.0)
            if 0 < F and k < N - F:
                assert bool(w[g].cpu()[tg > 0].all())
    for g in range(1, 5):
        tg = l2b[g][labels]
        F = int((tg > 0).sum())
        k = int(F * 8.0)
        if 0 < F and k < N - F:
            freq = counts[g][tg == 0] / trials
            p = k / (N - F)
            assert abs(freq.mean().item() - p) < 1e-6            # exact-k => exact mean
            assert freq.std().item() < 2.5 * np.sqrt(p * (1 - p) / trials)   # no row systematically favoured


def test_sampler_ratio_edge_cases(env):
    ops, t, dt, l2b, ps = env
    labels = torch.zeros(256, dtype=torch.long)
    w, a = ops.sample_others(labels.cuda(), dt, 8.0, 1)             # all background
    assert w[0].sum().item() == 256 and w[1:].sum().item() == 0 and a.cpu().tolist() == [256.0, 1.0, 1.0, 1.0, 1.0]
    labels[:200] = torch.randint(1, 1231, (200,), generator=torch.Generator().manual_seed(0))
    w, a = ops.sample_others(labels.cuda(), dt, 8.0, 1)             # k >= #others everywhere
    assert int(w.sum()) == 5 * 256
    w, a = ops.sample_others(labels.cuda(), dt, 0.0, 1)             # ratio 0: only in-bin rows
    for g in range(1, 5):
        assert torch.equal(w[g].cpu().bool(), l2b[g][labels] > 0)


def test_merge_scores_vs_oracle_and_rowsums(env):
    ops, t, dt, l2b, ps = env
    g = torch.Generator().manual_seed(1)
    z = torch.randn(1000, t.num_logits, generator=g) * 3
    ref = O.merge_score(z, ps, [torch.from_numpy(s) for s in t.fg_splits], t.num_classes)
    got = ops.merge_scores(z.cuda(), dt).cpu()
    assert (got - ref).abs().max().item() < 1e-6
    assert torch.equal(got.argmax(1), ref.argmax(1))
    # property: row sum = P(bg) + P(fg) * sum_g (1 - p_g[others])
    assert torch.allclose(got.sum(1), ref.sum(1), rtol=1e-5)


def test_empty_and_tiny_inputs(env):
    ops, t, dt, l2b, ps = env
    x = torch.zeros(0, 64, device='cuda', dtype=torch.bfloat16)
    W = torch.randn(t.num_logits, 64, device='cuda').bfloat16()
    labels = torch.zeros(0, dtype=torch.long, device='cuda')
    loss, logits, _, dz, colsum = ops.fused_fwd(x, W, None, labels, dt, None, None)
    dW, db, dX = ops.fused_bwd(dz, x, W, None, dt, colsum)
    torch.cuda.synchronize()
    assert loss.cpu().tolist() == [0.0] * 5 and dW.abs().max().item() == 0 and db.abs().max().item() == 0
    assert ops.merge_scores(torch.zeros(0, t.num_logits, device='cuda'), dt).shape == (0, 1231)


def test_full_size_properties_4096(env):
    """BASELINE size (4096 x 1024 x 1236), size-independent checks:
      * linearity of the backward in gout: bwd(a*g1 + b*g2) = a*bwd(g1) + b*bwd(g2)
      * sum_j dz[n, slice_g] = 0 for every row/bin (softmax - onehot sums to zero)
      * db = column sums of dz ; loss >= 0 ; dX rows of zero-weight RoIs in all bins are zero."""
    ops, t, dt, l2b, ps = env
    N = 4096
    x, W, b, labels, remapped = _problem(N, seed=11)
    xc, wc = x.cuda().bfloat16(), W.cuda().bfloat16()
    lab = labels.cuda()
    wmask, avg = ops.sample_others(lab, dt, 8.0, 7)
    loss, logits, lse, dz, colsum = ops.fused_fwd(xc, wc, b.cuda(), lab, dt, wmask, avg, want_lse=True,
                                                  materialize=True, want_colsum=True)
    # the fused kernel agrees with the two-kernel route on everything it outputs
    loss_f, none_logits, lse_f, dz_f, colsum_f = ops.fused_fwd(xc, wc, b.cuda(), lab, dt, wmask, avg, want_lse=True,
                                                               want_colsum=True)
    assert none_logits is None
    assert rel(loss_f, loss) < 1e-5 and rel(lse_f, lse) < 1e-6
    assert rel(dz_f[:, :t.num_logits].float(), dz[:, :t.num_logits].float()) < 4e-3
    assert rel(colsum_f.sum(0), colsum.sum(0)) < 2e-3 and colsum_f.shape[0] == 32
    assert (loss >= 0).all()
    dzf = dz[:, :t.num_logits].float()
    for g in range(5):
        s, l = int(ps[g, 0]), int(ps[g, 1])
        assert dzf[:, s:s + l].sum(1).abs().max().item() < 2e-5       # bf16 rounding of ~1e-4-sized terms
        # lse really is logsumexp of the slice
        assert torch.allclose(lse[:, g], torch.logsumexp(logits[:, s:s + l], dim=1), rtol=1e-5, atol=1e-5)
    assert rel(colsum.sum(0), dzf.sum(0)) < 2e-3
    g1 = torch.tensor([1.0, 0.0, 2.0, 0.0, 0.5], device='cuda')
    g2 = torch.tensor([0.0, 3.0, 0.0, 1.0, 0.25], device='cuda')
    r1 = ops.fused_bwd(dz, xc, wc, g1, dt, colsum)
    r2 = ops.fused_bwd(dz, xc, wc, g2, dt, colsum)
    r3 = ops.fused_bwd(dz, xc, wc, 2.0 * g1 - 0.5 * g2, dt, colsum)
    # db: forward partials (colsum) and the backward's own recomputation from dz agree
    db_a = ops.fused_bwd(dz, xc, wc, g1, dt, colsum, need_dw=False, need_dx=False)[1]
    db_b = ops.fused_bwd(dz, xc, wc, g1, dt, None, need_dw=False, need_dx=False)[1]
    assert rel(db_b, db_a) < 2e-3
    assert rel(r3[0], 2.0 * r1[0] - 0.5 * r2[0]) < 1e-5            # dW (fp32 atomics: order-dependent rounding)
    assert rel(r3[1], 2.0 * r1[1] - 0.5 * r2[1]) < 1e-6            # db
    assert rel(r3[2].float(), 2.0 * r1[2].float() - 0.5 * r2[2].float()) < 2e-2   # dX (bf16 out, bf16 W')
    # the fused dW agrees with a plain fp32 matmul of the saved dz
    dW_chk = (dzf * 1.0).t() @ xc.float()
    dW1 = ops.fused_bwd(dz, xc, wc, None, dt, colsum, need_dx=False)[0]
    assert rel(dW1, dW_chk) < 1e-5


def test_module_api_matches_oracle(env):
    """GSBBoxHeadWith0 through forward() -> loss() -> backward(), numpy ('reference') sampler so the
    masks are the reference's for the same numpy seed."""
    ops, t, dt, l2b, ps = env
    from balancedgroupsoftmax_b200.head import ClsScoreHandle, GSBBoxHeadWith0
    torch.manual_seed(0)
    head = GSBBoxHeadWith0(num_fcs=2, in_channels=8, fc_out_channels=256, roi_feat_size=2, num_classes=1231,
                           gs_config=dict(tables=t, others_sample_ratio=8.0, num_bins=5, sampler='numpy',
                                          compute_dtype='fp32',
                                          loss_bin=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0)))
    head.init_weights()
    with torch.no_grad():
        head.fc_cls.weight.normal_(0, 0.05)
    head = head.cuda().train()
    N = 384
    feats = torch.randn(N, 8, 2, 2, device='cuda')
    labels = torch.zeros(N, dtype=torch.long)
    labels[:96] = torch.randint(1, 1231, (96,))
    np.random.seed(21)
    cls_score, bbox_pred = head(feats)
    assert isinstance(cls_score, ClsScoreHandle) and tuple(bbox_pred.shape) == (N, 4924)
    losses = head.loss(cls_score, None, labels.cuda(), None, None, None)
    assert list(losses.keys()) == ['loss_cls_bin%d' % g for g in range(5)]
    sum(losses.values()).backward()
    x_cls = cls_score.x_cls.detach().cpu()
    W, b = head.fc_cls.weight.detach().cpu(), head.fc_cls.bias.detach().cpu()
    np.random.seed(21)
    lo, dW, db, dX = O.head_step(x_cls, W, b, labels, l2b, ps, 8.0)
    for k in losses:
        assert abs(losses[k].item() - lo[k].item()) <= 1e-3 * max(abs(lo[k].item()), 1e-2), k
    assert rel(head.fc_cls.weight.grad, dW) <= 1e-3 and rel(head.fc_cls.bias.grad, db) <= 1e-3
    # gradient reaches the trunk through dX
    assert head.shared_fcs[1].weight.grad is not None and head.shared_fcs[1].weight.grad.abs().sum().item() > 0
    # eval path: materialised logits + merged scores
    head.eval()
    with torch.no_grad():
        z, _ = head(feats)
        assert isinstance(z, torch.Tensor) and tuple(z.shape) == (N, 1236)
        assert rel(z, O.fc_cls(x_cls, W, b)) <= 1e-3
        bboxes, scores = head.get_det_bboxes(torch.zeros(N, 5, device='cuda'), [z, z], None, None, None)
        assert tuple(scores.shape) == (N, 1231)


def test_device_sampler_module_path_and_cascade_weights(env):
    """Default (device) sampler + per-stage loss weights (cascade_rcnn.py:248-250): scaling each per-bin
    loss by lw scales the fc_cls gradient by lw."""
    ops, t, dt, l2b, ps = env
    from balancedgroupsoftmax_b200.api import bags_head_loss
    x, W, b, labels, _ = _problem(512, seed=2)
    xc = x.cuda().bfloat16()
    lab = labels.cuda()
    grads = []
    for lw in (1.0, 0.25):
        w = torch.nn.Parameter(W.cuda())
        bb = torch.nn.Parameter(b.cuda())
        losses = bags_head_loss(xc, w, bb, lab, dt, 8.0, seed=77)
        (lw * losses.sum()).backward()
        grads.append((w.grad.clone(), bb.grad.clone()))
    assert rel(grads[1][0], 0.25 * grads[0][0]) < 1e-5 and rel(grads[1][1], 0.25 * grads[0][1]) < 1e-6


# --------------------------------------------------------------------------------------------------------------
# The benchmark configuration (4096 RoIs x 1024 x 1236) against the oracle itself -- the shape bench.py times -- plus
# neighbouring and ragged N.
# Reference to match: gs_bbox_head_with0.py:147-171 + autograd (dist_utils.py:53).
# --------------------------------------------------------------------------------------------------------------
GOUTS = {'uniform': [1.0] * 5, 'cascade': [0.5] * 5, 'nonuniform': [1.0, 0.5, 0.25, 2.0, 1.5]}


def _check_vs_oracle(ops, dt, l2b, ps, x, W, b, labels, remapped, mode, gout, loss, dW, db, dX):
    """fp32 mode: the TOL tolerances vs the fp32 oracle.  bf16 mode: those of TOL vs the fp32 oracle AND the tight
    ones vs the oracle fed the same bf16-rounded operands."""
    tol = TOL[mode]
    ref = O.bags_loss(O.fc_cls(x, W, b), labels, l2b, ps, remapped=remapped)
    _, dW_ref, db_ref, dX_ref = O.closed_form_grads(x, W, b, labels, l2b, ps, remapped, gout=gout)
    for g in range(5):
        r = ref['loss_cls_bin%d' % g].item()
        assert abs(loss[g].item() - r) <= tol['loss'] * max(abs(r), 1e-2), (g, loss[g].item(), r)
    errs = dict(dW=rel(dW, dW_ref), db=rel(db, db_ref), dX=rel(dX.float(), dX_ref))
    assert max(errs.values()) <= tol['grad'], errs
    if mode == torch.bfloat16:
        xo, Wo = x.bfloat16().float(), W.bfloat16().float()
        ref = O.bags_loss(O.fc_cls(xo, Wo, b), labels, l2b, ps, remapped=remapped)
        _, dW_r, db_r, dX_r = O.closed_form_grads(xo, Wo, b, labels, l2b, ps, remapped, gout=gout)
        for g in range(5):
            r = ref['loss_cls_bin%d' % g].item()
            assert abs(loss[g].item() - r) <= 1e-5 * max(abs(r), 1.0), (g, loss[g].item(), r)
        errs = dict(dW=rel(dW, dW_r), db=rel(db, db_r), dX=rel(dX.float(), dX_r))
        assert errs['dW'] <= 2e-3 and errs['db'] <= 2e-3 and errs['dX'] <= 4e-3, errs
    # dX row by row: a mis-mapped 256 x 256 unit would leave whole row blocks wrong while the Frobenius norm of a
    # single bad block of 16 could hide below a loose global bound -- so bound every 128-row block separately
    blk = 128
    for r0 in range(0, x.shape[0], blk):
        a, r = dX[r0:r0 + blk].float().cpu(), dX_ref[r0:r0 + blk]
        if r.norm() > 0:
            assert rel(a, r) <= 2 * tol['grad'], ('dX block', r0, rel(a, r))
    for c0 in range(0, W.shape[0], blk):
        assert rel(dW[c0:c0 + blk], dW_ref[c0:c0 + blk]) <= 2 * tol['grad'], ('dW block', c0)


@pytest.mark.parametrize('gname', ['uniform', 'nonuniform'])
@pytest.mark.parametrize('mode', [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('N', [3328, 3329, 4000, 4096])
def test_config2_full_size_vs_oracle(env, N, mode, gname):
    """loss, dW, db and dX of the benchmarked instantiation against the CPU oracle (closed-form gradients)."""
    ops, t, dt, l2b, ps = env
    x, W, b, labels, remapped = _problem(N, seed=100 + N)
    gout = GOUTS[gname]
    wmask = torch.stack([w.to(torch.uint8) for w in remapped[1]]).cuda()
    avg = ops.mask_avg(wmask)
    assert avg.cpu().tolist() == [float(a) for a in remapped[2]]
    xc, wc = x.cuda().to(mode), W.cuda().to(mode)
    loss, _, _, dz, _ = ops.fused_fwd(xc, wc, b.cuda(), labels.cuda(), dt, wmask, avg)
    dW, db, dX = ops.fused_bwd(dz, xc, wc, torch.tensor(gout, device='cuda'), dt, None)
    torch.cuda.synchronize()
    _check_vs_oracle(ops, dt, l2b, ps, x, W, b, labels, remapped, mode, gout, loss, dW, db, dX)


@pytest.mark.parametrize('splits', ['1', '5'])
@pytest.mark.parametrize('N', [512, 4096])
def test_backward_dw_splits_forced(env, monkeypatch, N, splits):
    """The merged backward with its dW units forced to one split (plain red.add of whole-K tiles) and to five (more dW
    than dX units in the work list), at a small and at the benchmark size."""
    ops, t, dt, l2b, ps = env
    from balancedgroupsoftmax_b200 import _native
    monkeypatch.setenv('BAGS_DW_SPLITS', splits)
    _native.reload_env()
    try:
        x, W, b, labels, remapped = _problem(N, seed=7 + N)
        gout = GOUTS['nonuniform']
        wmask = torch.stack([w.to(torch.uint8) for w in remapped[1]]).cuda()
        avg = ops.mask_avg(wmask)
        xc, wc = x.cuda().bfloat16(), W.cuda().bfloat16()
        loss, _, _, dz, _ = ops.fused_fwd(xc, wc, b.cuda(), labels.cuda(), dt, wmask, avg)
        dW, db, dX = ops.fused_bwd(dz, xc, wc, torch.tensor(gout, device='cuda'), dt, None)
        torch.cuda.synchronize()
        _check_vs_oracle(ops, dt, l2b, ps, x, W, b, labels, remapped, torch.bfloat16, gout, loss, dW, db, dX)
    finally:
        monkeypatch.delenv('BAGS_DW_SPLITS')
        _native.reload_env()


@pytest.mark.parametrize('need_dx', [True, False], ids=['dx', 'nodx'])
def test_graphed_step_config2_vs_oracle(env, need_dx):
    """The CUDA-graph step bench.py's e2e leg replays (GraphedHeadStep, N = 4096, bf16) against the oracle, with the
    masks its device sampler drew; need_dx=False is the shipped configs' case (selectp 1/3: dW + db only)."""
    ops, t, dt, l2b, ps = env
    from balancedgroupsoftmax_b200.api import GraphedHeadStep
    N = 4096
    x, W, b, labels, _ = _problem(N, seed=31)
    dev = torch.device('cuda', 0)
    Wp = torch.nn.Parameter(W.to(dev).bfloat16())
    bp = torch.nn.Parameter(b.to(dev))
    step = GraphedHeadStep(Wp, bp, dt, N, others_sample_ratio=8.0, seed=99, need_dx=need_dx)
    for it in range(2):
        losses = step(x.to(dev).bfloat16(), labels.to(dev)).clone()
        torch.cuda.synchronize()
        cnt = torch.tensor([it], dtype=torch.int64, device=dev)
        wmask, avg = ops.sample_others(labels.to(dev), dt, 8.0, 99, seed_step=cnt)
        remapped = ([l2b[g][labels] for g in range(5)], [wmask[g].cpu().long() for g in range(5)],
                    [float(a) for a in avg.cpu().tolist()])
        dX = step.grad_x if need_dx else None
        xo, Wo = x.bfloat16().float(), W.bfloat16().float()
        ref = O.bags_loss(O.fc_cls(xo, Wo, b), labels, l2b, ps, remapped=remapped)
        _, dW_r, db_r, dX_r = O.closed_form_grads(xo, Wo, b, labels, l2b, ps, remapped)
        for g in range(5):
            r = ref['loss_cls_bin%d' % g].item()
            assert abs(losses[g].item() - r) <= 1e-5 * max(abs(r), 1.0)
        # the parameter is bf16, so its gradient is returned in bf16 (one more rounding: 2^-9 relative per element)
        assert rel(step.grad_weight.float(), dW_r) <= 4e-3 and rel(step.grad_bias, db_r) <= 2e-3
        if need_dx:
            assert rel(dX.float(), dX_r) <= 4e-3
        else:
            assert step.grad_x is None


@pytest.mark.parametrize('gname', ['uniform', 'nonuniform'])
@pytest.mark.parametrize('mode', [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('N', [512, 4096])
def test_split_backward_matches_oracle(env, N, mode, gname):
    """The two launches of the in-step exchange schedule (dW + db first, then dX while the gradients travel): each half
    alone runs as a plain GEMM (with the preparation kernel where it has work) and must give the oracle's gradients."""
    ops, t, dt, l2b, ps = env
    x, W, b, labels, remapped = _problem(N, seed=55 + N)
    gout = GOUTS[gname]
    wmask = torch.stack([w.to(torch.uint8) for w in remapped[1]]).cuda()
    avg = ops.mask_avg(wmask)
    xc, wc = x.cuda().to(mode), W.cuda().to(mode)
    loss, _, _, dz, _ = ops.fused_fwd(xc, wc, b.cuda(), labels.cuda(), dt, wmask, avg)
    g = torch.tensor(gout, device='cuda')
    for _ in range(2):   # twice: the second call must not depend on state the first one left
        dW, db, none_dx = ops.fused_bwd(dz, xc, wc, g, dt, None, need_dx=False)
        none_dw, none_db, dX = ops.fused_bwd(dz, xc, wc, g, dt, None, need_dw=False, need_db=False)
    torch.cuda.synchronize()
    assert none_dx is None and none_dw is None and none_db is None
    _check_vs_oracle(ops, dt, l2b, ps, x, W, b, labels, remapped, mode, gout, loss, dW, db, dX)


@pytest.mark.parametrize('fwd_colsum', [False, True], ids=['bwdcolsum', 'fwdcolsum'])
@pytest.mark.parametrize('mode', [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('N', [200, 512, 4096])
def test_preparation_in_forward_matches_oracle(env, N, mode, fwd_colsum):
    """dW zeroed by the forward kernel's clear hook (bags_fwd's clear argument) -- and optionally the bias-gradient
    partials from the forward too -- then bags_bwd(DW_PREZEROED): same gradients as the oracle; the hook really zeroes a
    dirty buffer."""
    ops, t, dt, l2b, ps = env
    x, W, b, labels, remapped = _problem(N, seed=77 + N)
    gout = GOUTS['nonuniform']
    wmask = torch.stack([w.to(torch.uint8) for w in remapped[1]]).cuda()
    avg = ops.mask_avg(wmask)
    xc, wc = x.cuda().to(mode), W.cuda().to(mode)
    dW = torch.full((t.num_logits, 1024), 123.0, device='cuda')
    loss, _, _, dz, colsum = ops.fused_fwd(xc, wc, b.cuda(), labels.cuda(), dt, wmask, avg, clear=dW,
                                           want_colsum=fwd_colsum)
    torch.cuda.synchronize()
    assert dW.abs().max().item() == 0.0
    g = torch.tensor(gout, device='cuda')
    _, db, dX = ops.fused_bwd(dz, xc, wc, g, dt, colsum, dW=dW, dw_prezeroed=True)
    torch.cuda.synchronize()
    _check_vs_oracle(ops, dt, l2b, ps, x, W, b, labels, remapped, mode, gout, loss, dW, db, dX)
    # the split launches with a pre-zeroed dW
    dW2 = torch.full_like(dW, -7.0)
    loss, _, _, dz, colsum = ops.fused_fwd(xc, wc, b.cuda(), labels.cuda(), dt, wmask, avg, clear=dW2,
                                           want_colsum=fwd_colsum)
    _, db2, _ = ops.fused_bwd(dz, xc, wc, g, dt, colsum, dW=dW2, dw_prezeroed=True, need_dx=False)
    _, _, dX2 = ops.fused_bwd(dz, xc, wc, g, dt, None, need_dw=False, need_db=False)
    torch.cuda.synchronize()
    _check_vs_oracle(ops, dt, l2b, ps, x, W, b, labels, remapped, mode, gout, loss, dW2, db2, dX2)
