"""CPU: the sigmoid focal loss (FocalLoss; bags_focal_fwd on the GPU) without a GPU --

  * the float64 oracle (tests/focal_oracle.py) pinned to the reference's source text, and the reference's own
    FocalLoss.forward and heads run in place with its op replaced by that oracle (skipped where no reference checkout
    is reachable).  The reference's op cannot be built against current torch (THC API), so its math is pinned by the
    source text and the float64 restatement only;
  * this package's FocalLoss (the materialised route) against the oracle: the one-hot target quirk, avg_factor =
    N * 1231, the weight broadcast, the three reductions, the op's gradient, and the edge cases;
  * both focal configs' heads against the committed fixture tests/golden/focal_head_ref_n256.npz;
  * the registry building the bbox_head blocks of the three focal configs;
  * bags_focal_fwd's argument validation (error codes and messages, never exceptions).
"""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import focal_oracle as FO
from test_abi import check_fused_operand_rules
from balancedgroupsoftmax_b200 import _native as nat
from balancedgroupsoftmax_b200 import losses as L
from oracle import ref_shim

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason='no reference checkout reachable')


# --------------------------------------------------------------------------- the oracle and the reference
@needs_ref
def test_oracle_is_pinned_to_the_reference_source():
    assert FO.pin_reference_source() == {}


def _logits(N=300, C=1231, seed=0, scale=6.0):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(N, C, generator=g, dtype=torch.float64) * scale
    z[:, :8] = torch.tensor([-120., -40., -17.5, -1e-3, 0., 1e-3, 17.5, 40.], dtype=torch.float64)
    labels = torch.randint(0, C, (N,), generator=g)
    labels[0] = 5      # row 5 has column 0 positive (the one-hot quirk)
    labels[1] = 0
    weight = torch.rand(N, generator=g, dtype=torch.float64) + 0.5
    return z, labels, weight


def test_focal_targets_are_the_first_rows_of_the_flattened_one_hot():
    _, labels, _ = _logits()
    t = L.focal_targets(labels, labels.numel())
    assert t.dtype == torch.int64
    assert torch.equal(t, FO.targets_of(labels))
    assert torch.equal(t.nonzero().reshape(-1), torch.tensor([5]))


@pytest.mark.parametrize('reduction', ['mean', 'none', 'sum'])
@pytest.mark.parametrize('gamma,alpha', [(2.0, 0.25), (0.5, 1), (0.0, 0.25)])
def test_focal_loss_matches_oracle(gamma, alpha, reduction):
    """FocalLoss in float64 against the oracle: loss and the op's analytic gradient (not autograd of the loss); the
    caller's avg_factor is ignored."""
    z, labels, w = _logits()
    loss_mod = L.FocalLoss(gamma=gamma, alpha=alpha, loss_weight=0.5)
    zz = z.clone().requires_grad_(True)
    if reduction == 'sum':
        with pytest.raises(ValueError):
            loss_mod(zz, labels, w, avg_factor=3.0, reduction_override='sum')
        return
    out = loss_mod(zz, labels, w, avg_factor=3.0, reduction_override=reduction)
    ref, gref = FO.focal_loss(z, labels, w, gamma, alpha, reduction, loss_weight=0.5)
    torch.testing.assert_close(out, ref, rtol=1e-12, atol=1e-300)
    out.backward(torch.ones_like(out))
    torch.testing.assert_close(zz.grad, gref, rtol=1e-12, atol=1e-300)


def test_focal_loss_float32_edges():
    """float32 logits: gamma = 0 (x^0 = 1, 0^0 included), p saturating at |z| >= 17, and z beyond log(FLT_MIN)."""
    z = torch.tensor([[-200., -120., -88., -40., -17.5, 0., 17.5, 40., 120.]])
    for t in (0, 1):   # column 0 positive (t = 1), all negative (t = 0)
        for gamma, alpha in ((0.0, 0.25), (2.0, 0.25), (0.5, 1.0)):
            tt = torch.tensor([t])
            el, g = L.sigmoid_focal_elementwise(z, tt, gamma, alpha, with_grad=True)
            ref_el, ref_g = FO.op_forward(z, tt, gamma, alpha), FO.op_backward(z, tt, gamma, alpha)
            assert torch.isfinite(el).all() and torch.isfinite(g).all()
            torch.testing.assert_close(el.double(), ref_el, rtol=1e-5, atol=1e-6)
            torch.testing.assert_close(g.double(), ref_g, rtol=1e-5, atol=1e-6)
    # log(max(p, FLT_MIN)) caps the positive loss at alpha * 87.34
    el = L.sigmoid_focal_elementwise(torch.tensor([[-200.]]), torch.tensor([1]), 0.0, 1.0)
    assert el.item() == pytest.approx(87.3365447, rel=1e-6)


def test_negative_targets_ignore_the_row():
    z, _, _ = _logits(N=4, C=8)
    t = torch.tensor([-1, 0, 1, 9])
    el = L.sigmoid_focal_elementwise(z.float(), t, 2.0, 0.25)
    assert (el[0] == 0).all() and (el[1:].sum(1) > 0).all()
    torch.testing.assert_close(el.double(), FO.op_forward(z.float(), t, 2.0, 0.25), rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize('gamma,alpha', [(0.0, 0.25), (0.5, 1.0), (2.0, 0.25), (0.5, 0.25), (2.0, 1.0)])
def test_gradient_lipschitz_bound(gamma, alpha):
    """|d grad / dz| <= 1 for both element kinds: the GPU tests bound dz's error from the logits' error with it."""
    assert FO.lipschitz_bound(gamma, alpha) <= 1.0


@needs_ref
@pytest.mark.parametrize('reduction', ['mean', 'none', 'sum'])
def test_focal_loss_matches_reference(reduction):
    """The reference's FocalLoss.forward (its op replaced by the float64 oracle) against this package's, float64."""
    RefFocal = FO.load_reference_focal_loss()
    z, labels, w = _logits()
    ours, ref = L.FocalLoss(gamma=2.0, alpha=0.25), RefFocal(use_sigmoid=True, gamma=2.0, alpha=0.25)
    za, zb = z.clone().requires_grad_(True), z.clone().requires_grad_(True)
    if reduction == 'sum':
        for m, zz in ((ours, za), (ref, zb)):
            with pytest.raises(ValueError):
                m(zz, labels, w, avg_factor=7.0, reduction_override='sum')
        return
    a = ours(za, labels, w, avg_factor=7.0, reduction_override=reduction)
    b = ref(zb, labels, w, avg_factor=7.0, reduction_override=reduction)
    torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-300)
    a.sum().backward()
    b.sum().backward()
    torch.testing.assert_close(za.grad, zb.grad, rtol=1e-12, atol=1e-300)


def _our_heads(cls_weight_path):
    from balancedgroupsoftmax_b200 import head, registry  # noqa: F401  (importing head registers the heads)
    return {k: registry.build_head(cfg) for k, cfg in FO.head_blocks(cls_weight_path, **FO.fixture_sizes()).items()}


def _compare(got, want, key):
    for name in ('loss_cls', 'loss_bbox', 'db', 'dW4', 'dX'):
        a, b = got[name].double().numpy().reshape(-1), np.asarray(want['%s_%s' % (key, name)], np.float64).reshape(-1)
        np.testing.assert_allclose(a, b, rtol=2e-5, atol=1e-6 * np.abs(b).max(), err_msg='%s %s' % (key, name))
    assert got['acc'].item() == float(want['%s_acc' % key][0])


@pytest.mark.parametrize('key', ['shared', 'bfocal'])
def test_config_heads_match_fixture(key):
    """SharedFCBBoxHead (focalloss{,_all}) and ReweightBBoxHead (reweighthead_bfocal) built through the registry from
    their config blocks; losses and gradients on the fixture inputs (materialised logits, CPU, float64) equal the
    reference's."""
    inp = FO.fixture_inputs()
    fix = np.load(FO.FIXTURE)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'cls_weight_bf.pt')
        torch.save(inp['cls_weight'], path)
        head = _our_heads(path)[key]
    assert type(head.loss_cls) is L.FocalLoss
    _compare(FO.run_head(head, inp, materialise=key == 'bfocal', dtype=torch.float64), fix, key)


@needs_ref
def test_reference_heads_match_fixture():
    """The fixture is what the reference heads (float64 op) return today."""
    inp = FO.fixture_inputs()
    fix = np.load(FO.FIXTURE)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'cls_weight_bf.pt')
        torch.save(inp['cls_weight'], path)
        heads = FO.build_reference_heads(path, **FO.fixture_sizes())
    for key, head in heads.items():
        _compare(FO.run_head(head, inp, dtype=torch.float64), fix, key)


def test_registry_builds_the_three_focal_configs():
    """configs/transferred/faster_rcnn_r50_fpn_1x_lvis_{focalloss,focalloss_all,reweighthead_bfocal}.py: the first two
    share one bbox_head block.  Full sizes; the reweight head's class weights come from a file, as in the config."""
    from balancedgroupsoftmax_b200.head import ReweightBBoxHead, SharedFCBBoxHead
    from balancedgroupsoftmax_b200 import registry
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'cls_weight_bf.pt')
        torch.save(torch.rand(1231, dtype=torch.float64), path)
        heads = {k: registry.build_head(cfg) for k, cfg in FO.head_blocks(path).items()}
    assert type(heads['shared']) is SharedFCBBoxHead and type(heads['bfocal']) is ReweightBBoxHead
    for key, (gamma, alpha) in (('shared', (2.0, 0.25)), ('bfocal', (0.5, 1))):
        lc = heads[key].loss_cls
        assert isinstance(lc, L.FocalLoss) and (lc.gamma, lc.alpha, lc.reduction) == (gamma, alpha, 'mean')
    assert heads['bfocal']._fused_loss_ok() == 'focal'


def test_focal_reweight_head_rejects_sum_like_the_reference():
    from balancedgroupsoftmax_b200.head import ReweightBBoxHead
    head = ReweightBBoxHead(num_fcs=2, in_channels=4, fc_out_channels=16, roi_feat_size=1, num_classes=1231,
                            reweight_cfg=dict(cls_weights=torch.ones(1231)), loss_cls=dict(FO.FOCAL_BFOCAL_LOSS))
    z, labels, _ = _logits(N=20)
    lw = torch.ones(20)
    with pytest.raises(ValueError):
        head.loss(z.float(), None, labels, lw, None, None, reduction_override='sum')
    none = head.loss(z.float(), None, labels, lw, None, None, reduction_override='none')['loss_cls']
    assert none.shape == (20, 1231)


# --------------------------------------------------------------------------- ABI
def test_focal_fwd_invalid_arguments_return_error_codes():
    lib = nat.lib()
    buf = (C.c_char * 64)()
    p = C.addressof(buf)
    ws = lib.bags_workspace_bytes()

    base = (p + 15) // 16 * 16

    def call(N=4, K=8, C_=1231, targets=p, labels=None, loss=p, acc=None, dz=None, ldd=0, dtype=nat.DTYPE_BF16,
             wsb=ws, norm=4 * 1231.0, x=base, colsum=None, tiles=0, ldx=None, w=base, ldw=None):
        return lib.bags_focal_fwd(x, K if ldx is None else ldx, w, K if ldw is None else ldw, None, targets, labels,
                                  None, norm, 2.0, 0.25, N, K, C_, dtype, loss, acc, dz, ldd, colsum, tiles, p, wsb,
                                  None, 0, None)

    for c in (0, 1281):
        assert call(C_=c) == -1 and b'bad shape' in lib.bags_last_error(), c
    assert call(K=0) == -1 and b'bad shape' in lib.bags_last_error()
    assert call(loss=None) == -1 and b'NULL' in lib.bags_last_error()
    assert call(targets=None) == -1 and b'NULL' in lib.bags_last_error()
    assert call(x=None) == -1 and b'NULL' in lib.bags_last_error()
    assert call(acc=p) == -1 and b'NULL' in lib.bags_last_error()            # the accuracy needs the labels
    assert call(N=(1 << 24) + 1, acc=p, labels=p) == -1 and b'2^24' in lib.bags_last_error()
    assert call(dz=p, ldd=1236) == -1 and b'ldd' in lib.bags_last_error()    # not a multiple of 8
    assert call(dz=p, ldd=1224) == -1 and b'ldd' in lib.bags_last_error()    # < C
    assert call(dtype=7) == -1 and b'dtype' in lib.bags_last_error()
    assert call(wsb=16) == -1 and b'workspace' in lib.bags_last_error()
    for bad in (0.0, -1.0, float('inf'), float('nan')):
        assert call(norm=bad) == -1 and b'norm' in lib.bags_last_error(), bad
    assert call(colsum=p, tiles=2) == -1 and b'colsum' in lib.bags_last_error()
    check_fused_operand_rules(lib, 'bags_focal_fwd', call, base)
