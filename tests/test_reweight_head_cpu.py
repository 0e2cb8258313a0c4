"""CPU: the class-reweighted softmax head (ReweightBBoxHead) without a GPU --

  * bags_ce_fwd's argument validation (error codes and messages, never exceptions);
  * the oracle restatements (weighted CE, accuracy, the three class-weight formulas) and the package's own
    ``tables.class_weights`` / ``losses.accuracy`` pinned to the reference's source run in place (skipped where no
    reference checkout is reachable);
  * ``BBoxHead.loss`` and ReweightBBoxHead's materialised-logits loss against the reference heads;
  * the tables CLI's --cls-weight files, and a config block of faster_rcnn_r50_fpn_1x_lvis_reweighthead.py built through
    ``registry.build_head`` whose losses match the committed reference fixture.
"""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import reweight_oracle as R
from test_abi import check_fused_operand_rules
from balancedgroupsoftmax_b200 import _native as nat
from balancedgroupsoftmax_b200 import losses as L
from balancedgroupsoftmax_b200 import tables as T
from oracle import ref_shim

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason='no reference checkout reachable')


# --------------------------------------------------------------------------- ABI
def test_ce_fwd_invalid_arguments_return_error_codes():
    lib = nat.lib()
    buf = (C.c_char * 64)()
    p = C.addressof(buf)
    ws = lib.bags_workspace_bytes()

    base = (p + 15) // 16 * 16

    def call(N=4, K=8, C_=1231, loss=p, acc=None, dz=None, ldd=0, dtype=nat.DTYPE_BF16, wsb=ws, x=base, ldx=None, w=base,
             ldw=None):
        return lib.bags_ce_fwd(x, K if ldx is None else ldx, w, K if ldw is None else ldw, None, p, None, None, N, K, C_,
                               dtype, loss, acc, dz, ldd, None, 0, p, wsb, None, 0, None)

    for c in (0, 1281):
        assert call(C_=c) == -1 and b'bad shape' in lib.bags_last_error(), c
    assert call(loss=None) == -1 and b'NULL' in lib.bags_last_error()
    assert call(N=(1 << 24) + 1, acc=p) == -1 and b'2^24' in lib.bags_last_error()
    assert call(dz=p, ldd=1236) == -1 and b'ldd' in lib.bags_last_error()      # not a multiple of 8
    assert call(dz=p, ldd=1224) == -1 and b'ldd' in lib.bags_last_error()      # < C
    assert call(dtype=7) == -1 and b'dtype' in lib.bags_last_error()
    assert call(wsb=16) == -1 and b'workspace' in lib.bags_last_error()
    check_fused_operand_rules(lib, 'bags_ce_fwd', call, base)


def test_fused_eligibility_keeps_its_multiple_of_4_rule():
    """bags_ce_fwd takes any C; the grouped entry points keep theirs."""
    lib = nat.lib()
    assert lib.bags_fused_eligible(nat.int32_array([0, 1231]), 1, 1231) == 0
    assert lib.bags_fused_eligible(nat.int32_array([0, 1232]), 1, 1232) == 1


# --------------------------------------------------------------------------- class weights
def _counts():
    return T.synthetic_instance_counts(1230, seed=3)


@pytest.mark.parametrize('kind', ['inv', 'bf', 'bours'])
def test_class_weights_match_oracle(kind):
    fn = dict(inv=R.class_weights_inv, bf=R.class_weights_bf, bours=R.class_weights_bours)[kind]
    got = T.class_weights(_counts(), 1231, kind)
    assert got.dtype == np.float64 and got.shape == (1231,)
    np.testing.assert_allclose(got, fn(_counts()), rtol=1e-12, atol=0)
    if kind != 'bf':
        assert got[0] == 1.0 and got.min() >= 0.1 and got.max() <= 5.0


@needs_ref
@pytest.mark.parametrize('kind', ['inv', 'bf', 'bours'])
def test_class_weights_match_reference(kind):
    ref = R.reference_class_weights(_counts(), kind)
    assert ref.dtype == np.float64
    np.testing.assert_array_equal(T.class_weights(_counts(), 1231, kind), ref)


def test_tables_cli_writes_the_weight_files():
    with tempfile.TemporaryDirectory() as d:
        assert T.main(['--synthetic', '3', '--cls-weight', 'inv', 'bf', 'bours', '--out', d]) == 0
        for kind, name in T.CLS_WEIGHT_FILES.items():
            w = torch.load(os.path.join(d, name))
            assert w.dtype == torch.float64 and w.shape == (1231,)
            np.testing.assert_array_equal(w.numpy(), T.class_weights(_counts(), 1231, kind))


# --------------------------------------------------------------------------- loss and accuracy
def _logits(N=200, C=1231, seed=0):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(N, C, generator=g) * 2
    labels = torch.randint(0, C, (N,), generator=g)
    labels[: N // 2] = 0
    z[: N // 3, 0] += 8.0                               # some rows correct
    label_weights = torch.ones(N)
    label_weights[-7:] = 0
    return z, labels, label_weights


def test_accuracy_matches_oracle_and_counts_rows():
    z, labels, _ = _logits()
    a = L.accuracy(z, labels)
    assert a.shape == (1,)
    assert torch.equal(a, R.accuracy(z, labels))
    assert a.item() == pytest.approx(100.0 * R.correct_rows(z, labels).sum().item() / z.shape[0])


@needs_ref
def test_accuracy_and_loss_match_reference():
    z, labels, lw = _logits()
    cw = torch.from_numpy(T.class_weights(_counts(), 1231, 'inv'))
    assert torch.equal(R.accuracy(z, labels), R.reference_accuracy()(z, labels))
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'cls_weight.pt')
        torch.save(cw, path)
        ref = R.build_reference_reweight_bbox_head(path, in_channels=4, fc_out_channels=16, roi_feat_size=1)
    out = ref.loss(z, None, labels, lw, None, None)
    assert torch.equal(out['acc'], R.accuracy(z, labels))
    assert out['loss_cls'].item() == pytest.approx(R.reweight_ce_loss(z, labels, cw, lw).item(), rel=1e-6)


def _reweight_head(cls_weight, **kw):
    from balancedgroupsoftmax_b200.head import ReweightBBoxHead
    return ReweightBBoxHead(num_fcs=2, in_channels=4, fc_out_channels=16, roi_feat_size=1, num_classes=1231,
                            reweight_cfg=dict(cls_weights=cls_weight), **kw)


def test_reweight_head_materialised_loss_matches_oracle():
    """A plain logits tensor (or a reduction override) takes the reference's op sequence; no host sync is needed for
    the normaliser, which stays a tensor."""
    z, labels, lw = _logits()
    cw = torch.from_numpy(T.class_weights(_counts(), 1231, 'bours'))
    head = _reweight_head(cw)
    assert head.cls_weight.dtype == torch.float32 and not head.cls_weight.is_cuda
    out = head.loss(z, None, labels, lw, None, None)
    assert sorted(out) == ['acc', 'loss_cls']
    assert out['loss_cls'].item() == pytest.approx(R.reweight_ce_loss(z, labels, cw, lw).item(), rel=1e-6)
    assert torch.equal(out['acc'], R.accuracy(z, labels))
    none = head.loss(z, None, labels, lw, None, None, reduction_override='none')['loss_cls']
    assert none.shape == (z.shape[0],)
    ce = F.cross_entropy(z, labels, reduction='none') * cw.float()[labels]
    assert torch.allclose(none, ce)
    s = head.loss(z, None, labels, lw, None, None, reduction_override='sum')['loss_cls']
    assert s.item() == pytest.approx(ce.sum().item(), rel=1e-6)


@needs_ref
def test_bbox_head_loss_matches_reference():
    """BBoxHead.loss (inherited by SharedFCBBoxHead) against the reference's bbox_head.py:97-129."""
    import sys
    from balancedgroupsoftmax_b200.head import SharedFCBBoxHead
    ref_shim.load()
    RefShared = sys.modules['mmdet.models.bbox_heads.convfc_bbox_head'].SharedFCBBoxHead
    kw = dict(num_fcs=2, in_channels=4, fc_out_channels=16, roi_feat_size=1, num_classes=1231)
    ours, ref = SharedFCBBoxHead(**kw), RefShared(**kw)
    torch.manual_seed(0)
    ours.init_weights()
    ref.load_state_dict(ours.state_dict())
    inp = R.fixture_inputs()
    feats = torch.randn(256, 4, 1, 1)
    a, b = ours(feats), ref(feats)
    args = (inp['labels'], inp['label_weights'], inp['bbox_targets'], inp['bbox_weights'])
    lo, lr = ours.loss(*a, *args), ref.loss(*b, *args)
    assert sorted(lo) == sorted(lr) == ['acc', 'loss_bbox', 'loss_cls']
    for k in lr:
        assert torch.allclose(lo[k], lr[k], rtol=1e-6, atol=0), k


def test_reweighthead_config_block_matches_fixture():
    """The bbox_head block of faster_rcnn_r50_fpn_1x_lvis_reweighthead.py (sizes reduced to the fixture's), with a
    class-weight file written by the tables CLI, built through registry.build_head; its losses on the fixture inputs
    (materialised logits: no GPU here) equal the reference head's."""
    from balancedgroupsoftmax_b200 import registry
    inp = R.fixture_inputs()
    fix = np.load(R.FIXTURE)
    with tempfile.TemporaryDirectory() as d:
        T.main(['--synthetic', '0', '--cls-weight', 'inv', '--out', d])
        cfg = dict(
            type='ReweightBBoxHead', num_fcs=2, in_channels=R.FIX_IN, fc_out_channels=R.FIX_FC,
            reweight_cfg=dict(cls_weight=os.path.join(d, 'cls_weight.pt')), roi_feat_size=R.FIX_ROI,
            num_classes=1231, target_means=[0., 0., 0., 0.], target_stds=[0.1, 0.1, 0.2, 0.2],
            reg_class_agnostic=False, loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0),
            loss_bbox=dict(type='SmoothL1Loss', beta=1.0, loss_weight=1.0))
        head = registry.build_head(cfg)
    assert torch.equal(head.cls_weight, inp['cls_weight'].float())
    head.load_state_dict(inp['params'])
    head.train()
    x_cls, x_reg = head._trunk(inp['feats'])
    out = head.loss(head.fc_cls(x_cls), head.fc_reg(x_reg), inp['labels'], inp['label_weights'], inp['bbox_targets'],
                    inp['bbox_weights'])
    assert sorted(out) == ['acc', 'loss_bbox', 'loss_cls']
    assert out['loss_cls'].item() == pytest.approx(float(fix['loss_cls']), rel=1e-5)
    assert out['loss_bbox'].item() == pytest.approx(float(fix['loss_bbox']), rel=1e-5)
    assert out['acc'].item() == float(fix['acc'][0])
