"""CPU: the fused class-specific box loss (fuse_bbox_loss; bags_box_fwd / bags_box_bwd on the GPU) without a GPU --

  * the float64 oracle (tests/box_oracle.py) against the reference's own BBoxHead.loss run in place (skipped where no
    reference checkout is reachable), and against the committed fixture tests/golden/box_loss_ref_n256.npz;
  * the heads' materialised route on CPU against the fixture, and the reference heads against it;
  * BoxPredHandle's lazy mechanics, and ``forward`` returning a plain tensor on CPU or with the key unset;
  * bags_box_fwd / bags_box_bwd argument validation (error codes and messages, before any launch);
  * the box kernels' registers: no spills (ptxas -v).
"""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import box_oracle as BO
from balancedgroupsoftmax_b200 import _native as nat
from oracle import ref_shim

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason='no reference checkout reachable')


def _problem(N=40, K=8, C_=13, beta=1.0, seed=0):
    """float64 x, W, b, labels (0, 1, C - 1 and an out-of-range label among them), targets, weights; rows 0-3 are
    class C - 1, whose W rows and bias are zero, so pred = 0 there and the targets put d exactly at 0, +-beta."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, K, generator=g, dtype=torch.float64)
    W = torch.randn(4 * C_, K, generator=g, dtype=torch.float64) * 0.7
    b = torch.randn(4 * C_, generator=g, dtype=torch.float64) * 0.3
    W[4 * (C_ - 1):] = 0.
    b[4 * (C_ - 1):] = 0.
    labels = torch.randint(0, C_, (N,), generator=g)
    labels[:4] = C_ - 1
    labels[4], labels[5] = 0, 1
    targets = torch.randn(N, 4, generator=g, dtype=torch.float64) * 1.5
    targets[:4] = torch.tensor([[0., beta, -beta, 0.5 * beta]] * 4, dtype=torch.float64)
    weights = (torch.rand(N, 4, generator=g, dtype=torch.float64) > 0.2).double() * 1.5
    return x, W, b, labels, targets, weights


# --------------------------------------------------------------------------- the oracle and the reference
@needs_ref
@pytest.mark.parametrize('beta', [1.0, 1.0 / 9])
def test_oracle_matches_reference_bbox_loss(beta):
    """The reference's BBoxHead.loss (gather + SmoothL1Loss, float64, autograd) on fc_reg(x) gives the oracle's loss
    and gradients -- including |d| exactly at 0 and at beta."""
    x, W, b, labels, targets, weights = _problem(beta=beta)
    xr, Wr, br = (t.clone().requires_grad_(True) for t in (x, W, b))
    pred = xr @ Wr.t() + br
    pred.retain_grad()
    loss = BO.reference_bbox_loss()(pred, labels, targets, weights, beta=beta)
    (loss * 1.75).backward()
    ref = BO.box_terms(x, W, b, labels, targets, weights, beta, float(x.shape[0]), gout=1.75)
    torch.testing.assert_close(ref['loss'], loss.detach(), rtol=1e-13, atol=0)
    rows = (4 * labels).reshape(-1, 1) + torch.arange(4).reshape(1, 4)
    torch.testing.assert_close(ref['g'] * 1.75, pred.grad.gather(1, rows), rtol=1e-13, atol=1e-300)
    torch.testing.assert_close(ref['pred'][labels > 0], pred.detach().gather(1, rows)[labels > 0], rtol=1e-13, atol=0)
    for name, t in (('dW', Wr), ('db', br), ('dX', xr)):
        torch.testing.assert_close(ref[name], t.grad, rtol=1e-12, atol=1e-15, msg=name)
    # the exact cases: d = 0 -> g = 0; |d| = beta -> sign(d) (the |d| - beta / 2 branch)
    g0 = ref['g'][:4] * float(x.shape[0])
    w0 = weights[:4]
    torch.testing.assert_close(g0, w0 * torch.tensor([[0., -1., 1., -0.5]], dtype=torch.float64))


@needs_ref
def test_reference_heads_match_fixture():
    """The fixture is what the reference's GSBBoxHeadWith0 and ReweightBBoxHead return today."""
    import importlib.util
    spec = importlib.util.spec_from_file_location('make_box_golden', os.path.join(os.path.dirname(BO.FIXTURE),
                                                                                    'make_box_golden.py'))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    fix = np.load(BO.FIXTURE)
    inp = BO.fixture_inputs()
    with tempfile.TemporaryDirectory() as d:
        for key, head in mk.reference_heads(d).items():
            _compare(BO.run_box_loss(head, inp, dtype=torch.float64), fix, key)


def _compare(got, fix, key, rtol=2e-6):
    for name in ('loss_bbox', 'dW', 'db', 'dX'):
        a = got[name].double().cpu().numpy().reshape(-1)
        b = np.asarray(fix['%s_%s' % (key, name)], np.float64).reshape(-1)
        np.testing.assert_allclose(a, b, rtol=rtol, atol=rtol * np.abs(b).max(), err_msg='%s %s' % (key, name))


def _our_heads(**execution):
    from balancedgroupsoftmax_b200.head import GSBBoxHeadWith0, ReweightBBoxHead
    from balancedgroupsoftmax_b200.tables import synthetic_tables
    tables = synthetic_tables()
    sizes = dict(num_fcs=2, in_channels=BO.FIX_IN, fc_out_channels=BO.FIX_FC, roi_feat_size=BO.FIX_ROI,
                 num_classes=1231, reg_class_agnostic=False,
                 loss_bbox=dict(type='SmoothL1Loss', beta=1.0, loss_weight=1.0))
    gs = GSBBoxHeadWith0(gs_config=dict(tables=tables, others_sample_ratio=8.0, num_bins=tables.num_bins,
                                        loss_bin=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0),
                                        **execution), **sizes)
    rw = ReweightBBoxHead(reweight_cfg=dict(cls_weights=torch.ones(1231), **execution), **sizes)
    return {'gs': gs, 'reweight': rw}


@pytest.mark.parametrize('key', ['gs', 'reweight'])
def test_our_heads_and_the_oracle_match_fixture(key):
    """On CPU (float64) the heads take the materialised route, even with fuse_bbox_loss set, and reproduce the fixture;
    the oracle's closed form on the same trunk output does too."""
    fix = np.load(BO.FIXTURE)
    inp = BO.fixture_inputs()
    head = _our_heads(fuse_bbox_loss=True)[key]
    _compare(BO.run_box_loss(head, inp, dtype=torch.float64), fix, key)
    with torch.no_grad():
        x_reg = head._trunk(inp['feats'].double())[1]
    ref = BO.box_terms(x_reg, head.fc_reg.weight.detach(), head.fc_reg.bias.detach(), inp['labels'],
                       inp['bbox_targets'], inp['bbox_weights'], 1.0, float(BO.FIX_N))
    np.testing.assert_allclose(ref['loss'].item(), fix['%s_loss_bbox' % key][0], rtol=2e-6)
    np.testing.assert_allclose(ref['dW'][BO.FIX_ROWS].numpy(), fix['%s_dW' % key], rtol=2e-6,
                               atol=2e-6 * np.abs(fix['%s_dW' % key]).max())
    np.testing.assert_allclose(ref['db'].numpy(), fix['%s_db' % key], rtol=2e-6, atol=1e-9)


# --------------------------------------------------------------------------- the head on CPU
def test_forward_returns_a_plain_tensor_on_cpu_or_without_the_key():
    for execution in ({}, {'fuse_bbox_loss': True}):
        for key, head in _our_heads(**execution).items():
            assert head.fuse_bbox_loss is bool(execution), key
            head.train()
            _, bbox_pred = head(torch.randn(8, BO.FIX_IN, BO.FIX_ROI, BO.FIX_ROI))
            assert type(bbox_pred) is torch.Tensor and bbox_pred.shape == (8, 4 * 1231), (key, execution)


def test_box_pred_handle_materialises_like_the_projection():
    from balancedgroupsoftmax_b200.head import BoxPredHandle, ClsScoreHandle
    head = _our_heads(fuse_bbox_loss=True)['reweight']
    x_reg = torch.randn(5, BO.FIX_FC)
    want = head.fc_reg(x_reg)
    h = BoxPredHandle(head, x_reg)
    assert h.shape == (5, 4 * 1231) and h.size(1) == 4 * 1231 and h.dim() == 2 and h.device == x_reg.device
    assert h._pred is None
    torch.testing.assert_close(h[1:3], want[1:3])
    assert h._pred is not None and h.tensor() is h._pred and h.tensor().requires_grad
    torch.testing.assert_close(torch.cat([BoxPredHandle(head, x_reg), want]), torch.cat([want, want]))
    torch.testing.assert_close(BoxPredHandle(head, x_reg).float(), want)
    # the classifier's handle keeps its own behaviour
    c = ClsScoreHandle(head, x_reg)
    assert c.shape == (5, 1231) and c._logits is None
    with pytest.raises(AttributeError):
        c._missing


def test_fused_route_recognises_mean_smooth_l1_only():
    from balancedgroupsoftmax_b200 import losses as L
    head = _our_heads(fuse_bbox_loss=True)['gs']
    assert head._fused_bbox_loss_ok(None) and head._fused_bbox_loss_ok('mean')
    assert not head._fused_bbox_loss_ok('sum') and not head._fused_bbox_loss_ok('none')
    head.loss_bbox = L.SmoothL1Loss(beta=1.0, reduction='sum')
    assert not head._fused_bbox_loss_ok(None)
    head.loss_bbox = torch.nn.L1Loss()
    assert not head._fused_bbox_loss_ok(None)


# --------------------------------------------------------------------------- ABI
def test_box_entry_points_reject_bad_arguments():
    lib = nat.lib()
    buf = (C.c_char * 256)()
    p = (C.addressof(buf) + 15) // 16 * 16
    ws = lib.bags_workspace_bytes()

    def fwd(N=4, K=8, classes=1231, x=p, ldx=8, dtype=nat.DTYPE_BF16, w=p, ldw=8, labels=p, targets=p, weights=p,
            beta=1.0, avg=4.0, loss=p, g=p, pred=None, index=p, wsb=ws):
        return lib.bags_box_fwd(x, ldx, dtype, w, ldw, None, labels, targets, weights, beta, avg, N, K, classes, loss,
                                g, pred, index, p, wsb, None)

    def err():
        return lib.bags_last_error()

    assert fwd(N=-1) == -1 and b'bad shape' in err()
    for kw in ('loss', 'index', 'w', 'x', 'labels', 'targets', 'weights', 'g'):
        assert fwd(**{kw: None}) == -1 and b'NULL' in err(), kw
    assert fwd(dtype=7) == -1 and b'dtype' in err()
    for K in (0, 6):
        assert fwd(K=K, ldx=8, ldw=8) == -1 and b'K=' in err(), K
    for c in (0, 8193):
        assert fwd(classes=c) == -1 and b'classes' in err(), c
    assert fwd(x=p + 4) == -1 and b'x rows' in err()                                 # bf16 needs 8-byte rows
    assert fwd(x=p + 8, dtype=nat.DTYPE_F32) == -1 and b'x rows' in err()           # fp32 needs 16
    assert fwd(ldx=6) == -1 and b'x rows' in err()
    assert fwd(ldx=4) == -1 and b'x rows' in err()                                   # < K
    assert fwd(w=p + 8) == -1 and b'W rows' in err()
    assert fwd(ldw=10) == -1 and b'W rows' in err()
    for bad in (0.0, -1.0, float('inf'), float('nan')):
        assert fwd(beta=bad) == -1 and b'beta' in err(), bad
        assert fwd(avg=bad) == -1 and b'avg' in err(), bad
    assert fwd(targets=p + 4) == -1 and b'16-byte' in err()
    assert fwd(pred=p + 4) == -1 and b'16-byte' in err()
    assert fwd(wsb=16) == -1 and b'workspace' in err()

    def bwd(N=4, K=8, classes=1231, g=p, x=p, ldx=8, dtype=nat.DTYPE_BF16, w=p, ldw=8, labels=p, index=p, dW=p,
            lddw=8, db=p, dX=p, lddx=8):
        return lib.bags_box_bwd(g, None, x, ldx, dtype, w, ldw, labels, index, N, K, classes, dW, lddw, db, dX, lddx,
                                None)

    assert bwd(N=-1) == -1 and b'bad shape' in err()
    for kw in ('index', 'g', 'x', 'w', 'labels'):
        assert bwd(**{kw: None}) == -1 and b'NULL' in err(), kw
    assert bwd(dtype=3) == -1 and b'dtype' in err()
    assert bwd(K=12, ldx=12, ldw=12, lddw=12, lddx=12 + 2) == -1 and b'dX rows' in err()
    assert bwd(lddw=4) == -1 and b'dW rows' in err()
    assert bwd(dW=p + 4) == -1 and b'dW rows' in err()
    assert bwd(dX=p + 4) == -1 and b'dX rows' in err()
    assert bwd(g=p + 4) == -1 and b'g must' in err()
    assert bwd(classes=0) == -1 and b'classes' in err()
    assert bwd(x=p + 4) == -1 and b'x rows' in err()
    assert bwd(w=p + 4) == -1 and b'W rows' in err()


# --------------------------------------------------------------------------- registers
BOX = re.compile(r'bags_box_(fwd|bwd)_kernel')


def test_box_kernels_do_not_spill():
    """ptxas: the four bags_box_* instantiations (forward, backward x bf16, fp32) without spills."""
    from balancedgroupsoftmax_b200 import build as B
    try:
        nvcc = B._nvcc()
    except RuntimeError:
        pytest.skip('nvcc not found')
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-cubin', '-Xptxas', '-v',
               '-o', os.path.join(tmp, 'bags_api.cubin')] + B.SOURCES
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    found, cur = {}, None
    for line in res.stdout.splitlines():
        m = re.search(r'Function properties for (\S+)', line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if m and cur is not None:
            if BOX.search(cur):
                found[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    assert len(found) == 4, found
    assert all(v == (0, 0) for v in found.values()), found
