"""CPU: the LVIS mask heads and their fused mask loss (bags_mask_fwd / bags_mask_bwd on the GPU) without a GPU --

  * the float64 oracle (tests/mask_oracle.py) against the reference's own mask_cross_entropy run in place (skipped where
    no reference checkout is reachable), and the materialised CrossEntropyLoss(use_mask=True) against the same;
  * FCNMaskHead / HTCMaskHead: the config blocks build through the registry; state-dict keys and parameter shapes
    equal the reference heads'; on CPU they reproduce the committed fixture tests/golden/mask_loss_ref_p12.npz;
  * the restated mask_target against the reference's on seeded masks and boxes;
  * MaskPredHandle's lazy mechanics;
  * bags_mask_fwd / bags_mask_bwd argument validation (error codes and messages, before any launch);
  * the mask kernels' registers: no spills (ptxas -v).
"""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import mask_oracle as MO
from balancedgroupsoftmax_b200 import _native as nat
from balancedgroupsoftmax_b200 import mask_head as MH
from oracle import ref_shim

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason='no reference checkout reachable')


def _problem(P=9, Cin=5, H=6, W=7, C_=13, seed=0):
    g = torch.Generator().manual_seed(seed)
    y = torch.randn(P, Cin, H, W, generator=g, dtype=torch.float64)
    Wt = torch.randn(C_, Cin, 1, 1, generator=g, dtype=torch.float64) * 2.0
    b = torch.randn(C_, generator=g, dtype=torch.float64)
    labels = torch.randint(0, C_, (P,), generator=g)
    labels[:4] = torch.tensor([0, C_ - 1, 4, 4])[:P]
    t = (torch.rand(P, H, W, generator=g, dtype=torch.float64) > 0.5).double()
    t[-1] = torch.rand(H, W, generator=g, dtype=torch.float64)
    return y, Wt, b, labels, t


# --------------------------------------------------------------------------- the oracle and the reference
@needs_ref
@pytest.mark.parametrize('P', [1, 9])
def test_oracle_matches_reference_mask_cross_entropy(P):
    """The reference's mask_cross_entropy (float64, autograd) on conv_logits(y) gives the oracle's loss and
    gradients."""
    ref = MO.reference()
    y, Wt, b, labels, t = _problem(P=P)
    yr, Wr, br = (v.clone().requires_grad_(True) for v in (y, Wt, b))
    pred = torch.nn.functional.conv2d(yr, Wr, br)
    loss = ref.mask_cross_entropy(pred, t, labels)
    assert loss.shape == (1,)
    (loss * 1.75).sum().backward()
    o = MO.mask_terms(y, Wt, b, labels, t, gout=1.75)
    torch.testing.assert_close(o['loss'].reshape(1), loss.detach(), rtol=1e-13, atol=0)
    torch.testing.assert_close(o['dW'], Wr.grad.reshape(Wr.shape[0], -1), rtol=1e-12, atol=1e-16)
    torch.testing.assert_close(o['db'], br.grad, rtol=1e-12, atol=1e-16)
    torch.testing.assert_close(o['dY'], yr.grad, rtol=1e-12, atol=1e-16)


@needs_ref
@pytest.mark.parametrize('loss_weight', [1.0, 0.5])
def test_materialised_mask_loss_matches_reference(loss_weight):
    from balancedgroupsoftmax_b200.losses import CrossEntropyLoss
    ref = MO.reference()
    y, Wt, b, labels, t = _problem()
    pred = torch.nn.functional.conv2d(y, Wt, b)
    a = pred.clone().requires_grad_(True)
    r = pred.clone().requires_grad_(True)
    ours = CrossEntropyLoss(use_mask=True, loss_weight=loss_weight)(a, t, labels)
    theirs = ref.CrossEntropyLoss(use_mask=True, loss_weight=loss_weight)(r, t, labels)
    assert ours.shape == theirs.shape == (1,)
    torch.testing.assert_close(ours, theirs, rtol=0, atol=0)
    ours.sum().backward()
    theirs.sum().backward()
    torch.testing.assert_close(a.grad, r.grad, rtol=0, atol=0)


def test_materialised_mask_loss_asserts_like_the_reference():
    from balancedgroupsoftmax_b200.losses import CrossEntropyLoss
    y, Wt, b, labels, t = _problem()
    pred = torch.nn.functional.conv2d(y, Wt, b)
    with pytest.raises(AssertionError):
        CrossEntropyLoss(use_mask=True)(pred, t, labels, reduction_override='sum')
    with pytest.raises(AssertionError):
        CrossEntropyLoss(use_mask=True)(pred, t, labels, avg_factor=3.0)
    o = MO.mask_terms(y, Wt, b, labels, t)
    torch.testing.assert_close(CrossEntropyLoss(use_mask=True)(pred, t, labels)[0], o['loss'], rtol=1e-13, atol=0)


# --------------------------------------------------------------------------- the heads
CONFIG_BLOCKS = {
    # configs/bags/gs_mask_rcnn_r50_fpn_1x_lvis.py:65-72
    'FCNMaskHead': dict(type='FCNMaskHead', num_convs=4, in_channels=256, conv_out_channels=256, num_classes=1231,
                        loss_mask=dict(type='CrossEntropyLoss', use_mask=True, loss_weight=1.0)),
    # configs/bags/gs_htc_x101_64x4d_fpn_20e_16gpu_lvis.py:124-131 (and gs_htc_dconv_c3-c5_*)
    'HTCMaskHead': dict(type='HTCMaskHead', num_convs=4, in_channels=256, conv_out_channels=256, num_classes=1231,
                        loss_mask=dict(type='CrossEntropyLoss', use_mask=True, loss_weight=1.0)),
}


@pytest.mark.parametrize('name', list(CONFIG_BLOCKS))
def test_config_blocks_build_through_the_registry(name):
    from balancedgroupsoftmax_b200.registry import build_head
    head = build_head(dict(CONFIG_BLOCKS[name]))
    assert type(head) is getattr(MH, name)
    head.init_weights()
    assert head.conv_logits.weight.shape == (1231, 256, 1, 1)
    assert type(head.loss_mask).__name__ == 'CrossEntropyLoss' and head.loss_mask.use_mask
    head.eval()
    with torch.no_grad():
        out = head(torch.randn(2, 256, 14, 14))
    pred = out[0] if name == 'HTCMaskHead' else out
    assert type(pred) is torch.Tensor and pred.shape == (2, 1231, 28, 28)


@needs_ref
@pytest.mark.parametrize('name', list(CONFIG_BLOCKS))
@pytest.mark.parametrize('agnostic', [False, True])
def test_state_dict_matches_reference(name, agnostic):
    ref = MO.reference()
    kw = {k: v for k, v in CONFIG_BLOCKS[name].items() if k != 'type'}
    kw['class_agnostic'] = agnostic
    ours = getattr(MH, name)(**kw).state_dict()
    theirs = getattr(ref, name)(**kw).state_dict()
    assert list(ours) == list(theirs)
    assert all(ours[k].shape == theirs[k].shape for k in ours)


def test_conv_module_refuses_norms_and_other_convs():
    with pytest.raises(NotImplementedError):
        MH.ConvModule(4, 4, 3, norm_cfg=dict(type='GN', num_groups=2))
    with pytest.raises(NotImplementedError):
        MH.FCNMaskHead(num_convs=1, in_channels=4, conv_out_channels=4, conv_cfg=dict(type='ConvWS'))


@pytest.mark.parametrize('kind', ['fcn', 'htc'])
def test_our_heads_and_the_oracle_match_fixture(kind):
    """On CPU (float64) the heads take the materialised route and reproduce the fixture; the oracle's closed form on
    the same conv_logits input does too."""
    fix = np.load(MO.FIXTURE)
    inp = MO.fixture_inputs()
    cls = MH.HTCMaskHead if kind == 'htc' else MH.FCNMaskHead
    got = MO.run_mask_loss(cls(**MO.head_kwargs(kind)), inp, kind, dtype=torch.float64)
    for name in ('loss_mask', 'dW', 'db', 'dY'):
        np.testing.assert_allclose(got[name].numpy().reshape(-1), fix['%s_%s' % (kind, name)].reshape(-1), rtol=2e-6,
                                   atol=2e-6 * np.abs(fix['%s_%s' % (kind, name)]).max(), err_msg=name)
    W, b = inp['logits'][kind]
    labels = torch.zeros_like(inp['labels']) if kind == 'htc' else inp['labels']
    o = MO.mask_terms(got['y'], W, b, labels, inp['targets'])
    np.testing.assert_allclose(o['loss'].item(), fix['%s_loss_mask' % kind][0], rtol=2e-6)
    np.testing.assert_allclose(o['dW'][MO.FIX_ROWS].numpy(), fix['%s_dW' % kind], rtol=2e-6,
                               atol=2e-6 * np.abs(fix['%s_dW' % kind]).max())
    np.testing.assert_allclose(o['dY'].numpy(), fix['%s_dY' % kind], rtol=2e-6, atol=2e-6 * np.abs(fix['%s_dY' % kind]).max())


@needs_ref
def test_reference_heads_match_fixture():
    import importlib.util
    spec = importlib.util.spec_from_file_location('make_mask_golden', os.path.join(os.path.dirname(MO.FIXTURE),
                                                                                     'make_mask_golden.py'))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    fix = np.load(MO.FIXTURE)
    inp = MO.fixture_inputs()
    for kind, head in mk.reference_heads().items():
        got = MO.run_mask_loss(head, inp, kind, dtype=torch.float64)
        for name in ('loss_mask', 'dW', 'db', 'dY'):
            np.testing.assert_allclose(got[name].numpy().reshape(-1), fix['%s_%s' % (kind, name)].reshape(-1),
                                       rtol=2e-6, atol=2e-6 * np.abs(fix['%s_%s' % (kind, name)]).max())


def test_forward_returns_a_plain_tensor_on_cpu_and_in_eval():
    for cls in (MH.FCNMaskHead, MH.HTCMaskHead):
        head = cls(num_convs=1, in_channels=4, conv_out_channels=4, num_classes=11)
        for train in (True, False):
            head.train(train)
            out = head(torch.randn(3, 4, 7, 7))
            pred = out[0] if cls is MH.HTCMaskHead else out
            assert type(pred) is torch.Tensor and pred.shape == (3, 11, 14, 14)


def test_mask_pred_handle_materialises_like_the_conv():
    head = MH.FCNMaskHead(num_convs=1, in_channels=4, conv_out_channels=4, num_classes=11)
    y = torch.randn(3, 4, 14, 14)
    want = head.conv_logits(y)
    h = MH.MaskPredHandle(head, y)
    assert h.shape == (3, 11, 14, 14) and h.size(1) == 11 and h.dim() == 4 and h.device == y.device
    assert h._pred is None
    torch.testing.assert_close(h[1:3], want[1:3])
    assert h._pred is not None and h.tensor() is h._pred and h.tensor().requires_grad
    torch.testing.assert_close(torch.cat([MH.MaskPredHandle(head, y), want]), torch.cat([want, want]))
    torch.testing.assert_close(MH.MaskPredHandle(head, y).float(), want)


def test_fused_route_recognises_mean_mask_cross_entropy_only():
    from balancedgroupsoftmax_b200 import losses as L
    head = MH.FCNMaskHead(num_convs=1, in_channels=4, conv_out_channels=4, num_classes=11)
    assert head._fused_loss_ok()
    head.loss_mask = L.CrossEntropyLoss(use_mask=True, reduction='sum')
    assert not head._fused_loss_ok()
    head.loss_mask = L.CrossEntropyLoss(use_sigmoid=True)
    assert not head._fused_loss_ok()
    head.loss_mask = torch.nn.BCEWithLogitsLoss()
    assert not head._fused_loss_ok()


def _seg_inputs(num_classes, n=9, seed=0, channels=None):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(n, channels or num_classes, 14, 14, generator=g) * 3
    # inside a 56 x 70 image, and inside 80 x 100 after division by 0.7
    x1 = torch.rand(n, generator=g) * 30
    y1 = torch.rand(n, generator=g) * 20
    boxes = torch.stack([x1, y1, x1 + torch.rand(n, generator=g) * 20, y1 + torch.rand(n, generator=g) * 15,
                         torch.rand(n, generator=g)], 1)
    labels = torch.randint(0, num_classes - 1, (n,), generator=g)
    return logits, boxes, labels


def _fake_encode(arr):
    """Stands in for pycocotools.mask.encode: a lossless record of the [H, W, 1] Fortran-ordered uint8 array."""
    assert arr.dtype == np.uint8 and arr.ndim == 3 and arr.flags.f_contiguous
    return [{'size': list(arr.shape[:2]), 'counts': arr.tobytes(order='F')}]


def test_seg_masks_name_the_missing_dependency(monkeypatch):
    import sys
    monkeypatch.setitem(sys.modules, 'pycocotools', None)
    monkeypatch.setitem(sys.modules, 'pycocotools.mask', None)
    head = MH.FCNMaskHead(num_convs=1, in_channels=4, conv_out_channels=4, num_classes=11)
    logits, boxes, labels = _seg_inputs(11, n=2)
    for fn in (head.get_seg_masks, head.get_seg_masks_without):
        with pytest.raises(ImportError, match='pycocotools'):
            fn(logits, boxes, labels, dict(mask_thr_binary=0.5), (80, 100, 3), 1.0, True)


@needs_ref
@pytest.mark.parametrize('agnostic', [False, True])
@pytest.mark.parametrize('rescale', [True, False])
def test_seg_masks_match_reference_with_the_drop_in_registered(monkeypatch, agnostic, rescale):
    """With this package's heads registered under the reference's names (the documented drop-in) and the reference's
    fcn_mask_head module no longer importable, get_seg_masks / get_seg_masks_without run and give the reference
    methods' output."""
    import sys
    pytest.importorskip('cv2')
    ref = MO.reference()
    heads = sys.modules['mmdet.models.registry'].HEADS
    monkeypatch.setitem(heads._module_dict, 'FCNMaskHead', MH.FCNMaskHead)
    monkeypatch.setitem(heads._module_dict, 'HTCMaskHead', MH.HTCMaskHead)
    monkeypatch.setattr(sys.modules['pycocotools.mask'], 'encode', _fake_encode, raising=False)
    kw = dict(num_convs=1, in_channels=4, conv_out_channels=4, num_classes=11, class_agnostic=agnostic)
    theirs = ref.FCNMaskHead(**kw)
    logits, boxes, labels = _seg_inputs(11, channels=1 if agnostic else 11)
    cfg = ref_shim.AttrDict(mask_thr_binary=0.5)
    args = (boxes, labels, cfg, (80, 100, 3), 0.7, rescale)
    want = [theirs.get_seg_masks(logits, *args), theirs.get_seg_masks_without(logits, *args),
            theirs.get_seg_masks(torch.sigmoid(logits).numpy().astype(np.float16), *args)]
    monkeypatch.setitem(sys.modules, 'mmdet.models.mask_heads.fcn_mask_head', None)
    ours = MH.FCNMaskHead(**kw)
    got = [ours.get_seg_masks(logits, *args), ours.get_seg_masks_without(logits, *args),
           ours.get_seg_masks(torch.sigmoid(logits).numpy().astype(np.float16), *args)]
    assert got == want
    assert sum(len(v) for v in got[0]) == len(labels)


# --------------------------------------------------------------------------- mask targets
def _target_inputs(seed, num_pos=17, num_gt=5, shape=(61, 83)):
    g = torch.Generator().manual_seed(seed)
    gt_masks = (torch.rand(num_gt, *shape, generator=g) > 0.6).numpy().astype(np.uint8)
    x1 = torch.rand(num_pos, generator=g) * (shape[1] - 2)
    y1 = torch.rand(num_pos, generator=g) * (shape[0] - 2)
    x2 = x1 + torch.rand(num_pos, generator=g) * (shape[1] - x1)
    y2 = y1 + torch.rand(num_pos, generator=g) * (shape[0] - y1)
    boxes = torch.stack([x1, y1, x2, y2], 1)
    boxes[0] = torch.tensor([3., 4., 3.4, 4.2])           # a box narrower than one pixel
    inds = torch.randint(0, num_gt, (num_pos,), generator=g)
    return boxes, inds, gt_masks


@needs_ref
@pytest.mark.parametrize('mask_size', [28, 14])
def test_restated_mask_target_matches_reference(mask_size):
    pytest.importorskip('cv2')
    ref = MO.reference()
    cfg = ref_shim.AttrDict(mask_size=mask_size)
    imgs = [_target_inputs(s) for s in (0, 1, 2)]
    imgs.append((torch.zeros(0, 4), torch.zeros(0, dtype=torch.long), imgs[0][2]))      # an image without positives
    props, inds, masks = zip(*imgs)
    want = ref.mask_target(list(props), list(inds), list(masks), cfg)
    got = MH.mask_target(list(props), list(inds), list(masks), cfg)
    assert got.dtype == want.dtype == torch.float32 and got.shape == want.shape == (51, mask_size, mask_size)
    assert torch.equal(got, want)
    assert 0 < float(got.mean()) < 1


# --------------------------------------------------------------------------- ABI
def test_mask_entry_points_reject_bad_arguments():
    lib = nat.lib()
    buf = (C.c_char * 256)()
    p = (C.addressof(buf) + 15) // 16 * 16
    ws = lib.bags_workspace_bytes()

    def fwd(P=4, Cin=8, HW=784, classes=1231, y=p, dtype=nat.DTYPE_BF16, w=p, ldw=8, labels=p, targets=p, loss=p, g=p,
            rsum=p, rsum_floats=4 * 13 * 10, index=p, wsb=ws):
        return lib.bags_mask_fwd(y, dtype, w, ldw, None, labels, targets, P, Cin, HW, classes, loss, g, rsum,
                                 rsum_floats, index, p, wsb, None)

    def err():
        return lib.bags_last_error()

    for kw in (dict(P=-1), dict(Cin=0), dict(HW=0)):
        assert fwd(**kw) == -1 and b'bad shape' in err(), kw
    for kw in ('loss', 'index', 'y', 'w', 'labels', 'targets', 'g', 'rsum'):
        assert fwd(**{kw: None}) == -1 and b'NULL' in err(), kw
    assert fwd(dtype=7) == -1 and b'dtype' in err()
    for c in (0, 8193):
        assert fwd(classes=c) == -1 and b'classes' in err(), c
    assert fwd(ldw=7) == -1 and b'ldw' in err()
    assert fwd(rsum_floats=4 * 13 * 10 - 1) == -1 and b'rsum too small' in err()
    assert fwd(HW=833) == -1 and b'rsum too small' in err()      # one more tile
    assert fwd(wsb=16) == -1 and b'workspace' in err()

    def bwd(P=4, Cin=8, HW=784, classes=1231, g=p, rsum=p, dtype=nat.DTYPE_F32, w=p, ldw=8, labels=p, index=p, dW=p,
            lddw=8, db=p, dY=p):
        return lib.bags_mask_bwd(g, rsum, None, dtype, w, ldw, labels, index, P, Cin, HW, classes, dW, lddw, db, dY,
                                 None)

    assert bwd(P=-1) == -1 and b'bad shape' in err()
    assert bwd(Cin=0) == -1 and b'bad shape' in err()
    for kw in ('index', 'rsum', 'g', 'w', 'labels'):
        assert bwd(**{kw: None}) == -1 and b'NULL' in err(), kw
    assert bwd(dtype=3) == -1 and b'dtype' in err()
    assert bwd(classes=0) == -1 and b'classes' in err()
    assert bwd(ldw=4) == -1 and b'ldw' in err()
    assert bwd(lddw=4) == -1 and b'lddw' in err()


# --------------------------------------------------------------------------- registers
MASK = re.compile(r'bags_mask_(fwd|bwd|sort)_kernel')


def test_mask_kernels_do_not_spill():
    """ptxas: the nine bags_mask_* kernels (class sort; forward and backward x bf16, fp32 x vector width 1, 4) without
    spills."""
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
            if MASK.search(cur):
                found[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    assert len(found) == 9, found
    assert all(v == (0, 0) for v in found.values()), found
