"""The mask heads' test-time logits computed for each detection's channel only -- bags_mask_logits,
ops.mask_channel_logits and the eval MaskPredHandle -- against float64 and against the dense conv_logits route.

Every reference is plain torch (float64 for the kernel, the head's own conv_logits for the routes), never this
library.  Inputs come from mask_oracle.tier_inputs:
  * exact: small-integer y and W, b a multiple of 2^-3, every partial sum below 2^20 (asserted), so the logits are
    exact in fp32 in any summation order: the kernel equals float64 rounded once to y's dtype, bit for bit, and y one
    element off a 16-byte boundary (one pixel a thread although H W % 4 == 0) gives the same bits as the aligned call.
  * numeric: y = relu(normal), W and b normal.  z = b[c] + sum_k W[c,k] y[k,q] is formed by mask_logit: NG channel
    groups each run an fma chain over their ceil(Cin / NG) channels, the NG group sums are added in order, then the
    bias.  A product passes through at most ceil(Cin / NG) + min(Cin, NG) - 1 <= Cin roundings (adding a group sum of
    zero is exact) and the bias through one, each
    of relative size u = 2^-24 of a partial sum bounded by S = sum_k |W y| + |b|; so |fp32 z - z| <= gamma_{Cin+1} S
    with gamma_m = m u / (1 - m u) (Higham, Accuracy and Stability of Numerical Algorithms, 3.1).  A bf16 output adds
    its own rounding, at most 2^-8 |fp32 z| (8 significant bits).  y is given to float64 already in its operand dtype, so y's rounding to
    bf16 is no error of the kernel.
W's padding columns [Cin, ldw) and the elements of y's buffer past y hold NaN: a read of them would turn a valid map
into NaN.  The elements past ``out`` hold a sentinel that must survive.  A channel outside [0, classes) gives a map of
NaN (the dense route's torch.gather would raise a device-side assert there).
"""
import ctypes as C
import sys
import types

import numpy as np
import pytest
import torch

import mask_oracle as MO
import segm_oracle as SO
from balancedgroupsoftmax_b200 import _native as nat
from balancedgroupsoftmax_b200 import mask_head as MH

DEV = torch.device('cuda', 0)
BF, F32 = torch.bfloat16, torch.float32
SENT = -7.0
NAN = float('nan')
PAD = 64
U = 2.0 ** -24
CLASSES = 1231
CFG = dict(mask_thr_binary=0.5)


def _bits(x):
    x = x.contiguous().cpu()
    return x.view(torch.int32) if x.dtype == F32 else x.view(torch.int16) if x.dtype == BF else x


def _same_bits(got, want, what):
    a, b = _bits(got), _bits(want)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    bad = (a != b).reshape(-1)
    if bad.any():
        i = int(bad.nonzero()[0])
        raise AssertionError('%s: %d of %d elements differ; first at flat %d: got %r, want %r' % (
            what, int(bad.sum()), bad.numel(), i, got.reshape(-1)[i].item(), want.reshape(-1)[i].item()))


# ------------------------------------------------------------------------------------------------ the kernel
def _launch(y, W, b, channels, classes, ldw=None, offset=0):
    """bags_mask_logits on the current stream through ctypes; y at ``offset`` elements from an aligned buffer whose
    other elements are NaN, W padded with NaN to ``ldw`` columns.  Returns (out [n, HW], the sentinel tail)."""
    lib = nat.lib()
    n, Cin, HW = y.shape
    ldw = ldw or Cin
    dtype = y.dtype
    Wp = torch.full((classes, ldw), NAN, device=DEV)
    Wp[:, :Cin] = W.to(DEV)
    numel = n * Cin * HW
    yb = torch.full((numel + offset + PAD,), NAN, dtype=dtype, device=DEV)
    yb[offset:offset + numel] = y.reshape(-1).to(DEV)
    bd = None if b is None else b.to(DEV)
    ch = channels.to(DEV).contiguous()
    out = torch.full((n * HW + PAD,), SENT, dtype=dtype, device=DEV)
    code = nat.DTYPE_BF16 if dtype == BF else nat.DTYPE_F32
    nat.check(lib.bags_mask_logits(yb[offset:].data_ptr(), code, Wp.data_ptr(), ldw, nat.ptr(bd), ch.data_ptr(), n,
                                   Cin, HW, classes, out.data_ptr(), torch.cuda.current_stream(DEV).cuda_stream),
              'bags_mask_logits')
    torch.cuda.synchronize()
    return out[:n * HW].reshape(n, HW).cpu(), out[n * HW:].cpu()


def _reference(y, W, b, channels, classes):
    """(z float64 [n, HW] with NaN rows for invalid channels, S = sum_k |W y| + |b|, valid [n]) on the CPU, computed
    in float64 on the GPU."""
    n, Cin, HW = y.shape
    yd = y.to(DEV).double()
    valid = (channels >= 0) & (channels < classes)
    c = torch.where(valid, channels, torch.zeros_like(channels)).to(DEV)
    Wc = W.to(DEV).double()[c]
    bc = torch.zeros(n, dtype=torch.float64, device=DEV) if b is None else b.to(DEV).double()[c]
    z = torch.einsum('nk,nkq->nq', Wc, yd) + bc[:, None]
    S = torch.einsum('nk,nkq->nq', Wc.abs(), yd.abs()) + bc.abs()[:, None]
    z[~valid.to(DEV)] = NAN
    return z.cpu(), S.cpu(), valid


def _channels(n, classes, invalid, seed):
    """n channels: 0 and classes - 1 first, then -1, classes and 2^40 when ``invalid``, then random valid ones."""
    g = torch.Generator().manual_seed(seed)
    head = [0, classes - 1] + ([-1, classes, 2 ** 40] if invalid else [])
    ch = torch.randint(0, classes, (n,), generator=g)
    k = min(n, len(head))
    ch[:k] = torch.tensor(head[:k])
    return ch


def _case(n, HW, Cin, classes, dtype, tier, invalid=True, bias=True, pad=3, seed=0):
    y, W, b, _, _ = MO.tier_inputs(tier, n, Cin, HW, classes, dtype=dtype, seed=seed)
    channels = _channels(n, classes, invalid, seed)
    if tier == 'exact':
        vy, vW, vb = y.double(), W.double(), b.double()
        ok = (channels >= 0) & (channels < classes)
        lab = torch.where(ok, channels, torch.full_like(channels, -1))
        assert MO.exact_partial_max(vy, vW, vb if bias else None, lab) < MO.EXACT_LIMIT
    return y, W, (b if bias else None), channels, dict(ldw=Cin + pad)


def _check(got, tail, y, W, b, channels, classes, tier, what):
    assert bool((tail == SENT).all()), '%s: a sentinel past out was overwritten' % what
    z, S, valid = _reference(y, W, b, channels, classes)
    if (~valid).any():
        assert bool(torch.isnan(got[~valid].float()).all()), '%s: an invalid channel is not an all-NaN map' % what
    got, z, S = got[valid], z[valid], S[valid]
    if tier == 'exact':
        _same_bits(got, z.to(got.dtype), what)
        return
    m = y.shape[1] + 1
    bound = m * U / (1 - m * U) * S
    if got.dtype == BF:
        bound = bound + 2.0 ** -8 * (z.abs() + bound)
    err = (got.double() - z).abs()
    bad = ~(err <= bound)
    assert not bad.any(), '%s: %d elements outside the bound, worst err %g bound %g' % (
        what, int(bad.sum()), err[bad].max().item(), bound[bad].max().item())


GRID = [(HW, Cin, classes) for HW in (784, 64, 49, 4) for Cin, classes in ((256, CLASSES), (5, 1))]


@pytest.mark.gpu
@pytest.mark.parametrize('tier', ['exact', 'numeric'])
@pytest.mark.parametrize('dtype', [BF, F32], ids=['bf16', 'fp32'])
@pytest.mark.parametrize('shape', GRID, ids=['HW%d-Cin%d-C%d' % s for s in GRID])
def test_kernel_vs_float64(shape, dtype, tier):
    """n = 3 and 7 (0, classes - 1, then -1, classes and 2^40, then a valid one), W padded to ldw = Cin + 3, with
    and without a bias; n = 1."""
    HW, Cin, classes = shape
    for n, bias in ((3, True), (7, False), (1, True)):
        y, W, b, ch, kw = _case(n, HW, Cin, classes, dtype, tier, bias=bias, seed=n + HW)
        got, tail = _launch(y, W, b, ch, classes, **kw)
        _check(got, tail, y, W, b, ch, classes, tier, 'n=%d HW=%d Cin=%d classes=%d' % (n, HW, Cin, classes))


@pytest.mark.gpu
@pytest.mark.parametrize('tier', ['exact', 'numeric'])
@pytest.mark.parametrize('dtype', [BF, F32], ids=['bf16', 'fp32'])
def test_kernel_at_the_test_time_shape(dtype, tier):
    """n = 300 detections, 256 channels, 1231 classes, 28 x 28 pixels (12 full tiles and a tail of 16), ldw = Cin."""
    y, W, b, ch, _ = _case(300, 784, 256, CLASSES, dtype, tier, seed=300)
    got, tail = _launch(y, W, b, ch, CLASSES)
    _check(got, tail, y, W, b, ch, CLASSES, tier, 'n=300')


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [BF, F32], ids=['bf16', 'fp32'])
@pytest.mark.parametrize('HW', [784, 64, 4])
def test_misaligned_y_gives_the_aligned_bits(dtype, HW):
    """y one element off a 16-byte boundary takes one pixel a thread; in the exact tier its bits equal the aligned
    call's (four pixels a thread) and float64's."""
    y, W, b, ch, kw = _case(5, HW, 256, CLASSES, dtype, 'exact', seed=HW)
    aligned, _ = _launch(y, W, b, ch, CLASSES, **kw)
    off, tail = _launch(y, W, b, ch, CLASSES, offset=1, **kw)
    _check(off, tail, y, W, b, ch, CLASSES, 'exact', 'offset 1')
    _same_bits(off, aligned, 'offset 1 against aligned')


@pytest.mark.gpu
def test_no_detections_launches_nothing():
    y, W, b, ch, kw = _case(0, 784, 256, CLASSES, F32, 'numeric')
    got, tail = _launch(y, W, b, ch, CLASSES, **kw)
    assert got.shape == (0, 784) and bool((tail == SENT).all())
    from balancedgroupsoftmax_b200 import ops
    out = ops.mask_channel_logits(torch.zeros(0, 256, 28, 28, device=DEV), W.to(DEV), b.to(DEV),
                                  torch.zeros(0, dtype=torch.int64, device=DEV))
    assert out.shape == (0, 1, 28, 28)


def test_abi_rejects_bad_arguments():
    """NULL operands, a dtype other than bf16 / fp32, ldw < Cin and negative sizes: error codes and messages, reported
    before anything touches a device; n = 0 returns 0 without a launch."""
    lib = nat.lib()
    buf = (C.c_char * 256)()
    p = (C.addressof(buf) + 15) // 16 * 16

    def call(y=p, dtype=nat.DTYPE_F32, w=p, ldw=8, bias=None, ch=p, n=2, Cin=8, HW=16, classes=4, out=p):
        return lib.bags_mask_logits(y, dtype, w, ldw, bias, ch, n, Cin, HW, classes, out, None)

    for kw in (dict(y=None), dict(w=None), dict(ch=None), dict(out=None)):
        assert call(**kw) == -1 and b'NULL' in lib.bags_last_error(), kw
    for dt in (2, 7, -1):
        assert call(dtype=dt) == -1 and b'dtype' in lib.bags_last_error()
    assert call(ldw=7) == -1 and b'ldw' in lib.bags_last_error()
    for kw in (dict(n=-1), dict(Cin=-3, ldw=8), dict(Cin=0), dict(HW=-16), dict(HW=0)):
        assert call(**kw) == -1 and b'bad shape' in lib.bags_last_error(), kw
    assert call(classes=0) == -1 and b'classes' in lib.bags_last_error()
    assert call(n=0) == 0 and call(n=0, y=None, w=None, ch=None, out=None) == 0


# ------------------------------------------------------------------------------------------------ the head routes
@pytest.fixture
def host_encoder(monkeypatch):
    """pycocotools.mask.encode for the host loop: the real one if installed, else the oracle's."""
    if SO.installed_pycocotools_mask(monkeypatch) is None:
        mod = types.ModuleType('pycocotools.mask')
        mod.encode = SO.encode
        pkg = types.ModuleType('pycocotools')
        pkg.mask = mod
        monkeypatch.setitem(sys.modules, 'pycocotools', pkg)
        monkeypatch.setitem(sys.modules, 'pycocotools.mask', mod)
    monkeypatch.setenv('BAGS_SEGM_NATIVE', '1')


@pytest.fixture
def no_tf32():
    """cuDNN's fp32 conv without TF32, so that the dense route's exact-tier logits are exact too."""
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32 = old


def _detections(n, img_h, img_w, seed, outside=False):
    """det_bboxes [n, 5] inside an img_h x img_w canvas (one leaving it on the right with ``outside``), det_labels
    [n] in [0, CLASSES - 1), on cuda:0."""
    rng = np.random.default_rng(seed)
    w = rng.integers(1, img_w // 2, n)
    h = rng.integers(1, img_h // 2, n)
    x0 = rng.integers(0, img_w - w + 1)
    y0 = rng.integers(0, img_h - h + 1)
    xyxy = np.stack([x0, y0, x0 + w - 1, y0 + h - 1], 1).astype(np.float64) + 0.25
    if outside:
        xyxy[n // 2, 2] = img_w + 6.25
    det = np.concatenate([xyxy, rng.random((n, 1))], 1).astype(np.float32)
    labels = torch.from_numpy(rng.integers(0, CLASSES - 1, n)).long()
    return torch.from_numpy(det).to(DEV), labels.to(DEV)


def _exact_head(cls, Cin, seed, **kw):
    """A head whose conv_logits reads its input directly (no convs, no upsampling), with exact-tier conv_logits
    parameters (and an integer conv_res for HTC), in eval mode on cuda:0."""
    head = cls(num_convs=0, upsample_method=None, in_channels=Cin, conv_out_channels=Cin, num_classes=CLASSES, **kw)
    _, W, b, _, _ = MO.tier_inputs('exact', 1, Cin, 1, head.conv_logits.out_channels, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        head.conv_logits.weight.copy_(W.reshape(head.conv_logits.weight.shape))
        head.conv_logits.bias.copy_(b)
        if cls is MH.HTCMaskHead:
            head.conv_res.conv.weight.copy_(torch.randint(-1, 2, head.conv_res.conv.weight.shape, generator=g).float())
            head.conv_res.conv.bias.zero_()
    return head.to(DEV).eval()


def _exact_feats(n, Cin, seed):
    y, _, _, _, _ = MO.tier_inputs('exact', n, Cin, 28 * 28, 1, seed=seed)
    return y.reshape(n, Cin, 28, 28).to(DEV)


def _outcome(fn, *args):
    """fn(*args), or the type and message of what it raised (both routes must fail alike)."""
    try:
        return fn(*args)
    except Exception as e:  # noqa: BLE001
        return type(e), str(e)


@pytest.mark.gpu
@pytest.mark.parametrize('agnostic', [False, True], ids=['class_specific', 'class_agnostic'])
@pytest.mark.parametrize('route', ['native', 'host_loop', 'box_outside'])
def test_seg_masks_on_an_eval_handle_equal_the_dense_route(host_encoder, no_tf32, monkeypatch, agnostic, route):
    """The native route, the host loop (BAGS_SEGM_NATIVE=0) and a box that leaves the image (the host loop, whose
    numpy paste raises there on both routes alike)."""
    img_h, img_w = 480, 640
    if route == 'host_loop':
        monkeypatch.setenv('BAGS_SEGM_NATIVE', '0')
    head = _exact_head(MH.FCNMaskHead, 16, seed=3, class_agnostic=agnostic)
    x = _exact_feats(37, 16, seed=4)
    det, labels = _detections(37, img_h, img_w, seed=5, outside=route == 'box_outside')
    with torch.no_grad():
        pred = head(x)
        assert isinstance(pred, MH.MaskPredHandle) and pred.label_only()
        dense = head.conv_logits(pred.input)
        for fn in (head.get_seg_masks, head.get_seg_masks_without):
            for rescale in (True, False):
                args = (det, labels, CFG, (img_h, img_w, 3), 1.0, rescale)
                got = _outcome(fn, pred, *args)
                want = _outcome(fn, dense, *args)
                assert isinstance(want, list) == (route != 'box_outside')
                assert got == want, (fn.__name__, rescale)
                assert pred.pending
    # the label-only logits themselves: bit-identical to the dense channel
    ch = (labels + 1) if not agnostic else torch.zeros_like(labels)
    _same_bits(pred.channel_logits(ch), dense[torch.arange(37, device=DEV), ch][:, None], 'channel logits')


def _htc_heads(Cin):
    return [_exact_head(MH.HTCMaskHead, Cin, seed=10 + i) for i in range(3)]


@pytest.mark.gpu
def test_htc_sequence_gathers_equal_the_dense_gather(host_encoder, no_tf32):
    """htc.py:403-421 with mask_info_flow: each stage's gather of its label channels, bit for bit, then the merge
    (np.mean of the sigmoids) and get_seg_masks_without."""
    img_h, img_w = 480, 640
    heads = _htc_heads(16)
    x = _exact_feats(29, 16, seed=6)
    det, det_labels = _detections(29, img_h, img_w, seed=7)
    labels = (det_labels.unsqueeze(1) + 1).unsqueeze(2).unsqueeze(3).expand(-1, -1, 28, 28)
    aug, aug_dense = [], []
    last_feat = None
    with torch.no_grad():
        for head in heads:
            pred, last_feat = head(x, last_feat)
            assert isinstance(pred, MH.MaskPredHandle)
            dense = head.conv_logits(pred.input).gather(1, labels)
            g1 = pred.gather(1, labels)
            g2 = torch.gather(pred, 1, labels)
            g3 = torch.gather(pred, dim=1, index=labels)
            assert pred.pending
            for g in (g1, g2, g3):
                _same_bits(g, dense, 'gather')
            aug.append(g1.sigmoid().cpu().numpy())
            aug_dense.append(dense.sigmoid().cpu().numpy())
        merged, merged_dense = np.mean(aug, axis=0), np.mean(aug_dense, axis=0)
        assert np.array_equal(merged, merged_dense)
        args = (det, det_labels, CFG, (img_h, img_w, 3), 1.0, True)
        assert heads[-1].get_seg_masks_without(merged, *args) == heads[-1].get_seg_masks_without(merged_dense, *args)
    # a later dense use still materialises (multi-scale testing's mask_pred.sigmoid())
    torch.testing.assert_close(pred.sigmoid(), heads[-1].conv_logits(pred.input).sigmoid(), rtol=0, atol=0)
    assert not pred.pending


@pytest.mark.gpu
def test_fallbacks_materialise_and_equal_the_dense_results(host_encoder, no_tf32):
    img_h, img_w = 480, 640
    head = _exact_head(MH.FCNMaskHead, 16, seed=8)
    x = _exact_feats(11, 16, seed=9)
    det, det_labels = _detections(11, img_h, img_w, seed=10)
    args = (det, det_labels, CFG, (img_h, img_w, 3), 1.0, True)
    with torch.no_grad():
        want = head.get_seg_masks(head.conv_logits(x), *args)
    # an eval forward with autograd on and parameters that require grad: the dense, autograd-connected logits
    with torch.enable_grad():
        pred = head(x)
        assert isinstance(pred, MH.MaskPredHandle) and not pred.label_only()
        assert head.get_seg_masks(pred, *args) == want
        assert not pred.pending and pred.tensor().requires_grad
        labels = (det_labels + 1)[:, None, None, None].expand(-1, -1, 28, 28)
        g = MH.MaskPredHandle(head, x).gather(1, labels)
        assert g.requires_grad
        _same_bits(g.detach(), head.conv_logits(x).detach().gather(1, labels), 'gather with autograd')
    with torch.no_grad():
        dense = head.conv_logits(x)
        # an index that is not constant along H and W
        varying = labels.clone()
        varying[:, :, 3, 5] = 7
        pred = head(x)
        _same_bits(pred.gather(1, varying), dense.gather(1, varying), 'varying index')
        assert not pred.pending
        # dim != 1
        rows = torch.randint(0, 28, (11, 1, 28, 28), device=DEV)
        pred = head(x)
        _same_bits(torch.gather(pred, 2, rows), dense.gather(2, rows), 'dim 2')
        assert not pred.pending


@pytest.mark.gpu
def test_label_only_routes_never_allocate_the_logits():
    """n = 300, 1231 classes, 256 channels, 28 x 28: after y exists, get_seg_masks on an eval handle and the HTC
    gather each add less than 64 MB to the peak; the dense conv_logits adds at least its [n, 1231, 28, 28] fp32
    output (1.16 GB)."""
    n, Cin = 300, 256
    head = MH.FCNMaskHead(num_convs=0, upsample_method=None, in_channels=Cin, num_classes=CLASSES).to(DEV).eval()
    img_h, img_w = 800, 1333
    det, det_labels = _detections(n, img_h, img_w, seed=11)
    labels = (det_labels + 1)[:, None, None, None].expand(-1, -1, 28, 28)
    args = (det, det_labels, CFG, (img_h, img_w, 3), 1.0, True)
    with torch.no_grad():
        y = torch.relu(torch.randn(n, Cin, 28, 28, device=DEV))
        pred = head(y)
        head.get_seg_masks(pred, *args)         # warm-up

        def peak(fn):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            fn()
            torch.cuda.synchronize()
            return torch.cuda.max_memory_allocated() - base

        assert peak(lambda: head.get_seg_masks(pred, *args)) < 64 << 20
        assert peak(lambda: pred.gather(1, labels)) < 64 << 20
        assert pred.pending
        assert peak(lambda: head.conv_logits(y)) >= n * CLASSES * 28 * 28 * 4
