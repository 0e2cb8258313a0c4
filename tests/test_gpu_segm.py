"""GPU: FCNMaskHead.get_seg_masks / get_seg_masks_without on the native route (bags_segm_rle) against the host loop
(cv2 resize, numpy paste, COCO RLE), which is the reference's own code path.  The host loop's encoder is
pycocotools.mask.encode, or tests/segm_oracle.py's restatement of it where pycocotools is not installed.

The masks must be identical: the kernel restates OpenCV's float32 INTER_LINEAR arithmetic operation by operation (see
test_segm_cpu.py for the restatement against cv2.resize itself).  Also: three host syncs per call whatever n is.
"""
import sys
import types
import warnings

import numpy as np
import pytest
import torch

import segm_oracle as SO
from balancedgroupsoftmax_b200 import mask_head as MH

pytestmark = pytest.mark.gpu
CLASSES = 1231
CFG = dict(mask_thr_binary=0.5)


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


def _special_boxes(img_h, img_w):
    """(left, top, w, h) boxes on the canvas: edges, one pixel, the 14 x 14 and 28 x 28 sizes, large boxes."""
    out = [(0, 0, 30, 20), (img_w - 25, 0, 25, 40), (0, img_h - 17, 33, 17), (img_w - 9, img_h - 11, 9, 11),
           (0, 0, img_w, img_h), (0, 5, 7, img_h - 5), (10, 0, 40, img_h), (3, 4, 1, 1), (img_w - 1, img_h - 1, 1, 1),
           (100, 50, 14, 14), (200, 80, 28, 28), (0, 0, 28, 28), (50, 60, 1, 30), (70, 90, 45, 1)]
    if img_w >= 700:
        out += [(img_w - 650, 100, 650, 600), (30, img_h - 700, 640, 700)]
    else:
        out += [(20, 10, min(600, img_w - 20), min(400, img_h - 10))]
    return out


def _inputs(n, img_h, img_w, dtype, seed, scale=1.0, outside=False):
    """det_bboxes [n, 5] (scaled by ``scale``), det_labels [n], logits [n, CLASSES, 28, 28] on cuda:0."""
    g = torch.Generator().manual_seed(seed)
    rng = np.random.default_rng(seed)
    special = _special_boxes(img_h, img_w)
    boxes = []
    for k in range(n):
        if k < len(special):
            boxes.append(special[k])
            continue
        w, h = int(rng.integers(1, min(img_w, 500))), int(rng.integers(1, min(img_h, 500)))
        boxes.append((int(rng.integers(0, img_w - w + 1)), int(rng.integers(0, img_h - h + 1)), w, h))
    b = np.array(boxes, dtype=np.float64).reshape(-1, 4)
    xyxy = np.stack([b[:, 0], b[:, 1], b[:, 0] + b[:, 2] - 1, b[:, 1] + b[:, 3] - 1], 1) + 0.25
    if outside and n:
        xyxy[n // 2, 2] = img_w + 6.25                  # leaves the canvas on the right
    det = np.concatenate([xyxy * scale, rng.random((n, 1))], 1).astype(np.float32)
    dev = torch.device('cuda', 0)
    labels = torch.randint(0, CLASSES - 1, (n,), generator=g)
    # logits around 0 with sharp and flat regions: many pixels near the threshold of 0.5
    logits = torch.randn(n, CLASSES, 28, 28, generator=torch.Generator(dev).manual_seed(seed), device=dev) * 3
    logits[:, :, :7] *= 0.01
    return torch.from_numpy(det).to(dev), labels.to(dev), logits.to(dtype)


def _run(fn, monkeypatch, native, *args):
    monkeypatch.setenv('BAGS_SEGM_NATIVE', '1' if native else '0')
    try:
        return fn(*args), None
    except Exception as e:  # noqa: BLE001  (both routes must fail alike)
        return None, e


def _compare(got, want, img_h, img_w):
    assert got is not None and want is not None
    assert len(got) == len(want) == CLASSES - 1
    assert [len(v) for v in got] == [len(v) for v in want]
    for g_list, w_list in zip(got, want):
        for g, w in zip(g_list, w_list):
            assert g['size'] == w['size'] == [img_h, img_w]
            if g['counts'] != w['counts']:
                diff = int((SO.decode(g) != SO.decode(w)).sum())
                raise AssertionError('RLE differs: %d pixels' % diff)


@pytest.mark.parametrize('n', [0, 1, 37, 300])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('canvas', [(480, 640), (800, 1333)])
def test_get_seg_masks_native_equals_host(host_encoder, monkeypatch, n, dtype, canvas):
    img_h, img_w = canvas
    head = MH.FCNMaskHead(num_convs=1, in_channels=4, conv_out_channels=4, num_classes=CLASSES)
    det, labels, logits = _inputs(n, img_h, img_w, dtype, seed=n + img_h)
    for fn, rescale, sf in ((head.get_seg_masks, True, 1.0), (head.get_seg_masks_without, True, np.float64(1.0)),
                            (head.get_seg_masks, False, 1.0)):
        args = (logits, det, labels, CFG, (img_h, img_w, 3), sf, rescale)
        want, err_w = _run(fn, monkeypatch, False, *args)
        got, err_g = _run(fn, monkeypatch, True, *args)
        assert err_w is None and err_g is None, (err_w, err_g)
        _compare(got, want, img_h, img_w)


@pytest.mark.parametrize('rescale', [True, False])
@pytest.mark.parametrize('scale_factor', [0.7, np.float64(1.6)])
def test_scale_factor_and_rescale(host_encoder, monkeypatch, rescale, scale_factor):
    ori = (480, 640, 3)
    img_h, img_w = (ori[0], ori[1]) if rescale else (int(np.round(ori[0] * scale_factor)),
                                                     int(np.round(ori[1] * scale_factor)))
    # boxes on the canvas, given to the head in the scaled image's coordinates when rescaling
    det, labels, logits = _inputs(37, img_h, img_w, torch.float16, seed=3, scale=scale_factor if rescale else 1.0)
    head = MH.FCNMaskHead(num_convs=1, in_channels=4, conv_out_channels=4, num_classes=CLASSES)
    for fn in (head.get_seg_masks, head.get_seg_masks_without):
        args = (logits, det, labels, CFG, ori, scale_factor, rescale)
        want, err_w = _run(fn, monkeypatch, False, *args)
        got, err_g = _run(fn, monkeypatch, True, *args)
        assert err_w is None and err_g is None, (err_w, err_g)
        _compare(got, want, img_h, img_w)


@pytest.mark.parametrize('rescale', [True, False])
def test_class_agnostic_and_ndarray_inputs(host_encoder, monkeypatch, rescale):
    """A class-agnostic head, and the ndarray probabilities HTC passes to get_seg_masks_without ([n, 1, 28, 28] fp32,
    htc.py:403-421) and multi-scale testing passes to get_seg_masks ([n, C, 28, 28])."""
    img_h, img_w = 800, 1333
    det, labels, logits = _inputs(37, img_h, img_w, torch.float32, seed=11)
    agnostic = MH.FCNMaskHead(num_convs=1, in_channels=4, conv_out_channels=4, num_classes=CLASSES,
                              class_agnostic=True)
    head = MH.HTCMaskHead(num_convs=1, in_channels=4, conv_out_channels=4, num_classes=CLASSES)
    one = logits[:, :1].contiguous()
    cases = [(agnostic.get_seg_masks, one), (agnostic.get_seg_masks_without, one),
             (head.get_seg_masks_without, torch.sigmoid(one).cpu().numpy()),
             (head.get_seg_masks, torch.sigmoid(logits).cpu().numpy().astype(np.float16))]
    for fn, pred in cases:
        args = (pred, det, labels, CFG, (img_h, img_w, 3), 1.0, rescale)
        want, err_w = _run(fn, monkeypatch, False, *args)
        got, err_g = _run(fn, monkeypatch, True, *args)
        assert err_w is None and err_g is None, (err_w, err_g)
        _compare(got, want, img_h, img_w)


def test_box_outside_the_canvas_takes_the_host_loop(host_encoder, monkeypatch):
    img_h, img_w = 480, 640
    det, labels, logits = _inputs(37, img_h, img_w, torch.float32, seed=5, outside=True)
    head = MH.FCNMaskHead(num_convs=1, in_channels=4, conv_out_channels=4, num_classes=CLASSES)
    args = (logits, det, labels, CFG, (img_h, img_w, 3), 1.0, True)
    want, err_w = _run(head.get_seg_masks, monkeypatch, False, *args)
    got, err_g = _run(head.get_seg_masks, monkeypatch, True, *args)
    assert type(err_g) is type(err_w), (err_g, err_w)
    if want is not None:
        assert got == want


@pytest.mark.parametrize('n', [1, 300])
def test_three_host_syncs_per_call(monkeypatch, n):
    """The native route synchronises with the device three times (boxes, sizes, bytes) whatever n is; the count is
    taken by torch's sync debug mode, and bags_segm_rle itself never synchronises."""
    monkeypatch.setenv('BAGS_SEGM_NATIVE', '1')
    det, labels, logits = _inputs(n, 800, 1333, torch.float16, seed=n)
    head = MH.FCNMaskHead(num_convs=1, in_channels=4, conv_out_channels=4, num_classes=CLASSES)
    head.get_seg_masks(logits, det, labels, CFG, (800, 1333, 3), 1.0, True)   # warm-up
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            head.get_seg_masks(logits, det, labels, CFG, (800, 1333, 3), 1.0, True)
        finally:
            torch.cuda.set_sync_debug_mode('default')
    syncs = [w for w in caught if 'called a synchronizing CUDA operation' in str(w.message)]
    print('host syncs with n = %d: %d' % (n, len(syncs)))
    assert len(syncs) == 3, [str(w.message) for w in syncs]
