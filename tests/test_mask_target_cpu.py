"""CPU: the training mask targets' oracle and the argument checks of their kernel (bags_mask_target) --

  * tests/mask_target_oracle.py's uint8 resize against cv2.resize(INTER_LINEAR), bitwise, for every crop width and
    height in 1..130 (and a spread up to 1344) into 28 x 28, 14 x 14 and 28 x 14 targets, on 0/1 and full-range masks,
    including cv2's copy (crop == target) and INTER_AREA (crop == 2 x target) cases;
  * its per-image semantics (int32 truncation, numpy slicing, boxes that leave the mask) against the host loop
    mask_target_single wherever the host loop does not raise, and NaN rows where it does;
  * bags_mask_target's argument validation (error codes and messages before any device work).
"""
import ctypes as C
import re

import numpy as np
import pytest
import torch

import mask_target_oracle as MO
from balancedgroupsoftmax_b200 import _native as nat
from balancedgroupsoftmax_b200 import mask_head as MH

SIZES = list(range(1, 131)) + [131, 199, 256, 259, 333, 512, 800, 1024, 1333, 1344]
TARGETS = [(28, 28), (14, 14), (28, 14)]        # (out_h, out_w)


def _cv2_resize(img, out_w, out_h):
    cv2 = pytest.importorskip('cv2')
    return cv2.resize(img, (out_w, out_h), interpolation=cv2.INTER_LINEAR)


@pytest.mark.parametrize('out_h,out_w', TARGETS)
@pytest.mark.parametrize('content', ['binary', 'full'])
def test_resize_restatement_is_bitwise_cv2(out_h, out_w, content):
    pytest.importorskip('cv2')
    rng = np.random.default_rng(out_h * 100 + out_w + (content == 'full'))
    big = max(SIZES)
    if content == 'binary':
        src = (rng.random((big, big)) > 0.5).astype(np.uint8)
    else:
        src = rng.integers(0, 256, (big, big)).astype(np.uint8)
    bad = []
    for w in SIZES:
        for h in (SIZES if w <= 130 else SIZES[::5]):
            crop = src[:h, :w]
            if not np.array_equal(MO.resize_u8(crop, out_w, out_h), _cv2_resize(crop, out_w, out_h)):
                bad.append((w, h))
    assert not bad, bad[:20]


@pytest.mark.parametrize('out_h,out_w', TARGETS)
def test_copy_and_area_cases(out_h, out_w):
    """cv2 copies a crop of exactly the target size and averages 2 x 2 blocks of one exactly twice it; the oracle takes
    the same two branches (and the general formula would give the same values on these inputs too)."""
    rng = np.random.default_rng(7)
    for w, h in ((out_w, out_h), (2 * out_w, 2 * out_h)):
        for crop in ((rng.random((h, w)) > 0.5).astype(np.uint8), rng.integers(0, 256, (h, w)).astype(np.uint8),
                     np.full((h, w), 255, np.uint8)):
            want = _cv2_resize(crop, out_w, out_h)
            assert np.array_equal(MO.resize_u8(crop, out_w, out_h), want), (w, h)
            if w == out_w:
                assert np.array_equal(want, crop)
            else:
                assert np.array_equal(want, (crop.astype(int).reshape(out_h, 2, out_w, 2).sum((1, 3)) + 2) >> 2)
    # only both axes at 2x take INTER_AREA; one axis at 2x is the linear formula
    crop = rng.integers(0, 256, (out_h, 2 * out_w)).astype(np.uint8)
    assert np.array_equal(MO.resize_u8(crop, out_w, out_h), _cv2_resize(crop, out_w, out_h))


def _host_single(boxes, gt_inds, masks, out_h, out_w):
    cfg = dict(mask_size=(out_h, out_w))
    return MH.mask_target_single(torch.from_numpy(np.asarray(boxes, np.float32)),
                                 torch.from_numpy(np.asarray(gt_inds, np.int64)), masks, cfg).numpy()


def test_oracle_per_image_semantics_match_host_loop():
    pytest.importorskip('cv2')
    rng = np.random.default_rng(11)
    H, W = 61, 83
    masks = rng.integers(0, 256, (4, H, W)).astype(np.uint8)
    masks[1] = rng.random((H, W)) > 0.4
    boxes = [
        (10.7, 5.2, 40.9, 30.1), (0, 0, W - 1, H - 1), (0, 0, W + 30, H + 30),     # whole mask, past the edges
        (W - 1, H - 1, W - 1, H - 1), (W - 1.5, 3, W + 9, 20),                       # last pixel, ending on the edge
        (12.9, 7.9, 12.1, 7.2), (20, 20, 10, 10),                                    # sub-pixel, inverted: 1 pixel
        (-0.9, -0.5, 13, 14), (-20.0, -10.0, -3, -2), (-70, -50, -60, -45),          # negative: counts from the end
        (3, 4, 3 + 27, 4 + 27), (3, 4, 3 + 55, 4 + 55), (5, 6, 5 + 13, 6 + 13),      # 28, 56, 14 pixels
        (0, 9, 0, 50), (9, 0, 70, 0),                                                # 1 pixel wide, 1 pixel high
    ]
    gt = rng.integers(0, 4, len(boxes))
    for out_h, out_w in TARGETS:
        want = _host_single(boxes, gt, masks, out_h, out_w)
        assert np.array_equal(MO.target_single(np.array(boxes, np.float32), gt, masks, out_h, out_w), want)


def test_oracle_nan_rows_where_host_loop_raises():
    pytest.importorskip('cv2')
    masks = np.ones((2, 30, 40), np.uint8)
    good = (2.0, 3.0, 20.0, 25.0)
    for bad_box, bad_gt in (((45, 3, 50, 9), 0), ((2, 33, 9, 40), 1), ((-100, 3, -90, 9), 0), (good, 2),
                            ((np.nan, 3, 9, 9), 0), ((3e9, 3, 9, 9), 1),
                            ((-5, -3, 20, 9), 0)):                     # a negative start, a positive stop
        boxes, gt = np.array([good, bad_box, good], np.float32), np.array([0, bad_gt, 1])
        got = MO.target_single(boxes, gt, masks, 28, 28)
        assert np.isnan(got[1]).all() and not np.isnan(got[[0, 2]]).any()
        assert np.array_equal(got[[0, 2]], _host_single(boxes[[0, 2]], gt[[0, 2]], masks, 28, 28))
        with pytest.raises(Exception):
            _host_single(boxes[1:2], gt[1:2], masks, 28, 28)


# --------------------------------------------------------------------------- C ABI
def test_mask_target_rejects_bad_arguments():
    lib = nat.lib()
    fake, fake8 = C.c_void_p(256), C.c_void_p(264)         # never dereferenced: the checks fail first

    def call(n=1, mh=28, mw=28, sizes=(4, 3, 20, 30), boxes=fake, gt=fake8, masks=fake, out=fake, tables=True):
        sz = (C.c_int32 * (4 * n))(*(list(sizes) * n)) if n > 0 else None
        arr = lambda p: (C.c_void_p * max(n, 1))(*([p] * max(n, 1)))    # noqa: E731
        args = (arr(boxes), arr(gt), arr(masks), sz) if tables else (None, None, None, None)
        return lib.bags_mask_target(*args, n, mh, mw, out, None)

    def rejects(match, **kw):
        assert call(**kw) == -1, kw
        assert re.search(match, lib.bags_last_error().decode()), (kw, lib.bags_last_error())

    rejects('n_images = -1', n=-1)
    for mh, mw in ((0, 28), (28, 0), (257, 28), (28, -1)):
        rejects('mask size', mh=mh, mw=mw)
    rejects('NULL argument', tables=False)
    for k in range(4):
        s = [4, 3, 20, 30]
        s[k] = -1
        rejects('negative size', sizes=s)
    rejects('NULL boxes or gt_inds', boxes=None)
    rejects('NULL boxes or gt_inds', gt=None)
    rejects('NULL masks', masks=None)
    rejects('aligned', boxes=C.c_void_p(258))
    rejects('aligned', gt=C.c_void_p(260))
    rejects('NULL argument', out=None)
    rejects('at most 2', n=2, sizes=(2 ** 30 + 1, 3, 20, 30))
    # nothing to do: no images, or no positives (NULL boxes, gt indices, masks and output are then fine)
    assert call(n=0, tables=False) == 0
    assert call(sizes=(0, 3, 20, 30), boxes=None, gt=None, out=None) == 0
    assert call(sizes=(0, 0, 20, 30), boxes=None, gt=None, masks=None, out=None) == 0
