"""CPU: the test-time mask path's oracles and the argument checks of its kernel (bags_segm_rle) --

  * tests/segm_oracle.py's resize restatement against cv2.resize(INTER_LINEAR), bitwise, over every box size the
    28 x 28 and 14 x 14 maps meet up to 200 pixels and a spread up to 1333;
  * its COCO RLE encoder and decoder: round trips, pycocotools' own output where pycocotools is installed;
  * bags_segm_rle's argument validation (error codes and messages before any device work).
"""
import ctypes as C
import re
from fractions import Fraction

import numpy as np
import pytest

import segm_oracle as SO
from balancedgroupsoftmax_b200 import _native as nat

SIZES = list(range(1, 201)) + [233, 256, 301, 333, 400, 512, 600, 640, 777, 800, 999, 1024, 1200, 1333]


@pytest.mark.parametrize('src_size', [28, 14])
def test_resize_restatement_is_bitwise_cv2(src_size):
    cv2 = pytest.importorskip('cv2')
    rng = np.random.default_rng(src_size)
    src = rng.random((src_size, src_size), dtype=np.float32)
    src[0, :3] = [0.0, 1.0, 0.5]                      # exact values next to arbitrary ones
    bad = []
    for w in SIZES:
        for h in (SIZES if w <= 200 or w % 3 == 0 else SIZES[::7]):
            want = cv2.resize(src, (w, h), interpolation=cv2.INTER_LINEAR)
            got = SO.resize_linear(src, w, h)
            if want.shape != got.shape or not np.array_equal(want.view(np.uint32), got.view(np.uint32)):
                bad.append((w, h))
    assert not bad, bad[:20]


def test_resize_of_non_square_maps():
    """Maps of at least two rows and two columns (OpenCV resizes one-row and one-column maps by other arithmetic,
    which bags_segm_rle rejects and the head leaves to the host loop)."""
    cv2 = pytest.importorskip('cv2')
    rng = np.random.default_rng(5)
    for H, W in ((28, 14), (7, 28), (2, 28), (28, 2), (2, 2)):
        src = rng.random((H, W), dtype=np.float32)
        for w, h in ((1, 1), (W, H), (2 * W, H), (W, 3 * H), (37, 53), (600, 13)):
            want = cv2.resize(src, (w, h), interpolation=cv2.INTER_LINEAR)
            assert np.array_equal(want, SO.resize_linear(src, w, h)), (H, W, w, h)


def _round_f32(exact):
    """float32 nearest to a Fraction (ties to even)."""
    r = np.float32(float(exact))
    cands = [np.nextafter(r, np.float32(-np.inf)), r, np.nextafter(r, np.float32(np.inf))]
    return min(cands, key=lambda v: (abs(Fraction(float(v)) - exact), int(v.view(np.uint32)) & 1))


def test_fma32_rounds_once():
    # (1 + 2^-23) (2^-24 - 2^-47) + (1 + 2^-23) = 1 + 2^-23 + 2^-24 - 2^-70: float64 rounds it to the float32 midpoint
    # 1 + 2^-23 + 2^-24, which a second rounding takes up to 1 + 2^-22; the true value is below it
    a, b, c = np.float32(1 + 2 ** -23), np.float32(2 ** -24 - 2 ** -47), np.float32(1 + 2 ** -23)
    assert SO.fma32(a, b, c) == np.float32(1 + 2 ** -23)
    assert np.float32(np.float64(a) * np.float64(b) + np.float64(c)) == np.float32(1 + 2 ** -22)
    rng = np.random.default_rng(0)
    x, y, z = (rng.random(3000, dtype=np.float32) - np.float32(0.5) for _ in range(3))
    want = [_round_f32(Fraction(float(p)) * Fraction(float(q)) + Fraction(float(r))) for p, q, r in zip(x, y, z)]
    assert np.array_equal(SO.fma32(x, y, z), np.array(want, dtype=np.float32))


# --------------------------------------------------------------------------- RLE
def _canvases():
    rng = np.random.default_rng(1)
    out = [np.zeros((7, 5), np.uint8), np.ones((7, 5), np.uint8), np.zeros((1, 1), np.uint8),
           np.ones((1, 1), np.uint8), (rng.random((480, 640)) > 0.5).astype(np.uint8)]
    for (t, l, h, w) in ((0, 0, 1, 1), (479, 639, 1, 1), (10, 20, 1, 1), (0, 5, 480, 3), (100, 0, 50, 640)):
        m = np.zeros((480, 640), np.uint8)
        m[t:t + h, l:l + w] = 1
        out.append(m)
    big = np.zeros((800, 1333), np.uint8)
    big[3:797, 600:1333] = (rng.random((794, 733)) > 0.02)
    out.append(big)
    return out


def test_rle_round_trips():
    for m in _canvases():
        counts = SO.rle_counts(m)
        assert sum(counts) == m.size and all(c > 0 for c in counts[1:])
        s = SO.rle_string(counts)
        assert all(48 <= ch < 48 + 64 for ch in s)
        assert SO.rle_from_string(s) == counts
        rle = SO.encode(np.asfortranarray(m[:, :, None]))[0]
        assert rle['size'] == list(m.shape)
        assert np.array_equal(SO.decode(rle), m)


def test_rle_known_strings():
    assert SO.rle_counts(np.zeros((1, 1), np.uint8)) == [1]
    assert SO.rle_counts(np.ones((1, 1), np.uint8)) == [0, 1]
    assert SO.rle_string([1]) == b'1'
    assert SO.rle_string([0, 1]) == b'01'
    assert SO.rle_string([5, 3, 7, 1]) == b'537N'         # the fourth is 1 - 3 = -2: the group 30, + 48
    assert SO.rle_string([40]) == b'X1'                   # 40 = 8 + 32: 8 | 0x20, then 1
    assert SO.rle_from_string(SO.rle_string([100000, 1, 2, 99999, 7])) == [100000, 1, 2, 99999, 7]


def test_encoder_matches_pycocotools(monkeypatch):
    mask = SO.installed_pycocotools_mask(monkeypatch)
    if mask is None:
        pytest.skip('pycocotools is not installed')
    for m in _canvases():
        want = mask.encode(np.asfortranarray(m[:, :, None]))
        assert SO.encode(np.asfortranarray(m[:, :, None])) == want


# --------------------------------------------------------------------------- C ABI
def test_segm_rle_rejects_bad_arguments():
    lib = nat.lib()
    fake = C.c_void_p(256)                             # never dereferenced: the checks fail first
    good = (C.c_int32 * 4)(2, 3, 4, 5)

    def call(probs=fake, n=1, mh=28, mw=28, boxes_host=good, boxes=fake, img_h=20, img_w=30, lengths=fake):
        return lib.bags_segm_rle(probs, n, mh, mw, boxes_host, boxes, img_h, img_w, 0.5, lengths, None, None)

    def rejects(match, **kw):
        assert call(**kw) != 0, kw
        assert re.search(match, lib.bags_last_error().decode()), (kw, lib.bags_last_error())

    rejects('n = -1', n=-1)
    for k in ('probs', 'boxes_host', 'boxes', 'lengths'):
        rejects('NULL', **{k: None})
    rejects('mask size', mh=1)
    rejects('mask size', mw=-3)
    rejects('canvas', img_h=0)
    rejects('canvas', img_w=-1)
    rejects('canvas', img_h=65536, img_w=65536)
    for bad, what in (((2, 3, 0, 5), 'empty box'), ((2, 3, 4, -1), 'empty box'), ((-1, 3, 4, 5), 'leaves'),
                      ((2, -1, 4, 5), 'leaves'), ((27, 3, 4, 5), 'leaves'), ((2, 16, 4, 5), 'leaves')):
        rejects(what, boxes_host=(C.c_int32 * 4)(*bad))
    two = (C.c_int32 * 8)(0, 0, 30, 20, 0, 0, 31, 20)  # the second of two detections
    rejects('detection 1', n=2, boxes_host=two)
    rejects('aligned', boxes=C.c_void_p(260))
    assert call(n=0, probs=None, boxes_host=None, boxes=None, lengths=None) == 0   # nothing to do
