"""Oracles of the test-time mask path (FCNMaskHead.get_seg_masks, fcn_mask_head.py:125-239) in numpy:

  * ``resize_linear``: cv2.resize(src, (w, h), interpolation=cv2.INTER_LINEAR) of a float32 map, bitwise.  OpenCV's
    default build hands float32 linear resizes to IPP, whose arithmetic is: per axis the source coordinate
    (d + 0.5) * (S / D) - 0.5 in float64, its fraction rounded once to float32, the index clamped to [0, S - 1] with
    the fraction zeroed at both borders; then a horizontal pass and a vertical pass of a + t * (b - a), each one fused
    multiply-add in float32.  ``dsize == ssize`` is a copy (cv2.resize returns before any interpolation).
  * COCO run-length encoding as pycocotools' maskApi.c: ``rle_counts`` (rleEncode: column-major runs, the first one of
    zeros), ``rle_string`` / ``rle_from_string`` (rleToString / rleFrString), ``encode`` / ``decode`` with the
    signatures of pycocotools.mask.encode / decode.
"""
import sys

import numpy as np

f32, f64 = np.float32, np.float64


def fma32(a, b, c):
    """float32 fma(a, b, c), correctly rounded: a * b is exact in float64; the float64 sum is rounded to float32
    unless it lands on a float32 midpoint, where the two-sum error decides the side."""
    a, b, c = (np.asarray(v, dtype=f32) for v in (a, b, c))
    p = a.astype(f64) * b.astype(f64)
    s = p + c.astype(f64)
    bb = s - p
    err = (p - (s - bb)) + (c.astype(f64) - bb)
    r = s.astype(f32)
    up = np.nextafter(r, f32(np.inf))
    dn = np.nextafter(r, f32(-np.inf))
    nb = np.where(s > r.astype(f64), up, dn)
    mid = (r.astype(f64) + nb.astype(f64)) / 2
    tie = (s == mid) & (err != 0)
    toward_nb = np.where(nb > r, err > 0, err < 0)
    return np.where(tie & toward_nb, nb, r).astype(f32)


def _axis(S, D):
    x = (np.arange(D, dtype=f64) + 0.5) * (S / D) - 0.5
    i0 = np.floor(x)
    t = (x - i0).astype(f32)
    i0 = i0.astype(np.int64)
    lo, hi = i0 < 0, i0 >= S - 1
    t[lo | hi] = 0
    i0[lo], i0[hi] = 0, S - 1
    return i0, np.minimum(i0 + 1, S - 1), t


def _lerp(a, b, t):
    return fma32(t, (b - a).astype(f32), a)


def resize_linear(src, w, h):
    """cv2.resize(src, (w, h), interpolation=cv2.INTER_LINEAR) of a float32 [H, W] map, bitwise."""
    src = np.asarray(src, dtype=f32)
    H, W = src.shape
    if (w, h) == (W, H):
        return src.copy()
    x0, x1, tx = _axis(W, w)
    y0, y1, ty = _axis(H, h)
    rows = _lerp(src[:, x0], src[:, x1], tx[None, :])
    return _lerp(rows[y0], rows[y1], ty[:, None])


# --------------------------------------------------------------------------- COCO RLE
def rle_counts(mask):
    """rleEncode of a [h, w] mask: run lengths over its column-major pixels, alternating 0-runs and 1-runs from a
    (possibly empty) 0-run."""
    flat = np.asarray(mask).astype(bool).ravel(order='F').astype(np.int8)
    change = np.flatnonzero(np.diff(np.concatenate([[0], flat])) != 0)
    edges = np.concatenate([[0], change, [flat.size]])
    return np.diff(edges).astype(np.int64).tolist()


def rle_string(counts):
    """rleToString: each count minus the count two before (from the fourth on), 5-bit groups, low first, 0x20 when
    more follow, + 48."""
    out = bytearray()
    for i, c in enumerate(counts):
        x = int(c) - (int(counts[i - 2]) if i > 2 else 0)
        more = True
        while more:
            ch = x & 0x1f
            x >>= 5
            more = x != -1 if ch & 0x10 else x != 0
            out.append((ch | 0x20 if more else ch) + 48)
    return bytes(out)


def rle_from_string(s):
    """rleFrString: the counts of a compressed RLE string."""
    counts, p = [], 0
    while p < len(s):
        x, k, more = 0, 0, True
        while more:
            c = s[p] - 48
            x |= (c & 0x1f) << (5 * k)
            more = bool(c & 0x20)
            p += 1
            k += 1
            if not more and c & 0x10:
                x |= -1 << (5 * k)
        if len(counts) > 2:
            x += counts[-2]
        counts.append(x)
    return counts


def encode(masks):
    """pycocotools.mask.encode of a uint8 [h, w, k] array: [{'size': [h, w], 'counts': bytes}] * k."""
    h, w, k = masks.shape
    return [{'size': [h, w], 'counts': rle_string(rle_counts(masks[:, :, i]))} for i in range(k)]


def decode(rle):
    """pycocotools.mask.decode of one RLE dict: the uint8 [h, w] mask."""
    h, w = rle['size']
    counts = rle_from_string(rle['counts'])
    assert sum(counts) == h * w, (sum(counts), h, w)
    flat = np.repeat(np.arange(len(counts)) % 2, counts).astype(np.uint8)
    return flat.reshape((w, h)).T.copy()


def installed_pycocotools_mask(monkeypatch):
    """The installed pycocotools.mask, or None where pycocotools is not installed.  Other test helpers put file-less
    stand-ins for pycocotools into sys.modules (so that the reference's modules import); those are set aside for the
    test with ``monkeypatch`` and put back after it."""
    for name in ('pycocotools', 'pycocotools.mask'):
        mod = sys.modules.get(name)
        if mod is not None and getattr(mod, '__file__', None) is None:
            monkeypatch.delitem(sys.modules, name)
    try:
        import pycocotools.mask as mask
    except ImportError:
        return None
    return mask
