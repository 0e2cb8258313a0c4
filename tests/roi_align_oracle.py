"""Restatements of the reference's RoIAlign op and FPN extractor -- TEST ORACLE.

``roi_samples`` places one RoI's samples with the op's fp32 rounding sequence (the one its sm_90a build has: fused
multiply-adds rounded once, computed exactly here), so that they land on the same pixels as on the device; ``forward``
and ``backward`` then pool and scatter in float64.  ``backward`` also returns, per pixel, the sum of the absolute
values of the terms it added, which bounds how far an fp32 scatter in any order can be from it.

``extractor`` is mmdet's SingleRoIExtractor.forward loop (level mapping, one op call per level on the RoIs of that
level, scatter into the output) with the RoIAlign op passed in, so that it runs on the reference's compiled op.
"""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np
import torch

f32 = np.float32


def _round32(q: Fraction) -> np.float32:
    """q rounded once to fp32, to nearest even."""
    r = f32(float(q))
    if not np.isfinite(r) or q == 0:
        return r
    best = None
    for c in (np.nextafter(r, f32(-np.inf)), r, np.nextafter(r, f32(np.inf))):
        if not np.isfinite(c):
            continue
        key = (abs(Fraction(float(c)) - q), int(np.array(c, dtype=np.float32).view(np.int32)) & 1)
        if best is None or key < best[0]:
            best = (key, c)
    return f32(best[1])


def fma32(a, b, c) -> np.float32:
    """fp32 fused multiply-add: a * b + c rounded once."""
    a, b, c = float(a), float(b), float(c)
    if not (math.isfinite(a) and math.isfinite(b) and math.isfinite(c)):
        return f32(a * b + c)
    return _round32(Fraction(a) * Fraction(b) + Fraction(c))


def axis_sample(start, bin_, p: int, i: int, s: int, size: int):
    """(valid, lo, hi, l, h) of sample i of bin p on one axis of ``size`` pixels; l, h as fp32."""
    with np.errstate(all='ignore'):
        c = f32(fma32(f32(p), bin_, start) + f32(f32(f32(i) + f32(0.5)) * bin_) / f32(s))
        valid = not (c < -1 or c > size)
        v = f32(0) if c <= 0 else c
        lo = 0 if np.isnan(v) else int(min(v, f32(2 ** 31 - 1)))
        if lo >= size - 1:
            lo = hi = size - 1
            v = f32(lo)
        else:
            hi = lo + 1
        l = f32(v - f32(lo))
        return valid, lo, hi, l, f32(f32(1) - l)


def roi_samples(roi, scale: float, out_h: int, out_w: int, sample_num: int, H: int, W: int):
    """The samples of one RoI (batch, x1, y1, x2, y2) on a level of H x W with the given spatial_scale:
    (ys, xs, count), ys[ph][iy] and xs[pw][ix] as axis_sample returns them."""
    s = f32(scale)
    x1, y1, x2, y2 = (f32(v) for v in roi[1:5])
    with np.errstate(all='ignore'):
        start_w, start_h = f32(x1 * s), f32(y1 * s)
        roi_w = fma32(f32(x2 + f32(1)), s, -start_w)
        roi_h = fma32(f32(y2 + f32(1)), s, -start_h)
        roi_w = f32(0) if not roi_w > 0 else roi_w          # fmaxf(x, 0): NaN -> 0
        roi_h = f32(0) if not roi_h > 0 else roi_h
        bin_h, bin_w = f32(roi_h / f32(out_h)), f32(roi_w / f32(out_w))
    sh = sample_num if sample_num > 0 else int(math.ceil(bin_h))
    sw = sample_num if sample_num > 0 else int(math.ceil(bin_w))
    ys = [[axis_sample(start_h, bin_h, p, i, sh, H) for i in range(sh)] for p in range(out_h)]
    xs = [[axis_sample(start_w, bin_w, p, i, sw, W) for i in range(sw)] for p in range(out_w)]
    return ys, xs, sh * sw


def _corners(ys, xs, ph, pw):
    for y in ys[ph]:
        for x in xs[pw]:
            if y[0] and x[0]:
                yield ((y[1], x[1], float(y[4]) * float(x[4])), (y[1], x[2], float(y[4]) * float(x[3])),
                       (y[2], x[1], float(y[3]) * float(x[4])), (y[2], x[2], float(y[3]) * float(x[3])))


def forward(feat: np.ndarray, rois: np.ndarray, out_h: int, out_w: int, scale: float, sample_num: int) -> np.ndarray:
    """float64 RoIAlign of every RoI on one level feat [B, C, H, W] (no level mapping); a batch index outside
    [0, B) gives a zero row.  [k, C, out_h, out_w]."""
    feat = np.asarray(feat, dtype=np.float64)
    B, Cc, H, W = feat.shape
    out = np.zeros((len(rois), Cc, out_h, out_w))
    for r, roi in enumerate(np.asarray(rois, dtype=np.float32)):
        b = int(roi[0]) if np.isfinite(roi[0]) else 0
        if not 0 <= b < B:
            continue
        ys, xs, cnt = roi_samples(roi, scale, out_h, out_w, sample_num, H, W)
        for ph in range(out_h):
            for pw in range(out_w):
                acc = np.zeros(Cc)
                for quad in _corners(ys, xs, ph, pw):
                    for yy, xx, w in quad:
                        acc += w * feat[b, :, yy, xx]
                out[r, :, ph, pw] = acc / cnt if cnt else np.nan
    return out


def backward(gout: np.ndarray, rois: np.ndarray, scale: float, sample_num: int, shape):
    """float64 gradient of ``forward`` for gout [k, C, out_h, out_w] on a level of ``shape`` [B, C, H, W], and the
    sum of the absolute values of the terms (gout w / count) added to each element."""
    gout = np.asarray(gout, dtype=np.float64)
    B, Cc, H, W = shape
    _, _, out_h, out_w = gout.shape
    grad, absum = np.zeros(shape), np.zeros(shape)
    for r, roi in enumerate(np.asarray(rois, dtype=np.float32)):
        b = int(roi[0]) if np.isfinite(roi[0]) else 0
        if not 0 <= b < B:
            continue
        ys, xs, cnt = roi_samples(roi, scale, out_h, out_w, sample_num, H, W)
        for ph in range(out_h):
            for pw in range(out_w):
                g = gout[r, :, ph, pw] / cnt if cnt else None
                for quad in _corners(ys, xs, ph, pw):
                    for yy, xx, w in quad:
                        grad[b, :, yy, xx] += g * w
                        absum[b, :, yy, xx] += np.abs(g * w)
    return grad, absum


# ----------------------------------------------------------------------------------------- the extractor's loop
def map_roi_levels(rois: torch.Tensor, num_levels: int, finest_scale) -> torch.Tensor:
    """SingleRoIExtractor.map_roi_levels: the reference's torch ops, on the RoIs' device."""
    scale = torch.sqrt((rois[:, 3] - rois[:, 1] + 1) * (rois[:, 4] - rois[:, 2] + 1))
    return torch.floor(torch.log2(scale / finest_scale + 1e-6)).clamp(min=0, max=num_levels - 1).long()


def extractor(op, feats, rois, out_size, strides, sample_num, finest_scale=56, out_channels=None,
              roi_scale_factor=None, rescale=None):
    """SingleRoIExtractor.forward with ``op(feat, rois, out_h, out_w, spatial_scale, sample_num)`` as the RoIAlign
    layer of each level (spatial_scale = 1 / stride), ``rescale(rois, factor)`` as roi_rescale."""
    out_h, out_w = out_size
    if len(feats) == 1:
        return op(feats[0], rois, out_h, out_w, 1 / strides[0], sample_num)
    lvls = map_roi_levels(rois, len(feats), finest_scale)
    out = feats[0].new_zeros(rois.shape[0], out_channels or feats[0].shape[1], out_h, out_w)
    if roi_scale_factor is not None:
        rois = rescale(rois, roi_scale_factor)
    for i in range(len(feats)):
        inds = lvls == i
        if inds.any():
            out[inds] = op(feats[i], rois[inds, :], out_h, out_w, 1 / strides[i], sample_num)
    return out
