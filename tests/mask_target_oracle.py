"""numpy restatement of the mask heads' training targets as bags_mask_target computes them.

``resize_u8`` is cv2.resize(uint8 [h, w], (D_w, D_h), INTER_LINEAR) as OpenCV computes it for 8-bit images: per axis
the source coordinate (d + 0.5) * (1 / (D / S)) - 0.5 in double, rounded once to float, its floor and fraction, and
11-bit weights rint((1 - f) * 2048), rint(f * 2048).  The horizontal axis is clamped at both borders (the edge tap is
the edge pixel with weight 2048); the vertical axis keeps its fraction and clamps only the row index.  Then a
horizontal pass R = src[x0] a0 + src[x1] a1 and a vertical pass ((b0 (R0 >> 4)) >> 16) + ((b1 (R1 >> 4)) >> 16),
rounded by (+ 2) >> 2.  A source of exactly the output size is copied; one of exactly twice it on both axes takes
cv2's INTER_AREA path, (sum of 2 x 2 + 2) >> 2.

``targets`` is mask_target for a batch: the host loop's box truncation and numpy slicing, with a row of NaN where
the host loop raises (a gt index outside [0, num_gt), an empty crop).
"""
import numpy as np


def taps(S, D, clamp):
    """(i0, i1, a0, a1) int64 arrays of one axis: source size S -> destination size D."""
    scale = 1.0 / (D / S)
    i0, i1, a0, a1 = (np.zeros(D, np.int64) for _ in range(4))
    for d in range(D):
        f = np.float32((d + 0.5) * scale - 0.5)
        s = int(np.floor(f))
        f = np.float32(f - np.float32(s))
        if clamp:
            if s < 0:
                f, s = np.float32(0), 0
            if s >= S - 1:
                f, s = np.float32(0), S - 1
        a0[d] = int(np.rint(np.float32(np.float32(1) - f) * np.float32(2048)))
        a1[d] = int(np.rint(f * np.float32(2048)))
        i0[d], i1[d] = min(max(s, 0), S - 1), min(max(s + 1, 0), S - 1)
    return i0, i1, a0, a1


def resize_u8(img, out_w, out_h):
    h, w = img.shape
    if (w, h) == (out_w, out_h):
        return img.copy()
    if (w, h) == (2 * out_w, 2 * out_h):
        s = img.astype(np.int64).reshape(out_h, 2, out_w, 2).sum((1, 3))
        return ((s + 2) >> 2).astype(np.uint8)
    x0, x1, ax0, ax1 = taps(w, out_w, True)
    y0, y1, by0, by1 = taps(h, out_h, False)
    src = img.astype(np.int64)
    rows = src[:, x0] * ax0 + src[:, x1] * ax1
    v = (((by0[:, None] * (rows[y0] >> 4)) >> 16) + ((by1[:, None] * (rows[y1] >> 4)) >> 16) + 2) >> 2
    return np.minimum(v, 255).astype(np.uint8)


def target_single(boxes, gt_inds, masks, out_h, out_w):
    """float32 [P, out_h, out_w] of one image: boxes float32 [P, 4], gt_inds int [P], masks uint8 [num_gt, H, W]."""
    out = np.full((len(gt_inds), out_h, out_w), np.nan, np.float32)
    with np.errstate(over='ignore', invalid='ignore'):
        ib = np.asarray(boxes, np.float32)[:, :4].astype(np.int32)
        for r, ((left, top, right, bottom), gt) in enumerate(zip(ib, gt_inds)):
            w = max(right - left + np.int32(1), np.int32(1))
            h = max(bottom - top + np.int32(1), np.int32(1))
            if not 0 <= gt < masks.shape[0]:
                continue
            crop = masks[gt][top:top + h, left:left + w]
            if crop.size == 0:
                continue
            out[r] = resize_u8(crop, out_w, out_h)
    return out


def targets(boxes_list, gt_inds_list, masks_list, out_h, out_w):
    return np.concatenate([target_single(b, g, m, out_h, out_w) for b, g, m in zip(boxes_list, gt_inds_list,
                                                                                   masks_list)])
