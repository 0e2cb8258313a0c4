"""Inputs and exact references for the class-aware hard NMS tests (tests/test_nms_ref_cpu.py,
tests/test_gpu_nms_vs_reference.py).

The NMS under test is greedy: candidates are visited in descending score order and box j is removed when an earlier
box that is still alive has IoU(i, j) > fp32(iou_thr), IoU with "+1" widths in fp32 (devIoU, the reference's
mmdet/ops/nms/src/nms_kernel.cu:13-21; restated as oracle.bags_oracle.iou_plus1_fp32 / greedy_keep).

Three tiers of input:
  * exact: integer coordinates in [0, 2047].  Every width, area, intersection and union is an integer below 2^23, so
    exact in fp32, and the only rounding is the IEEE division.  exact_iou gives the rational IoU, fp32_round its
    correctly rounded fp32 value; keep bits must then agree bit for bit between every implementation.
    NEAR_PAIRS holds, per threshold, box pairs (a, b) whose rational IoU lies within 1/8 ulp of an fp32 rounding
    boundary next to fp32(thr) (between the neighbours two below and two above it), on both sides where one
    exists.  They come from an exhaustive search over nested pairs -- b of size wb x hb inside a of size wa x ha,
    IoU = wb hb / (wa ha), wa, ha in [600, 2000], hb in [1, 2000], wb the two integers around the boundary -- with
    fractions.Fraction deciding each candidate.  A boundary that is missing has no such pair: near a rational p/q of
    small q (0.3 = 3/10, 0.5 = 1/2, ...) an IoU with union U differs from p/q by at least 1/(q U), more than 1/8 ulp.
    0.5 is the one representable threshold; its pairs have IoU exactly 1/2 and the nearest nested IoUs on each side.
  * kernel level: the same integer boxes handed straight to bags_class_nms_dense with crafted order / counts.
  * realistic: decoded float boxes at the LVIS test shape.  Rounding can then differ in the last place between fp32
    evaluations (an FMA contraction, an operation order), so a class is compared exactly only when it is DECIDED:
    every IoU its greedy scan acts on lies, in float64, more than DECIDED_MARGIN * thr from fp32(thr) (decided()).
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np
import torch

from oracle import bags_oracle as O

THRESHOLDS = (0.3, 0.45, 0.5, 0.6, 0.7)
DECIDED_MARGIN = 2.0 ** -20

NEAR_PAIRS = {
    0.3: [
        ((78, 88, 1804, 2018), (660, 139, 1222, 1915)),
        ((127, 176, 1929, 2004), (492, 478, 1564, 1399)),
        ((264, 47, 1423, 1332), (496, 261, 1191, 903)),
        ((885, 560, 2044, 1845), (1143, 756, 1785, 1451)),
        ((49, 94, 1991, 2024), (178, 515, 1862, 1182)),
        ((35, 69, 1977, 1999), (171, 488, 1840, 1161)),
        ((58, 243, 1976, 1949), (187, 614, 1846, 1205)),
        ((74, 78, 1992, 1784), (293, 425, 1772, 1088)),
        ((468, 38, 1416, 2014), (496, 486, 1387, 1116)),
        ((773, 29, 1721, 2005), (932, 390, 1562, 1281)),
    ],
    0.45: [
        ((105, 870, 1850, 1882), (491, 935, 1463, 1752)),
        ((47, 782, 1792, 1794), (511, 795, 1328, 1767)),
        ((589, 472, 1675, 1978), (856, 530, 1408, 1862)),
        ((420, 393, 1652, 1745), (598, 558, 1474, 1413)),
        ((175, 367, 1485, 1865), (185, 638, 1475, 1322)),
        ((58, 30, 1368, 1528), (371, 99, 1055, 1389)),
        ((118, 8, 1967, 1947), (118, 363, 1967, 1235)),
        ((125, 66, 1974, 2005), (177, 404, 1922, 1328)),
        ((317, 65, 1947, 2026), (417, 383, 1846, 1389)),
        ((381, 0, 2011, 1961), (507, 305, 1884, 1349)),
    ],
    0.5: [
        ((0, 0, 2047, 2047), (0, 0, 2047, 1023)),         # IoU = 2^21 / 2^22 = 1/2 exactly
        ((5, 9, 1204, 1408), (5, 9, 604, 1408)),          # 600 x 1400 / (1200 x 1400) = 1/2 exactly
        ((0, 0, 2046, 2046), (0, 0, 1023, 2045)),         # 1/2 - 1/(2 * 2047^2)
        ((0, 0, 2044, 2046), (0, 0, 1022, 2045)),         # 1/2 + 1/(2 * 2045 * 2047)
    ],
    0.6: [
        ((174, 13, 1825, 1958), (187, 266, 1811, 1452)),
        ((256, 24, 1907, 1969), (488, 131, 1674, 1755)),
        ((582, 697, 1355, 1771), (582, 840, 1355, 1484)),
        ((936, 457, 1709, 1531), (1000, 557, 1644, 1330)),
        ((3, 47, 1973, 1989), (96, 265, 1879, 1552)),
        ((5, 102, 1975, 2044), (210, 259, 1770, 1730)),
        ((6, 187, 1997, 1945), (38, 409, 1964, 1499)),
        ((197, 8, 2033, 1896), (294, 215, 1935, 1482)),
        ((56, 94, 1928, 1059), (258, 169, 1726, 907)),
        ((44, 669, 1826, 1674), (80, 794, 1790, 1422)),
    ],
    0.7: [
        ((156, 141, 1904, 1921), (413, 145, 1646, 1911)),
        ((700, 164, 1452, 1564), (767, 233, 1385, 1425)),
        ((274, 525, 1894, 1857), (312, 643, 1856, 1621)),
        ((418, 339, 2038, 1671), (561, 405, 1895, 1537)),
        ((14, 447, 1974, 1869), (270, 471, 1717, 1819)),
        ((104, 21, 1652, 1877), (167, 168, 1589, 1582)),
        ((653, 535, 1793, 1731), (700, 629, 1745, 1542)),
        ((226, 342, 1366, 1538), (339, 392, 1252, 1437)),
    ],
}


def fp32_round(x: Fraction) -> Fraction:
    """The fp32 value nearest to a rational x (ties to even), exactly; normal range only, NaN-free."""
    if x == 0:
        return Fraction(0)
    sign = -1 if x < 0 else 1
    x = abs(x)
    e = x.numerator.bit_length() - x.denominator.bit_length()
    if Fraction(2) ** e > x:
        e -= 1
    ulp = Fraction(2) ** (e - 23)
    q, r = divmod(x, ulp)
    q = int(q)
    if r > ulp / 2 or (r == ulp / 2 and q % 2):
        q += 1
    return sign * q * ulp


def exact_iou(a, b) -> Fraction:
    """The rational devIoU of two integer boxes (x1, y1, x2, y2) with "+1" widths; union must be non-zero."""
    a, b = [int(v) for v in a], [int(v) for v in b]
    w = max(min(a[2], b[2]) - max(a[0], b[0]) + 1, 0)
    h = max(min(a[3], b[3]) - max(a[1], b[1]) + 1, 0)
    inter = w * h
    sa = (a[2] - a[0] + 1) * (a[3] - a[1] + 1)
    sb = (b[2] - b[0] + 1) * (b[3] - b[1] + 1)
    return Fraction(inter, sa + sb - inter)


def brute_greedy(boxes, iou_thr: float) -> np.ndarray:
    """Greedy NMS stated the slow way, independent of greedy_keep: walk the boxes in order, keep a box when no box
    kept so far has IoU > fp32(thr) with it.  -> bool keep."""
    boxes = np.asarray(boxes, dtype=np.float32).reshape(-1, 4)
    thr = np.float32(iou_thr)
    kept = []
    for j in range(boxes.shape[0]):
        if all(not (O.iou_plus1_fp32(boxes[i], boxes[j]) > thr) for i in kept):
            kept.append(j)
    out = np.zeros(boxes.shape[0], dtype=bool)
    out[kept] = True
    return out


def random_int_boxes(g: np.random.Generator, n: int, span: int = 2047, max_wh: int = 400) -> np.ndarray:
    """n integer boxes inside [0, span]^2, sizes in [1, max_wh] (fp32 [n, 4])."""
    wh = g.integers(1, max_wh + 1, (n, 2))
    x1 = g.integers(0, span - wh[:, 0] + 2)
    y1 = g.integers(0, span - wh[:, 1] + 2)
    return np.stack([x1, y1, x1 + wh[:, 0] - 1, y1 + wh[:, 1] - 1], 1).astype(np.float32)


def clustered_int_boxes(g: np.random.Generator, n: int, clusters: int = 6) -> np.ndarray:
    """n integer boxes jittered around a few centres: many IoUs between 0.2 and 0.9, so suppression chains form."""
    base = random_int_boxes(g, clusters, span=1700, max_wh=300)
    pick = base[g.integers(0, clusters, n)]
    jit = g.integers(-12, 13, (n, 4)).astype(np.float32)
    b = np.clip(pick + jit, 0, 2047)
    b[:, 2] = np.maximum(b[:, 2], b[:, 0])
    b[:, 3] = np.maximum(b[:, 3], b[:, 1])
    return b.astype(np.float32)


def chain() -> np.ndarray:
    """Three integer boxes A, B, C in visiting order with IoU(A, B) = 0.6, IoU(B, C) = 0.6 and IoU(A, C) = 1/3 (at
    iou_thr 0.5): A removes B, so C survives although B would have removed it."""
    return np.array([[0, 0, 99, 99], [25, 0, 124, 99], [50, 0, 149, 99]], dtype=np.float32)


def place(background: np.ndarray, at: dict) -> np.ndarray:
    """Copy of background [n, 4] with rows replaced: at = {position: box}."""
    b = background.copy()
    for p, box in at.items():
        b[p] = box
    return b


def edge_sets(g: np.random.Generator):
    """(name, boxes [n, 4] in visiting order, thresholds) for the exact tier's hand-made edges; boxes that are far
    apart fill the rows around the crafted ones.  Integer coordinates except where a name says NaN / inf."""
    far = lambda n: np.array([[40 * (i % 50), 40 * (i // 50) + 1000, 40 * (i % 50) + 20, 40 * (i // 50) + 1020]
                              for i in range(n)], dtype=np.float32)
    a, b, c = chain()
    out = []
    for p in (30, 31, 32, 62, 63, 64):          # A, B, C at p, p+1, p+2: across word edges 31|32 and 63|64
        out.append(('chain@%d' % p, place(far(100), {p: a, p + 1: b, p + 2: c}), (0.5,)))
    # a row in word 0 suppressing a column in word 2 and one in word 3; a suppressed row in word 1 whose box would
    # have suppressed a column in word 3 -- only the alive row may act
    out.append(('long_range', place(far(130), {3: a, 70: a, 40: b, 100: c, 120: b}), (0.5,)))
    out.append(('identical', np.tile(np.array([[10, 10, 60, 90]], np.float32), (40, 1)), (0.5, 0.999999, 1.0)))
    touch = np.array([[0, 0, 9, 9], [10, 0, 19, 9], [9, 0, 18, 9], [0, 10, 9, 19], [0, 9, 9, 18]], np.float32)
    out.append(('touching', touch, (-0.5, 0.0, 0.05, 0.5)))
    degenerate = np.array([[5, 5, 4, 4], [5, 5, 4, 4],             # 0 x 0 twice: union 0, IoU 0/0 = NaN
                           [5, 5, 4, 20], [5, 5, 4, 20],           # zero width
                           [30, 30, 20, 20], [30, 30, 20, 20],     # inverted: negative widths
                           [0, 0, 40, 40], [10, 10, 5, 50],        # inverted inside a box
                           [3, 3, 3, 3]], np.float32)              # 1 x 1
    out.append(('degenerate', degenerate, (-0.5, 0.0, 0.5, 1.0)))
    nan, inf = np.float32('nan'), np.float32('inf')
    special = np.array([[0, 0, 50, 50], [nan, 0, 50, 50], [0, 0, 50, 50], [0, 0, inf, 50], [0, 0, inf, 50],
                        [-inf, 0, 50, 50], [0, -inf, 50, inf], [0, 0, nan, nan], [0, 0, 50, 50], [inf, inf, inf, inf],
                        [-inf, -inf, -inf, -inf], [0, 0, 50, 50]], np.float32)
    out.append(('nan_inf_coords', special, (-0.5, 0.0, 0.5, 1.0)))
    for thr in (-0.5, 0.0, 1.0, 0.999999):
        out.append(('random_thr%g' % thr, clustered_int_boxes(g, 200), (thr,)))
    return out


def realistic_inputs(g: torch.Generator, n: int = 1000, classes: int = 1231):
    """Decoded float boxes and merged-score-like class scores at the LVIS test shape: (boxes [n, 4], scores
    [n, classes] with column 0 the background).  Proposals cluster around a few dozen objects, so every class
    has IoUs all over (0, 1)."""
    obj = torch.rand(40, 2, generator=g) * 1000
    owh = torch.rand(40, 2, generator=g) * 250 + 16
    pick = torch.randint(0, 40, (n,), generator=g)
    ctr = obj[pick] + torch.randn(n, 2, generator=g) * owh[pick] * 0.15
    wh = owh[pick] * (1 + 0.2 * torch.randn(n, 2, generator=g)).clamp_min(0.3)
    boxes = torch.cat([ctr - wh / 2, ctr + wh / 2], 1).clamp(0, 1332)
    logits = torch.randn(n, classes, generator=g) * 2
    logits[:, 0] += 3
    scores = torch.softmax(logits, 1)
    return boxes.float(), scores.float()


def iou_matrix64(boxes: np.ndarray) -> np.ndarray:
    """float64 "+1" IoU of every pair of boxes [m, 4] -> [m, m]."""
    b = np.asarray(boxes, dtype=np.float64)
    x1, y1, x2, y2 = b[:, 0], b[:, 1], b[:, 2], b[:, 3]
    w = np.maximum(np.minimum(x2[:, None], x2[None]) - np.maximum(x1[:, None], x1[None]) + 1, 0)
    h = np.maximum(np.minimum(y2[:, None], y2[None]) - np.maximum(y1[:, None], y1[None]) + 1, 0)
    inter = w * h
    area = (x2 - x1 + 1) * (y2 - y1 + 1)
    return inter / (area[:, None] + area[None] - inter)


def decided(iou64: np.ndarray, keep: np.ndarray, iou_thr: float) -> bool:
    """A class's NMS is DECIDED when every IoU the greedy scan acts on -- row i kept, column j > i, in visiting order
    (iou64 [m, m] of the candidates in that order, keep [m] bool) -- lies, in float64, more than DECIDED_MARGIN * thr
    from fp32(thr).  devIoU's fp32 error is a few ulps (2^-22 relative or less), so no fp32 evaluation order or
    contraction can flip one of those comparisons, and by induction over the scan every correct implementation keeps
    the same rows.  Comparisons of removed rows never act, so they need no margin."""
    t = float(np.float32(iou_thr))
    rows = np.flatnonzero(keep)
    if rows.size == 0:
        return True
    sub = iou64[rows]
    after = np.arange(iou64.shape[0])[None, :] > rows[:, None]
    return bool(np.all(np.abs(sub[after] - t) > DECIDED_MARGIN * abs(t)))
