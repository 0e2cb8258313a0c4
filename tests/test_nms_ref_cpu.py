"""CPU: the NMS restatement (oracle.bags_oracle: iou_plus1_fp32, greedy_keep, nms_plus1, multiclass_nms) against exact
rational arithmetic, a brute-force greedy NMS and the reference's own bbox_nms.py loop.  Inputs: tests/nms_oracle.py."""
from fractions import Fraction

import numpy as np
import pytest
import torch

import nms_oracle as NO
from oracle import bags_oracle as O
from oracle import ref_shim


def _f32_neighbours(t: np.float32):
    lo = np.nextafter(t, np.float32(0), dtype=np.float32)
    hi = np.nextafter(t, np.float32(1), dtype=np.float32)
    return [np.nextafter(lo, np.float32(0), dtype=np.float32), lo, t, hi, np.nextafter(hi, np.float32(1), dtype=np.float32)]


@pytest.mark.parametrize('thr', NO.THRESHOLDS)
def test_near_pairs_lie_next_to_a_rounding_boundary(thr):
    """Away from 0.5 each pair's rational IoU rounds to fp32(thr) or a neighbour and lies within 1/8 ulp of a rounding
    boundary among the five fp32 values around fp32(thr); at 0.5 it is 1/2 exactly or 1/(2 union) away from it.  The
    table hits fp32(thr) itself and at least one other value.  The fp32 restatement gives the correctly rounded quotient both ways round."""
    t = np.float32(thr)
    r = _f32_neighbours(t)
    rounded = set()
    assert len(NO.NEAR_PAIRS[thr]) >= 4
    for a, b in NO.NEAR_PAIRS[thr]:
        assert all(0 <= v <= 2047 and float(v).is_integer() for v in a + b)
        x = NO.exact_iou(a, b)
        assert NO.exact_iou(b, a) == x
        fx = NO.fp32_round(x)
        rounded.add(float(fx))
        if thr == 0.5:                                  # exactly 1/2, or as close as a union of this size gets
            assert x == Fraction(1, 2) or abs(x - Fraction(1, 2)) == Fraction(1, 2 * x.denominator), (a, b)
        else:
            assert fx in (Fraction(float(r[1])), Fraction(float(t)), Fraction(float(r[3]))), (a, b, float(x))
            dist = min(abs(x - (Fraction(float(r[i])) + Fraction(float(r[i + 1]))) / 2) for i in range(4))
            spacing = Fraction(float(r[3])) - Fraction(float(t))
            assert 0 < dist < spacing / 8, (a, b)
        for p, q in ((a, b), (b, a)):
            got = O.iou_plus1_fp32(np.array(p, np.float32), np.array(q, np.float32))
            assert Fraction(float(got)) == fx, (p, q, float(got), float(fx))
    assert float(t) in rounded and len(rounded) >= 2


def test_restatement_iou_equals_rational_rounding_across_exact_tier():
    """iou_plus1_fp32 = fp32_round(exact rational IoU) for every pair of integer boxes of the exact tier (random,
    clustered, the hand-made edges with finite coordinates); a union of 0 gives NaN."""
    g = np.random.default_rng(7)
    sets = [NO.random_int_boxes(g, 60), NO.clustered_int_boxes(g, 80)]
    sets += [b for name, b, _ in NO.edge_sets(g) if np.isfinite(b).all()]
    checked = nan = 0
    for boxes in sets:
        m = O.iou_plus1_fp32(boxes[:, None, :], boxes[None, :, :])
        for i in range(len(boxes)):
            for j in range(len(boxes)):
                a, b = boxes[i].tolist(), boxes[j].tolist()
                w = max(min(a[2], b[2]) - max(a[0], b[0]) + 1, 0)
                h = max(min(a[3], b[3]) - max(a[1], b[1]) + 1, 0)
                union = (a[2] - a[0] + 1) * (a[3] - a[1] + 1) + (b[2] - b[0] + 1) * (b[3] - b[1] + 1) - w * h
                if union == 0:
                    assert np.isnan(m[i, j]) if w * h == 0 else np.isinf(m[i, j])
                    nan += 1
                    continue
                assert Fraction(float(m[i, j])) == NO.fp32_round(NO.exact_iou(a, b)), (a, b)
                checked += 1
    assert checked > 10000 and nan > 0


def test_greedy_scan_equals_brute_force():
    """greedy_keep (removal bits ORed by alive rows) = brute_greedy (compare with every kept box) on the exact tier,
    NaN / inf coordinates and the thresholds -0.5, 0, 1, 0.999999 included, and on float boxes."""
    g = np.random.default_rng(11)
    cases = [(b, thrs) for _, b, thrs in NO.edge_sets(g)]
    cases += [(NO.clustered_int_boxes(g, 150), (0.3, 0.5, 0.7)), (NO.random_int_boxes(g, 150, max_wh=900), (0.45, 0.6))]
    fb, _ = NO.realistic_inputs(torch.Generator().manual_seed(2), n=200, classes=2)
    cases.append((fb.numpy(), (0.5,)))
    for thr in NO.THRESHOLDS:
        cases.append((np.array([q for pair in NO.NEAR_PAIRS[thr] for q in pair], np.float32), (thr,)))
    for boxes, thrs in cases:
        for thr in thrs:
            assert np.array_equal(O.greedy_keep(boxes, thr), NO.brute_greedy(boxes, thr)), thr


def test_nms_plus1_returns_ascending_indices_after_score_order_visit():
    """nms_plus1 visits by descending score (ties: lower index first) and returns the kept rows ascending."""
    g = np.random.default_rng(3)
    boxes = NO.clustered_int_boxes(g, 120)
    scores = g.permutation(120).astype(np.float32) / 120
    scores[::7] = 0.5                                  # ties
    dets = torch.from_numpy(np.concatenate([boxes, scores[:, None]], 1))
    kept, inds = O.nms_plus1(dets, 0.5)
    order = np.argsort(-scores, kind='stable')
    want = np.sort(order[NO.brute_greedy(boxes[order], 0.5)])
    assert inds.tolist() == want.tolist() and torch.equal(kept, dets[inds])


needs_ref = pytest.mark.skipif(not ref_shim.available(), reason='no reference checkout')


def _mc_inputs(seed, n, classes, per_class, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    xy = torch.randint(0, 300, (n, 2), generator=g).float()
    wh = torch.randint(1, 90, (n, 2), generator=g).float()
    b4 = torch.cat([xy, xy + wh], 1)
    boxes = (b4[:, None, :] + torch.randint(0, 6, (n, classes, 4), generator=g)).reshape(n, 4 * classes) \
        if per_class else b4
    scores = (torch.rand(n, classes, generator=g) ** 2).to(dtype)
    return boxes, scores


@needs_ref
@pytest.mark.parametrize('per_class', [False, True])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float16, torch.bfloat16])
def test_reference_loop_equals_oracle_order_included(per_class, dtype):
    """The reference's bbox_nms.py (with the restatement as its NMS op) = O.multiclass_nms, dets bit for bit, labels
    and order, with and without a cut, for fp32 / fp16 / bf16 scores -- including scores equal to the threshold
    rounded to the scores' dtype (fp16(0.3) = 0.30004883 is not > 0.3 in fp16, though it is > 0.3 in fp32)."""
    ref_mc = ref_shim.load_multiclass_nms(O.nms_plus1)
    boxes, scores = _mc_inputs(5, 80, 12, per_class, dtype)
    scores[::5, 3] = torch.tensor(0.3).to(dtype)
    scores[::4, 5] = torch.tensor(0.05).to(dtype)
    scores[1, 2] = float('nan')
    for thr, iou, k in ((0.3, 0.5, 10 ** 6), (0.05, 0.45, 10 ** 6), (0.3, 0.6, 15), (0.05, 0.5, -1), (0.0, 0.7, 0)):
        want = ref_mc(boxes, scores.clone(), thr, dict(type='nms', iou_thr=iou), k)
        got = O.multiclass_nms(boxes, scores.clone(), thr, iou, k)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), (thr, iou, k)
    half_thr = O.multiclass_nms(boxes, scores, 0.3, 0.5, 10 ** 6)
    if dtype != torch.float32:                          # the rows at exactly dtype(0.3) are not candidates
        assert not any(r[4] == float(torch.tensor(0.3).to(dtype)) for r in half_thr[0].tolist())
