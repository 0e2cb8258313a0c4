"""GPU: the class-aware hard NMS -- bags_class_nms_dense and its host glue ops.multiclass_nms -- against the reference's
own compiled NMS op (oracle/_ref/, built by oracle/ref_build.py from mmdet/ops/nms) and the fp32 restatement
(oracle.bags_oracle.greedy_keep / multiclass_nms), at its edges.  Inputs: tests/nms_oracle.py.

  * exact tier: integer coordinates, so the IEEE division is the only rounding; keep bits equal the restatement and
    the reference op bit for bit -- the near-threshold pair table, suppression chains across the 32-bit word edges,
    a row suppressing a column two and three words on, identical / touching / zero-width / inverted boxes, a union of
    0 (NaN IoU), NaN and +-inf coordinates, iou_thr -0.5, 0, 1 and 0.999999.
  * kernel level: bags_class_nms_dense called directly with crafted order and counts; the keep buffer is filled with
    a sentinel and framed by a sentinel row on each side, so every byte it must write (0 past a class's count) and
    every byte it must not are checked.  Counts at every word edge up to 1024, above 1024 (the overflow flag is set
    and the first 1024 candidates are still exact), above n and below 0; n above 1024; 1, 7 and 1230 classes in one
    launch with 4 or 4 (S + 1) box columns.
  * ops level: ops.multiclass_nms against O.multiclass_nms with the reference op plugged in and with the restatement:
    dets bit for bit, labels, and their order.  Equal scores inside a class are visited lower RoI index first (ops'
    stable sort); the reference op's unstable sort leaves that order open, so tie cases compare with the
    restatement only, and a cut that splits a group of equal scores compares that group as a multiset.
  * realistic tier: decoded float boxes at the LVIS test shape (1000 RoIs x 1231 classes); every DECIDED class
    (nms_oracle.decided) must keep exactly what the reference op and the restatement keep.
"""
import numpy as np
import pytest
import torch

import nms_oracle as NO
from balancedgroupsoftmax_b200 import _native as nat
from balancedgroupsoftmax_b200 import ops
from oracle import bags_oracle as O
from oracle import ref_nms

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
SENT = 0xA5
MAX_SEG = 1024


def _ref_available():
    assert ref_nms.available(), 'the reference NMS op is not built (oracle/ref_build.py)'


def kernel_keep(boxes: np.ndarray, order: np.ndarray, counts, thr: float):
    """bags_class_nms_dense on boxes [n, cols] fp32, order [S, n], counts [S] -> (keep [S, n] uint8, overflow)."""
    S, n = order.shape
    b = torch.from_numpy(np.ascontiguousarray(boxes, dtype=np.float32)).to(DEV)
    o = torch.from_numpy(np.ascontiguousarray(order, dtype=np.int32)).to(DEV)
    c = torch.tensor(np.asarray(counts, dtype=np.int32)).to(DEV)
    frame = torch.full((S + 2, n), SENT, dtype=torch.uint8, device=DEV)
    ovf = torch.zeros(1, dtype=torch.int32, device=DEV)
    keep = frame[1:S + 1]
    nat.check(nat.lib().bags_class_nms_dense(b.data_ptr(), b.shape[1], o.data_ptr(), c.data_ptr(), S, n, float(thr),
                                             keep.data_ptr(), ovf.data_ptr(), torch.cuda.current_stream().cuda_stream),
              'bags_class_nms_dense')
    f = frame.cpu().numpy()
    assert (f[0] == SENT).all() and (f[-1] == SENT).all(), 'keep written outside its rows'
    return f[1:S + 1], int(ovf.item())


def expected_keep(boxes: np.ndarray, order: np.ndarray, counts, thr: float) -> np.ndarray:
    S, n = order.shape
    cols = boxes.shape[1]
    out = np.zeros((S, n), dtype=np.uint8)
    for s in range(S):
        cnt = max(min(int(counts[s]), n, MAX_SEG), 0)
        coff = 0 if cols == 4 else 4 * (s + 1)
        out[s, :cnt] = O.greedy_keep(boxes[order[s, :cnt], coff:coff + 4], thr)
    return out


def ref_keep(boxes4: np.ndarray, thr: float) -> np.ndarray:
    """The reference op on boxes visited in row order (distinct descending scores) -> bool keep."""
    m = boxes4.shape[0]
    scores = (m - np.arange(m)).astype(np.float32)
    dets = torch.from_numpy(np.concatenate([boxes4.astype(np.float32), scores[:, None]], 1)).to(DEV)
    inds = ref_nms.nms(dets, thr).cpu().numpy()
    assert np.array_equal(inds, np.sort(inds)), 'the reference op returns ascending indices'
    keep = np.zeros(m, dtype=bool)
    keep[inds] = True
    return keep


def _one_class(boxes4, thr):
    n = boxes4.shape[0]
    return kernel_keep(boxes4, np.arange(n)[None, :], [n], thr)


# ------------------------------------------------------------------------------------------------ exact tier
EDGE_NAMES = [name for name, _, _ in NO.edge_sets(np.random.default_rng(0))]


@pytest.mark.parametrize('name', EDGE_NAMES)
def test_exact_edges_keep_bits(name):
    _ref_available()
    boxes, thrs = {nm: (b, t) for nm, b, t in NO.edge_sets(np.random.default_rng(0))}[name]
    for thr in thrs:
        want = O.greedy_keep(boxes, thr)
        got, ovf = _one_class(boxes, thr)
        assert ovf == 0
        assert np.array_equal(got[0].astype(bool), want), (name, thr, np.flatnonzero(got[0].astype(bool) != want))
        assert np.array_equal(ref_keep(boxes, thr), want), (name, thr)


@pytest.mark.parametrize('thr', NO.THRESHOLDS)
def test_near_threshold_pairs_one_class_each(thr):
    """Every NEAR_PAIRS pair, both ways round, as its own class of one launch (per-class box columns): the second box
    survives exactly when fp32_round(rational IoU) <= fp32(thr); the reference op agrees pair by pair."""
    _ref_available()
    pairs = [(a, b) for a, b in NO.NEAR_PAIRS[thr]] + [(b, a) for a, b in NO.NEAR_PAIRS[thr]]
    S = len(pairs)
    boxes = np.zeros((2, 4 * (S + 1)), dtype=np.float32)
    for s, (a, b) in enumerate(pairs):
        boxes[0, 4 * (s + 1):4 * (s + 2)] = a
        boxes[1, 4 * (s + 1):4 * (s + 2)] = b
    got, _ = kernel_keep(boxes, np.tile(np.arange(2), (S, 1)), [2] * S, thr)
    t = NO.fp32_round(NO.Fraction(float(np.float32(thr))))
    for s, (a, b) in enumerate(pairs):
        survives = NO.fp32_round(NO.exact_iou(a, b)) <= t
        assert got[s].tolist() == [1, int(survives)], (a, b)
        assert ref_keep(np.array([a, b], np.float32), thr).tolist() == [True, survives], (a, b)


@pytest.mark.parametrize('n', [1, 2, 31, 32, 33, 64, 65, 300, 1024])
def test_exact_random_boxes_keep_bits(n):
    _ref_available()
    g = np.random.default_rng(n)
    for boxes in (NO.clustered_int_boxes(g, n), NO.random_int_boxes(g, n, max_wh=1200)):
        for thr in (0.3, 0.5, 0.7):
            want = O.greedy_keep(boxes, thr)
            got, _ = _one_class(boxes, thr)
            assert np.array_equal(got[0].astype(bool), want), (n, thr)
            assert np.array_equal(ref_keep(boxes, thr), want), (n, thr)


# ------------------------------------------------------------------------------------------------ kernel level
COUNTS = [0, 1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 992, 1000, 1023, 1024]


@pytest.mark.parametrize('cnt', COUNTS)
def test_kernel_counts_at_word_edges(cnt):
    """Three classes of one launch with their own visiting orders: counts cnt, cnt // 3 and n + 5 (> n, so clamped);
    n = cnt + 9 so there is a tail of zeros to write after every count."""
    g = np.random.default_rng(100 + cnt)
    n = cnt + 9
    boxes = NO.clustered_int_boxes(g, n, clusters=max(2, n // 40))
    order = np.stack([g.permutation(n) for _ in range(3)])
    counts = [cnt, cnt // 3, n + 5]
    for thr in (0.5, 0.3):
        got, ovf = kernel_keep(boxes, order, counts, thr)
        assert ovf == (1 if n > MAX_SEG else 0)
        assert np.array_equal(got, expected_keep(boxes, order, counts, thr)), (cnt, thr)


@pytest.mark.parametrize('cnt', [1025, 2048])
def test_kernel_overflow_flags_and_keeps_first_1024_exact(cnt):
    g = np.random.default_rng(cnt)
    n = 2048
    boxes = NO.clustered_int_boxes(g, n, clusters=40)
    order = np.stack([g.permutation(n), g.permutation(n)])
    counts = [cnt, 17]
    got, ovf = kernel_keep(boxes, order, counts, 0.5)
    assert ovf == 1
    assert np.array_equal(got, expected_keep(boxes, order, counts, 0.5))
    assert not got[0, MAX_SEG:].any()


def test_kernel_n_above_1024_counts_above_n_and_negative():
    g = np.random.default_rng(5)
    for n, counts in ((1500, [1024, 700, 0, 1]), (300, [500, -3, 300, 299]), (40, [-3, 2 ** 31 - 1, 40, 39])):
        boxes = NO.clustered_int_boxes(g, n, clusters=10)
        order = np.stack([g.permutation(n) for _ in counts])
        got, ovf = kernel_keep(boxes, order, counts, 0.45)
        assert ovf == 0, (n, counts)
        assert np.array_equal(got, expected_keep(boxes, order, counts, 0.45)), (n, counts)


@pytest.mark.parametrize('S', [1, 7, 1230])
@pytest.mark.parametrize('per_class', [False, True])
def test_kernel_many_classes_mixed_counts(S, per_class):
    """S classes with counts from 0 to n in one launch; with per-class columns every class has its own boxes (class
    0, the background, holds boxes that would suppress everything, so a one-class-off column shows)."""
    g = np.random.default_rng(S * 2 + per_class)
    n = 96 if S == 1230 else 400
    if per_class:
        boxes = np.concatenate([np.tile(np.array([[0, 0, 2047, 2047]], np.float32), (n, 1))] +
                               [NO.clustered_int_boxes(g, n, clusters=4) for _ in range(S)], 1)
    else:
        boxes = NO.clustered_int_boxes(g, n, clusters=8)
    order = np.stack([g.permutation(n) for _ in range(S)])
    counts = g.integers(0, n + 1, S)
    counts[:min(S, 3)] = [n, 0, 33][:min(S, 3)]
    got, ovf = kernel_keep(boxes, order, counts, 0.5)
    assert ovf == 0
    assert np.array_equal(got, expected_keep(boxes, order, counts, 0.5))


# ------------------------------------------------------------------------------------------------ ops level
def _ops_inputs(seed, n=120, classes=9, per_class=False, quant=None):
    g = torch.Generator().manual_seed(seed)
    xy = torch.randint(0, 400, (n, 2), generator=g).float()
    wh = torch.randint(8, 120, (n, 2), generator=g).float()
    b4 = torch.cat([xy, xy + wh], 1)
    boxes = (b4[:, None, :] + torch.randint(0, 9, (n, classes, 4), generator=g)).reshape(n, 4 * classes) \
        if per_class else b4
    if quant is None:     # distinct scores everywhere
        scores = (torch.randperm(n * classes, generator=g).float() / (n * classes)).reshape(n, classes)
    else:
        scores = torch.randint(0, quant, (n, classes), generator=g).float() / quant
    return boxes, scores


def _run_ops(boxes, scores, thr, iou, k):
    d, l = ops.multiclass_nms(boxes.to(DEV), scores.to(DEV), thr, iou, k)
    return d.cpu(), l.cpu()


def _assert_same(got, want, what):
    assert got[0].shape == want[0].shape, (what, got[0].shape, want[0].shape)
    assert torch.equal(got[1], want[1].cpu()), what
    assert np.array_equal(got[0].numpy().view(np.int32), want[0].cpu().float().numpy().view(np.int32)), what


def _both(boxes, scores, thr, iou, k, ref=True):
    got = _run_ops(boxes, scores, thr, iou, k)
    _assert_same(got, O.multiclass_nms(boxes, scores, thr, iou, k), ('restatement', thr, iou, k))
    if ref:
        want = O.multiclass_nms(boxes.to(DEV), scores.to(DEV), thr, iou, k, nms_op=ref_nms.nms_wrapper_op)
        _assert_same(got, want, ('reference op', thr, iou, k))
    return got


@pytest.mark.parametrize('per_class', [False, True])
def test_ops_no_cut_and_distinct_cut_order_included(per_class):
    """Without a cut the output is class-major, ascending RoI index inside a class; with a cut, descending score."""
    _ref_available()
    boxes, scores = _ops_inputs(1, per_class=per_class)
    for thr, iou, k in ((0.05, 0.5, 10 ** 6), (0.0, 0.3, 10 ** 6), (0.0, 0.5, 40), (0.5, 0.7, 25), (0.2, 0.45, 0),
                        (0.2, 0.45, -1), (0.2, 0.45, -2), (0.999, 0.5, 10 ** 6)):
        got = _both(boxes, scores, thr, iou, k)
        if 0 < k < 10 ** 6:
            assert got[0].shape[0] == k
    got = _both(boxes, scores, 0.05, 0.5, 10 ** 6)
    lab = got[1].numpy()
    assert (np.diff(lab) >= 0).all() and got[0].shape[0] > 50


def test_ops_cut_through_tied_scores():
    """Scores on a grid of 1/16: a cut at k splits a group of equal scores.  The scores match in order; each group of
    equal scores above the cut matches as a multiset, and the group at the cut is drawn from that score's survivors."""
    boxes, scores = _ops_inputs(2, quant=16)
    full = O.multiclass_nms(boxes, scores, 0.1, 0.5, 10 ** 6)
    for k in (7, 30, 61):
        got = _run_ops(boxes, scores, 0.1, 0.5, k)
        want = O.multiclass_nms(boxes, scores, 0.1, 0.5, k)
        assert torch.equal(got[0][:, 4], want[0][:, 4]) and got[0].shape[0] == k
        key = lambda d, l, m: sorted((int(a), tuple(r)) for a, r, keep in zip(l.tolist(), d.tolist(), m) if keep)
        v = float(want[0][-1, 4])
        above_g, above_w = (got[0][:, 4] > v).tolist(), (want[0][:, 4] > v).tolist()
        assert key(*got, above_g) == key(*want, above_w)
        at_g = key(*got, (got[0][:, 4] == v).tolist())
        pool = key(*full, (full[0][:, 4] == v).tolist())
        for item in at_g:
            pool.remove(item)                          # raises if a tied survivor is missing or repeated


def test_ops_ties_inside_a_class_follow_the_stable_convention():
    """Equal scores inside a class (no cut): visited lower RoI index first, as the restatement does."""
    boxes, scores = _ops_inputs(3, quant=8)
    for thr, iou in ((0.0, 0.5), (0.3, 0.3), (0.6, 0.7)):
        got = _run_ops(boxes, scores, thr, iou, 10 ** 6)
        _assert_same(got, O.multiclass_nms(boxes, scores, thr, iou, 10 ** 6), (thr, iou))


def test_ops_scores_at_the_threshold_nan_and_inf():
    """A score equal to fp32(score_thr) is not a candidate; NaN never is (it must not push out a genuine candidate);
    +inf is, and -inf is not.  One +inf in all, so no ties."""
    _ref_available()
    boxes, base = _ops_inputs(4)
    n, c = base.shape
    base[1::2, 3] = float('nan')
    base[:, 6] = float('nan')
    base[7, 1] = float('inf')
    for j in range(1, c):
        base[(5 * j + 1) % n, j] = float('-inf')
    for thr, iou, k in ((0.05, 0.5, 10 ** 6), (0.3, 0.5, 10 ** 6), (0.05, 0.5, 30), (0.3, 0.45, -1)):
        scores = base.clone()
        scores[::3, 2] = scores[::4, 4] = float(np.float32(thr))
        got = _both(boxes, scores, thr, iou, k)
        assert not torch.isnan(got[0]).any() and torch.isinf(got[0][:, 4]).sum() == 1
        assert (got[0][:, 4] != float(np.float32(thr))).all()


@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
def test_ops_half_precision_scores_compare_in_their_dtype(dtype):
    """score > score_thr in the scores' dtype: dtype(0.3) > 0.3 in fp32 but not in fp16 / bf16, so those rows are no
    candidates.  Scores distinct in fp32 would collide in half precision, so the restatement alone judges ties."""
    _ref_available()
    boxes, scores = _ops_inputs(5, classes=7)
    scores = scores.to(dtype)
    for thr in (0.3, 0.05):
        scores[::5, 2] = torch.tensor(thr).to(dtype)
        scores[1::7, 5] = torch.tensor(thr).to(dtype)
    for thr, iou, k in ((0.3, 0.5, 10 ** 6), (0.05, 0.5, 10 ** 6)):        # no cut: ties across classes stay apart
        got = _run_ops(boxes, scores, thr, iou, k)
        _assert_same(got, O.multiclass_nms(boxes, scores, thr, iou, k), (dtype, thr, k))
        assert (got[0][:, 4] > float(torch.tensor(thr).to(dtype))).all()
    # distinct half-precision scores below 0.5 (consecutive bit patterns of the dtype, permuted): the reference op
    # agrees, with rows at exactly dtype(0.3) in one class
    n, c = scores.shape
    top = 0x3F00 if dtype == torch.bfloat16 else 0x3800                  # the pattern of 0.5
    pats = top - 1 - torch.randperm(n * c, generator=torch.Generator().manual_seed(9))
    grid = pats.to(torch.int16).view(dtype).reshape(n, c)
    _both(boxes, grid, 0.1, 0.5, 33)
    grid[::5, 2] = torch.tensor(0.3).to(dtype)
    _both(boxes, grid, 0.3, 0.5, 10 ** 6)


def test_ops_accepts_a_misaligned_box_view():
    """A contiguous fp32 [n, 4] view one float into its storage (not 16-byte aligned) gives the aligned result."""
    boxes, scores = _ops_inputs(6)
    store = torch.empty(boxes.numel() + 1, device=DEV)
    view = store[1:].view(-1, 4)
    view.copy_(boxes.to(DEV))
    assert view.is_contiguous() and view.data_ptr() % 16
    for thr, iou, k in ((0.05, 0.5, 10 ** 6), (0.0, 0.5, 40)):
        got = ops.multiclass_nms(view, scores.to(DEV), thr, iou, k)
        _assert_same((got[0].cpu(), got[1].cpu()), _run_ops(boxes, scores, thr, iou, k), (thr, k))


def test_ops_more_than_1024_candidates_raises():
    boxes, scores = _ops_inputs(7, n=1100, classes=3)
    with pytest.raises(nat.BagsNativeError):
        ops.multiclass_nms(boxes.to(DEV), scores.to(DEV), -1.0, 0.5, 100)


# ------------------------------------------------------------------------------------------------ realistic tier
def _greedy_from_matrix(sup: np.ndarray) -> np.ndarray:
    m = sup.shape[0]
    removed = np.zeros(m, dtype=bool)
    for i in range(m):
        if not removed[i]:
            removed[i + 1:] |= sup[i, i + 1:]
    return ~removed


@pytest.mark.parametrize('score_thr', [0.0, 0.05])
def test_realistic_lvis_shape_decided_classes_exact(score_thr):
    """1000 decoded float boxes x 1231 classes.  Per class: kernel keep bits (ops' order and counts) = reference op
    = restatement in every decided class, and at least 99 % of classes are decided (on an H100 all 1230 are, at both
    thresholds; the floor sits just below that).  ops.multiclass_nms with
    max_per_img 10^6 (no cut) and 300 equals the reference loop on the decided classes, order included."""
    _ref_available()
    iou_thr = 0.5
    boxes, scores = NO.realistic_inputs(torch.Generator().manual_seed(1231))
    n, C = scores.shape
    S = C - 1
    sd = scores.to(DEV)
    cand = (sd[:, 1:] > score_thr).t()
    counts = cand.sum(1, dtype=torch.int32)
    key = torch.where(cand, sd[:, 1:].t(), float('-inf'))
    order = key.sort(dim=1, descending=True, stable=True).indices.to(torch.int32).cpu().numpy()
    counts = counts.cpu().numpy()
    bnp = boxes.numpy()
    got, ovf = kernel_keep(bnp, order, counts, iou_thr)
    assert ovf == 0
    sup32 = O.iou_plus1_fp32(bnp[:, None, :], bnp[None, :, :]) > np.float32(iou_thr)
    iou64 = NO.iou_matrix64(bnp)
    decided = np.zeros(S, dtype=bool)
    for s in range(S):
        o = order[s, :counts[s]]
        want = _greedy_from_matrix(sup32[np.ix_(o, o)])
        decided[s] = NO.decided(iou64[np.ix_(o, o)], want, iou_thr)
        if decided[s]:
            assert np.array_equal(got[s, :counts[s]].astype(bool), want), s
            assert np.array_equal(ref_keep(bnp[o], iou_thr), want), s
        assert not got[s, counts[s]:].any()
    frac = decided.mean()
    print('score_thr %g: %d of %d classes decided (%.4f); undecided: %s'
          % (score_thr, decided.sum(), S, frac, np.flatnonzero(~decided).tolist()[:50]))
    assert frac >= 0.99
    for k in (10 ** 6, 300):
        g_d, g_l = ops.multiclass_nms(boxes.to(DEV), sd, score_thr, iou_thr, k)
        w_d, w_l = O.multiclass_nms(boxes.to(DEV), sd, score_thr, iou_thr, k, nms_op=ref_nms.nms_wrapper_op)
        if decided.all():
            _assert_same((g_d.cpu(), g_l.cpu()), (w_d, w_l), k)
        elif k == 10 ** 6:
            mg, mw = decided[g_l.cpu().numpy()], decided[w_l.cpu().numpy()]
            _assert_same((g_d.cpu()[mg], g_l.cpu()[mg]), (w_d.cpu()[mw], w_l.cpu()[mw]), k)
