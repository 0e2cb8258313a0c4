"""CPU: the float64 references of tests/test_gpu_fused_fwd_vs_float64.py (tests/fused_fwd_ref.py) against the oracle
(oracle/bags_oracle.py: GSBBoxHeadWith0's sliced cross entropy and its closed-form dz; tests/reweight_oracle.py:
mmdet's accuracy), and the GPU file's case table against the parameter space it claims to sample.  The GPU tests run
on an H100 only, so their reference is checked where it can be."""
import math

import torch

import focal_oracle as FO
import fused_fwd_ref as R
import reweight_oracle as RW
from oracle import bags_oracle as O


def _grouped_case(seed=0):
    g = torch.Generator().manual_seed(seed)
    slices = [(0, 3), (3, 1), (4, 5), (9, 3)]
    C, G, N, classes = 12, 4, 40, 9
    lens = torch.tensor([ln for _, ln in slices])
    l2b = (torch.rand(G, classes, generator=g) * lens[:, None]).long()
    labels = torch.randint(0, classes, (N,), generator=g)
    z = torch.randn(N, C, generator=g, dtype=torch.float64) * 3
    wm = (torch.rand(G, N, generator=g) < 0.6).long()
    wm[1] = 0
    avg = [max(float(wm[i].sum()), 1.0) for i in range(G)]
    return z, slices, l2b, labels, classes, wm, avg


def test_softmax_ce_matches_the_oracle():
    """Loss per bin and dz of a grouped case with in-range labels and table entries: equal to the oracle's
    bags_loss (F.cross_entropy over the slices, weight_reduce_loss with avg_factor) and closed_form_grads."""
    z, slices, l2b, labels, classes, wm, avg = _grouped_case()
    G = len(slices)
    targets = R.bin_targets(labels, l2b, slices, classes)
    for i in range(G):
        assert torch.equal(targets[i], l2b[i][labels])
    coef = wm.double() / torch.tensor(avg, dtype=torch.float64)[:, None]
    dz, lse, loss, coef_col, terms = R.softmax_ce(z, slices, targets, coef)
    remapped = ([l2b[i][labels] for i in range(G)], [wm[i] for i in range(G)], avg)
    ps = torch.tensor(slices, dtype=torch.long)
    ref = O.bags_loss(z, labels, l2b, ps, remapped=remapped)
    for i in range(G):
        r = ref['loss_cls_bin%d' % i].item()
        assert abs(loss[i].item() - r) <= 1e-12 * max(1.0, abs(r)), (i, loss[i].item(), r)
    # closed_form_grads computes z = x W^T + b; x = I, W = z^T, b = 0 gives z itself
    N, C = z.shape
    dz_ref = O.closed_form_grads(torch.eye(N, dtype=torch.float64), z.t().contiguous(), torch.zeros(C, dtype=torch.float64),
                                 labels, l2b, ps, remapped)[0]
    assert torch.allclose(dz, dz_ref, rtol=0, atol=1e-14)
    for i, (s, ln) in enumerate(slices):
        assert torch.allclose(lse[:, i], torch.logsumexp(z[:, s:s + ln], 1), rtol=0, atol=1e-14)
        assert bool((coef_col[:, s:s + ln] == coef[i][:, None]).all())


def test_out_of_range_labels_and_entries_take_the_first_column():
    """A label outside [0, classes) and a table entry outside [0, len_g) are scored against the bin's column 0."""
    _, slices, l2b, labels, classes, _, _ = _grouped_case(1)
    l2b[:, 0] = torch.tensor([ln for _, ln in slices])
    l2b[:, 1] = -1
    labels[:6] = torch.tensor([0, 1, -1, classes, classes + 5, 2])
    t = R.bin_targets(labels, l2b, slices, classes)
    assert bool((t[:, :5] == 0).all())
    assert torch.equal(t[:, 5], l2b[:, 2])
    t1 = R.bin_targets(torch.tensor([-1, 0, 3, 4]), None, [(0, 4)], 4)
    assert t1.tolist() == [[0, 0, 3, 0]]


def test_top1_count_is_mmdets_accuracy_without_ties():
    """Without ties top1_count is mmdet's accuracy count (pred.topk(1) == target): labels -1, C and C + 5 never count,
    even where column 0 is the row maximum."""
    g = torch.Generator().manual_seed(2)
    N, C = 300, 17
    z = torch.randn(N, C, generator=g, dtype=torch.float64)
    labels = torch.randint(0, C, (N,), generator=g)
    labels[::2] = z[::2].argmax(1)
    z[5::7, 0] = 10.0
    labels[5::21], labels[12::21], labels[19::21] = -1, C, C + 5
    want = RW.accuracy(z, labels).item() * N / 100.0
    assert R.top1_count(z, labels) == round(want)
    assert R.top1_count(z, labels) > 0
    # a tie with the row maximum counts
    zt = torch.zeros(2, 4, dtype=torch.float64)
    assert R.top1_count(zt, torch.tensor([3, -1])) == 1


def test_focal_matches_the_op_oracle_where_it_is_well_conditioned():
    """fused_fwd_ref.focal against the op's float64 restatement for |z| <= 12, where the oracle's 1 - p keeps at
    least 10 digits; every target convention (in range, 1, C, 0, negative, past C) and gamma 0 included."""
    g = torch.Generator().manual_seed(4)
    N, C = 64, 9
    z = (torch.rand(N, C, generator=g, dtype=torch.float64) * 24 - 12)
    z[:, 0] = 0.0
    t = torch.randint(1, C + 1, (N,), generator=g)
    t[:7] = torch.tensor([1, C, 0, -1, -3, C + 1, C + 5])
    for gamma, alpha in ((2.0, 0.25), (0.5, 1.0), (0.0, 0.25), (1.5, 0.75)):
        l, gr = R.focal(z, t, gamma, alpha)
        assert torch.allclose(l, FO.op_forward(z, t, gamma, alpha), rtol=1e-9, atol=1e-300)
        assert torch.allclose(gr, FO.op_backward(z, t, gamma, alpha), rtol=1e-9, atol=1e-300)
        assert bool((l[3:5] == 0).all()) and bool((gr[3:5] == 0).all())
    # far out, where the oracle's 1 - p is 0, q = exp(-z) / (1 + exp(-z)) keeps the positive element's gradient
    l, gr = R.focal(torch.tensor([[60.0]], dtype=torch.float64), torch.tensor([1]), 0.0, 0.25)
    assert abs(gr.item() + 0.25 * math.exp(-60.0)) <= 1e-12 * 0.25 * math.exp(-60.0)


def test_colsum_is_the_row_ordered_fp32_sum():
    g = torch.Generator().manual_seed(3)
    N, C = 300, 5
    dz = (torch.randn(N, C, generator=g) * 1e3).to(torch.bfloat16)
    got = R.colsum_fp32(dz, N)
    assert got.shape == (3, C) and got.dtype == torch.float32
    for t in range(3):
        for c in range(C):
            s = torch.zeros((), dtype=torch.float32)
            for r in range(128 * t, min(N, 128 * t + 128)):
                s = s + dz[r, c].float()
            assert got[t, c].item() == s.item()


def test_case_table_covers_the_parameter_space():
    """Every C of its entry point, every K and every N in both operand dtypes for each entry point, and the knobs the
    GPU file claims to sample."""
    import test_gpu_fused_fwd_vs_float64 as T
    for entry, cs in (('grouped', sorted(T.GROUPED_TABLES)), ('ce', T.SINGLE_CS), ('focal', T.SINGLE_CS)):
        for dt in ('fp32', 'bf16'):
            sub = [c for c in T.CASES if c['entry'] == entry and c['dtype'] == dt]
            assert sorted(c['C'] for c in sub) == sorted(cs), (entry, dt)
            assert set(T.KS) <= {c['K'] for c in sub}, (entry, dt)
            assert set(map(str, T.NS)) <= {str(c['N']) for c in sub}, (entry, dt)
            for knob in ('wide', 'ldx_pad', 'clear', 'bias'):
                assert {c[knob] for c in sub} == {True, False}, (entry, dt, knob)
            assert {c['ldd'] for c in sub} == {'pad64', 'r8p8'}
            if entry != 'grouped':
                assert {c['acc'] for c in sub} == {True, False}
    g = [c for c in T.CASES if c['entry'] == 'grouped']
    assert {(c['weights'], c['avg']) for c in g} >= {('u8', True), ('f32', True), (None, True), (None, False)}
    for C, (a, b) in T.GROUPED_TABLES.items():
        for starts in (a, b):
            assert starts[0] == 0 and starts == sorted(set(starts)) and starts[-1] < C and C % 4 == 0
            assert len(starts) <= 6
    edges = {s for a, b in T.GROUPED_TABLES.values() for s in a + b}
    assert {319, 320, 321, 639, 640, 641, 959, 960, 961} <= edges
    assert {s % 8 for s in edges if s % 320} == set(range(8))
