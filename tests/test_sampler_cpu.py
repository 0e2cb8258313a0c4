"""CPU: the restatement of the device sampler (tests/sampler_oracle.py) against the reference's rule and the quality
of its draws.

  * Against oracle/bags_oracle.sample_others (the reference's np.random.choice sampler): F, k, avg, the in-bin rows
    kept and exactly k others set agree over a few hundred seeded label vectors covering every mode; which others
    are chosen is the only difference.
  * The keys of one (seed, bin) are distinct over 2^20 rows, so "the k smallest keys" is well defined.
  * The draws of consecutive seeds (as the head's _next_seed gives them), of consecutive device step counters and
    of two bins on the same rows behave like independent uniform k-subsets: per-row inclusion, co-inclusion of row
    pairs (n^1, n+1, n^2048, n^4095: the key is mix32(h ^ n), so XOR partners matter), and overlaps, each held
    to 5 sigma on fixed seeds (the test is deterministic).
"""
import numpy as np
import pytest
import torch

import sampler_oracle as S
from oracle import bags_oracle as O


def _table(rng, G, classes):
    """label2bin [G, classes] with entries in {-2, ..., 3}: a class is in bin g when its entry is > 0."""
    t = rng.integers(-2, 4, size=(G, classes))
    t[:, 0] = 0
    return t


def _labels(rng, N, classes, p_bg):
    lab = rng.integers(1, classes, size=N)
    lab[rng.random(N) < p_bg] = 0
    return lab


def test_restatement_agrees_with_the_reference_sampler_except_for_the_draw():
    rng = np.random.default_rng(2024)
    ratios = [0.0, 0.5, 0.7, 1.0, 2.0, 8.0, 1e300]
    modes_seen = set()
    for case in range(300):
        G = int(rng.integers(2, 9))
        classes = int(rng.integers(2, 40))
        N = int(rng.integers(0, 300))
        table = _table(rng, G, classes)
        if case % 7 == 3:
            table[1] = 1                       # a bin that owns every class
        if case % 7 == 5:
            table[G - 1] = 0                   # a bin that owns none
        labels = _labels(rng, N, classes, p_bg=float(rng.choice([0.0, 0.5, 0.95])))
        ratio = ratios[case % len(ratios)]
        seed = int(rng.integers(0, 2 ** 63)) * 2 + case % 2
        wm, avg = S.sample(labels, table, ratio, seed)
        assert wm.shape == (G, N) and avg.dtype == np.float32
        assert (wm[0] == 1).all() and avg[0] == max(N, 1)
        np.random.seed(case)
        lab_t = torch.from_numpy(labels)
        for g in range(1, G):
            bin_label = torch.from_numpy(table[g])[lab_t]
            ref = O.sample_others(bin_label, ratio).numpy()
            ref_avg = max(float(ref.sum()), 1.0)
            F, Oth, k, mode = S.bin_counts(labels, table, ratio, g)
            modes_seen.add(mode)
            fg = S.in_bin(labels, table, g)
            assert F == int((bin_label > 0).sum())
            assert avg[g] == np.float32(ref_avg), (case, g, avg[g], ref_avg)
            assert int(wm[g].sum()) == int(ref.sum())
            assert (wm[g][fg] == ref[fg]).all()                      # in-bin rows: kept by both (or all zero)
            if mode == 3:
                assert (wm[g][fg] == 1).all() and int(wm[g][~fg].sum()) == k == int(F * ratio)
    assert modes_seen == {0, 1, 2, 3}


def test_restatement_edge_rules():
    """Out-of-range labels are others, an infinite ratio takes every other, and k truncates in float64."""
    table = np.array([[0, 0, 0], [0, 1, -1], [0, 0, 2], [0, 0, -4]])
    labels = np.array([1, -1, -2 ** 63, 3, 2 ** 40, 2, 0, 1])
    fg1 = S.in_bin(labels, table, 1)
    assert fg1.tolist() == [True, False, False, False, False, False, False, True]
    wm, avg = S.sample(labels, table, float('inf'), 5)                # bin 3 owns no row: zeros, avg 1
    assert (wm[:3] == 1).all() and (wm[3] == 0).all() and avg.tolist() == [8.0, 8.0, 8.0, 1.0]
    wm, avg = S.sample(labels, table, 0.0, 5)
    assert wm[1].tolist() == fg1.astype(np.uint8).tolist() and avg[1] == 2.0
    assert 90 * 0.7 < 63 and S.count_k(90, 0.7, 1000) == 62
    assert S.count_k(3, 0.5, 1000) == 1 and S.count_k(3, 1e300, 10) == 10
    assert S.effective_seed(7, -1) == (7 - 0x9E3779B97F4A7C15) % 2 ** 64
    assert S.effective_seed(7, None) == S.effective_seed(7, 0) == 7


@pytest.mark.parametrize('seed', [0, 1, 2 ** 64 - 1, 0x123456789ABCDEF0])
def test_keys_of_one_bin_are_distinct(seed):
    n = np.arange(1 << 20)
    for g in (1, 7):
        k = S.keys(seed, g, n)
        assert np.unique(k).size == n.size, (seed, g)


# ------------------------------------------------------------------------------------------------ quality
N_Q, F_Q, RATIO_Q, DRAWS = 4096, 400, 2.0, 4000
Z_MAX = 5.0


@pytest.fixture(scope='module')
def draws():
    rng = np.random.default_rng(0)
    fg = np.zeros(N_Q, dtype=bool)
    fg[rng.choice(N_Q, F_Q, replace=False)] = True
    others = np.nonzero(~fg)[0]
    k = int(F_Q * RATIO_Q)

    def draw(seed, g=1):
        kk = S.keys(seed, g, others)
        m = np.zeros(N_Q, dtype=bool)
        m[others[np.argpartition(kk, k - 1)[:k]]] = True
        return m

    base = (12345 * S.STEP_MUL) & S.MASK64
    seeds = [(base + s) & S.MASK64 for s in range(DRAWS)]                 # head._next_seed: consecutive seeds
    A = np.stack([draw(s) for s in seeds])
    B = np.stack([draw(S.effective_seed(base, s)) for s in range(DRAWS)])  # consecutive device step counters
    C = np.stack([draw(s, g=2) for s in seeds])                            # bin 2 on the same in-bin rows
    return dict(fg=fg, others=others, k=k, O=others.size, A=A, B=B, C=C)


def _chi2_z(D, others, p):
    cnt = D[:, others].sum(0)
    S_ = D.shape[0]
    chi = ((cnt - S_ * p) ** 2 / (S_ * p * (1 - p))).sum()
    df = others.size
    return (chi - df) / np.sqrt(2 * df)


def _overlap_z(X, Y, k, O):
    ov = (X & Y).sum(1)
    mean = k * k / O
    var = k * (k / O) * ((O - k) / O) * ((O - k) / (O - 1))     # hypergeometric
    return (ov.mean() - mean) / np.sqrt(var / ov.size)


def test_draws_are_exact_k_and_keep_the_in_bin_rows(draws):
    for D in (draws['A'], draws['B'], draws['C']):
        assert (D.sum(1) == draws['k']).all() and not D[:, draws['fg']].any()


@pytest.mark.parametrize('which', ['A', 'B'], ids=['consecutive_seeds', 'consecutive_steps'])
def test_per_row_inclusion_is_uniform(draws, which):
    z = _chi2_z(draws[which], draws['others'], draws['k'] / draws['O'])
    assert abs(z) < Z_MAX, z


@pytest.mark.parametrize('pair', ['n^1', 'n+1', 'n^2048', 'n^4095'])
def test_pairs_of_rows_are_co_included_at_the_uniform_rate(draws, pair):
    others, fg, A, k, Oth = draws['others'], draws['fg'], draws['A'], draws['k'], draws['O']
    partner = {'n^1': others ^ 1, 'n+1': others + 1, 'n^2048': others ^ 2048, 'n^4095': others ^ 4095}[pair]
    ok = (partner < N_Q) & ~fg[np.minimum(partner, N_Q - 1)]
    a, b = others[ok], partner[ok]
    q = k * (k - 1) / (Oth * (Oth - 1))
    co = (A[:, a] & A[:, b]).mean()
    z = (co - q) / np.sqrt(q * (1 - q) / (A.shape[0] * ok.sum()))
    assert abs(z) < Z_MAX, (pair, co, q, z)


def test_consecutive_draws_and_bins_overlap_like_independent_subsets(draws):
    A, B, C, k, Oth = draws['A'], draws['B'], draws['C'], draws['k'], draws['O']
    for what, X, Y in (('consecutive seeds', A[1:], A[:-1]), ('consecutive steps', B[1:], B[:-1]),
                       ('bins 1 and 2', A, C)):
        z = _overlap_z(X, Y, k, Oth)
        assert abs(z) < Z_MAX, (what, z)
