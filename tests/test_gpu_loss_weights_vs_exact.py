"""GPU: the loss-weight stage -- sample_others_kernel (all three instantiations), reweight_kernel and mask_avg_kernel,
which make the per-bin weights w[g, n] and normalisers avg[g] every loss of a training step divides by -- against exact
references.

Every reference is the numpy restatement in tests/sampler_oracle.py or float64, never this library.  The raw C ABI
is called through ctypes wherever the wrappers hide something: label2bin tables of any G and class count, the
seed_step pointer, and output buffers with room past their end.  The wmask / wfloat buffer has 256 bytes (64 floats)
past [G, N] filled with 0xA5 (-7.0), avg has kMaxG + 4 floats of -7.0; everything past [G, N] and avg[G:] must
survive.  Comparisons called bit-exact compare bit patterns.

Sampler (bags_sample_others), bit-exact: the wmask bytes and the avg bits equal sampler_oracle.sample.  N runs over
every instantiation -- <4> for N <= 4096 (0, 1, 31, 1000, 1023, 1024, 1025, 4095, 4096), <16> for N <= 16384 (4097,
10000, 16384), <0>, which re-reads its labels, above (16385, 65543, 2^20) -- with realistic tables (the synthetic
LVIS tables, G = 1, G = 8 over 1 and 3 classes, a bin owning every class and one owning none) and label mixes
(mostly background, all in one bin, labels -1 and INT64_MIN, labels classes and 2^40), and with tables built to
put bins exactly on every mode: F = 0, O = 0, k = 0, k = 1, k = O - 1, k = O, a truncated k (F = 90 at ratio 0.7 is
62, not 63), ratios 8, 1e300 and inf.  Seeds 0, 1, 2^64 - 1 and a pair differing only in the high word; the device
step counter absent, 0, 1, 2^40 and -1.  NaN or negative ratios and G outside [1, 8] are refused and launch nothing.
Captured in a CUDA graph, the sampler follows its step counter replay by replay, and GraphedHeadStep's first
replays draw what the restatement draws for its seed at steps 0, 1, 2 (checked through its per-bin losses on exact
logits: the float64 loss of the restated masks, within the fused forward's bound, which the loss of the next step's
masks is shown to miss).

Programmatic dependent launch, write after read: the sampler (and bags_mask_avg) launched right behind a fused
bags_fwd that reads the same wmask / avg buffers must not overwrite them while the forward reads them: the forward
matches the float64 reference built from the old buffers (the bounds of tests/test_gpu_fused_fwd_vs_float64.py),
and the buffers end up equal to the restatement.

bags_mask_avg, bit-exact: avg[g] = fp32(max(sum_n wmask[g, n], 1)) of the exact integer sum, bytes 0, 1 and 255 as
their values, including a sum above 2^24, which rounds once.

bags_reweight: wfloat = fp32(wmask byte * cls_weight[g, t]) bit-exact (one correctly rounded product; exact for a
0/1 mask), with t = label2bin[g, label] for a label in [0, classes) and 0 otherwise, and t outside [0, wstride)
read as 0 (the "others" weight); bin 0 keeps the mask itself; no mask means ones.  avg[g] = max(sum, 1):
  * exact tier: weights multiples of 2^-6 in [2^-6, 4], 0/1 masks, N <= 2^14: every partial sum is a multiple of
    2^-6 below 2^16 (asserted per case), 22 bits, so every fp32 addition is exact and avg equals float64 bit for bit;
  * numeric tier: |avg - ref| <= gamma_m sum_n |w|, gamma_m = m u / (1 - m u), u = 2^-24, m = ceil(N / 256) + 13.
    Every weight reaches avg through at most m fp32 additions: its thread's chain over rows t, t + 256, ... (at most
    ceil(N / 256)), the warp's 5 butterfly steps, and thread 0's chain over the 8 warp partials (8); a sum whose
    every addend passes through at most m roundings errs by at most gamma_m times the sum of magnitudes (Higham,
    Accuracy and Stability of Numerical Algorithms, 4.2).  The clamp to 1 does not widen the difference.
"""

import numpy as np
import pytest
import torch

import fused_fwd_ref as R
import sampler_oracle as S
import test_gpu_fused_fwd_vs_float64 as FF
from balancedgroupsoftmax_b200 import _native as nat
from balancedgroupsoftmax_b200.tables import synthetic_tables

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
KMAXG = nat.MAX_BINS
PAD_BYTES = 256
BYTE_SENT = 0xA5
SENT = -7.0
U = 2.0 ** -24
INT64_MIN = -2 ** 63
EPT4_MAX, EPT16_MAX = 4096, 16384       # bags_sample_others' dispatch: <4> up to 4096 rows, <16> up to 16384, else <0>
NS = [0, 1, 31, 1000, 1023, 1024, 1025, 4095, 4096, 4097, 10000, 16384, 16385, 65543, 1 << 20]
SEEDS = [0, 1, 2 ** 64 - 1, 0x0000000500000007, 0x0000000600000007]
STEPS = [None, 0, 1, 2 ** 40, -1]


def _stream():
    return torch.cuda.current_stream(DEV).cuda_stream


def instantiation(N):
    return 'ept4' if N <= EPT4_MAX else 'ept16' if N <= EPT16_MAX else 'ept0'


def test_sizes_cover_every_instantiation():
    by = {}
    for N in NS:
        by.setdefault(instantiation(N), []).append(N)
    assert sorted(by) == ['ept0', 'ept16', 'ept4']
    for inst, ns in by.items():
        assert any(n % 1024 for n in ns), inst
    assert EPT4_MAX in NS and EPT4_MAX + 1 in NS and EPT16_MAX in NS and EPT16_MAX + 1 in NS


# ------------------------------------------------------------------------------------------------ buffers
class Out:
    """A [G, N] output in a buffer with PAD_BYTES of sentinel past it, and avg [kMaxG + 4] of -7."""

    def __init__(self, G, N, dtype=torch.uint8):
        self.G, self.N, self.dtype = G, N, dtype
        if dtype == torch.uint8:
            self.buf = torch.full((G * N + PAD_BYTES,), BYTE_SENT, dtype=torch.uint8, device=DEV)
        else:
            self.buf = torch.full((G * N + PAD_BYTES // 4,), SENT, dtype=torch.float32, device=DEV)
        self.avg = torch.full((KMAXG + 4,), SENT, dtype=torch.float32, device=DEV)

    def values(self):
        return self.buf[:self.G * self.N].view(self.G, self.N).cpu().numpy()

    def avg_values(self):
        return self.avg[:self.G].cpu().numpy()

    def check_sentinels(self, what):
        tail = self.buf[self.G * self.N:].cpu()
        if self.dtype == torch.uint8:
            assert bool((tail == BYTE_SENT).all()), '%s: a byte past [G, N] was written' % what
        else:
            assert bool((tail == SENT).all()), '%s: a float past [G, N] was written' % what
        assert bool((self.avg[self.G:].cpu() == SENT).all()), '%s: avg past G was written' % what

    def untouched(self, what):
        self.G, self.N = 0, 0
        self.check_sentinels(what)


def same_bits(got, want, what):
    got, want = np.ascontiguousarray(got), np.ascontiguousarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if got.dtype == np.float32:
        got, want = got.view(np.int32), want.astype(np.float32).view(np.int32)
    bad = np.nonzero((got != want).reshape(-1))[0]
    if bad.size:
        i = int(bad[0])
        raise AssertionError('%s: %d of %d elements differ; first at %s: got %r, want %r' % (
            what, bad.size, got.size, np.unravel_index(i, got.shape), got.reshape(-1)[i], want.reshape(-1)[i]))


def run_sampler(labels, table, ratio, seed, step=None, G=None):
    """bags_sample_others through ctypes into sentinel buffers; returns (rc, Out)."""
    table = np.ascontiguousarray(table, dtype=np.int32)
    G = table.shape[0] if G is None else G
    classes = table.shape[1]
    N = len(labels)
    lab = torch.as_tensor(np.asarray(labels, dtype=np.int64), device=DEV)
    l2b = torch.as_tensor(table, device=DEV)
    out = Out(G, N)
    st = None if step is None else torch.tensor([step], dtype=torch.int64, device=DEV)
    rc = nat.lib().bags_sample_others(lab.data_ptr(), l2b.data_ptr(), N, G, classes, float(ratio),
                                      int(seed) & S.MASK64, nat.ptr(st), out.buf.data_ptr(), out.avg.data_ptr(),
                                      _stream())
    torch.cuda.synchronize()
    return rc, out


def check_sampler(labels, table, ratio, seed, step, what):
    rc, out = run_sampler(labels, table, ratio, seed, step)
    nat.check(rc, what)
    wm, avg = S.sample(labels, table, ratio, seed, step)
    same_bits(out.values(), wm, '%s: wmask' % what)
    same_bits(out.avg_values(), avg, '%s: avg' % what)
    out.check_sentinels(what)
    return wm


# ------------------------------------------------------------------------------------------------ sampler cases
def _realistic_table(name, rng):
    if name == 'lvis':
        return synthetic_tables().label2binlabel.astype(np.int32)
    if name == 'g1':
        return np.zeros((1, 7), dtype=np.int32)
    if name == 'g8c1':
        return np.array([[0], [1], [0], [2], [-1], [1], [0], [3]], dtype=np.int32)
    if name == 'g8c3':
        t = np.array([[0, 0, 0], [0, 1, 0], [0, 0, 1], [0, 2, 5], [0, -1, 1], [1, 1, 1], [0, 0, 0], [-3, 7, 0]])
        return t.astype(np.int32)
    if name == 'every_none':        # bin 1 owns every class, bin 2 none (zeros and negatives), bin 3 some
        t = np.zeros((4, 50), dtype=np.int32)
        t[1] = rng.integers(1, 9, 50)
        t[2, ::2] = -1
        t[3, 10:30] = np.arange(1, 21)
        return t
    raise KeyError(name)


def _realistic_labels(style, N, table, rng):
    classes = table.shape[1]
    lab = rng.integers(0, classes, N)
    if style == 'mostly_bg':
        lab[rng.random(N) < 0.8] = 0
    elif style == 'one_bin':
        g = table.shape[0] - 1
        owned = np.nonzero(table[g] > 0)[0]
        if owned.size:
            lab = owned[rng.integers(0, owned.size, N)]
    elif style == 'negative':
        r = rng.random(N)
        lab[r < 0.3] = -1
        lab[(r >= 0.3) & (r < 0.5)] = INT64_MIN
    elif style == 'too_large':
        r = rng.random(N)
        lab[r < 0.3] = classes
        lab[(r >= 0.3) & (r < 0.5)] = 2 ** 40
    return lab.astype(np.int64)


TABLES = ['lvis', 'g1', 'g8c1', 'g8c3', 'every_none']
STYLES = ['mostly_bg', 'one_bin', 'negative', 'too_large']
RATIOS = [8.0, 0.5, 0.7, 2.0, 0.0, 1e300, float('inf')]


def _realistic_cases():
    cases = []
    i = 0
    for N in NS:
        for tname in TABLES:
            cases.append(dict(N=N, table=tname, style=STYLES[i % len(STYLES)], ratio=RATIOS[i % len(RATIOS)],
                              seed=SEEDS[i % len(SEEDS)], step=STEPS[(i // 2) % len(STEPS)]))
            i += 1
    return cases


REALISTIC = _realistic_cases()


def _rid(c):
    return '%s-N%d-%s-%s-r%g-s%x-step%s' % (instantiation(c['N']), c['N'], c['table'], c['style'], c['ratio'],
                                             c['seed'], c['step'])


@pytest.mark.parametrize('case', REALISTIC, ids=[_rid(c) for c in REALISTIC])
def test_sampler_bit_exact_on_realistic_tables(case):
    rng = np.random.default_rng(case['N'] * 31 + TABLES.index(case['table']))
    table = _realistic_table(case['table'], rng)
    labels = _realistic_labels(case['style'], case['N'], table, rng)
    check_sampler(labels, table, case['ratio'], case['seed'], case['step'], _rid(case))


def _find_F(N, ratio, pred, guess):
    """An F in [1, N] within 8 of ``guess`` with pred(F, k = int(F ratio), O = N - F), or None."""
    for F in range(max(1, guess - 8), min(N, guess + 8) + 1):
        if pred(F, S.count_k(F, ratio, 1 << 62), N - F):
            return F
    return None


MODE_TARGETS = {
    'F=0': lambda N, r: 0,
    'O=0': lambda N, r: N if N else None,
    'k=0': lambda N, r: _find_F(N, r, lambda F, k, O: k == 0 and O > 0, 1),
    'k=1': lambda N, r: _find_F(N, r, lambda F, k, O: k == 1 and O > 1, int(1 / r) if r else 1),
    'k=O-1': lambda N, r: _find_F(N, r, lambda F, k, O: k == O - 1 and O > 1, int(N / (1 + r))),
    'k=O': lambda N, r: _find_F(N, r, lambda F, k, O: k == O and O > 0, int(N / (1 + r))),
    'trunc': lambda N, r: (90 if r == 0.7 and N > 153 else
                           _find_F(N, r, lambda F, k, O: F * r != int(F * r) and 1 < k < O - 1, N // 4)),
}
MODE_RATIOS = [0.7, 1.0, 0.5, 3.0]


def mode_problem(N, ratio, rng):
    """labels = a permutation of [0, N) (classes = N), G = 8: bin g owns a random F_g classes chosen to put it on
    the mode MODE_TARGETS[g - 1], so its in-bin rows are a random F_g-subset of the rows.  Owned entries are in
    [1, 1000], the others 0 or negative.  Returns (labels, table, {bin: target name})."""
    labels = rng.permutation(N).astype(np.int64)
    table = np.zeros((KMAXG, max(N, 1)), dtype=np.int32)
    table[:, ::3] = -rng.integers(1, 5, table[:, ::3].shape)
    hit = {}
    for g, (name, fn) in enumerate(MODE_TARGETS.items(), start=1):
        F = fn(N, ratio)
        if F is None:
            F = int(rng.integers(0, N + 1))
        else:
            hit[g] = name
        owned = rng.choice(N, F, replace=False) if F else np.zeros(0, dtype=np.int64)
        table[g, owned] = rng.integers(1, 1001, F)
    return labels, table, hit


@pytest.mark.parametrize('ratio', MODE_RATIOS)
@pytest.mark.parametrize('N', NS, ids=['%s-N%d' % (instantiation(n), n) for n in NS])
def test_sampler_bit_exact_on_every_mode(N, ratio):
    rng = np.random.default_rng(N + int(ratio * 10))
    labels, table, hit = mode_problem(N, ratio, rng)
    for g, name in hit.items():                       # the construction really puts bin g on its mode
        F, O, k, mode = S.bin_counts(labels, table, ratio, g)
        expect = {'F=0': F == 0, 'O=0': O == 0 and mode == 1, 'k=0': mode == 2, 'k=1': mode == 3 and k == 1,
                  'k=O-1': mode == 3 and k == O - 1, 'k=O': mode == 1 and int(F * ratio) == O,
                  'trunc': mode == 3 and F * ratio != k}[name]
        assert expect, (N, ratio, g, name, F, O, k, mode)
    if N > 153 and ratio == 0.7:
        assert 'trunc' in hit.values() and S.count_k(90, 0.7, N) == 62
    seed = SEEDS[(N + int(ratio * 10)) % len(SEEDS)]
    step = STEPS[N % len(STEPS)]
    check_sampler(labels, table, ratio, seed, step, 'modes N=%d ratio=%g' % (N, ratio))


def test_every_mode_is_reached_in_every_instantiation():
    for inst in ('ept4', 'ept16', 'ept0'):
        names = set()
        for N in NS:
            if instantiation(N) != inst:
                continue
            for r in MODE_RATIOS:
                names |= set(mode_problem(N, r, np.random.default_rng(0))[2].values())
        assert names == set(MODE_TARGETS), (inst, set(MODE_TARGETS) - names)


@pytest.mark.parametrize('N', [1000, 10000, 65543], ids=['ept4', 'ept16', 'ept0'])
def test_sampler_mixes_the_high_seed_word(N):
    rng = np.random.default_rng(5)
    table = synthetic_tables().label2binlabel.astype(np.int32)
    labels = _realistic_labels('mostly_bg', N, table, rng)
    a = check_sampler(labels, table, 2.0, SEEDS[3], None, 'seed lo')
    b = check_sampler(labels, table, 2.0, SEEDS[4], None, 'seed hi')
    assert any(S.bin_counts(labels, table, 2.0, g)[3] == 3 for g in range(1, 5))
    assert not np.array_equal(a, b), 'seeds that differ only in the high word drew the same masks'


@pytest.mark.parametrize('bad', ['nan', 'negative', 'G=0', 'G=9'])
def test_sampler_refuses_bad_arguments_and_launches_nothing(bad):
    table = np.ones((9, 4), dtype=np.int32)
    labels = np.arange(100) % 4
    ratio = {'nan': float('nan'), 'negative': -0.5}.get(bad, 2.0)
    G = {'G=0': 0, 'G=9': 9}.get(bad, 5)
    rc, out = run_sampler(labels, table, ratio, 3, None, G=G)
    assert rc != 0, bad
    out.untouched(bad)


# ------------------------------------------------------------------------------------------------ CUDA graphs
def test_captured_sampler_follows_its_step_counter():
    from balancedgroupsoftmax_b200 import ops
    t = synthetic_tables()
    dt = ops.DeviceTables.from_tables(t, DEV)
    rng = np.random.default_rng(11)
    N, ratio, seed = 3000, 4.0, 0xDEADBEEF12345678
    labels_np = _realistic_labels('mostly_bg', N, t.label2binlabel, rng)
    labels = torch.as_tensor(labels_np, device=DEV)
    c = torch.zeros((1,), dtype=torch.int64, device=DEV)
    ops.sample_others(labels, dt, ratio, seed, seed_step=c)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            wm, avg = ops.sample_others(labels, dt, ratio, seed, seed_step=c)
    torch.cuda.current_stream(DEV).wait_stream(side)
    seen = []
    for v in (0, 1, 7, -1, 2 ** 40, 1):
        c.fill_(v)
        graph.replay()
        torch.cuda.synchronize()
        want_wm, want_avg = S.sample(labels_np, t.label2binlabel, ratio, seed, v)
        same_bits(wm.cpu().numpy(), want_wm, 'replay at step %d: wmask' % v)
        same_bits(avg.cpu().numpy(), want_avg, 'replay at step %d: avg' % v)
        seen.append(want_wm)
    assert not np.array_equal(seen[0], seen[1]) and np.array_equal(seen[1], seen[-1])


def test_graphed_head_step_draws_the_restated_masks():
    """GraphedHeadStep's replays 0, 1, 2 on exact logits: each replay's per-bin losses equal the float64 losses of
    the masks the restatement draws for the step's seed at that step (within the fused forward's bound), and miss
    those of the following step."""
    from balancedgroupsoftmax_b200 import ops
    from balancedgroupsoftmax_b200.api import GraphedHeadStep
    t = synthetic_tables()
    dt = ops.DeviceTables.from_tables(t, DEV)
    slices = [tuple(int(v) for v in r) for r in t.pred_slice]
    C, classes, N, K, ratio = t.num_logits, t.num_classes, 1000, 128, 2.0
    X, Wm, b, _ = FF.make_problem(N, K, C, False, seed=31)
    z = FF._z(X, Wm, b, True)
    rng = np.random.default_rng(3)
    labels_np = _realistic_labels('mostly_bg', N, t.label2binlabel, rng)
    labels = torch.as_tensor(labels_np, device=DEV)
    W = torch.nn.Parameter(Wm.to(torch.bfloat16))
    bias = torch.nn.Parameter(b.float())
    step = GraphedHeadStep(W, bias, dt, N, others_sample_ratio=ratio, seed=0x0123456789ABCDEF)
    targets = R.bin_targets(labels, dt.label2bin, slices, classes)
    eps = R.eps_softmax(z.abs().max(1).values)

    def ref(s):
        wm, avg = S.sample(labels_np, t.label2binlabel, ratio, step.seed, s)
        coef = torch.as_tensor(wm, device=DEV).double() / torch.as_tensor(avg, device=DEV).double()[:, None]
        _, _, loss, _, terms = R.softmax_ce(z, slices, targets, coef)
        tol = (coef * eps).sum(1) + (4 + N + 300) * U * terms.sum(0)
        return loss, tol

    x = X.to(torch.bfloat16)
    for s in range(3):
        got = step(x, labels).double().clone()
        torch.cuda.synchronize()
        want, tol = ref(s)
        nxt, _ = ref(s + 1)
        assert bool(((got - want).abs() <= tol).all()), (s, got, want, tol)
        sampled = [g for g in range(1, t.num_bins) if S.bin_counts(labels_np, t.label2binlabel, ratio, g)[3] == 3]
        assert sampled and all(abs(float(nxt[g] - want[g])) > 10 * float(tol[g]) for g in sampled), (s, nxt, want)


# ------------------------------------------------------------------------------------------------ PDL write after read
@pytest.mark.parametrize('succ', ['sample_others', 'mask_avg'])
def test_pdl_successor_writes_after_the_forward_reads(succ):
    """bags_fwd (fused route) reads masks M1 and avg A1; bags_sample_others (or bags_mask_avg) is launched right
    behind it on the same stream and writes the same buffers.  The forward must have read M1 / A1 and the buffers
    must end as the restatement (or the mask sum)."""
    from balancedgroupsoftmax_b200 import ops
    t = synthetic_tables()
    dt = ops.DeviceTables.from_tables(t, DEV)
    slices = [tuple(int(v) for v in r) for r in t.pred_slice]
    G, C, classes = dt.G, t.num_logits, t.num_classes
    N, K, ratio, seed = 4096 + 77, 1028, 8.0, 77
    case = dict(dtype='bf16', C=C, K=K, wide=False, ldx_pad=True, ldd='pad64', bias=True)
    dtype, x, w, ld, bias, z, _, ldd = FF._operands(case, N)
    gen = torch.Generator(device=DEV).manual_seed(321)
    labels = torch.randint(0, classes, (N,), generator=gen, device=DEV)
    labels[::3] = 0
    m1 = (torch.rand(G, N, generator=gen, device=DEV) < 0.4).to(torch.uint8)
    a1 = torch.tensor([5.0, 3.0, 0.75, 2.0, 9.0], dtype=torch.float32, device=DEV)
    wm, avg = m1.clone(), a1.clone()
    out = FF.Outputs(N, C, G, dtype, ldd, True, False, 0)
    ws = ops._workspace(DEV)
    args = (x.data_ptr(), ld, w.data_ptr(), ld, bias.data_ptr(), labels.data_ptr(), dt.label2bin.data_ptr(),
            dt.slices_host, wm.data_ptr(), nat.WEIGHTS_U8, avg.data_ptr(), N, K, C, G, classes, FF._code(dtype), None,
            0, out.loss.data_ptr(), out.lse.data_ptr()) + out.tail(ws)
    torch.cuda.synchronize()
    lib = nat.lib()
    rc = lib.bags_fwd(*args)
    if succ == 'sample_others':      # immediately behind the forward, on the same stream
        rc2 = lib.bags_sample_others(labels.data_ptr(), dt.label2bin.data_ptr(), N, G, classes, ratio, seed, None,
                                     wm.data_ptr(), avg.data_ptr(), _stream())
    else:
        rc2 = lib.bags_mask_avg(wm.data_ptr(), N, G, avg.data_ptr(), _stream())
    nat.check(rc, 'bags_fwd')
    nat.check(rc2, succ)
    torch.cuda.synchronize()
    coef = m1.double() / a1.double()[:, None]
    targets = R.bin_targets(labels, dt.label2bin, slices, classes)
    out.check_layout('before %s' % succ)
    FF.check_softmax(out, z, slices, targets, coef, dtype, 'before %s' % succ)
    if succ == 'sample_others':
        want_wm, want_avg = S.sample(labels.cpu().numpy(), t.label2binlabel, ratio, seed)
        assert not np.array_equal(want_wm, m1.cpu().numpy())
    else:
        want_wm = m1.cpu().numpy()
        want_avg = S.mask_avg(want_wm).astype(np.float32)
    assert not np.array_equal(want_avg, a1.cpu().numpy())
    same_bits(wm.cpu().numpy(), want_wm, '%s: wmask' % succ)
    same_bits(avg.cpu().numpy(), want_avg, '%s: avg' % succ)


# ------------------------------------------------------------------------------------------------ bags_mask_avg
MASK_AVG_CASES = [(G, N, kind) for G, N, kind in [
    (1, 0, 'bytes'), (8, 0, 'bytes'), (1, 1, 'bytes'), (2, 255, 'bytes'), (3, 257, 'zeros'), (4, 1000, 'bytes'),
    (5, 4097, 'ones'), (6, 65543, 'bytes'), (7, 1 << 20, 'bytes'), (8, 70001, 'all255'), (8, 300001, 'all255')]]


@pytest.mark.parametrize('G,N,kind', MASK_AVG_CASES, ids=['G%d-N%d-%s' % c for c in MASK_AVG_CASES])
def test_mask_avg_bit_exact(G, N, kind):
    rng = np.random.default_rng(G * 7 + N)
    if kind == 'bytes':
        m = rng.choice(np.array([0, 1, 255], dtype=np.uint8), size=(G, N), p=[0.45, 0.45, 0.1])
    elif kind == 'zeros':
        m = np.zeros((G, N), dtype=np.uint8)
        m[0, 5] = 1
    elif kind == 'ones':
        m = np.ones((G, N), dtype=np.uint8)
    else:
        m = np.full((G, N), 255, dtype=np.uint8)
        m[1:, ::7] = 1
    out = Out(G, N)
    out.buf[:G * N] = torch.as_tensor(m.reshape(-1), device=DEV)
    nat.check(nat.lib().bags_mask_avg(out.buf.data_ptr(), N, G, out.avg.data_ptr(), _stream()), 'bags_mask_avg')
    torch.cuda.synchronize()
    exact = S.mask_avg(m)
    if kind == 'all255':
        assert (exact > 2 ** 24).any() and (exact.astype(np.float32).astype(np.int64) != exact).any()
    same_bits(out.avg_values(), exact.astype(np.float32), 'mask_avg G=%d N=%d' % (G, N))
    same_bits(out.values(), m, 'mask_avg input')
    out.check_sentinels('mask_avg')


def test_empty_batch_gives_unit_normalisers():
    """A batch without RoIs: the wrappers' empty tensors (and NULL pointers) are accepted and every avg is 1."""
    from balancedgroupsoftmax_b200 import ops
    dt = ops.DeviceTables.from_tables(synthetic_tables(), DEV)
    wm, avg = ops.sample_others(torch.zeros(0, dtype=torch.int64, device=DEV), dt, 8.0, 3)
    assert wm.shape == (dt.G, 0) and avg.tolist() == [1.0] * dt.G
    assert ops.mask_avg(torch.zeros((dt.G, 0), dtype=torch.uint8, device=DEV)).tolist() == [1.0] * dt.G
    out = Out(KMAXG, 0)
    l2b = torch.ones((KMAXG, 3), dtype=torch.int32, device=DEV)
    nat.check(nat.lib().bags_sample_others(None, l2b.data_ptr(), 0, KMAXG, 3, 2.0, 1, None, None,
                                           out.avg.data_ptr(), _stream()), 'bags_sample_others')
    torch.cuda.synchronize()
    same_bits(out.avg_values(), np.ones(KMAXG, dtype=np.float32), 'empty sampler: avg')
    out.check_sentinels('empty sampler')
    out = Out(KMAXG, 0)
    nat.check(nat.lib().bags_mask_avg(None, 0, KMAXG, out.avg.data_ptr(), _stream()), 'bags_mask_avg')
    torch.cuda.synchronize()
    same_bits(out.avg_values(), np.ones(KMAXG, dtype=np.float32), 'empty mask_avg: avg')
    out.check_sentinels('empty mask_avg')


@pytest.mark.parametrize('G', [0, 9])
def test_mask_avg_refuses_bad_bin_counts(G):
    out = Out(max(G, 1), 100)
    rc = nat.lib().bags_mask_avg(out.buf.data_ptr(), 100, G, out.avg.data_ptr(), _stream())
    torch.cuda.synchronize()
    assert rc != 0
    out.untouched('mask_avg G=%d' % G)


# ------------------------------------------------------------------------------------------------ bags_reweight
def run_reweight(labels, table, wmask, cls_weight):
    table = np.ascontiguousarray(table, dtype=np.int32)
    G, classes = table.shape
    wstride = cls_weight.shape[1]
    N = len(labels)
    lab = torch.as_tensor(np.asarray(labels, dtype=np.int64), device=DEV)
    l2b = torch.as_tensor(table, device=DEV)
    wm = None if wmask is None else torch.as_tensor(np.ascontiguousarray(wmask, dtype=np.uint8), device=DEV)
    cw = torch.as_tensor(np.ascontiguousarray(cls_weight, dtype=np.float32), device=DEV)
    out = Out(G, N, torch.float32)
    nat.check(nat.lib().bags_reweight(lab.data_ptr() if N else None, l2b.data_ptr(), nat.ptr(wm), cw.data_ptr(),
                                      wstride, N, G, classes, out.buf.data_ptr(), out.avg.data_ptr(), _stream()),
              'bags_reweight')
    torch.cuda.synchronize()
    return out


def reweight_problem(G, N, classes, wstride, tier, mask, rng):
    """Labels with out-of-range values (-1, INT64_MIN, classes, 2^40), a table whose entries reach past wstride and
    below 0, per-class weights of the tier, and the mask kind."""
    labels = rng.integers(0, classes, N).astype(np.int64)
    r = rng.random(N)
    labels[r < 0.05] = -1
    labels[(r >= 0.05) & (r < 0.08)] = INT64_MIN
    labels[(r >= 0.08) & (r < 0.11)] = classes
    labels[(r >= 0.11) & (r < 0.13)] = 2 ** 40
    table = rng.integers(0, min(wstride, 40), (G, classes)).astype(np.int32)
    table[:, ::5] = wstride + rng.integers(0, 3, table[:, ::5].shape)       # >= wstride: the "others" weight
    table[:, 1::7] = -rng.integers(1, 4, table[:, 1::7].shape)              # negative: the "others" weight
    if tier == 'exact':
        cw = rng.integers(1, 257, (G, wstride)) / 64.0                      # multiples of 2^-6 in [2^-6, 4]
    else:
        cw = rng.uniform(0.0, 2.0, (G, wstride))
    cw = cw.astype(np.float32)
    if mask == 'none':
        wmask = None
    elif mask == '01':
        wmask = (rng.random((G, N)) < 0.6).astype(np.uint8)
    else:
        wmask = rng.choice(np.array([0, 1, 2, 255], dtype=np.uint8), size=(G, N))
    return labels, table, wmask, cw


REWEIGHT_CASES = [
    # (G, N, classes, wstride, tier, mask)
    (1, 0, 5, 3, 'exact', '01'), (5, 0, 1231, 300, 'exact', 'none'), (2, 1, 3, 2, 'exact', '01'),
    (5, 255, 1231, 300, 'exact', '01'), (5, 256, 1231, 300, 'exact', 'none'), (8, 257, 40, 7, 'exact', '01'),
    (3, 1000, 100, 2000, 'exact', '01'), (8, 4097, 1231, 64, 'exact', 'none'), (5, 1 << 14, 1231, 300, 'exact', '01'),
    (4, 1000, 60, 30, 'numeric', 'bytes'), (5, 4097, 1231, 300, 'numeric', '01'), (8, 65543, 200, 2000, 'numeric', 'none'),
    (5, 1 << 20, 1231, 300, 'numeric', '01'), (2, 1 << 20, 50, 9, 'numeric', 'bytes')]


@pytest.mark.parametrize('case', REWEIGHT_CASES, ids=['G%d-N%d-c%d-ws%d-%s-%s' % c for c in REWEIGHT_CASES])
def test_reweight_vs_float64(case):
    G, N, classes, wstride, tier, mask = case
    rng = np.random.default_rng(N * 13 + G)
    labels, table, wmask, cw = reweight_problem(G, N, classes, wstride, tier, mask, rng)
    out = run_reweight(labels, table, wmask, cw)
    w, avg = S.reweight(labels, table, wmask, cw)
    what = 'reweight %r' % (case,)
    same_bits(out.values(), w.astype(np.float32), '%s: wfloat' % what)    # byte * fp32 weight: one rounding
    got = out.avg_values().astype(np.float64)
    if tier == 'exact':
        assert wmask is None or wmask.max(initial=0) <= 1
        assert N <= 1 << 14 and (w * 64 == np.round(w * 64)).all() and (w.sum(1) < 2 ** 16).all(), what
        same_bits(out.avg_values(), avg.astype(np.float32), '%s: avg' % what)
    else:
        m = -(-N // 256) + 13
        bound = m * U / (1 - m * U) * np.abs(w).sum(1)
        err = np.abs(got - avg)
        assert (err <= bound).all(), (what, got, avg, err, bound)
    if N == 0:
        assert (got == 1.0).all()
    out.check_sentinels(what)


def test_reweight_conventions_on_named_rows():
    """One row per convention, bin by bin: a label out of range, a table entry >= wstride and a negative one all take
    cls_weight[g, 0]; an in-range entry takes its own weight; bin 0 keeps the mask byte."""
    table = np.array([[9, 9, 9, 9], [0, 2, 5, -1], [0, 1, 3, 2]], dtype=np.int32)      # wstride 4: 5 is out
    cw = np.array([[100.0, 200.0, 300.0, 400.0], [0.5, 1.5, 2.5, 3.5], [0.25, 0.75, 1.25, 1.75]], dtype=np.float32)
    labels = np.array([1, 2, 3, -1, 4, 2 ** 40, INT64_MIN, 0], dtype=np.int64)
    wmask = np.array([[1, 2, 255, 0, 1, 1, 1, 1], [1] * 8, [1, 1, 1, 1, 0, 1, 1, 1]], dtype=np.uint8)
    out = run_reweight(labels, table, wmask, cw)
    want = np.array([[1, 2, 255, 0, 1, 1, 1, 1],
                     [2.5, 0.5, 0.5, 0.5, 0.5, 0.5, 0.5, 0.5],
                     [0.75, 1.75, 1.25, 0.25, 0.0, 0.25, 0.25, 0.25]], dtype=np.float32)
    same_bits(out.values(), want, 'named rows: wfloat')
    same_bits(out.avg_values(), want.sum(1).astype(np.float32), 'named rows: avg')
    same_bits(S.reweight(labels, table, wmask, cw)[0].astype(np.float32), want, 'named rows: restatement')
    out.check_sentinels('named rows')
