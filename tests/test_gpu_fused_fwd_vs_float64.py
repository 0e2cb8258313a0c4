"""GPU: the fused fc_cls forward -- bags_fwd's fused route, bags_ce_fwd and bags_focal_fwd, the three entry points of
fused_fwd_body -- against float64 at its edges.

Every reference is plain torch in float64 on the device (tests/fused_fwd_ref.py, tests/focal_oracle.py), never this
library.  Arguments the Python wrappers hide (ldx, ldw, ldd, colsum_tiles, clear, lse, acc) go through ctypes.
Operand padding (columns [K, ld) and rows past N / C) holds NaN, and every output byte the kernel must not write
holds the sentinel -7.

Exact logits.  x and W are small integers (exact in bf16 and TF32), the bias is a multiple of 2^-3, and every
partial sum of z = x W^T + b is a multiple of 2^-3 below 2^20 in magnitude (asserted per case).  So z is exact in
fp32 in any summation order, and so is the difference of any two logits (a multiple of 2^-3 below 2^21 needs at most
24 bits).  What remains is the kernel's own fp32 softmax, bounded below against the float64 softmax of the same z.
"Moderate" cases keep |z| around 16; "wide" ones add a constant column of x (8) times an integer column of W
(|W| <= 64), so |z| reaches about 2^9 and most of a bin's exponentials underflow.

Bounds of the softmax CE (u = 2^-24, Z = max_c |z[n, c]| of the row, L = fp32(log2 e) = log2 e (1 + dL), |dL| <= u;
exp2f errs by at most 2 ulp, logf by 1 ulp, a correctly rounded operation by u relative; first order throughout,
the second-order terms are below 0.3 % of the first up to Z = 2^11 and covered by the rounding up of the constants):
  * pass B, e = exp2f(fma(z, L, -fl(m L))), m the CTA's bin maximum: fl(m L) errs by |m| L u <= 1.45 Z u, the fma's
    rounding by |(z - m) L| u <= 2.9 Z u, and L's own error contributes |z - m| log2e u <= 2.9 Z u: 7.2 Z u in the
    base-2 exponent, i.e. ln 2 * 7.2 Z u = 5 Z u relative, plus exp2f's 4 u.  rho_e = (5 Z + 4) u.
  * the CTA's sum of e: at most 80 sequential additions per thread and two quad shuffles of positive terms, 82 u.
  * the exchange, S = sum_s sum_s * exp2f((max_s - M) L): max_s - M is exact, the product with L errs by
    2 * 2 Z * 1.45 u in the exponent (its rounding and dL), 4 Z u relative, exp2f 4 u, the product u, and the sum of
    four terms 3 u.  rho_S = rho_e + 82 u + (4 Z + 4) u + 4 u = (9 Z + 94) u.
  * lse = fl(M + logf(S)), 1 <= S <= 1280: rho_S, logf's ulp of a value below 8 (8 u), the addition (Z + 8) u:
    eps_lse = (10 Z + 110) u.
  * pass C, scale = fl(exp2f(fl(fl(m - lse) L)) * cf), cf = fl(w * fl(1 / avg)) (2 u from w/avg): eps_lse, the
    subtraction (2 Z + 8) u, the product with L 2 (2 Z + 8) u, exp2f 4 u, the product u, cf 2 u:
    rho_scale = (16 Z + 141) u.
  * dz = fl(e * scale) - [target] cf: rho_e + rho_scale + u relative to w/avg * p <= w/avg, and for the target
    column cf's 2 u and the subtraction's u: (21 Z + 149) u * w/avg.
So eps(Z) = (24 Z + 192) u (fused_fwd_ref.eps_softmax; 3.4e-5 at Z = 16), and
  * dz:   |got - ref| <= w/avg * eps(Z) in fp32; a bf16 dz adds its rounding to 8 significant bits, 2^-8 |ref| (and
          2^-8 of the fp32 error);
  * lse:  |got - ref| <= eps(Z) (eps_lse <= eps);
  * loss: each row's term cf * (lse - z[target]) errs by w/avg * eps(Z) plus 4 u of the term (cf, the subtraction,
          the product); the terms are summed with shared-memory atomics, the per-CTA partials and a warp sum: at
          most N + 300 additions in a chain, (N + 300) u * sum |terms|;
  * colsum: bit for bit.  colsum[t, c] is the fp32 sum of the stored dz of rows 128 t ... 128 t + 127 in row order
          from 0 (rows >= N add 0); the build has no fast-math and the loop only adds, so 128 sequential fp32 torch
          additions reproduce it exactly;
  * acc:  an exact count (ties are exact): rows whose label lies in [0, C) and whose label logit equals the row
          maximum, times fp32(100 / N) in fp32.

The focal loss (bags_focal_fwd) reuses tests/test_gpu_focal.py's derivation with the logit error gone: its fp32
per-element math errs by at most 2^-18 relative to |g| (and |l|), cf by 2 u; an exponential that underflows in fp32
errs by less than 2^-100 absolute; the loss's sums add 2^-14 relative (a few hundred additions per chain).  The
reference is fused_fwd_ref.focal, the oracle's formulas with 1 - p formed from exp(-|z|) as the kernel forms it (the
oracle's own 1 - p is 0 in float64 for z > 37, so it cannot bound a positive element's gradient there).

Conventions pinned here: a label outside [0, classes) or a label2bin entry outside [0, len_g) is scored against the
bin's first column, as bags_group_ce does, and never counts as correct for the accuracy; a focal target t puts the
positive at column t - 1, t <= 0 or t > C gives no positive column and t < 0 a row without loss and with zero dz.
"""
import numpy as np
import pytest
import torch

import focal_oracle as FO
import fused_fwd_ref as R
from balancedgroupsoftmax_b200 import _native as nat

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
BF, F32 = torch.bfloat16, torch.float32
SENT = -7.0
NAN = float('nan')
U = R.U
EXACT_LIMIT = 2.0 ** 20


def _ops():
    from balancedgroupsoftmax_b200 import ops
    return ops


def _stream():
    return torch.cuda.current_stream(DEV).cuda_stream


def _code(dtype):
    return nat.DTYPE_BF16 if dtype == BF else nat.DTYPE_F32


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _big_n():
    """Enough rows that every CTA group walks two or three row tiles (both exchange slots): 2 (SMs / 4) 128 + 77."""
    return 2 * (torch.cuda.get_device_properties(DEV).multi_processor_count // 4) * 128 + 77


# ------------------------------------------------------------------------------------------------ the cases
KS = [4, 8, 60, 64, 68, 128, 200, 1028]                 # 1, 2, 3 (= STAGES), 4 and many k-blocks, K tails
NS = [1, 2, 127, 128, 129, 4096 + 77, 'big']
# bin starts per C on the grouped route (C % 4 == 0), one table per operand dtype (fp32, bf16); bins tile [0, C)
GROUPED_TABLES = {
    4: ([0], [0, 1, 2, 3]),                                        # one-column bins
    8: ([0, 4], [0, 3, 7]),
    12: ([0, 5, 6, 11], [0, 8]),                                   # an edge on an 8-column chunk boundary
    316: ([0, 1, 50, 101, 200, 315], [0, 16, 104, 200, 312]),      # six bins in rank 0; chunk-boundary edges
    320: ([0, 7, 64, 128, 256, 319], [0, 319]),
    324: ([0, 320], [0, 319, 320, 321, 322, 323]),                 # one-column bins around the CTA edge
    636: ([0, 240, 360, 635], [0, 318, 319, 633]),
    644: ([0, 46, 167, 240, 360, 641], [0, 639, 640, 643]),        # edges at chunk offsets 6, 7, 0, 0, 1
    960: ([0, 320, 639, 641, 959], [0, 25, 330, 483, 644, 805]),   # offsets 1 ... 5
    964: ([0, 25, 330, 483, 644, 805], [0, 959, 960, 961, 963]),
    1236: ([0, 319, 640, 961], [0, 2, 303, 701, 1201]),
    1276: ([0, 1, 320, 641, 960, 1275], [0, 2, 1274]),             # edges 320 / 641 / 960; a bin over all four CTAs
    1280: ([0, 961, 1000, 1100, 1200, 1279], [0, 321, 639, 959]),  # bins 1-5 inside rank 3; edges 321 / 639 / 959
}
SINGLE_CS = [1, 3, 7, 9, 319, 321, 641, 1231, 1279, 1280]         # both sides of the TMA / plain-store split of dz
GA = [(2.0, 0.25), (0.5, 1.0), (0.0, 0.25), (1.5, 0.75)]


def _build_cases():
    """The sampled parameter space: every C, K and N in both operand dtypes for each entry point; the other knobs
    cycle independently over the cases of a dtype."""
    cases = []
    for entry, cs in (('grouped', sorted(GROUPED_TABLES)), ('ce', SINGLE_CS), ('focal', SINGLE_CS)):
        for di, dtype in enumerate(('fp32', 'bf16')):
            for i, C in enumerate(cs):
                j = i + 3 * di
                case = dict(entry=entry, dtype=dtype, C=C, K=KS[(i + 5 * di) % len(KS)], N=NS[(i + 2 * di) % len(NS)],
                            wide=(j % 4 == 1), ldx_pad=(j % 2 == 0), ldd=('pad64', 'r8p8')[(j // 2) % 2],
                            clear=(j % 3 == 2), bias=(j % 5 != 4))
                if entry == 'grouped':
                    case['starts'] = GROUPED_TABLES[C][di]
                    case['weights'] = ('u8', 'f32', None)[j % 3]
                    case['avg'] = j % 2 == 0
                elif entry == 'ce':
                    case['weights'] = ('f32', None)[j % 2]
                    case['avg'] = (j // 2) % 2 == 0
                    case['acc'] = j % 3 != 1
                else:
                    case['weights'] = ('f32', None)[(j // 2) % 2]
                    case['acc'] = j % 3 != 1
                    case['gamma'], case['alpha'] = GA[j % len(GA)]
                cases.append(case)
    return cases


CASES = _build_cases()


def case_id(c):
    s = '%s-%s-C%d-K%d-N%s-%s' % (c['entry'], c['dtype'], c['C'], c['K'], c['N'], 'wide' if c['wide'] else 'mod')
    if c['entry'] == 'grouped':
        s += '-G%d-%s%s' % (len(c['starts']), c['weights'] or 'noweights', '-avg' if c['avg'] else '')
    elif c['entry'] == 'ce':
        s += '-%s%s%s' % (c['weights'] or 'noweights', '-avg' if c['avg'] else '', '-acc' if c['acc'] else '')
    else:
        s += '-%s%s-g%g-a%g' % (c['weights'] or 'noweights', '-acc' if c['acc'] else '', c['gamma'], c['alpha'])
    return s


# ------------------------------------------------------------------------------------------------ operands
def _ints(shape, gen, lim, density):
    v = torch.randint(-lim, lim + 1, shape, generator=gen, device=DEV)
    v = v * (torch.rand(shape, generator=gen, device=DEV) < density)
    return v.double()


def _ld(K, dtype, pad):
    """Row stride in elements: K itself where its rows are whole 16-byte pieces (and ``pad`` is off), otherwise the
    next 16-byte multiple plus one more piece."""
    a = 8 if dtype == BF else 4
    if not pad and K % a == 0:
        return K
    return (K + a - 1) // a * a + a


def _padded(values, dtype, ld, extra_rows=8):
    """values [rows, cols] in a buffer of rows + extra_rows rows of ld elements, NaN everywhere else."""
    rows, cols = values.shape
    buf = torch.full((rows + extra_rows, ld), NAN, dtype=dtype, device=DEV)
    buf[:rows, :cols] = values.to(dtype)
    return buf


def tie_columns(C):
    """Columns that carry identical W rows and bias: (5, 6) share a CTA, (319, 320) and (5, 1000) do not."""
    return [c for c in (5, 6, 319, 320, 1000) if c < C]


def make_problem(N, K, C, wide, seed):
    """Exact integer operands X [N, K], Wm [C, K] and bias [C] (float64 values), and labels [N] with rows that tie
    at the row maximum and rows whose out-of-range label is scored against a column-0 maximum:
      rows n % 10 == 3: x[n, 1] = 4 and W[tie, 1] = 16 lift the tie columns above every other column; the label is
                        one of the tie columns;
      rows n % 10 == 7: x[n, 2] = 4 and W[0, 2] = 16 make column 0 the row maximum; the label is -1, C or C + 5.
    Wide problems add x[:, 0] = 8 times W[:, 0] in [-64, 64] (64 for column 0 and the tie columns)."""
    assert K >= 3
    gen = _gen(seed)
    d = min(1.0, (6.0 / K) ** 0.5)
    X = _ints((N, K), gen, 1, d)
    Wm = _ints((C, K), gen, 1, d)
    b = torch.randint(-16, 17, (C,), generator=gen, device=DEV).double() / 8
    ties = tie_columns(C)
    labels = torch.randint(0, C, (N,), generator=gen, device=DEV)
    if wide:
        X[:, 0] = 8
        Wm[:, 0] = torch.randint(-64, 65, (C,), generator=gen, device=DEV).double()
        Wm[0, 0] = 64
    if ties:
        Wm[ties] = Wm[ties[0]].clone()
        b[ties] = b[ties[0]].item()
        if K > 1:
            Wm[ties, 1] = 16
        if wide:
            Wm[ties, 0] = 64
    rows = torch.arange(N, device=DEV)
    Wm[0, 2] = 16
    tie_rows = rows % 10 == 3
    if ties:
        X[tie_rows, 1] = 4
        tl = torch.tensor(ties, device=DEV)
        labels = torch.where(tie_rows, tl[rows % len(ties)], labels)
    oor = rows % 10 == 7
    X[oor, 2] = 4
    oor_lab = torch.tensor([-1, C, C + 5], device=DEV)[(rows // 10) % 3]
    return X, Wm, b, torch.where(oor, oor_lab, labels)


def _z(X, Wm, b, use_bias):
    z = X @ Wm.t() + (b if use_bias else 0.0)
    S = X.abs() @ Wm.abs().t() + (b.abs() if use_bias else 0.0)
    assert float(S.max()) < EXACT_LIMIT, 'operands too large for exact logits: max |x||W| + |b| = %g' % float(S.max())
    assert bool(((b * 8) == (b * 8).round()).all())
    return z


def _first_bad(bad):
    return tuple(bad.nonzero()[0].tolist())


def check_bound(got, ref, tol, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= tol)
    if bool(bad.any()):
        i = _first_bad(bad)
        raise AssertionError('%s: %d of %d elements over the bound, first at %s: got %r, ref %r, bound %r' % (
            what, int(bad.sum()), bad.numel(), i, got[i].item(), ref[i].item(), tol[i].item()))


def check_sentinel(buf, what):
    bad = ~(buf.double() == SENT)
    if bool(bad.any()):
        raise AssertionError('%s: %d bytes written that must not be, first at %s (%r)' % (
            what, int(bad.sum()), _first_bad(bad), buf[_first_bad(bad)].item()))


def _bits(t):
    return t.contiguous().view(torch.int32)


class Outputs:
    """Every output buffer of one fused call, surrounded by sentinel: dz [N + 3, ldd], colsum [tiles + 1, C],
    lse [(N + 2) G], loss [G + 2], acc [2], and a clear buffer with 64 sentinel bytes either side."""

    def __init__(self, N, C, G, dtype, ldd, want_lse, want_acc, clear_floats):
        self.N, self.C, self.G = N, C, G
        self.tiles = (N + 127) // 128
        self.ldd = ldd
        self.dz = torch.full((N + 3, ldd), SENT, dtype=dtype, device=DEV)
        self.colsum = torch.full((self.tiles + 1, C), SENT, dtype=F32, device=DEV)
        self.loss = torch.full((G + 2,), SENT, dtype=F32, device=DEV)
        self.lse = torch.full(((N + 2) * G,), SENT, dtype=F32, device=DEV) if want_lse else None
        self.acc = torch.full((2,), SENT, dtype=F32, device=DEV) if want_acc else None
        self.clear_floats = clear_floats
        self.clear = torch.full((clear_floats + 32,), SENT, dtype=F32, device=DEV) if clear_floats else None

    def clear_args(self):
        if self.clear is None:
            return None, 0
        return self.clear.data_ptr() + 64, 4 * self.clear_floats

    def tail(self, ws):
        cptr, cbytes = self.clear_args()
        return (self.dz.data_ptr(), self.ldd, self.colsum.data_ptr(), self.tiles, ws.data_ptr(), ws.numel(), cptr,
                cbytes, _stream())

    def check_layout(self, what):
        """Everything outside the written ranges still holds the sentinel; the cleared range is zero."""
        N, C, G = self.N, self.C, self.G
        check_sentinel(self.dz[:, C:], '%s: dz padding columns [C, ldd)' % what)
        check_sentinel(self.dz[N:], '%s: dz rows >= N' % what)
        check_sentinel(self.colsum[self.tiles:], '%s: colsum past its row tiles' % what)
        check_sentinel(self.loss[G:], '%s: loss past G' % what)
        if self.lse is not None:
            check_sentinel(self.lse[N * G:], '%s: lse rows >= N' % what)
        if self.acc is not None:
            check_sentinel(self.acc[1:], '%s: acc[1]' % what)
        if self.clear is not None:
            check_sentinel(self.clear[:16], '%s: before the cleared range' % what)
            check_sentinel(self.clear[16 + self.clear_floats:], '%s: after the cleared range' % what)
            assert bool((self.clear[16:16 + self.clear_floats] == 0).all()), '%s: cleared range not zero' % what

    def results(self):
        r = dict(dz=self.dz[:self.N, :self.C].clone(), colsum=self.colsum[:self.tiles].clone(), loss=self.loss[:self.G].clone())
        if self.lse is not None:
            r['lse'] = self.lse[:self.N * self.G].clone()
        if self.acc is not None:
            r['acc'] = self.acc[:1].clone()
        return r


def _clear_floats(case, N):
    # 4 * (odd) floats: not a multiple of grid * 256 float4, so the last CTAs clear a partial stride
    return 4 * (2 * N + 1237) if case.get('clear') else 0


# ------------------------------------------------------------------------------------------------ checks
def check_softmax(out, z, slices, targets, coef, dtype, what, lse=True):
    dz_ref, lse_ref, loss_ref, coef_col, terms = R.softmax_ce(z, slices, targets, coef)
    N = z.shape[0]
    eps = R.eps_softmax(z.abs().max(1).values)
    got = out.dz[:N, :out.C]
    tol = coef_col * eps[:, None]
    if dtype == BF:
        tol = tol * (1 + 2.0 ** -8) + 2.0 ** -8 * dz_ref.abs()
    check_bound(got, dz_ref, tol, '%s: dz' % what)
    if lse:
        check_bound(out.lse[:N * len(slices)].view(N, -1), lse_ref, eps[:, None].expand_as(lse_ref), '%s: lse' % what)
    for g in range(len(slices)):
        ltol = float((coef[g] * eps).sum()) + (4 + N + 300) * U * float(terms[:, g].sum())
        assert abs(out.loss[g].item() - loss_ref[g].item()) <= ltol, '%s: loss bin %d: got %r, ref %r, bound %r' % (
            what, g, out.loss[g].item(), loss_ref[g].item(), ltol)
    check_colsum(out, what)


def check_colsum(out, what):
    want = R.colsum_fp32(out.dz[:out.N, :out.C], out.N)
    got = out.colsum[:out.tiles]
    same = _bits(got) == _bits(want)
    if not bool(same.all()):
        i = _first_bad(~same)
        raise AssertionError('%s: colsum differs from the row-ordered fp32 sum of the stored dz at %s: got %r, want %r' %
                             (what, i, got[i].item(), want[i].item()))


def check_acc(out, z, labels, what):
    N = z.shape[0]
    count = R.top1_count(z, labels)
    want = torch.tensor(float(count), dtype=F32) * torch.tensor(100.0 / N, dtype=F32)
    got = out.acc[0].item()
    assert got == want.item(), '%s: acc %r, want %r (%d correct rows of %d)' % (what, got, want.item(), count, N)


def _weights(kind, shape, gen):
    if kind == 'u8':
        return (torch.rand(shape, generator=gen, device=DEV) < 0.7).to(torch.uint8)
    if kind == 'f32':
        vals = torch.tensor([0.0, 0.25, 0.5, 1.0, 2.0, 4.0, 0.375], device=DEV)
        return vals[torch.randint(0, len(vals), shape, generator=gen, device=DEV)]
    return None


# ------------------------------------------------------------------------------------------------ entry points
def _operands(case, N):
    dtype = BF if case['dtype'] == 'bf16' else F32
    K, C = case['K'], case['C']
    X, Wm, b, labels = make_problem(N, K, C, case['wide'], seed=C * 7919 + K * 31 + N + (dtype == BF))
    ld = _ld(K, dtype, case['ldx_pad'])
    x, w = _padded(X, dtype, ld), _padded(Wm, dtype, ld)
    bias = None
    if case['bias']:
        bias = torch.full((C + 4,), NAN, dtype=F32, device=DEV)
        bias[:C] = b.float()
    z = _z(X, Wm, b, case['bias'])
    ldd = _ops().pad_cols(C) if case['ldd'] == 'pad64' else (C + 7) // 8 * 8 + 8
    return dtype, x, w, ld, bias, z, labels, ldd


def run_grouped(case, N, ws, seed=0):
    """bags_fwd's fused route: returns (Outputs, z, slices, targets, coef)."""
    dtype, x, w, ld, bias, z, labels, ldd = _operands(case, N)
    C, K = case['C'], case['K']
    starts = case['starts']
    slices = [(s, e - s) for s, e in zip(starts, starts[1:] + [C])]
    G, classes = len(slices), 40
    gen = _gen(seed + 17 * C + N)
    lens = torch.tensor([ln for _, ln in slices], device=DEV)
    l2b = (torch.rand(G, classes, generator=gen, device=DEV) * lens[:, None]).long()
    l2b[:, 0] = lens          # entries outside [0, len_g): scored against the bin's first column
    l2b[:, 1] = -1
    # the problem's labels are columns; here they index the class table (-1 / C / C + 5 stay out of range)
    labels = torch.where(labels >= 0, labels % (classes + 6), labels)
    wm = _weights(case['weights'], (G, N), gen)
    if case['weights'] == 'u8' and G > 1:
        wm[G - 1] = 0         # a bin without any row: avg clamps to 1, loss and dz are 0
    wd = wm.double() if wm is not None else torch.ones(G, N, dtype=torch.float64, device=DEV)
    avg = wd.sum(1).clamp_min(1.0).float() if case['avg'] else None
    avg_d = avg.double() if avg is not None else torch.full((G,), float(N), dtype=torch.float64, device=DEV)
    coef = wd / avg_d[:, None]
    targets = R.bin_targets(labels, l2b, slices, classes)
    out = Outputs(N, C, G, dtype, ldd, True, False, _clear_floats(case, N))
    l2b32 = l2b.int().contiguous()
    wcode = nat.WEIGHTS_F32 if case['weights'] == 'f32' else nat.WEIGHTS_U8
    nat.check(nat.lib().bags_fwd(
        x.data_ptr(), ld, w.data_ptr(), ld, nat.ptr(bias), labels.data_ptr(), l2b32.data_ptr(),
        nat.int32_array([v for sl in slices for v in sl]), nat.ptr(wm), wcode, nat.ptr(avg), N, K, C, G, classes,
        _code(dtype), None, 0, out.loss.data_ptr(), out.lse.data_ptr(), *out.tail(ws)), 'bags_fwd')
    return out, z, slices, targets, coef, labels


def run_ce(case, N, ws):
    dtype, x, w, ld, bias, z, labels, ldd = _operands(case, N)
    C, K = case['C'], case['K']
    gen = _gen(C + 3 * N)
    wv = _weights(case['weights'], (N,), gen)
    wd = wv.double() if wv is not None else torch.ones(N, dtype=torch.float64, device=DEV)
    avg = torch.tensor([max(float(wd.sum()), 1.0) * 0.75], dtype=F32, device=DEV) if case['avg'] else None
    avg_d = float(avg.item()) if avg is not None else float(N)
    out = Outputs(N, C, 1, dtype, ldd, False, case['acc'], _clear_floats(case, N))
    nat.check(nat.lib().bags_ce_fwd(
        x.data_ptr(), ld, w.data_ptr(), ld, nat.ptr(bias), labels.data_ptr(), nat.ptr(wv), nat.ptr(avg), N, K, C,
        _code(dtype), out.loss.data_ptr(), nat.ptr(out.acc), *out.tail(ws)), 'bags_ce_fwd')
    targets = R.bin_targets(labels, None, [(0, C)], C)
    return out, z, [(0, C)], targets, (wd / avg_d)[None], labels


def focal_targets(N, C, gen):
    """The op's targets: in range (column t - 1 positive, t = 1 and t = C among them), 0, -1, -3, C + 1, C + 5."""
    t = torch.randint(1, C + 1, (N,), generator=gen, device=DEV)
    special = torch.tensor([1, C, 0, -1, -3, C + 1, C + 5], device=DEV)
    pick = torch.randint(0, 2 * len(special), (N,), generator=gen, device=DEV)
    return torch.where(pick < len(special), special[pick.clamp_max(len(special) - 1)], t)


def run_focal(case, N, ws):
    dtype, x, w, ld, bias, z, labels, ldd = _operands(case, N)
    C, K = case['C'], case['K']
    gen = _gen(5 * C + N)
    t = focal_targets(N, C, gen)
    wv = _weights(case['weights'], (N,), gen)
    wd = wv.double() if wv is not None else torch.ones(N, dtype=torch.float64, device=DEV)
    norm = float(N * FO.ONE_HOT)
    out = Outputs(N, C, 1, dtype, ldd, False, case['acc'], _clear_floats(case, N))
    nat.check(nat.lib().bags_focal_fwd(
        x.data_ptr(), ld, w.data_ptr(), ld, nat.ptr(bias), t.data_ptr(), labels.data_ptr() if case['acc'] else None,
        nat.ptr(wv), norm, case['gamma'], case['alpha'], N, K, C, _code(dtype), out.loss.data_ptr(), nat.ptr(out.acc),
        *out.tail(ws)), 'bags_focal_fwd')
    coef = wd / float(np.float32(norm))
    return out, z, t, coef, labels


def check_focal(out, z, t, coef, case, dtype, what):
    gamma, alpha = case['gamma'], case['alpha']
    el, g = R.focal(z, t, gamma, alpha)
    ref = coef[:, None] * g
    tol = coef[:, None] * (2.0 ** -18 * g.abs() + 2.0 ** -100)
    if dtype == BF:
        tol = tol * (1 + 2.0 ** -8) + 2.0 ** -8 * ref.abs()
    check_bound(out.dz[:out.N, :out.C], ref, tol, '%s: dz' % what)
    ignored = t < 0
    assert bool((out.dz[:out.N][ignored, :out.C] == 0).all()), '%s: a row with t < 0 has a nonzero dz' % what
    terms = coef[:, None] * el
    loss_ref = float(terms.sum())
    ltol = float((coef[:, None] * (2.0 ** -18 * el.abs() + 2.0 ** -100)).sum()) + 2.0 ** -14 * float(terms.abs().sum())
    assert abs(out.loss[0].item() - loss_ref) <= ltol, '%s: loss %r, ref %r, bound %r' % (
        what, out.loss[0].item(), loss_ref, ltol)
    check_colsum(out, what)


@pytest.mark.parametrize('case', CASES, ids=[case_id(c) for c in CASES])
def test_fused_forward_vs_float64(case):
    N = _big_n() if case['N'] == 'big' else case['N']
    ws = _ops()._workspace(DEV)
    what = case_id(case)
    dtype = BF if case['dtype'] == 'bf16' else F32
    if case['entry'] == 'grouped':
        out, z, slices, targets, coef, _ = run_grouped(case, N, ws)
        torch.cuda.synchronize()
        out.check_layout(what)
        check_softmax(out, z, slices, targets, coef, dtype, what)
    elif case['entry'] == 'ce':
        out, z, slices, targets, coef, labels = run_ce(case, N, ws)
        torch.cuda.synchronize()
        out.check_layout(what)
        check_softmax(out, z, slices, targets, coef, dtype, what, lse=False)
        if case['acc']:
            check_acc(out, z, labels, what)
    else:
        out, z, t, coef, labels = run_focal(case, N, ws)
        torch.cuda.synchronize()
        out.check_layout(what)
        check_focal(out, z, t, coef, case, dtype, what)
        if case['acc']:
            check_acc(out, z, labels, what)


def test_accuracy_ties_and_out_of_range_labels():
    """bags_ce_fwd and bags_focal_fwd count a label tied with the row maximum -- in the same CTA (columns 5 / 6) and
    across CTAs (319 / 320, 5 / 1000) -- and rows of zero weight, and never count a label -1, C or C + 5, even where
    column 0, which such a row is scored against, is the row maximum."""
    C, K, N = 1231, 64, 1000
    for entry in ('ce', 'focal'):
        for dt in ('bf16', 'fp32'):
            case = dict(entry=entry, dtype=dt, C=C, K=K, N=N, wide=False, ldx_pad=False, ldd='pad64', clear=False,
                        bias=True, weights='f32', avg=True, acc=True, gamma=2.0, alpha=0.25)
            run = run_ce if entry == 'ce' else run_focal
            res = run(case, N, _ops()._workspace(DEV))
            out, z, labels = res[0], res[1], res[-1]
            torch.cuda.synchronize()
            rows = torch.arange(N, device=DEV)
            zmax = z.max(1).values
            ties = torch.tensor(tie_columns(C), device=DEV)
            tie_rows = rows % 10 == 3
            # the construction: every tie row's tie columns are its maximum, every out-of-range row's column 0 is
            assert bool((z[tie_rows][:, ties] == zmax[tie_rows][:, None]).all())
            oor = rows % 10 == 7
            assert bool((z[oor, 0] == zmax[oor]).all()) and bool(((labels[oor] < 0) | (labels[oor] >= C)).all())
            check_acc(out, z, labels, '%s %s' % (entry, dt))
            count = R.top1_count(z, labels)
            assert count >= int(tie_rows.sum()), 'every tie row counts'


# ------------------------------------------------------------------------------------------------ PDL predecessor
@pytest.mark.parametrize('pred', ['sample_others', 'mask_avg'])
def test_pdl_predecessor_masks_are_read_after_it(pred):
    """The fused bags_fwd launched right behind the kernel that writes its masks / avg (programmatic dependent launch):
    the buffers first hold a pattern unlike the predecessor's output, and the outputs must match the float64
    reference built from the predecessor's final masks, read after a synchronisation."""
    from balancedgroupsoftmax_b200.tables import synthetic_tables
    ops = _ops()
    t = synthetic_tables()
    dt = ops.DeviceTables.from_tables(t, DEV)
    slices = [tuple(int(v) for v in r) for r in t.pred_slice]
    G, C, classes = dt.G, t.num_logits, t.num_classes
    N, K = 4096 + 77, 1028
    case = dict(dtype='bf16', C=C, K=K, wide=False, ldx_pad=True, ldd='pad64', bias=True)
    dtype, x, w, ld, bias, z, _, ldd = _operands(case, N)
    gen = _gen(123)
    labels = torch.randint(0, classes, (N,), generator=gen, device=DEV)
    labels[::3] = 0
    wm = torch.ones((G, N), dtype=torch.uint8, device=DEV)
    wm[0] = 0
    avg = torch.full((G,), 3.0, dtype=F32, device=DEV)
    if pred == 'mask_avg':
        wm = (torch.rand(G, N, generator=gen, device=DEV) < 0.3).to(torch.uint8)
    pattern_wm, pattern_avg = wm.clone(), avg.clone()
    out = Outputs(N, C, G, dtype, ldd, True, False, 0)
    ws = ops._workspace(DEV)
    args = (x.data_ptr(), ld, w.data_ptr(), ld, bias.data_ptr(), labels.data_ptr(), dt.label2bin.data_ptr(),
            dt.slices_host, wm.data_ptr(), nat.WEIGHTS_U8, avg.data_ptr(), N, K, C, G, classes, _code(dtype), None, 0,
            out.loss.data_ptr(), out.lse.data_ptr()) + out.tail(ws)
    torch.cuda.synchronize()
    lib = nat.lib()
    if pred == 'sample_others':
        rc = lib.bags_sample_others(labels.data_ptr(), dt.label2bin.data_ptr(), N, G, classes, 8.0, 77, None,
                                    wm.data_ptr(), avg.data_ptr(), _stream())
    else:
        rc = lib.bags_mask_avg(wm.data_ptr(), N, G, avg.data_ptr(), _stream())
    rc2 = lib.bags_fwd(*args)     # immediately behind the predecessor, on the same stream
    nat.check(rc, pred)
    nat.check(rc2, 'bags_fwd')
    torch.cuda.synchronize()
    assert not torch.equal(avg, pattern_avg), 'the predecessor left avg as it was: nothing to tell apart'
    if pred == 'sample_others':
        assert not torch.equal(wm, pattern_wm)
    coef = wm.double() / avg.double()[:, None]
    targets = R.bin_targets(labels, dt.label2bin, slices, classes)
    out.check_layout(pred)
    check_softmax(out, z, slices, targets, coef, dtype, 'after %s' % pred)


# ------------------------------------------------------------------------------------------------ shared workspace
def test_one_workspace_across_entry_points_and_grid_sizes():
    """One stream and its one workspace: the fused bags_fwd (looping row tiles), bags_ce_fwd with acc (fewer groups),
    bags_focal_fwd with and without acc, bags_group_ce, bags_box_fwd, bags_mask_fwd, and the first bags_fwd again.
    Each fused call's dz, lse, colsum and acc are bitwise those of the same call on a fresh zeroed workspace (the
    exchange's arrival counters are never reset); its loss, summed with atomics, is within 1e-6 relative."""
    ops = _ops()
    big = _big_n()
    grouped = dict(entry='grouped', dtype='bf16', C=1236, K=200, wide=False, ldx_pad=True, ldd='pad64', clear=True,
                   bias=True, starts=[0, 2, 303, 701, 1201], weights='u8', avg=True)
    ce = dict(entry='ce', dtype='fp32', C=1231, K=68, wide=False, ldx_pad=False, ldd='r8p8', clear=False, bias=True,
              weights='f32', avg=False, acc=True)
    focal = dict(entry='focal', dtype='bf16', C=1231, K=128, wide=False, ldx_pad=False, ldd='pad64', clear=False,
                 bias=True, weights='f32', acc=True, gamma=2.0, alpha=0.25)
    fused = [('grouped', lambda ws: run_grouped(grouped, big, ws)[0]),
             ('ce', lambda ws: run_ce(ce, 300, ws)[0]),
             ('focal_acc', lambda ws: run_focal(focal, 700, ws)[0]),
             ('focal', lambda ws: run_focal(dict(focal, acc=False), 700, ws)[0])]
    fresh = {}
    for name, call in fused:
        ws = torch.zeros(nat.lib().bags_workspace_bytes(), dtype=torch.uint8, device=DEV)
        fresh[name] = call(ws).results()
        torch.cuda.synchronize()

    gen = _gen(99)
    # the other users of the workspace, with small valid arguments
    logits = torch.randn(500, 1236, generator=gen, device=DEV)
    slices = [(0, 2), (2, 301), (303, 398), (701, 500), (1201, 35)]
    l2b = torch.zeros(5, 50, dtype=torch.int32, device=DEV)
    dtab = ops.DeviceTables(5, 50, 1236, l2b, torch.zeros(50, dtype=torch.int32, device=DEV),
                            nat.int32_array([v for sl in slices for v in sl]), np.array(slices, dtype=np.int64))
    glabels = torch.randint(0, 50, (500,), generator=gen, device=DEV)
    bx = torch.randn(400, 64, generator=gen, device=DEV)
    bw = torch.randn(4 * 30, 64, generator=gen, device=DEV)
    blabels = torch.randint(0, 31, (400,), generator=gen, device=DEV)
    bt, bwt = torch.randn(400, 4, generator=gen, device=DEV), torch.ones(400, 4, device=DEV)
    my = torch.randn(40, 16, 14, 14, generator=gen, device=DEV)
    mw = torch.randn(30, 16, generator=gen, device=DEV)
    mlabels = torch.randint(0, 30, (40,), generator=gen, device=DEV)
    mt = (torch.rand(40, 14, 14, generator=gen, device=DEV) < 0.5).float()
    torch.cuda.synchronize()

    ws = ops._workspace(DEV)
    shared = {}
    shared['grouped'] = fused[0][1](ws).results()
    for name, call in fused[1:]:
        shared[name] = call(ws).results()
    ops.group_ce(logits, glabels, dtab, None, None)
    ops.box_fwd(bx, bw, None, blabels, bt, bwt, 1.0, 400.0)
    ops.mask_fwd(my, mw, None, mlabels, mt)
    again = fused[0][1](ws).results()
    torch.cuda.synchronize()
    for name, got in list(shared.items()) + [('grouped again', again)]:
        want = fresh[name.split()[0]]
        for key in ('dz', 'lse', 'colsum', 'acc'):
            if key in want:
                a, b = got[key], want[key]
                a = a.view(torch.int16) if a.dtype == BF else a.view(torch.int32)
                b = b.view(torch.int16) if b.dtype == BF else b.view(torch.int32)
                assert torch.equal(a, b), '%s: %s differs from the fresh-workspace call' % (name, key)
        for g in range(want['loss'].numel()):
            lw, lg = want['loss'][g].item(), got['loss'][g].item()
            assert abs(lg - lw) <= 1e-6 * abs(lw) + 1e-30, '%s: loss bin %d %r vs %r' % (name, g, lg, lw)
