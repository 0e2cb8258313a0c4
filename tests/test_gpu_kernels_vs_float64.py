"""GPU: the wgmma GEMM, the linear layer, the backward, the grouped CE and the score merge against float64, at their edges.

Every reference here is plain torch in float64 on the device (cuBLAS DGEMM, torch.logsumexp), never this library.
Arguments the Python wrappers do not expose (leading dimensions, colsum_tiles, BAGS_BWD_DW_PREZEROED, odd output
strides, padded output buffers) go through ctypes; the backward's dW split count is forced with BAGS_DW_SPLITS and
_native.reload_env().

Exact tier (most cases).  Operands are small integers, exact in bf16, fp32 and TF32; upstream gradients and scales
are powers of two, 0 and -1 included; every partial sum is a multiple of 2^-2 whose magnitude stays below 2^12
(asserted on each case).  Then every tensor-core product and every fp32 addition is exact in any order, so the
outputs must equal the float64 result bit for bit, and a bf16 output its round-to-nearest-even ``ref.to(bf16)``.
At zero tolerance this catches any error in tile mapping, K tails, split-K ranges, transposed loads, swizzles, row
scales or the ``+=`` of a reduce-add.  Operand padding columns hold NaN, so a kernel that reads them poisons its
output; output buffers get extra rows and columns holding a sentinel that must survive.

Numeric tier (a few cases per kernel).  Operands are random normal; each element is bounded against
S = |A| |B|^T in float64: bf16 operands |got - ref| <= (K + splits) 2^-23 S, fp32 operands (TF32 products)
(2^-8 + (K + splits) 2^-23) S, and a bf16 output another 2^-8 |ref|.  The grouped CE and the score merge are
bounded elementwise as stated at their tests.

Conventions of bags_group_ce checked here: a label outside [0, classes), or a label2bin entry outside [0, len_g), is
scored against in-bin label 0 of that bin, as the kernel does; dz is exactly 0 in columns that lie in no bin.
"""
import contextlib
import itertools
import os

import numpy as np
import pytest
import torch

from balancedgroupsoftmax_b200 import _native as nat

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
BF, F32 = torch.bfloat16, torch.float32
DTYPES, DT_IDS = [F32, BF], ['fp32', 'bf16']
SENT = -7.0            # output sentinel, exact in bf16 and fp32
NAN = float('nan')     # operand padding
EXACT_LIMIT = 2.0 ** 12


def _ops():
    from balancedgroupsoftmax_b200 import ops
    return ops


def _stream():
    return torch.cuda.current_stream(DEV).cuda_stream


def _code(dtype):
    return nat.DTYPE_BF16 if dtype == BF else nat.DTYPE_F32


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


@contextlib.contextmanager
def _env(**switches):
    """The library's BAGS_* switches set (None: unset) for the calls inside the block."""
    old = {k: os.environ.get(k) for k in switches}
    try:
        for k, v in switches.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = str(v)
        nat.reload_env()
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
        nat.reload_env()


def _padded(values, dtype, fill=NAN):
    """`values` [rows, cols] in a buffer with a row stride of pad8(cols) + 8 whose padding columns hold `fill`."""
    rows, cols = values.shape
    buf = torch.full((rows, (cols + 7) // 8 * 8 + 8), fill, dtype=dtype, device=DEV)
    buf[:, :cols] = values.to(dtype)
    return buf[:, :cols]


def _ints(shape, gen, lim=2, density=1.0):
    """float64 integers in [-lim, lim], each nonzero with probability `density`."""
    v = torch.randint(-lim, lim + 1, shape, generator=gen, device=DEV)
    if density < 1.0:
        v = v * (torch.rand(shape, generator=gen, device=DEV) < density)
    return v.double()


def _exact_operands(shape, contraction, gen):
    # dense {-2..2} up to K = 1024, sparser {-1, 0, 1} beyond: the partial sums stay far below 2^12
    return _ints(shape, gen) if contraction <= 1024 else _ints(shape, gen, 1, 1024.0 / contraction)


def _assert_exact_range(S, what):
    assert float(S.max()) < EXACT_LIMIT, '%s: operands too large for the exact tier (max |A||B|^T = %g)' % (
        what, float(S.max()))


def _first_bad(bad):
    return tuple(bad.nonzero()[0].tolist())


def _check_exact(buf, rows, cols, ref, what):
    """buf[:rows, :cols] == ref rounded to buf's dtype (nearest even), and the sentinel everywhere else in buf."""
    got = buf[:rows, :cols]
    want = ref.to(buf.dtype)
    bad = got.double() != want.double()
    if bool(bad.any()):
        i = _first_bad(bad)
        raise AssertionError('%s: %d of %d elements differ from float64, first at %s: got %r, want %r' % (
            what, int(bad.sum()), bad.numel(), i, got[i].item(), want[i].item()))
    outside = torch.ones(buf.shape, dtype=torch.bool, device=DEV)
    outside[:rows, :cols] = False
    assert bool((buf[outside] == SENT).all()), '%s: written outside [%d, %d) x [%d, %d)' % (what, 0, rows, 0, cols)


def _check_bound(got, ref, tol, what):
    err = (got.double() - ref).abs()
    bad = err > tol
    if bool(bad.any()):
        i = _first_bad(bad)
        raise AssertionError('%s: %d elements over the bound, first at %s: got %r, ref %r, bound %r' % (
            what, int(bad.sum()), i, got[i].item(), ref[i].item(), tol[i].item() if torch.is_tensor(tol) else tol))


# ------------------------------------------------------------------------------------------------ GEMM (bags_gemm_probe)
GEMM_KINDS = {   # A MN-major, B MN-major, epilogue for (bf16, fp32) operands -- the six instantiations the product uses
    'kk': (False, False, {BF: 0, F32: 0}),    # forward z = x W^T: fp32 store
    'kmn': (False, True, {BF: 1, F32: 0}),    # dX = dz W (the merged backward's dX units): bf16 / fp32 store
    'mnmn': (True, True, {BF: 2, F32: 2}),    # dW = dz^T x (its dW units): split-K reduce-add
}
# (M, N, K): every M in {1, 127, 128, 129, 300}, N in {1, 255, 256, 257, 1236} and K in {BLOCK_K - 8, BLOCK_K,
# BLOCK_K + 8, 1000, 12544} at least once, around the 128 x 256 tile edges
GEMM_SHAPES = [
    (1, 1, 'bk-8'), (127, 255, 'bk'), (128, 256, 'bk+8'), (129, 257, 1000), (300, 1236, 'bk-8'), (300, 1, 1000),
    (1, 1236, 12544), (129, 256, 12544), (128, 257, 'bk'), (127, 1236, 'bk+8'),
]


def _k(spec, bk):
    return {'bk-8': bk - 8, 'bk': bk, 'bk+8': bk + 8}.get(spec, spec)


def _gemm_case(kind, dtype, M, N, K, gen, exact):
    """(A [M,K], B [N,K] float64 values, a, b device operands in the layouts of `kind`)."""
    a_mn, b_mn, _ = GEMM_KINDS[kind]
    if exact:
        A, B = _exact_operands((M, K), K, gen), _exact_operands((N, K), K, gen)
    else:
        A = torch.randn(M, K, generator=gen, device=DEV, dtype=torch.float64).to(dtype).double()
        B = torch.randn(N, K, generator=gen, device=DEV, dtype=torch.float64).to(dtype).double()
    a = _padded(A.t() if a_mn else A, dtype)
    b = _padded(B.t() if b_mn else B, dtype)
    return A, B, a, b


def _probe(kind, a, b, out, ldo, M, N, K, splits, epi):
    a_mn, b_mn, _ = GEMM_KINDS[kind]
    nat.check(nat.lib().bags_gemm_probe(a.data_ptr(), a.stride(0), int(a_mn), b.data_ptr(), b.stride(0), int(b_mn),
                                        out.data_ptr(), ldo, M, N, K, _code(a.dtype), 256, splits, epi, _stream()),
              'bags_gemm_probe')


def _gemm_out(M, N, ldo, dtype):
    """Output buffer of M + 2 rows of ldo elements (ldo >= N), all sentinel."""
    return torch.full((M + 2, ldo), SENT, dtype=dtype, device=DEV)


@pytest.mark.parametrize('shape', GEMM_SHAPES, ids=['%dx%dx%s' % s for s in GEMM_SHAPES])
@pytest.mark.parametrize('kind', sorted(GEMM_KINDS))
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
def test_gemm_exact(dtype, kind, shape):
    bk = 64 if dtype == BF else 32
    M, N, K = shape[0], shape[1], _k(shape[2], bk)
    epi = GEMM_KINDS[kind][2][dtype]
    out_dtype = BF if epi == 1 else F32
    gen = _gen(M * 7919 + N * 31 + K)
    A, B, a, b = _gemm_case(kind, dtype, M, N, K, gen, exact=True)
    ref = A @ B.t()
    _assert_exact_range(A.abs() @ B.abs().t(), kind)
    kblocks = (K + bk - 1) // bk
    # even ldo: paired stores / red.add.v2; odd ldo: the scalar path.  splits beyond kblocks are clamped.
    for ldo in ((N + 7) // 8 * 8 + 8, N + 5 if (N + 5) % 2 else N + 6):
        for splits in ([1, 2, 3, kblocks, kblocks + 5] if epi == 2 else [1]):
            out = _gemm_out(M, N, ldo, out_dtype)
            want = ref
            if epi == 2:   # reduce-add: out = prefill + A B^T
                pre = _ints((M, N), gen, lim=8)
                out[:M, :N] = pre.to(out_dtype)
                want = pre + ref
            _probe(kind, a, b, out, ldo, M, N, K, splits, epi)
            _check_exact(out, M, N, want, '%s %s M=%d N=%d K=%d ldo=%d splits=%d' % (kind, dtype, M, N, K, ldo, splits))


@pytest.mark.parametrize('kind', sorted(GEMM_KINDS))
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
def test_gemm_numeric(dtype, kind):
    bk = 64 if dtype == BF else 32
    epi = GEMM_KINDS[kind][2][dtype]
    out_dtype = BF if epi == 1 else F32
    for i, (M, N, K) in enumerate([(300, 1236, 1000), (129, 257, 12544), (127, 255, bk + 8)]):
        gen = _gen(1000 + i)
        A, B, a, b = _gemm_case(kind, dtype, M, N, K, gen, exact=False)
        splits = 3 if epi == 2 else 1
        eff = min(splits, (K + bk - 1) // bk)
        out = torch.zeros((M, (N + 7) // 8 * 8), dtype=out_dtype, device=DEV)
        _probe(kind, a, b, out, out.stride(0), M, N, K, splits, epi)
        ref, S = A @ B.t(), A.abs() @ B.abs().t()
        tol = (K + eff) * 2.0 ** -23 * S
        if dtype == F32:
            tol = tol + 2.0 ** -8 * S
        if out_dtype == BF:
            tol = tol + 2.0 ** -8 * ref.abs()
        _check_bound(out[:, :N], ref, tol, '%s %s M=%d N=%d K=%d' % (kind, dtype, M, N, K))


# ------------------------------------------------------------------------------------------------ linear layer
@pytest.mark.parametrize('C', [4, 1231, 1236])
@pytest.mark.parametrize('dtypes', [(F32, F32), (BF, F32), (BF, BF)], ids=['fp32', 'bf16_out_fp32', 'bf16_out_bf16'])
def test_linear_act_fwd_exact(dtypes, C):
    """bags_linear_act_fwd and bags_linear_act_fwd_splitk (splits 2, 3, 16), bias and ReLU on and off; ldo = C for
    odd C (1231: the scalar stores), C + 8 otherwise."""
    dtype, out_dtype = dtypes
    lib = nat.lib()
    ldo = C if C % 2 else C + 8
    for variant, (N, K) in (('single', (300, 264)), ('splitk', (129, 2000))):
        gen = _gen(C * 13 + N)
        X, Wm = _exact_operands((N, K), K, gen), _exact_operands((C, K), K, gen)
        x, w = _padded(X, dtype), _padded(Wm, dtype)
        bias_v = _ints((C,), gen, lim=8) / 2
        bias = torch.zeros(C + 4, dtype=F32, device=DEV)
        bias[:C] = bias_v.float()
        acc = X @ Wm.t()
        _assert_exact_range(X.abs() @ Wm.abs().t() + bias_v.abs(), 'linear')
        for use_bias, relu in itertools.product((False, True), (False, True)):
            ref = acc + bias_v if use_bias else acc
            if relu:
                ref = ref.clamp_min(0.0)
            for splits in ((1,) if variant == 'single' else (2, 3, 16)):
                out = _gemm_out(N, C, ldo, out_dtype)
                bptr = bias.data_ptr() if use_bias else None
                if splits == 1:
                    rc = lib.bags_linear_act_fwd(x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), bptr,
                                                 out.data_ptr(), ldo, N, K, C, _code(dtype), _code(out_dtype), int(relu),
                                                 _stream())
                else:
                    ws = torch.full((N, (C + 3) // 4 * 4 + 4), NAN, dtype=F32, device=DEV)   # zeroed by the call
                    rc = lib.bags_linear_act_fwd_splitk(x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), bptr,
                                                        out.data_ptr(), ldo, N, K, C, _code(dtype), _code(out_dtype),
                                                        int(relu), ws.data_ptr(), ws.stride(0), splits, _stream())
                nat.check(rc, 'linear_act_fwd')
                _check_exact(out, N, C, ref, '%s bias=%d relu=%d splits=%d' % (variant, use_bias, relu, splits))


def _bits(t):
    t = t.contiguous()
    return t.view(torch.int16) if t.dtype == BF else t.view(torch.int32)


@pytest.mark.parametrize('combo', list(itertools.product(DTYPES, DTYPES, DTYPES)),
                         ids=['dy_%s-y_%s-g_%s' % tuple('bf16' if d == BF else 'fp32' for d in c)
                              for c in itertools.product(DTYPES, DTYPES, DTYPES)])
def test_act_bwd_bit_exact(combo):
    """g = (y > 0 ? dy : 0) cast to g's dtype, bit for bit against torch; y = +0, -0 and NaN give +0.  With y's dtype
    fp32 the plain cast (y NULL) is checked as well."""
    dy_dt, y_dt, g_dt = combo
    rows, cols, ldg = 37, 1236, 1240
    gen = _gen(5)
    dy = _padded(torch.randn(rows, cols, generator=gen, device=DEV) * 3, dy_dt)
    yv = torch.randn(rows, cols, generator=gen, device=DEV)
    yv[:, 0::7] = 0.0
    yv[:, 1::7] = -0.0
    yv[:, 2::7] = NAN
    yv[:, 3::7] = float('-inf')
    y = _padded(yv, y_dt)
    for with_y in ((True, False) if y_dt == F32 else (True,)):
        g = torch.full((rows + 2, ldg), SENT, dtype=g_dt, device=DEV)
        nat.check(nat.lib().bags_act_bwd(dy.data_ptr(), dy.stride(0), _code(dy_dt), y.data_ptr() if with_y else None,
                                         y.stride(0), _code(y_dt), g.data_ptr(), ldg, _code(g_dt), rows, cols, _stream()),
                  'bags_act_bwd')
        want = torch.where(y > 0, dy, torch.zeros_like(dy)).to(g_dt) if with_y else dy.to(g_dt)
        assert torch.equal(_bits(g[:rows, :cols]), _bits(want)), 'with_y=%s' % with_y
        assert bool((g[rows:] == SENT).all()) and bool((g[:, cols:] == SENT).all()), 'g written outside [rows, cols)'


def test_cast_bf16_bit_exact():
    """bags_cast_bf16 against torch's .bfloat16(): random bit patterns plus +-0, +-inf, subnormals, round-to-even ties
    (down and up, in the subnormals and to infinity) and NaNs, which must stay NaN."""
    rows, cols = 33, 1236
    gen = _gen(9)
    raw = torch.randint(0, 2 ** 32, (rows, cols), generator=gen, device=DEV, dtype=torch.int64)
    special = [0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x00000001, 0x807FFFFF, 0x00008000, 0x00018000,
               0x3F808000, 0x3F818000, 0xBF808000, 0x7F7FFFFF, 0x7F7F8000, 0x7F7F7FFF, 0x7FC00000, 0xFFFFFFFF,
               0x7F800001, 0x3F80FFFF, 0x00800000]
    raw[:, :len(special)] = torch.tensor(special, dtype=torch.int64, device=DEV)
    ties = (torch.randint(0, 2 ** 16, (rows, 64), generator=gen, device=DEV, dtype=torch.int64) << 16) | 0x8000
    raw[:, 64:128] = ties   # exactly halfway between two bf16 values
    raw = torch.where(raw >= 2 ** 31, raw - 2 ** 32, raw).to(torch.int32)
    src = torch.full((rows, cols + 8), NAN, dtype=F32, device=DEV)
    src[:, :cols] = raw.view(F32)
    src = src[:, :cols]
    dst = torch.full((rows + 2, cols + 4), SENT, dtype=BF, device=DEV)
    nat.check(nat.lib().bags_cast_bf16(src.data_ptr(), src.stride(0), dst.data_ptr(), dst.stride(0), rows, cols,
                                       _stream()), 'bags_cast_bf16')
    got, want = dst[:rows, :cols], src.bfloat16()
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan), 'NaN must stay NaN (and nothing else become NaN)'
    same = _bits(got) == _bits(want)
    assert bool(same[~nan].all()), 'first difference at %s' % (_first_bad(~same & ~nan),)
    assert bool((dst[rows:] == SENT).all()) and bool((dst[:, cols:] == SENT).all()), 'dst written outside'


# ------------------------------------------------------------------------------------------------ bags_bwd
def _bwd_table(name, C):
    """[(start, len)] per bin."""
    if name == 'full':
        return [(0, C)]
    if name == 'front_gap':
        return [(4, C - 4)]
    if name == 'synthetic':
        from balancedgroupsoftmax_b200.tables import synthetic_tables
        t = synthetic_tables()
        assert t.num_logits == C
        return [tuple(int(v) for v in r) for r in t.pred_slice]
    if name == 'g8_edges':   # edges either side of the dW row tiles' 128 / 256, one-column bins, the last one included
        return [(0, 127), (127, 1), (128, 1), (129, 126), (255, 2), (257, 400), (657, C - 658), (C - 1, 1)]
    if name == 'gaps':       # gaps in the middle and at the end
        if C < 64:
            return [(0, 3), (5, 4)]
        return [(0, 100), (108, 21), (129, 1), (140, 500), (700, C - 712)]
    raise KeyError(name)


def _gout(mode, G):
    if mode is None:
        return None
    if mode == 'one':
        return [1.0] * G
    if mode == 'half':
        return [0.5] * G
    return [1.0, 0.0, -1.0, 2.0, 0.5, -0.5, 0.25, -2.0][:G] if G > 1 else [-1.0]   # 'mixed'


def _col_scale(slices, C, gout):
    """Scale of each dz column: gout of its bin, 0 outside every bin; all 1 without gout."""
    if gout is None:
        return torch.ones(C, dtype=torch.float64, device=DEV)
    s = torch.zeros(C, dtype=torch.float64, device=DEV)
    for (st, ln), g in zip(slices, gout):
        s[st:st + ln] = g
    return s


# C, K, N, operand dtype, table, ldd ('pad': pad64(C), 'tight': C, fp32 only), gout
BWD_CASES = [
    (12, 8, 1, F32, 'full', 'tight', None),
    (12, 264, 65, BF, 'front_gap', 'pad', 'mixed'),
    (12, 8, 63, F32, 'gaps', 'tight', 'one'),
    (12, 1024, 4097, BF, 'full', 'pad', 'mixed'),
    (1236, 1024, 4097, BF, 'synthetic', 'pad', 'mixed'),
    (1236, 264, 64, F32, 'synthetic', 'tight', 'half'),
    (1236, 264, 65, F32, 'full', 'tight', None),
    (1236, 1024, 4097, F32, 'full', 'tight', 'one'),
    (1236, 8, 4097, BF, 'gaps', 'pad', 'one'),
    (1284, 264, 4097, BF, 'g8_edges', 'pad', 'mixed'),
    (1284, 8, 63, F32, 'g8_edges', 'tight', 'half'),
    (1284, 264, 1, BF, 'gaps', 'pad', 'one'),
    (2052, 264, 65, F32, 'gaps', 'tight', 'half'),
    (2052, 1024, 4097, BF, 'g8_edges', 'pad', 'mixed'),
    (2052, 8, 64, BF, 'front_gap', 'pad', 'one'),
    (2052, 264, 63, F32, 'front_gap', 'pad', None),
]
# name, switches, dW, db, dX, caller colsum tiles (0: NULL, recomputed from dz), dW zeroed + BAGS_BWD_DW_PREZEROED
# (otherwise dW holds the sentinel and the flag is off)
BWD_ROUTES = [
    ('merged', {}, True, True, True, 0, False),
    ('merged_colsum3_prezeroed', {}, True, True, True, 3, True),
    ('merged_splits1_colsum1', {'BAGS_DW_SPLITS': 1}, True, True, True, 1, False),
    ('merged_splits16_prezeroed', {'BAGS_DW_SPLITS': 16}, True, True, True, 0, True),
    ('dw_db_splits16_colsum1_prezeroed', {'BAGS_DW_SPLITS': 16}, True, True, False, 1, True),
    ('dw_db', {}, True, True, False, 0, False),
    ('dw_db_splits1_colsum3_prezeroed', {'BAGS_DW_SPLITS': 1}, True, True, False, 3, True),
    ('dw', {}, True, False, False, 0, False),
    ('dx', {}, False, False, True, 0, False),
    ('db', {}, False, True, False, 0, False),
    ('db_colsum1', {}, False, True, False, 1, False),
]


def _bwd_id(c):
    C, K, N, dt, table, ldd, gout = c
    return 'C%d-K%d-N%d-%s-%s-%s-%s' % (C, K, N, 'bf16' if dt == BF else 'fp32', table, ldd, gout or 'nogout')


@pytest.mark.parametrize('case', BWD_CASES, ids=[_bwd_id(c) for c in BWD_CASES])
def test_bwd_exact_all_routes(case):
    """bags_bwd on arbitrary integer dz: dW, db and dX bit-exact against float64 on every route, and every route's
    bits equal to every other route's."""
    ops = _ops()
    C, K, N, dtype, table, ldd_mode, gout_mode = case
    slices = _bwd_table(table, C)
    G = len(slices)
    gout = _gout(gout_mode, G)
    gen = _gen(C * 100003 + K * 101 + N)
    DZ = _ints((N, C), gen, density=min(1.0, 300.0 / max(N, C)))
    X, Wm = _ints((N, K), gen), _ints((C, K), gen)
    if ldd_mode == 'tight':
        assert dtype == F32
        dz = torch.empty((N, C), dtype=dtype, device=DEV)
        dz.copy_(DZ)
    else:
        ldd = ops.pad_cols(C)
        dz = torch.full((N, ldd), NAN, dtype=dtype, device=DEV)
        dz[:, :C] = DZ.to(dtype)
    x, w = _padded(X, dtype), _padded(Wm, dtype)
    s = _col_scale(slices, C, gout)
    dzs = DZ * s
    ref = {'dW': dzs.t() @ X, 'db': dzs.sum(0), 'dX': dzs @ Wm}
    _assert_exact_range(dzs.abs().t() @ X.abs(), 'dW')
    _assert_exact_range(dzs.abs() @ Wm.abs(), 'dX')
    gout_t = torch.tensor(gout, dtype=F32, device=DEV) if gout is not None else None
    colsums = {t: torch.stack([p.sum(0) for p in torch.tensor_split(DZ, t)]).float() for t in (1, 3)}
    slices_host = nat.int32_array([v for sl in slices for v in sl])
    ws = ops.bwd_scratch(w)
    results = {}
    for name, switches, want_dw, want_db, want_dx, tiles, prezeroed in BWD_ROUTES:
        dW = torch.full((C + 2, K + 4), SENT, dtype=F32, device=DEV)
        if prezeroed:
            dW[:C, :K] = 0.0
        db = torch.full((C + 4,), SENT, dtype=F32, device=DEV)
        dX = torch.full((N + 2, K + 8), SENT, dtype=dtype, device=DEV)
        cs = colsums[tiles] if tiles else None
        with _env(BAGS_DW_SPLITS=switches.get('BAGS_DW_SPLITS')):
            nat.check(nat.lib().bags_bwd(
                dz.data_ptr(), dz.stride(0), x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), nat.ptr(gout_t),
                slices_host, nat.ptr(cs), tiles, dW.data_ptr() if want_dw else None, dW.stride(0),
                db.data_ptr() if want_db else None, dX.data_ptr() if want_dx else None, dX.stride(0), ws.data_ptr(),
                ws.numel(), N, K, C, G, _code(dtype), 1 if prezeroed else 0, _stream()), 'bags_bwd')
        outs = {}
        if want_dw:
            _check_exact(dW, C, K, ref['dW'], '%s: dW' % name)
            outs['dW'] = dW[:C, :K]
        if want_db:
            _check_exact(db.view(1, -1), 1, C, ref['db'].view(1, -1), '%s: db' % name)
            outs['db'] = db[:C]
        if want_dx:
            _check_exact(dX, N, K, ref['dX'], '%s: dX' % name)
            outs['dX'] = dX[:N, :K]
        results[name] = outs
    # the same bits on every route, signs of zeros included
    for out in ('dW', 'db', 'dX'):
        runs = [(name, _bits(r[out])) for name, r in results.items() if out in r]
        for name, t in runs[1:]:
            assert torch.equal(t, runs[0][1]), '%s: route %s differs in its bits from %s' % (out, name, runs[0][0])


@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
def test_bwd_numeric(dtype):
    """Random normal operands, synthetic table, non-uniform gout: the full call and the split pair (dW + db, then dX)
    within the numeric bounds (contractions over N for dW, over C for dX)."""
    ops = _ops()
    C, K, N = 1236, 264, 1000 + 77
    slices = _bwd_table('synthetic', C)
    gout = [1.0, 0.5, 0.25, 2.0, 4.0]   # powers of two: W' = gout-scaled W is exact in either operand dtype
    gen = _gen(77)
    DZ = torch.randn(N, C, generator=gen, device=DEV, dtype=torch.float64).to(dtype).double()
    X = torch.randn(N, K, generator=gen, device=DEV, dtype=torch.float64).to(dtype).double()
    Wm = torch.randn(C, K, generator=gen, device=DEV, dtype=torch.float64).to(dtype).double()
    ldd = ops.pad_cols(C)
    dz = torch.zeros((N, ldd), dtype=dtype, device=DEV)
    dz[:, :C] = DZ.to(dtype)
    x, w = _padded(X, dtype), _padded(Wm, dtype)
    s = _col_scale(slices, C, gout)
    gout_t = torch.tensor(gout, dtype=F32, device=DEV)
    dt = ops.DeviceTables(len(slices), 1, C, torch.zeros(len(slices), 1, dtype=torch.int32, device=DEV),
                          torch.zeros(1, dtype=torch.int32, device=DEV),
                          nat.int32_array([v for sl in slices for v in sl]), np.array(slices, dtype=np.int64))
    ttf = 2.0 ** -8 if dtype == F32 else 0.0
    for route in ('full', 'split'):
        if route == 'full':
            dW, db, dX = ops.fused_bwd(dz, x, w, gout_t, dt, None)
        else:
            dW, db, _ = ops.fused_bwd(dz, x, w, gout_t, dt, None, need_dx=False)
            _, _, dX = ops.fused_bwd(dz, x, w, gout_t, dt, None, need_dw=False, need_db=False)
        torch.cuda.synchronize()
        # dW: sum over N rows of the scaled dz; the splits of the reduce-add are at most 16
        S = (DZ.abs() * s.abs()).t() @ X.abs()
        _check_bound(dW, (DZ * s).t() @ X, (ttf + (N + 16) * 2.0 ** -23) * S, 'dW %s' % route)
        cs = (DZ * s).sum(0)
        _check_bound(db, cs, (N + 16) * 2.0 ** -23 * (DZ.abs() * s.abs()).sum(0), 'db %s' % route)
        S = (DZ.abs() * s.abs()) @ Wm.abs()
        ref = (DZ * s) @ Wm
        tol = (ttf + (C + 1) * 2.0 ** -23) * S + (2.0 ** -8 * ref.abs() if dtype == BF else 0.0)
        _check_bound(dX, ref, tol, 'dX %s' % route)


# ------------------------------------------------------------------------------------------------ bags_group_ce
def _ce_table(name, C):
    """[(start, len)] per bin for C >= 1236 (bins of the fused forward's tests at their own C)."""
    def tiling(starts, end):
        return [(s, e - s) for s, e in zip(starts, list(starts[1:]) + [end])]
    if name == 'one_bin':
        return [(0, C)]
    if name == 'contig5':
        return tiling([0, 2, 303, 701, 1201], C)
    if name == 'contig7':
        return tiling([0, 2, 129, 257, 511, 1023, C - 200], C)
    if name == 'onecol7':    # one-column bins at the front, in the middle and at the end
        return tiling([0, 1, 2, 3, 603, 604, C - 1], C)
    if name == 'mod4_8':     # bin edges at every offset inside a float4 chunk
        return tiling([0, 5, 10, 15, 400, 801, 1202, C - 3], C)
    if name == 'gaps8':      # gaps between bins (some inside a float4 chunk) and at the end
        return [(0, 2), (5, 120), (130, 1), (135, 300), (440, 3), (450, 500), (960, 250), (1221, C - 1230)]
    raise KeyError(name)


# the bin tables of test_fused_fwd_epilogue.TABLES, on the materialised route here
FUSED_TABLES = {'edges': ([0, 1, 3, 320, 640, 960], 1280), 'around_edges': ([0, 319, 321, 639, 959, 1279], 1280)}
for _o in range(1, 8):
    FUSED_TABLES['offset%d' % _o] = ([0] + [8 * j + _o for j in (3, 41, 80, 120, 150)], 1236)

# C (NV = 10 up to 1280 columns, 16 up to 2048, 32 beyond), table, N, weights, dz dtype, avg given
CE_CASES = [
    (1236, 'contig5', 1000, 'u8', BF, True),
    (1236, 'one_bin', 1, None, F32, False),
    (1236, 'gaps8', 9, 'f32', F32, True),
    (1284, 'contig7', 7, 'u8', F32, False),
    (1284, 'mod4_8', 1000, 'f32', BF, True),
    (1284, 'gaps8', 8, None, BF, False),
    (2048, 'mod4_8', 1000, 'u8', F32, True),
    (2048, 'onecol7', 9, None, BF, False),
    (2052, 'gaps8', 1000, 'f32', F32, False),
    (2052, 'contig5', 7, 'u8', BF, True),
    (2052, 'onecol7', 1000, 'u8', F32, True),
    (4096, 'one_bin', 1000, None, F32, False),
    (4096, 'mod4_8', 8 * 4096 + 3, 'u8', BF, True),     # every CTA walks many row octets
    (1236, 'contig5', 8 * 4096 + 3, 'f32', F32, False),
] + [(FUSED_TABLES[k][1], k, 1000, 'u8', BF, True) for k in sorted(FUSED_TABLES)]


def _ce_slices(C, table):
    if table in FUSED_TABLES:
        starts, end = FUSED_TABLES[table]
        return [(s, e - s) for s, e in zip(starts, starts[1:] + [end])]
    return _ce_table(table, C)


@pytest.mark.parametrize('case', CE_CASES, ids=['C%d-%s-N%d-%s-dz_%s-%s' % (c[0], c[1], c[2], c[3] or 'noweights',
                                                                          'bf16' if c[4] == BF else 'fp32',
                                                                          'avg' if c[5] else 'noavg') for c in CE_CASES])
def test_group_ce_vs_float64(case):
    """Loss relative error <= 1e-5, lse <= 2e-6 max(1, |lse|), dz elementwise <= 2e-6 w/avg (plus 2^-8 |dz| when dz
    is bf16: round-to-nearest into 8 significant bits errs by up to half a unit in the last place, 2^-8 relative);
    dz exactly 0 in gap columns, padding columns [C, ldd) untouched, colsum = sum_n dz."""
    ops = _ops()
    C, table, N, weights, dz_dtype, with_avg = case
    slices = _ce_slices(C, table)
    G, classes = len(slices), 300
    gen = _gen(C + 7 * N + G)
    z = _padded(torch.randn(N, C, generator=gen, device=DEV) * 1.5, F32)
    lens = torch.tensor([ln for _, ln in slices], device=DEV)
    l2b = (torch.rand(G, classes, generator=gen, device=DEV) * lens[:, None]).long()
    l2b[:, 0] = lens              # in-bin labels outside [0, len_g): scored against in-bin label 0
    l2b[:, 1] = -1
    l2b[:, 2] = lens + 7
    labels = torch.randint(0, classes, (N,), generator=gen, device=DEV)
    labels[1::11] = -1            # labels outside [0, classes): in-bin label 0 of every bin
    labels[4::13] = classes
    if weights == 'u8':
        wm = (torch.rand(G, N, generator=gen, device=DEV) < 0.7).to(torch.uint8)
    elif weights == 'f32':
        wm = torch.rand(G, N, generator=gen, device=DEV) * 2.0
    else:
        wm = None
    wd = wm.double() if wm is not None else torch.ones(G, N, dtype=torch.float64, device=DEV)
    avg = wd.sum(1).clamp_min(1.0).float() if with_avg else None
    avg_d = avg.double() if with_avg else torch.full((G,), float(N), dtype=torch.float64, device=DEV)
    ldd = ops.pad_cols(C) + (64 if C % 64 == 0 else 0)
    dz = torch.full((N, ldd), SENT, dtype=dz_dtype, device=DEV)
    loss = torch.empty(G, dtype=F32, device=DEV)
    lse = torch.empty((N, G), dtype=F32, device=DEV)
    colsum = torch.full((C,), NAN, dtype=F32, device=DEV)
    wptr, wcode = ops._weights_arg(wm)
    ws = ops._workspace(DEV)
    l2b32 = l2b.int().contiguous()
    nat.check(nat.lib().bags_group_ce(
        z.data_ptr(), z.stride(0), labels.data_ptr(), l2b32.data_ptr(),
        nat.int32_array([v for sl in slices for v in sl]), nat.ptr(wptr), wcode, nat.ptr(avg), N, C, G, classes,
        loss.data_ptr(), lse.data_ptr(), dz.data_ptr(), ldd, _code(dz_dtype), colsum.data_ptr(), ws.data_ptr(),
        ws.numel(), _stream()), 'bags_group_ce')

    zd = z.double()
    lab_ok = (labels >= 0) & (labels < classes)
    ref_dz = torch.zeros(N, C, dtype=torch.float64, device=DEV)
    coef_max = torch.zeros(N, C, dtype=torch.float64, device=DEV)
    in_bin = torch.zeros(C, dtype=torch.bool, device=DEV)
    for g, (s, ln) in enumerate(slices):
        zs = zd[:, s:s + ln]
        t = torch.where(lab_ok, l2b[g][labels.clamp(0, classes - 1)], torch.zeros_like(labels))
        t = torch.where((t >= 0) & (t < ln), t, torch.zeros_like(t))
        lse_ref = torch.logsumexp(zs, 1)
        coef = wd[g] / avg_d[g]
        ref_loss = (coef * (lse_ref - zs.gather(1, t[:, None])[:, 0])).sum()
        # relative 1e-5, and each row's lse bound (a one-column bin has loss 0 up to the rounding of its lse)
        loss_tol = 1e-5 * abs(ref_loss.item()) + 2e-6 * (coef * lse_ref.abs().clamp_min(1.0)).sum().item()
        assert abs(loss[g].item() - ref_loss.item()) <= loss_tol, (g, loss[g].item(), ref_loss.item())
        _check_bound(lse[:, g], lse_ref, 2e-6 * lse_ref.abs().clamp_min(1.0), 'lse bin %d' % g)
        onehot = torch.nn.functional.one_hot(t, ln).double()
        ref_dz[:, s:s + ln] = coef[:, None] * (torch.softmax(zs, 1) - onehot)
        coef_max[:, s:s + ln] = coef[:, None]
        in_bin[s:s + ln] = True
    got = dz[:, :C]
    tol = 2e-6 * coef_max + (2.0 ** -8 * ref_dz.abs() if dz_dtype == BF else 0.0)
    _check_bound(got, ref_dz, tol, 'dz')
    assert bool((got[:, ~in_bin] == 0).all()), 'dz is not 0 in the columns outside every bin'
    assert bool((dz[:, C:] == SENT).all()), 'dz padding columns were written'
    # colsum: the same per-element bound summed over the rows, plus fp32 summation along the kernel's longest chain
    # of additions (rows of one thread, 8 warps, one reduce-add per CTA: <= 320 here)
    cs_tol = 2e-6 * coef_max.sum(0) + 320 * 2.0 ** -24 * ref_dz.abs().sum(0)
    _check_bound(colsum, ref_dz.sum(0), cs_tol, 'colsum')


# ------------------------------------------------------------------------------------------------ bags_merge_scores
@pytest.mark.parametrize('C', [1284, 2048, 2052, 4096])
def test_merge_scores_vs_float64(C):
    """G = 8 with gaps (NV = 16 and 32), cls2col with -1 entries and columns in gaps: |error| <= 1e-6."""
    slices = _ce_table('gaps8', C)
    G, classes, N = len(slices), 1500, 1000
    gen = _gen(C)
    z = _padded(torch.randn(N, C, generator=gen, device=DEV) * 2.0, F32)
    c2c = torch.randint(0, C, (classes,), generator=gen, device=DEV).int()
    c2c[0] = 0
    c2c[3::17] = -1
    c2c[5] = 1
    c2c[6] = 3                   # a column in the first gap
    lds = classes + 3
    scores = torch.full((N + 2, lds), SENT, dtype=F32, device=DEV)
    nat.check(nat.lib().bags_merge_scores(z.data_ptr(), z.stride(0), nat.int32_array([v for sl in slices for v in sl]),
                                          c2c.data_ptr(), N, C, G, classes, scores.data_ptr(), lds, _stream()),
              'bags_merge_scores')
    zd = z.double()
    P = torch.zeros(N, C, dtype=torch.float64, device=DEV)
    binof = torch.full((C,), -1, dtype=torch.long, device=DEV)
    for g, (s, ln) in enumerate(slices):
        P[:, s:s + ln] = torch.softmax(zd[:, s:s + ln], 1)
        binof[s:s + ln] = g
    pfg = P[:, slices[0][0] + 1] if slices[0][1] > 1 else torch.zeros(N, dtype=torch.float64, device=DEV)
    col = c2c.long()
    valid = col >= 0
    colc = col.clamp_min(0)
    p = P[:, colc]
    ref = torch.where(binof[colc] == 0, p, pfg[:, None] * p)
    ref = torch.where((valid & (binof[colc] >= 0))[None, :], ref, torch.zeros_like(ref))
    _check_bound(scores[:N, :classes], ref, 1e-6, 'scores')
    assert bool((scores[N:] == SENT).all()) and bool((scores[:, classes:] == SENT).all()), 'scores written outside'


# ------------------------------------------------------------------------------------------------ end to end
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
def test_end_to_end_unfusable_table(dtype):
    """G = 8, C = 2052 (not fused-eligible): bags_fwd with materialised logits, then bags_bwd, against the oracle's
    closed form in float64 on the same rounded operands and masks.  Norm-relative tolerances of test_gpu_parity.py,
    except fp32 gradients: their contractions take both operands in TF32 (10 stored mantissa bits, up to 2^-10
    relative each), so 2^-8 as in the numeric tier."""
    ops = _ops()
    from oracle import bags_oracle as O
    C, K, N, classes = 2052, 256, 1000 + 77, 900
    slices = [(0, 2), (2, 129), (131, 127), (258, 1), (259, 500), (759, 600), (1359, 690), (2049, 3)]
    G = len(slices)
    g = torch.Generator().manual_seed(11)
    lens = torch.tensor([ln for _, ln in slices])
    l2b = (torch.rand(G, classes, generator=g) * lens[:, None]).long()
    l2b[:, 0] = 0
    ps = torch.tensor(slices, dtype=torch.long)
    dt = ops.DeviceTables(G, classes, C, l2b.int().to(DEV), torch.zeros(classes, dtype=torch.int32, device=DEV),
                          nat.int32_array([v for sl in slices for v in sl]), np.array(slices, dtype=np.int64))
    assert not ops.fused_eligible(dt)
    x = torch.relu(torch.randn(N, K, generator=g)).to(dtype)
    W = (torch.randn(C, K, generator=g) * 0.05).to(dtype)
    b = torch.randn(C, generator=g) * 0.1
    labels = torch.randint(0, classes, (N,), generator=g)
    wmask = (torch.rand(G, N, generator=g) < 0.7).to(torch.uint8)
    wmask[0] = 1
    gout = [1.0, 0.5, 0.25, 2.0, 1.5, 1.0, 0.75, 3.0]
    wm_d = wmask.to(DEV)
    avg = ops.mask_avg(wm_d)
    loss, logits, _, dz, _ = ops.fused_fwd(x.to(DEV), W.to(DEV), b.to(DEV), labels.to(DEV), dt, wm_d, avg)
    assert logits is not None
    dW, db, dX = ops.fused_bwd(dz, x.to(DEV), W.to(DEV), torch.tensor(gout, device=DEV), dt, None)
    torch.cuda.synchronize()
    xo, Wo, bo = x.double(), W.double(), b.double()
    remapped = ([l2b[i][labels] for i in range(G)], [wmask[i].long() for i in range(G)],
                [float(a) for a in avg.cpu().tolist()])
    ref = O.bags_loss(O.fc_cls(xo, Wo, bo), labels, l2b, ps, remapped=remapped)
    _, dW_ref, db_ref, dX_ref = O.closed_form_grads(xo, Wo, bo, labels, l2b, ps, remapped, gout=gout)
    tol = dict(loss=1e-3, grad=2.0 ** -8) if dtype == F32 else dict(loss=2e-3, grad=5e-3)
    for i in range(G):
        r = ref['loss_cls_bin%d' % i].item()
        assert abs(loss[i].item() - r) <= tol['loss'] * max(abs(r), 1e-3), (i, loss[i].item(), r)

    def rel(a, r):
        return ((a.double().cpu() - r).norm() / r.norm().clamp_min(1e-30)).item()
    assert rel(dW, dW_ref) <= tol['grad']
    assert rel(db, db_ref) <= tol['grad']
    assert rel(dX, dX_ref) <= tol['grad']
