"""GPU: the fused mask loss -- bags_mask_sort_kernel, bags_mask_fwd_kernel and bags_mask_bwd_kernel -- against float64 per
element at its edges.

Every reference is plain torch in float64 (tests/mask_oracle.py: mask_terms, and error_bounds / reduction_bounds,
whose derivation is in their docstrings), never this library.  Arguments the Python wrappers hide (ldw, lddw, a NULL
bias or gout, y and dY one element off a 16-byte boundary) go through ctypes.  W's padding columns [Cin, ldw) and the
elements of y's buffer around y hold NaN; every output byte the kernels must not write (dW columns [Cin, lddw), the
row and element past dW / db / g / dY / the loss / rsum, the class index past its valid RoIs, every output of a
gradient that is not asked for) holds a sentinel that must survive.  Comparisons called bit-exact compare bit
patterns, so a -0 where +0 is expected fails.

Three tiers of input (mask_oracle.tier_inputs):
  * exact: small-integer y and W, b a multiple of 2^-3, every partial sum of z below 2^20 (asserted per case), so z
    is exact in fp32 for four pixels a thread (16 channel groups) and for one (4 groups).  g, the loss, dW and db are
    held to error_bounds(z_exact=True): only the kernel's own expf / log1pf / division and its sums err.
  * saturated: one channel of +-1 times a W entry of +-256, the rest below 64, so |z| >= 128 and expf(-|z|) is 0:
    s is exactly 0 or 1, g is exactly 0 or +-fl(1 / n), the loss terms are multiples of 2^-3 whose sum is exact, so
    g and the loss are bit-exact; when n = P H W is a power of two, dW, db and dY equal float64 bit for bit too.
  * numeric: y = relu(normal), W and b normal, 0/1 and soft targets: everything within error_bounds.
In every tier:
  * dY is bit-exact against the kernel's own g: ((fp32(gout) g) W[l, c]) rounded to y's dtype, +0 on invalid rows --
    the mapping of every dY element at zero tolerance, whatever g's own bound;
  * dW and db are within reduction_bounds of float64 sums of the kernel's own g (an error of g cannot hide in a
    bound that allows for one);
  * g of an invalid row, dW rows and db of a class without RoIs are +0; labels -1, classes, classes + 7 and 2^40 are
    invalid (they count in n and contribute nothing; with P = 0 the loss is +0);
  * the class index (offsets, then RoI ids) equals torch.argsort(labels[valid], stable=True) with its counts;
  * the forward's arrival counter (word 17 of ops._workspace) is back at 0.
With y and dY one element off (one pixel a thread although H W % 4 == 0) the exact and saturated tiers give results
bit-identical to the aligned call on the same values; in the numeric tier both are held to the bounds.
"""
import pytest
import torch

import mask_oracle as MO
from balancedgroupsoftmax_b200 import _native as nat

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
BF, F32 = torch.bfloat16, torch.float32
SENT = -7.0
ISENT = -123457
NAN = float('nan')
PAD = 64                  # sentinel elements past every output
COUNTER_WORD = 17         # the forward's arrival counter in the workspace (kMaskCounterWord)
ALL = (True, True, True)


def _ops():
    from balancedgroupsoftmax_b200 import ops
    return ops


def _bits(x):
    x = x.contiguous()
    return x.view(torch.int32) if x.dtype == F32 else x.view(torch.int16) if x.dtype == BF else x


def _same_bits(got, want, what):
    a, b = _bits(got.cpu()), _bits(want.cpu())
    assert a.shape == b.shape, (what, a.shape, b.shape)
    bad = (a != b).reshape(-1)
    if bad.any():
        i = int(bad.nonzero()[0])
        raise AssertionError('%s: %d of %d elements differ; first at flat %d: got %r, want %r' % (
            what, int(bad.sum()), bad.numel(), i, got.reshape(-1)[i].item(), want.reshape(-1)[i].item()))


def _within(got, want, bound, what):
    got, want = got.double().to(DEV), want.double().to(DEV)
    err = (got - want).abs()
    bad = ~(err <= torch.as_tensor(bound, dtype=torch.float64, device=DEV))
    if bad.any():
        i = int(bad.reshape(-1).nonzero()[0])
        bd = torch.as_tensor(bound, dtype=torch.float64, device=DEV).expand_as(err).reshape(-1)[i].item()
        raise AssertionError('%s: %d of %d elements outside the bound; first at flat %d: got %r, want %r, err %g, '
                             'bound %g' % (what, int(bad.sum()), bad.numel(), i, got.reshape(-1)[i].item(),
                                           want.reshape(-1)[i].item(), err.reshape(-1)[i].item(), bd))


def _all_sent(x, what, sent=SENT):
    x = x.cpu()
    assert bool((_bits(x) == _bits(torch.full_like(x, sent))).all()), '%s: a sentinel was overwritten' % what


# ------------------------------------------------------------------------------------------------ the launches
def _enqueue(y, W, b, labels, t, classes, ldw=None, lddw=None, gout=None, need=ALL, offset=0):
    """bags_mask_fwd then bags_mask_bwd on the current stream through ctypes, into sentinel-filled buffers; y, dY at
    ``offset`` elements from an aligned buffer."""
    lib, ops = nat.lib(), _ops()
    P, Cin, HW = y.shape
    dtype = y.dtype
    ldw = ldw or Cin
    lddw = lddw or Cin
    code = nat.DTYPE_BF16 if dtype == BF else nat.DTYPE_F32
    tiles = -(-HW // MO.TILE)
    numel = P * Cin * HW
    bufs = dict(P=P, Cin=Cin, HW=HW, classes=classes, lddw=lddw, offset=offset, numel=numel, need=need, dtype=dtype)
    Wp = torch.full((classes, ldw), NAN, device=DEV)
    Wp[:, :Cin] = W.to(DEV)
    yb = torch.full((numel + offset + PAD,), NAN, dtype=dtype, device=DEV)
    yb[offset:offset + numel] = y.reshape(-1).to(DEV)
    bd = None if b is None else b.to(DEV)
    ld, td = labels.to(DEV), t.to(DEV).contiguous()
    rsum_floats = P * tiles * (Cin + 2)
    out = dict(loss=torch.full((1 + PAD,), SENT, device=DEV), g=torch.full((P * HW + PAD,), SENT, device=DEV),
               rsum=torch.full((rsum_floats + PAD,), SENT, device=DEV),
               index=torch.full((classes + 1 + P + PAD,), ISENT, dtype=torch.int32, device=DEV),
               dW=torch.full(((classes + 1) * lddw,), SENT, device=DEV),
               db=torch.full((classes + 1,), SENT, device=DEV),
               dY=torch.full((numel + offset + PAD,), SENT, dtype=dtype, device=DEV))
    ws = ops._workspace(DEV)
    stream = torch.cuda.current_stream(DEV).cuda_stream
    nat.check(lib.bags_mask_fwd(
        yb[offset:].data_ptr(), code, Wp.data_ptr(), ldw, nat.ptr(bd), ld.data_ptr(), td.data_ptr(), P, Cin, HW,
        classes, out['loss'].data_ptr(), out['g'].data_ptr(), out['rsum'].data_ptr(), rsum_floats,
        out['index'].data_ptr(), ws.data_ptr(), ws.numel(), stream), 'bags_mask_fwd')
    go = None if gout is None else torch.tensor([gout], dtype=F32, device=DEV)
    nat.check(lib.bags_mask_bwd(
        out['g'].data_ptr(), out['rsum'].data_ptr(), nat.ptr(go), code, Wp.data_ptr(), ldw, ld.data_ptr(),
        out['index'].data_ptr(), P, Cin, HW, classes, out['dW'].data_ptr() if need[0] else None, lddw,
        out['db'].data_ptr() if need[1] else None, out['dY'][offset:].data_ptr() if need[2] else None, stream),
        'bags_mask_bwd')
    bufs.update(out, keep=(Wp, yb, bd, ld, td, go), rsum_floats=rsum_floats)
    return bufs


def _collect(bufs, labels):
    """Synchronise; check the counter and every sentinel; the outputs on CPU ({loss, g, index, dW, db, dY} with
    None for what was not asked)."""
    torch.cuda.synchronize(DEV)
    assert _ops()._workspace(DEV).view(torch.int32)[COUNTER_WORD].item() == 0, 'arrival counter not reset'
    P, Cin, HW, C, lddw, off, numel = (bufs[k] for k in ('P', 'Cin', 'HW', 'classes', 'lddw', 'offset', 'numel'))
    need = bufs['need']
    cpu = {k: bufs[k].cpu() for k in ('loss', 'g', 'rsum', 'index', 'dW', 'db', 'dY')}
    _all_sent(cpu['loss'][1:], 'past the loss')
    _all_sent(cpu['g'][P * HW:], 'past g')
    _all_sent(cpu['rsum'][bufs['rsum_floats']:], 'past rsum')
    nvalid = int(MO.valid_rows(labels, C).sum())
    _all_sent(cpu['index'][C + 1 + nvalid:], 'past the class index', ISENT)
    dW = cpu['dW'].reshape(C + 1, lddw)
    _all_sent(dW[C], 'the row past dW')
    _all_sent(dW[:C, Cin:], 'dW columns [Cin, lddw)')
    _all_sent(cpu['db'][C:], 'past db')
    _all_sent(cpu['dY'][:off], 'before dY')
    _all_sent(cpu['dY'][off + numel:], 'past dY')
    if not need[0]:
        _all_sent(dW, 'dW not asked for')
    if not need[1]:
        _all_sent(cpu['db'], 'db not asked for')
    if not need[2]:
        _all_sent(cpu['dY'], 'dY not asked for')
    return dict(loss=cpu['loss'][0], g=cpu['g'][:P * HW].reshape(P, HW), index=cpu['index'][:C + 1 + nvalid],
                dW=dW[:C, :Cin] if need[0] else None, db=cpu['db'][:C] if need[1] else None,
                dY=cpu['dY'][off:off + numel].reshape(P, Cin, HW) if need[2] else None)


def _run(y, W, b, labels, t, classes, **kw):
    return _collect(_enqueue(y, W, b, labels, t, classes, **kw), labels)


# ------------------------------------------------------------------------------------------------ the checks
def _check_common(out, y, W, labels, classes, gout):
    P, Cin, HW = y.shape
    go = 1.0 if gout is None else gout
    valid = MO.valid_rows(labels, classes)
    vid = valid.nonzero().reshape(-1)
    # the class index: offsets, then the valid RoIs ordered by class and by id inside a class
    counts = torch.bincount(labels[vid], minlength=classes)
    offsets = torch.cat([torch.zeros(1, dtype=torch.int64), counts.cumsum(0)])
    order = vid[torch.argsort(labels[vid], stable=True)]
    assert torch.equal(out['index'], torch.cat([offsets, order]).int()), 'class index'
    # invalid rows and absent classes: +0
    _same_bits(out['g'][~valid], torch.zeros(int((~valid).sum()), HW), 'g of invalid rows')
    absent = counts == 0
    if out['dW'] is not None:
        _same_bits(out['dW'][absent], torch.zeros(int(absent.sum()), Cin), 'dW of absent classes')
    if out['db'] is not None:
        _same_bits(out['db'][absent], torch.zeros(int(absent.sum())), 'db of absent classes')
    # dY from the kernel's own g, bit for bit: two fp32 products, then y's dtype
    if out['dY'] is not None:
        lab = torch.where(valid, labels, torch.zeros_like(labels))
        want = ((torch.tensor(go, dtype=F32) * out['g']).unsqueeze(1) * W.float()[lab].unsqueeze(2)).to(y.dtype)
        want[~valid] = 0
        _same_bits(out['dY'], want, 'dY against the kernel g')
    # dW, db against float64 sums of the kernel's own g: the reduction's roundings only
    if P and (out['dW'] is not None or out['db'] is not None):
        red = MO.reduction_bounds(out['g'].to(DEV), y.to(DEV), labels, classes, go)
        gg = out['g'].double().to(DEV) * go
        lv, vd = labels[vid].to(DEV), vid.to(DEV)
        if out['dW'] is not None:
            dW = torch.zeros(classes, Cin, dtype=torch.float64, device=DEV).index_add_(
                0, lv, torch.einsum('pq,pcq->pc', gg[vd], y.to(DEV).double()[vd]))
            _within(out['dW'], dW, red['dW'], 'dW against the kernel g')
        if out['db'] is not None:
            db = torch.zeros(classes, dtype=torch.float64, device=DEV).index_add_(0, lv, gg[vd].sum(1))
            _within(out['db'], db, red['db'], 'db against the kernel g')


def _pow2(n):
    return n > 0 and n & (n - 1) == 0


def _check_tier(tier, out, y, W, b, labels, t, classes, gout):
    P, Cin, HW = y.shape
    go = 1.0 if gout is None else gout
    if P == 0:
        _same_bits(out['loss'], torch.zeros(()), 'loss with P = 0')
        return
    n = P * HW
    if tier == 'saturated':
        assert MO.saturated_min_abs_z(y, W, b, labels) >= 128
        o = MO.mask_terms(y.to(DEV), W, b, labels, t, gout=go)
        z = o['z'].cpu()
        valid = MO.valid_rows(labels, classes)
        nf = torch.tensor(float(n), dtype=F32)
        want_g = torch.where(valid.unsqueeze(1), ((z >= 0).float() - t) / nf, torch.zeros(()))
        _same_bits(out['g'], want_g, 'g (saturated)')
        terms = (torch.clamp(z, min=0) - z * t.double())[valid]      # exact: multiples of 2^-3
        S = terms.sum()
        assert S.abs() < 2 ** 21
        _same_bits(out['loss'], S.float() / nf, 'loss (saturated)')
        if _pow2(n):
            # float64's g is +-e^-|z|, not 0, where the kernel's s - t is exactly 0: what rounds to zero in fp32
            # has float64's sign.  A zero sum of dW or db is +0 (as for a class without RoIs); the sign of a zero dY
            # element is the product's, pinned against the kernel's g above, so zeros compare as values there
            for name in ('dW', 'db'):
                if out[name] is not None:
                    want = o[name].float().cpu()
                    want[want == 0] = 0.0
                    _same_bits(out[name], want, name + ' (saturated, n a power of two)')
            if out['dY'] is not None:
                want = o['dY'].reshape(P, Cin, HW).to(y.dtype).cpu()
                zero = want == 0
                assert bool((out['dY'][zero] == 0).all()), 'dY (saturated, n a power of two): a nonzero for 0'
                _same_bits(out['dY'][~zero], want[~zero], 'dY (saturated, n a power of two)')
        return
    if tier == 'exact':
        assert MO.exact_partial_max(y, W, b, labels) < MO.EXACT_LIMIT
    eb = MO.error_bounds(y.to(DEV), W, b, labels, t, gout=go, z_exact=tier == 'exact')
    o = eb['terms']
    _within(out['g'], o['g'], eb['g'], 'g')
    _within(out['loss'], o['loss'], eb['loss'], 'loss')
    for name in ('dW', 'db'):
        if out[name] is not None:
            _within(out[name], o[name], eb[name], name)


# ------------------------------------------------------------------------------------------------ the cases
HWS = [1, 2, 3, 4, 31, 32, 33, 60, 63, 64, 65, 96, 97, 127, 128, 129, 196, 221, 784, 3136]
CINS = [1, 3, 4, 5, 15, 16, 17, 31, 32, 33, 63, 64, 256]
CLASSES = [1, 2, 1231, 8192]
NEEDS = [ALL, (True, False, False), (False, True, False), (False, False, True), (True, True, False),
         (True, False, True), (False, True, True)]
TIERS = ['exact', 'saturated', 'numeric']
BUDGET = 1 << 21          # elements of y per sampled case


def _case(tier, dtype, P, Cin, HW, classes, gout=-0.5, bias=True, need=ALL, ldw_pad=0, lddw_pad=0, misalign=False,
          soft=False, invalid=False, one_class=False, seed=0):
    return dict(tier=tier, dtype=dtype, P=P, Cin=Cin, HW=HW, classes=classes, gout=gout, bias=bias, need=need,
                ldw_pad=ldw_pad, lddw_pad=lddw_pad, misalign=misalign, soft=soft, invalid=invalid,
                one_class=one_class, seed=seed)


def _name(c):
    s = '%s-%s-p%d-cin%d-hw%d-k%d' % (c['tier'], 'bf16' if c['dtype'] == BF else 'fp32', c['P'], c['Cin'], c['HW'],
                                     c['classes'])
    s += '-go%s' % ('null' if c['gout'] is None else c['gout'])
    if not c['bias']:
        s += '-nobias'
    if c['need'] != ALL:
        s += '-' + ''.join(k for k, w in zip(('dW', 'db', 'dY'), c['need']) if w)
    for k, tag in (('ldw_pad', 'ldw+'), ('lddw_pad', 'lddw+')):
        if c[k]:
            s += '-%s%d' % (tag, c[k])
    for k in ('misalign', 'soft', 'invalid', 'one_class'):
        if c[k]:
            s += '-' + k
    return s


def _build_cases():
    """Every H W, Cin and class count in each tier, the P, gout, bias, output-subset, padding and alignment knobs
    dealt over them; then the sort-batch, one-class, power-of-two and many-wave cases."""
    cases = []
    for ti, tier in enumerate(TIERS):
        gouts = [None, 1.0, -0.5, 0.0] + ([0.3] if tier != 'saturated' else [])
        for i, HW in enumerate(HWS):
            Cin = CINS[(3 * i + 5 * ti) % len(CINS)]
            classes = CLASSES[(i + ti) % len(CLASSES)]
            P = [7, 2, 33, 300, 1][(i + ti + i // 5) % 5]
            while P > 1 and P * Cin * HW > BUDGET:
                P //= 2
            if tier == 'saturated':
                while P > 1 and P * HW > 6000:        # the exact loss sum stays below 2^21
                    P //= 2
            cases.append(_case(
                tier, BF if (i + ti) % 2 else F32, P, Cin, HW, classes, gout=gouts[i % len(gouts)],
                bias=i % 6 != 5, need=NEEDS[i % len(NEEDS)], ldw_pad=5 if i % 3 == 1 else 0,
                lddw_pad=3 if i % 3 == 2 else 0, misalign=HW % 4 == 0 and i % 2 == 0,
                soft=tier != 'saturated' and i % 2 == 1, invalid=i % 3 == 0 and P >= 2,
                one_class=i % 5 == 4 and P >= 33, seed=100 * ti + i))
    # the class index past one sort batch (4096 labels), up to 8192 classes
    for j, (P, classes) in enumerate([(4095, 8192), (4096, 1231), (4097, 8192), (8193, 2), (8193, 8192)]):
        cases.append(_case(('exact', 'numeric')[j % 2], BF if j % 2 else F32, P, 3, 33 if j % 2 else 4, classes,
                           invalid=True, misalign=j == 0, seed=500 + j))
    for dtype in (BF, F32):
        cases.append(_case('exact', dtype, 0, 5, 33, 7, seed=600))
    # one class holding every RoI: its units spread over all 8 warps
    cases.append(_case('exact', BF, 300, 33, 64, 1231, one_class=True, misalign=True, seed=700))
    cases.append(_case('numeric', F32, 1000, 31, 4, 1231, one_class=True, soft=True, seed=701))
    cases.append(_case('saturated', F32, 2048, 32, 1, 1, gout=1.0, seed=702))
    # saturated with n = P H W a power of two: dW, db and dY bit for bit
    for j, (P, HW) in enumerate([(64, 1), (32, 4), (16, 16), (8, 64), (16, 256), (4, 1024), (1, 4096)]):
        cases.append(_case('saturated', BF if j % 2 else F32, P, [17, 64, 3, 33, 5, 16, 1][j], HW, [2, 1231, 1, 8192][j % 4],
                           gout=[None, -0.5, 1.0, 0.0][j % 4], bias=j != 3, misalign=HW % 4 == 0 and j % 2 == 0,
                           invalid=j == 1, ldw_pad=5 if j == 2 else 0, lddw_pad=3 if j == 5 else 0, seed=800 + j))
    # tens of thousands of CTAs: the last CTA's loss sum over many waves
    cases.append(_case('exact', BF, 4097, 3, 784, 1231, invalid=True, seed=900))
    return {_name(c): c for c in cases}


CASES = _build_cases()


def _inputs(c):
    y, W, b, labels, t = MO.tier_inputs(c['tier'], c['P'], c['Cin'], c['HW'], c['classes'], c['dtype'], seed=c['seed'],
                                        soft=c['soft'], invalid=c['invalid'], one_class=c['one_class'])
    return y, W, (b if c['bias'] else None), labels, t


@pytest.mark.parametrize('name', list(CASES))
def test_mask_loss_vs_float64(name):
    c = CASES[name]
    y, W, b, labels, t = _inputs(c)
    kw = dict(ldw=c['Cin'] + c['ldw_pad'], lddw=c['Cin'] + c['lddw_pad'], gout=c['gout'], need=c['need'])
    out = _run(y, W, b, labels, t, c['classes'], **kw)
    _check_common(out, y, W, labels, c['classes'], c['gout'])
    _check_tier(c['tier'], out, y, W, b, labels, t, c['classes'], c['gout'])
    if c['misalign']:
        # one pixel a thread although H W % 4 == 0
        off = _run(y, W, b, labels, t, c['classes'], offset=1, **kw)
        if c['tier'] == 'numeric':
            _check_common(off, y, W, labels, c['classes'], c['gout'])
            _check_tier(c['tier'], off, y, W, b, labels, t, c['classes'], c['gout'])
        else:
            for k in out:
                if out[k] is not None:
                    _same_bits(off[k], out[k], k + ': one pixel a thread against four')


def test_cases_cover_the_edges():
    cs = list(CASES.values())
    for tier in TIERS:
        mine = [c for c in cs if c['tier'] == tier]
        assert {c['HW'] for c in mine} >= set(HWS) and {c['Cin'] for c in mine} >= set(CINS)
        assert {c['classes'] for c in mine} >= set(CLASSES) and {c['dtype'] for c in mine} == {BF, F32}
        assert {c['need'] for c in mine} == set(NEEDS) and any(c['misalign'] for c in mine)
        assert any(not c['bias'] for c in mine) and any(c['ldw_pad'] for c in mine) and any(c['lddw_pad'] for c in mine)
        assert {None, 1.0, -0.5, 0.0} <= {c['gout'] for c in mine}
    assert {0, 1, 2, 7, 300, 4095, 4096, 4097, 8193} <= {c['P'] for c in cs}
    assert any(c['tier'] == 'numeric' and c['gout'] == 0.3 and c['need'][2] for c in cs)
    assert sum(c['tier'] == 'saturated' and _pow2(c['P'] * c['HW']) for c in cs) >= 7


def test_back_to_back_grids_on_one_workspace():
    """Forwards of 53k, 7 and 53k CTAs enqueued back to back on one workspace (one arrival counter) give what each
    gives alone."""
    cs = [CASES[n] for n in CASES if CASES[n]['P'] == 4097 and CASES[n]['HW'] == 784]
    cs = [cs[0], CASES[[n for n in CASES if CASES[n]['P'] == 7][0]], cs[0]]
    ins = [_inputs(c) for c in cs]
    alone = [_run(*i, c['classes'], gout=c['gout']) for c, i in zip(cs, ins)]
    bufs = [_enqueue(*i, c['classes'], gout=c['gout']) for c, i in zip(cs, ins)]
    torch.cuda.synchronize(DEV)
    for a, bf, i in zip(alone, bufs, ins):
        got = _collect(bf, i[3])
        for k in a:
            _same_bits(got[k], a[k], k + ' back to back')


@pytest.mark.parametrize('dtype', [BF, F32], ids=['bf16', 'fp32'])
def test_wrappers_with_a_storage_offset(dtype):
    """ops.mask_fwd / mask_bwd on a y one element into its storage (one pixel a thread) give the aligned call's
    results bit for bit in the exact tier, and the same as the ctypes launch."""
    ops = _ops()
    P, Cin, H, W_, C = 9, 17, 8, 8, 13
    y, W, b, labels, t = MO.tier_inputs('exact', P, Cin, H * W_, C, dtype, seed=31, invalid=True, soft=True)
    buf = torch.empty(y.numel() + 1, dtype=dtype, device=DEV)
    buf[1:] = y.reshape(-1).to(DEV)
    y_off = buf[1:].view(P, Cin, H, W_)
    assert y_off.storage_offset() == 1 and y_off.is_contiguous()
    Wd, bd, ld, td = W.to(DEV), b.to(DEV), labels.to(DEV), t.reshape(P, H, W_).to(DEV)
    go = torch.tensor([-0.5], device=DEV)
    res = []
    for yy in (y.reshape(P, Cin, H, W_).to(DEV), y_off):
        loss, g, rsum, index = ops.mask_fwd(yy, Wd, bd, ld, td)
        res.append((loss, g, index) + ops.mask_bwd(g, rsum, go, Wd, ld, index, tuple(yy.shape), dtype))
    ref = _run(y, W, b, labels, t, C, gout=-0.5)
    nidx = ref['index'].numel()          # the index past the valid RoIs is not written
    for a, b_, k in zip(res[0], res[1], ('loss', 'g', 'index', 'dW', 'db', 'dY')):
        if k == 'index':
            a, b_ = a[:nidx], b_[:nidx]
        _same_bits(b_, a, k + ' with a storage offset')
    _same_bits(res[1][2][:nidx], ref['index'], 'index against the ctypes launch')
    for k, v in zip(('loss', 'g', 'dW', 'db', 'dY'), (res[1][0][0], res[1][1], res[1][3], res[1][4], res[1][5])):
        _same_bits(v.reshape(ref[k].shape), ref[k], k + ' against the ctypes launch')
    _check_tier('exact', ref, y, W, b, labels, t, C, -0.5)
