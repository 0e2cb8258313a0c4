"""CPU: the float64 mask oracle and its per-element bounds (tests/mask_oracle.py), which the GPU tests of the fused mask
loss (tests/test_gpu_mask_loss_vs_float64.py, tests/test_gpu_mask_loss.py) rest on --

  * the bounds hold for an fp32 restatement of bags_mask_fwd / bags_mask_bwd's arithmetic in the kernels' order (the
    channel groups of both load widths, the expf / log1pf formulas, the xor warp sums, the last CTA's loss sum and the
    class units' warp order), in all three tiers of input: bounds too tight for the kernels would fail here first;
  * the tier constructions are what the GPU tests assume (exact partial sums below 2^20, |z| >= 128 when saturated);
  * the oracle's BCE is F.binary_cross_entropy_with_logits, soft targets included.
"""
import pytest
import torch
import torch.nn.functional as F

import mask_oracle as MO

F32, F64 = torch.float32, torch.float64
THREADS = 256


def _fma(a, b, c):
    """fp32 fma through float64 (the product of two fp32 values is exact there; one rounding to fp32 after)."""
    return (a.double() * b.double() + c.double()).float()


def _warp_sum(v):
    """bags::warp_sum over the last dimension (32 lanes): v += shfl_xor(v, o) for o = 16, 8, 4, 2, 1."""
    lanes = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., lanes ^ o]
    return v[..., 0]


def _tiles(x, HW):
    """[..., HW] -> [..., tiles, 64], zero-padded past HW."""
    tiles = -(-HW // MO.TILE)
    pad = torch.zeros(*x.shape[:-1], tiles * MO.TILE - HW, dtype=x.dtype)
    return torch.cat([x, pad], -1).reshape(*x.shape[:-1], tiles, MO.TILE)


def kernel_fp32(y, W, b, labels, t, V, gout=1.0):
    """loss, g [P, HW], dW, db in fp32, each operation rounded as bags_mask_fwd / bags_mask_bwd round it."""
    P, Cin, HW = y.shape
    C = W.shape[0]
    y, W, t = y.float(), W.float(), t.float()
    b = torch.zeros(C) if b is None else b.float()
    valid = MO.valid_rows(labels, C)
    lab = torch.where(valid, labels, torch.zeros_like(labels))
    Wl, bl = W[lab], b[lab]                                   # [P, Cin], [P]
    NG = THREADS // (MO.TILE // V)
    z = torch.zeros(P, HW)
    for k in range(NG):                                       # the groups' fma chains, then their sums in order
        acc = torch.zeros(P, HW)
        for c in range(k, Cin, NG):
            acc = _fma(Wl[:, c:c + 1], y[:, c], acc)
        z = z + acc
    z = z + bl.unsqueeze(1)
    e = torch.exp(-z.abs())
    s = torch.where(z >= 0, 1 / (1 + e), e / (1 + e))
    n = torch.tensor(float(P * HW))
    lq = (torch.clamp(z, min=0) - z * t) + torch.log1p(e)
    g = torch.where(valid.unsqueeze(1), (s - t) / n, torch.zeros(()))
    # the loss: each tile's two warps, then the last CTA's sum of the P * tiles partials
    lt = _tiles(torch.where(valid.unsqueeze(1), lq, torch.zeros(())), HW)      # [P, tiles, 64]
    part = (_warp_sum(lt[..., :32]) + _warp_sum(lt[..., 32:])).reshape(-1)
    grid = part.numel()
    per = torch.zeros(THREADS)
    for i0 in range(0, grid, THREADS):
        chunk = part[i0:i0 + THREADS]
        per[:chunk.numel()] = per[:chunk.numel()] + chunk
    warp_tot = _warp_sum(per.reshape(THREADS // 32, 32))
    total = torch.zeros(())
    for w in range(THREADS // 32):
        total = total + warp_tot[w]
    loss = total / n if P > 0 else torch.zeros(())
    # pass 2: rsum[p, tile, c] (lanes fma q = lane, lane + 32, then the warp sum) and the db column
    gt = _tiles(g, HW)                                        # [P, tiles, 64]
    yt = _tiles(y, HW)                                        # [P, Cin, tiles, 64]
    lane = _fma(gt[:, None, :, 32:], yt[..., 32:], _fma(gt[:, None, :, :32], yt[..., :32], torch.zeros(())))
    rsum = torch.cat([_warp_sum(lane), _warp_sum(gt[..., :32] + gt[..., 32:]).unsqueeze(1)], 1)  # [P, Cin+1, tiles]
    # class units: warp w adds pairs j = w, w + 8, ... (RoIs by ascending id, then tiles), then the warps in order
    tiles = rsum.shape[2]
    go = torch.tensor(float(gout))
    out = torch.zeros(C, Cin + 1)
    for l in range(C):
        rois = ((labels == l) & valid).nonzero().reshape(-1)
        rows = rsum[rois].permute(0, 2, 1).reshape(-1, Cin + 1)     # pair j = roi * tiles + tile
        tot = torch.zeros(Cin + 1)
        for w in range(THREADS // 32):
            acc = torch.zeros(Cin + 1)
            for j in range(w, rows.shape[0], THREADS // 32):
                acc = acc + rows[j]
            tot = tot + acc
        out[l] = _fma(go, tot, torch.zeros(()))
    return dict(loss=loss, g=g, dW=out[:, :Cin], db=out[:, Cin])


SHAPES = [   # P, Cin, HW, classes, extra
    (5, 3, 33, 4, dict(invalid=True)),
    (9, 17, 64, 3, dict(soft=True)),
    (3, 33, 97, 2, dict(one_class=True)),
    (17, 5, 4, 1, dict(soft=True)),
    (2, 40, 130, 5, dict(invalid=True, soft=True)),
]


@pytest.mark.parametrize('V', [4, 1])
@pytest.mark.parametrize('tier', ['exact', 'saturated', 'numeric'])
@pytest.mark.parametrize('shape', range(len(SHAPES)), ids=['P%dC%dHW%dK%d' % s[:4] for s in SHAPES])
def test_bounds_hold_for_the_kernels_arithmetic(shape, tier, V):
    P, Cin, HW, C, kw = SHAPES[shape]
    if V == 4 and HW % 4:
        pytest.skip('four pixels a thread only when H W % 4 == 0')
    for dtype, gout in ((F32, (1.0, -0.5, 0.3)[shape % 3]), (torch.bfloat16, (-0.5, 0.3, 1.0)[shape % 3])):
        y, W, b, labels, t = MO.tier_inputs(tier, P, Cin, HW, C, dtype, seed=shape, **kw)
        got = kernel_fp32(y, W, b, labels, t, V, gout=gout)
        eb = MO.error_bounds(y, W, b, labels, t, gout=gout, z_exact=tier != 'numeric')
        o = eb['terms']
        assert abs(got['loss'].double() - o['loss']).item() <= eb['loss'], (got['loss'], o['loss'], eb['loss'])
        for name in ('g', 'dW', 'db'):
            err = (got[name].double() - o[name]).abs()
            assert (err <= eb[name]).all(), (name, (err - eb[name]).max().item())
        # the reduction-only bound of dW / db against float64 of the restatement's own g
        red = MO.reduction_bounds(got['g'], y, labels, C, gout)
        gg = got['g'].double() * gout
        valid = MO.valid_rows(labels, C).nonzero().reshape(-1)
        dW = torch.zeros(C, Cin, dtype=F64).index_add_(0, labels[valid], torch.einsum(
            'pq,pcq->pc', gg[valid], y.double()[valid]))
        db = torch.zeros(C, dtype=F64).index_add_(0, labels[valid], gg[valid].sum(1))
        assert ((got['dW'].double() - dW).abs() <= red['dW']).all()
        assert ((got['db'].double() - db).abs() <= red['db']).all()
        if tier == 'saturated':       # s is exactly 0 or 1, the loss terms multiples of 2^-3
            n = torch.tensor(float(P * HW))
            s = (o['z'] >= 0).float()
            want_g = torch.where(MO.valid_rows(labels, C).unsqueeze(1), (s - t) / n, torch.zeros(()))
            assert torch.equal(got['g'], want_g)
            valid = MO.valid_rows(labels, C)
            S = (torch.clamp(o['z'], min=0) - o['z'] * t.double())[valid].sum()    # exact
            assert torch.equal(got['loss'], S.float() / n)


def test_bounds_are_not_vacuous():
    """The numeric tier's g bound is a few hundred u of |g| at Cin = 256, not a multiple of |g| itself."""
    y, W, b, labels, t = MO.tier_inputs('numeric', 4, 256, 64, 3)
    eb = MO.error_bounds(y, W, b, labels, t)
    g = eb['terms']['g'].abs()
    assert (eb['g'] <= 2e-4 * g + 1e-9 / g.numel()).float().mean() > 0.99


@pytest.mark.parametrize('Cin', [1, 4, 17, 64, 256])
@pytest.mark.parametrize('HW', [1, 33, 784])
def test_exact_tier_sums_stay_exact(Cin, HW):
    for seed in range(3):
        y, W, b, labels, t = MO.tier_inputs('exact', 7, Cin, HW, 11, torch.bfloat16, seed=seed, invalid=True)
        assert torch.equal(y.float().round(), y.float()) and torch.equal((b * 8).round(), b * 8)
        m = MO.exact_partial_max(y, W, b, labels)
        assert m < MO.EXACT_LIMIT
        z = MO.mask_terms(y, W, b, labels, t)['z']
        assert z.abs().max() > 15          # the exponentials reach far below 1


@pytest.mark.parametrize('Cin', [1, 3, 33, 256])
def test_saturated_tier_is_saturated(Cin):
    for seed in range(3):
        y, W, b, labels, t = MO.tier_inputs('saturated', 7, Cin, 65, 11, torch.bfloat16, seed=seed, invalid=True)
        assert MO.saturated_min_abs_z(y, W, b, labels) >= 128
        assert MO.exact_partial_max(y, W, b, labels) < 2 ** 9
        # expf(-128) is 0 in fp32, so s is exactly 0 or 1
        assert torch.exp(torch.tensor(-128.0)).item() == 0.0
        assert set(t.unique().tolist()) <= {0.0, 1.0}


def test_tier_labels():
    _, _, _, labels, _ = MO.tier_inputs('numeric', 9, 3, 4, 13, invalid=True)
    assert labels[1:9:2].tolist() == [-1, 13, 20, 2 ** 40]
    _, _, _, labels, _ = MO.tier_inputs('numeric', 9, 3, 4, 13, one_class=True)
    assert (labels == 6).all()
    _, _, _, labels, _ = MO.tier_inputs('numeric', 9, 3, 4, 1)
    assert (labels == 0).all()


@pytest.mark.parametrize('gout', [1.0, -0.75])
def test_oracle_bce_is_torch_bce_with_logits(gout):
    """mask_terms' loss and g are F.binary_cross_entropy_with_logits (mean over P H W, invalid rows 0) and its
    autograd gradient, in float64, on soft and 0/1 targets."""
    y, W, b, labels, t = MO.tier_inputs('numeric', 9, 6, 35, 5, F64, seed=4, soft=True, invalid=True)
    y, W, b = y.double() * 3, W.double(), b.double()
    o = MO.mask_terms(y, W, b, labels, t, gout=gout)
    valid = MO.valid_rows(labels, 5)
    z = torch.einsum('pc,pcq->pq', W[labels.clamp(0, 4)], y) + b[labels.clamp(0, 4)].unsqueeze(1)
    z = z.detach().requires_grad_(True)
    per = F.binary_cross_entropy_with_logits(z, t.double(), reduction='none')
    loss = (per * valid.unsqueeze(1)).sum() / z.numel()
    (loss * gout).backward()
    torch.testing.assert_close(o['loss'], loss.detach(), rtol=1e-14, atol=0)
    torch.testing.assert_close(o['g'] * gout, z.grad, rtol=1e-13, atol=1e-300)
    assert (t[::2] * 8).remainder(8).eq(0).all() and not (t * 8).remainder(8).eq(0).all()
